// The lio_rm handle's placement, for a caller that inserts into it on its own stream (lio_node_attach_registered_map, node.cu).
// The handle stays opaque otherwise (regmap.cu).
#pragma once
#include <cuda_runtime.h>
#include "../../include/lio_b200.h"

int rm_device(const lio_rm *m);
cudaStream_t rm_stream(const lio_rm *m);
