"""lio_mapping_b200: the reference LIO-mapping pipeline on the GPU, over the C-ABI in include/lio_b200.h."""
from .registered_map import RegisteredMap, write_pcd  # noqa: F401
from .node import TOPICS, LioNode, write_tum  # noqa: F401
