// lio_mapping_b200 — library-wide C-ABI helpers (error text, device probe, live-resource count).
#include "common.cuh"
#include <cstring>

static thread_local char g_err[512] = "";
std::atomic<long long> lio::g_live_resources{0};

void lio_set_last_error(const char *file, int line, const char *msg) {
  snprintf(g_err, sizeof(g_err), "%s:%d: %s", file, line, msg ? msg : "");
}

int lio::refuse_null_handle(const char *entry) {
  snprintf(g_err, sizeof(g_err), "%s: null handle", entry);
  return LIO_ERR_INVALID;
}

int lio::select_device(int device, int *sms) {
  if (lio_device_count() <= 0) return LIO_ERR_NO_DEVICE;
  LIO_CUDA_OK(cudaSetDevice(device));
  if (sms) cudaDeviceGetAttribute(sms, cudaDevAttrMultiProcessorCount, device);
  return LIO_OK;
}

extern "C" const char *lio_last_error(void) { return g_err; }
extern "C" int lio_version(void) { return 100; }
extern "C" long long lio_live_resources(void) { return lio::g_live_resources.load(); }
extern "C" int lio_device_count(void) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess) {
    lio_set_last_error(__FILE__, __LINE__, cudaGetErrorString(e));
    cudaGetLastError();
    return 0;
  }
  return n;
}
