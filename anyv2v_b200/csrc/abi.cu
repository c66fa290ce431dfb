// C-ABI plumbing: version, thread-local error text, device query.
#include "host_util.cuh"

namespace av2v {

char* last_error_buf() {
  static thread_local char buf[512] = {0};
  return buf;
}

int sm_count_cached() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cached[dev] = n;
  }
  return cached[dev];
}

}  // namespace av2v

extern "C" int av2v_abi_version(void) { return 1; }

extern "C" const char* av2v_last_error(void) { return av2v::last_error_buf(); }

extern "C" int av2v_device_info(int* sm_count, int* cc_major, int* cc_minor) {
  int dev = 0;
  AV2V_CHECK_CUDA(cudaGetDevice(&dev));
  int sm = 0, maj = 0, min = 0;
  AV2V_CHECK_CUDA(cudaDeviceGetAttribute(&sm, cudaDevAttrMultiProcessorCount, dev));
  AV2V_CHECK_CUDA(cudaDeviceGetAttribute(&maj, cudaDevAttrComputeCapabilityMajor, dev));
  AV2V_CHECK_CUDA(cudaDeviceGetAttribute(&min, cudaDevAttrComputeCapabilityMinor, dev));
  if (sm_count) *sm_count = sm;
  if (cc_major) *cc_major = maj;
  if (cc_minor) *cc_minor = min;
  if (maj != 9 || min != 0) return av2v::fail(AV2V_ENOSUP, "device compute capability %d.%d is not sm_90", maj, min);
  return AV2V_OK;
}
