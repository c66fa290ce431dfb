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

// 4-D fp16 tensor map for TMA tile loads: dims[0] (elements, contiguous) .. dims[3], byte strides of dims 1..3 (multiples of
// 16), a box of box[0] x .. x box[3] elements with box[0] = 64 (128-byte rows), 128-byte swizzle (the sw128 tile layout),
// zeros outside the tensor
int encode_map_4d(CUtensorMap* map, const void* base, const unsigned long long (&dims)[4],
                  const unsigned long long (&strides)[3], const unsigned (&box)[4]) {
  using Encode = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                              const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                              CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static Encode encode = nullptr;
  if (encode == nullptr) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    AV2V_CHECK_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q));
    AV2V_REQUIRE(q == cudaDriverEntryPointSuccess && fn != nullptr, AV2V_ECUDA, "cuTensorMapEncodeTiled not available");
    encode = reinterpret_cast<Encode>(fn);
  }
  const cuuint64_t d[4] = {dims[0], dims[1], dims[2], dims[3]}, st[3] = {strides[0], strides[1], strides[2]};
  const cuuint32_t bx[4] = {box[0], box[1], box[2], box[3]}, estr[4] = {1, 1, 1, 1};
  const CUresult r = encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), d, st, bx, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  AV2V_REQUIRE(r == CUDA_SUCCESS, AV2V_ECUDA, "cuTensorMapEncodeTiled failed (%d)", static_cast<int>(r));
  return AV2V_OK;
}

// [branches][sequences][tokens][cols] (row stride ld elements, branch stride in elements): a box of 64 columns x box_rows
// tokens
int encode_rows_map(CUtensorMap* map, const void* base, int cols, int tokens, int seqs, int branches, int ld,
                    long long branch_stride, int box_rows) {
  const unsigned long long seq_bytes = static_cast<unsigned long long>(tokens) * ld * 2;
  const unsigned long long dims[4] = {static_cast<unsigned long long>(cols), static_cast<unsigned long long>(tokens),
                                      static_cast<unsigned long long>(seqs), static_cast<unsigned long long>(branches)};
  const unsigned long long strides[3] = {static_cast<unsigned long long>(ld) * 2, seq_bytes,
                                         branches > 1 ? static_cast<unsigned long long>(branch_stride) * 2 : seq_bytes * seqs};
  const unsigned box[4] = {64, static_cast<unsigned>(box_rows), 1, 1};
  return encode_map_4d(map, base, dims, strides, box);
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
