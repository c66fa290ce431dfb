// Host-side helpers shared by the C-ABI translation units: error text, argument checks.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "../../include/anyv2v_b200.h"

namespace av2v {

char* last_error_buf();  // thread-local 512-byte buffer (defined in abi.cu)

inline int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(last_error_buf(), 512, fmt, ap);
  va_end(ap);
  return code;
}

#define AV2V_CHECK_CUDA(expr)                                                                   \
  do {                                                                                          \
    cudaError_t e__ = (expr);                                                                   \
    if (e__ != cudaSuccess)                                                                     \
      return ::av2v::fail(AV2V_ECUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), \
                          __FILE__, __LINE__);                                                  \
  } while (0)

#define AV2V_REQUIRE(cond, code, ...) \
  do {                                \
    if (!(cond)) return ::av2v::fail(code, __VA_ARGS__); \
  } while (0)

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

int sm_count_cached();  // abi.cu

// 4-D fp16 tensor maps for TMA tile loads, 128-byte swizzle, zeros outside the tensor (abi.cu): any dims, byte strides and
// box with 64-element rows; and the rows map of the GEMM and attention operands, boxes of 64 columns x box_rows rows
int encode_map_4d(CUtensorMap* map, const void* base, const unsigned long long (&dims)[4],
                  const unsigned long long (&strides)[3], const unsigned (&box)[4]);
int encode_rows_map(CUtensorMap* map, const void* base, int cols, int tokens, int seqs, int branches, int ld,
                    long long branch_stride, int box_rows);

}  // namespace av2v
