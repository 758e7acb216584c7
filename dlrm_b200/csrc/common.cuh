// Shared helpers for libdlrm_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/dlrm_b200.h"

namespace dlrm {

// thread-local error text behind dlrm_b200_last_error()
char* err_buf();
int set_error(const char* fmt, ...);
int get_tunable(int id);
// One 4-byte device error word per GPU (allocated on first use, never freed): bit 0 = an embedding index was
// outside its table.  Kernels only set bits; dlrm_b200_check_device_errors() reads and clears it.
unsigned* err_word_device();

enum Tunable {
  TUNE_EMB_BAGS_PER_GROUP = 0,  // bags processed back to back by one lane group
  TUNE_EMB_UNROLL = 1,          // rows in flight per lane group (4 or 8)
  TUNE_EMB_BLOCK = 2,           // threads per CTA in the gather
  TUNE_UPD_BLOCK = 3,
  TUNE_GEMM_SPLITK = 4,
  TUNE_GEMM_SMEM_KB = 5,        // operand-ring budget per GEMM CTA at plan creation (0 = 200 KB, the deepest ring)
  TUNE_HEAD_ROWS = 6,           // samples per CTA in the fused head (16 or 32; 0 = default)
  TUNE_INTERACT_BWD_COLS = 7,   // 1 = one column per thread (first kernel), else float2 columns
  TUNE_PDL = 8,                 // programmatic dependent launch on the dense chain: 0/1 = on, 2 = off
  TUNE_UPD_LEAN = 10,           // embedding update, dim <= 128: 0 = default lean variant, 1/3..7 = variants (emb_bwd.cu), 2 = general kernel
  TUNE_UPD_DEBUG = 11,          // timing experiments on the update kernel (see EmbBwdParams::debug); 0 = off
  TUNE_CHAIN_ORDER = 9,         // gemm_chain task order: 0/1 = layer by layer, 2 = m-tile major across layers
  TUNE_COUNT = 16
};

#define DLRM_CHECK_LAUNCH(name)                                                         \
  do {                                                                                  \
    cudaError_t e__ = cudaGetLastError();                                               \
    if (e__ != cudaSuccess)                                                             \
      return dlrm::set_error("%s: launch failed: %s", name, cudaGetErrorString(e__));   \
  } while (0)

#define DLRM_CUDA(call)                                                                 \
  do {                                                                                  \
    cudaError_t e__ = (call);                                                           \
    if (e__ != cudaSuccess)                                                             \
      return dlrm::set_error("%s failed: %s", #call, cudaGetErrorString(e__));          \
  } while (0)

// Programmatic dependent launch (griddepcontrol): a kernel launched through launch_chain() may become
// resident while its predecessor in the stream is still draining; it must not touch global memory
// before pdl_wait() (which returns once the predecessor grid has completed and its writes are visible).
// Every kernel launched this way executes BOTH calls, so completion stays transitive along the stream.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

template <typename... KArgs, typename... Args>
static inline cudaError_t launch_chain(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
                                       cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = get_tunable(TUNE_PDL) == 2 ? 0 : 1;   // on by default (r20: 0.518 -> 0.502 ms/step); 2 = off
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// 128-bit read-only load that does not allocate in L1 (rows are touched once per kernel)
__device__ __forceinline__ float4 ldg_stream_f4(const float* p) {
  float4 v;
  asm("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p));
  return v;
}

// slot of a (table,row) in the duplicate filter: the address of the row's list head is a unique key
__device__ __forceinline__ unsigned filter_slot(const int* head_of_row, int log2_size) {
  const unsigned long long key = reinterpret_cast<unsigned long long>(head_of_row) >> 2;
  return (unsigned)((key * 11400714819323198485ull) >> (64 - log2_size));
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

}  // namespace dlrm
