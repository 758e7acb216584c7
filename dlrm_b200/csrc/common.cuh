// Shared helpers for libdlrm_b200.so (sm_90a only).
#pragma once
#include <cuda_fp16.h>
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
  TUNE_UPD_LEAN = 10,           // embedding update, dim <= 128: 2 = the general kernel instead of the lean one
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

// ---- fp16 table rows (weight_dtype = DLRM_DTYPE_F16): widened to fp32 on load, stochastically rounded on store.
// The kernels are templated on the row type `wt` (float or __half); the float instantiations are the fp32 code.
template <typename wt>
struct is_f16 { static constexpr bool value = false; };
template <>
struct is_f16<__half> { static constexpr bool value = true; };

__device__ __forceinline__ float4 h4_to_f4(uint2 u) {
  const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
  const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
  return make_float4(a.x, a.y, b.x, b.y);
}

// 4 consecutive row elements as fp32 (16-byte fp32 / 8-byte fp16 load)
template <typename wt>
__device__ __forceinline__ float4 ld_row4(const wt* p) {
  if constexpr (is_f16<wt>::value) return h4_to_f4(*reinterpret_cast<const uint2*>(p));
  else return *reinterpret_cast<const float4*>(p);
}
// the same through the non-allocating read-only path (gather)
template <typename wt>
__device__ __forceinline__ float4 ldg_stream_row4(const wt* p) {
  if constexpr (is_f16<wt>::value) {
    uint2 u;
    asm("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(u.x), "=r"(u.y) : "l"(p));
    return h4_to_f4(u);
  } else {
    return ldg_stream_f4(p);
  }
}

// finaliser of splitmix64 (dlrm_b200/mlperf.py; the synthetic batches of shard_ops.cu use it too)
__device__ __forceinline__ unsigned long long splitmix64(unsigned long long x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
// key of a global row for the stochastic rounding of its columns (include/dlrm_b200.h, round_key)
__device__ __forceinline__ unsigned long long sr_row_key(unsigned long long round_key, long long global_row) {
  return round_key ^ ((unsigned long long)global_row * 0xC2B2AE3D27D4EB4Full);
}
// 64 random bits for columns [4 q, 4 q + 4) of a row: column 4 q + j uses bits [16 j, 16 j + 16)
__device__ __forceinline__ unsigned long long sr_bits(unsigned long long row_key, int q) {
  return splitmix64(row_key ^ ((unsigned long long)q * 0x165667B19E3779F9ull));
}

// Stochastic rounding of fp32 x to fp16 with the 16 random bits r (the definition in include/dlrm_b200.h).
__device__ __forceinline__ unsigned short f32_to_f16_sr(float x, unsigned r) {
  const float ax = fabsf(x);
  const unsigned short sign = (__float_as_uint(x) >> 16) & 0x8000u;
  if (!(ax <= 65504.f)) return (ax != ax) ? (unsigned short)(sign | 0x7e00u) : (unsigned short)(sign | 0x7c00u);
  const unsigned short lo = __half_as_ushort(__float2half_rz(x));   // the fp16 neighbour toward zero
  const float flo = fabsf(__half2float(__ushort_as_half(lo)));
  if (flo == ax) return lo;
  const float fhi = fabsf(__half2float(__ushort_as_half((unsigned short)(lo + 1))));   // away from zero
  const float t = floorf((ax - flo) / (fhi - flo) * 65536.f);       // exact: the step is a power of two
  return ((float)r < t) ? (unsigned short)(lo + 1) : lo;
}

// store 4 consecutive fp32 values as row elements: fp32 as is, fp16 with stochastic rounding from `bits`
template <typename wt>
__device__ __forceinline__ void st_row4(wt* p, float4 v, unsigned long long bits) {
  if constexpr (is_f16<wt>::value) {
    const unsigned a = f32_to_f16_sr(v.x, (unsigned)(bits & 0xffffu));
    const unsigned b = f32_to_f16_sr(v.y, (unsigned)((bits >> 16) & 0xffffu));
    const unsigned c = f32_to_f16_sr(v.z, (unsigned)((bits >> 32) & 0xffffu));
    const unsigned d = f32_to_f16_sr(v.w, (unsigned)(bits >> 48));
    *reinterpret_cast<uint2*>(p) = make_uint2(a | (b << 16), c | (d << 16));
  } else {
    (void)bits;
    *reinterpret_cast<float4*>(p) = v;
  }
}

// slot of a (table,row) in the duplicate filter: the address of the row's list head is a unique key
__device__ __forceinline__ unsigned filter_slot(const int* head_of_row, int log2_size) {
  const unsigned long long key = reinterpret_cast<unsigned long long>(head_of_row) >> 2;
  return (unsigned)((key * 11400714819323198485ull) >> (64 - log2_size));
}

// Element-wise Adagrad (DLRM_OPT_ADAGRAD) on one element, in the order include/dlrm_b200.h states: the accumulator
// takes g*g and the add as two roundings (torch's grad.pow(2) then the sparse add; no FMA contraction), then IEEE
// sqrt, + eps, an IEEE division and one fused update w + nlr * q.  nlr = -lr.  Returns w'; s is updated in place.
__device__ __forceinline__ float adagrad_ew(float g, float& s, float w, float nlr, float eps) {
  s = __fadd_rn(s, __fmul_rn(g, g));
  return fmaf(nlr, __fdiv_rn(g, __fadd_rn(__fsqrt_rn(s), eps)), w);
}
__device__ __forceinline__ float4 adagrad_ew4(float4 g, float4& s, float4 w, float nlr, float eps) {
  return make_float4(adagrad_ew(g.x, s.x, w.x, nlr, eps), adagrad_ew(g.y, s.y, w.y, nlr, eps),
                     adagrad_ew(g.z, s.z, w.z, nlr, eps), adagrad_ew(g.w, s.w, w.w, nlr, eps));
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

}  // namespace dlrm
