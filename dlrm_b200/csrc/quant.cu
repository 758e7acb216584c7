// Row-wise 8- / 4-bit quantization of embedding rows into fbgemm's packed rows (the bytes of
// torch.ops.quantized.embedding_bag_{byte,4bit}_prepack, used by DLRM_Net.quantize_embedding, dlrm_s_pytorch.py:465-481).
// One warp per row: the lanes stride over the columns for min / max, reduce with shuffles, then write the packed
// bytes (4-bit: lane j of a pass owns output byte j, i.e. columns 2j and 2j+1).  Every operation is the fp32 operation
// of the CPU op, rounded the same way (__f*_rn so that nothing is contracted), so the bytes are identical.
#include "common.cuh"

namespace dlrm {

template <typename st>
__device__ __forceinline__ float ld_elem(const st* p) {
  if constexpr (is_f16<st>::value) return __half2float(*p);
  else return *p;
}

__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// rint of x clamped to [0, hi]; NaN gives 0, like the CPU op's conversion of a non-finite row's products
__device__ __forceinline__ unsigned quant_level(float x, float hi) {
  const float r = rintf(x);
  return (r >= 0.f) ? (unsigned)fminf(r, hi) : 0u;
}

template <typename st, int BITS>
__global__ void __launch_bounds__(256) quantize_rows_kernel(const st* __restrict__ src, long long ld_src,
                                                            long long rows, int D, unsigned char* __restrict__ dst,
                                                            long long ld_dst) {
  const long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= rows) return;
  const st* x = src + r * ld_src;
  unsigned char* out = dst + r * ld_dst;
  float mn = INFINITY, mx = -INFINITY;
  for (int c = lane; c < D; c += 32) {
    const float v = ld_elem(x + c);
    mn = fminf(mn, v);
    mx = fmaxf(mx, v);
  }
  mn = warp_min(mn);
  mx = warp_max(mx);
  if constexpr (BITS == 8) {
    const float range = __fsub_rn(mx, mn);
    const float scale = __fdiv_rn(range, 255.f);
    const float inv = __fdiv_rn(255.f, __fadd_rn(range, 1e-8f));
    for (int c = lane; c < D; c += 32)
      out[c] = (unsigned char)quant_level(__fmul_rn(__fsub_rn(ld_elem(x + c), mn), inv), 255.f);
    if (lane == 0) {
      reinterpret_cast<float*>(out + D)[0] = scale;
      reinterpret_cast<float*>(out + D)[1] = mn;
    }
  } else {
    const __half bias16 = __float2half_rn(mn);
    const float bias = __half2float(bias16);
    const float range = __fsub_rn(mx, bias);
    float scale = range == 0.f ? 1.f : __fdiv_rn(range, 15.f);
    scale = __half2float(__float2half_rn(scale));
    if (scale == 0.f) scale = 1.f;
    float inv = __fdiv_rn(1.f, scale);
    if (isinf(inv)) scale = inv = 1.f;
    for (int j = lane; j < D / 2; j += 32) {
      const unsigned lo = quant_level(__fmul_rn(__fsub_rn(ld_elem(x + 2 * j), bias), inv), 15.f);
      const unsigned hi = quant_level(__fmul_rn(__fsub_rn(ld_elem(x + 2 * j + 1), bias), inv), 15.f);
      out[j] = (unsigned char)(lo | (hi << 4));
    }
    if (lane == 0) {
      __half2 sb;
      sb.x = __float2half_rn(scale);
      sb.y = bias16;
      *reinterpret_cast<__half2*>(out + D / 2) = sb;
    }
  }
}

}  // namespace dlrm

extern "C" int dlrm_b200_emb_quantize_rows(const void* src, int src_dtype, int64_t ld_src, int64_t rows, int dim,
                                           void* dst, int dst_dtype, int64_t ld_dst, void* stream) {
  using namespace dlrm;
  if (src_dtype != DLRM_DTYPE_F32 && src_dtype != DLRM_DTYPE_F16)
    return set_error("emb_quantize_rows: src_dtype=%d (fp32 or fp16 rows)", src_dtype);
  if (dst_dtype != DLRM_DTYPE_Q8 && dst_dtype != DLRM_DTYPE_Q4)
    return set_error("emb_quantize_rows: dst_dtype=%d (DLRM_DTYPE_Q8 or DLRM_DTYPE_Q4)", dst_dtype);
  if (dim <= 0 || (dst_dtype == DLRM_DTYPE_Q8 && dim % 4) || (dst_dtype == DLRM_DTYPE_Q4 && dim % 8))
    return set_error("emb_quantize_rows: dim=%d (8-bit rows need dim %% 4 == 0, 4-bit rows dim %% 8 == 0)", dim);
  const int64_t width = dst_dtype == DLRM_DTYPE_Q8 ? dim + 8 : dim / 2 + 4;
  if (ld_dst == 0) ld_dst = width;
  if (ld_src == 0) ld_src = dim;
  if (rows < 0 || ld_dst < width || ld_dst % 4 || ld_src < dim)
    return set_error("emb_quantize_rows: rows=%lld ld_src=%lld ld_dst=%lld", (long long)rows, (long long)ld_src,
                     (long long)ld_dst);
  if (rows == 0) return 0;
  if (!src || !dst || (reinterpret_cast<uintptr_t>(dst) & 3))
    return set_error("emb_quantize_rows: NULL pointer or dst not 4-byte aligned");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const dim3 grid((unsigned)((rows * 32 + 255) / 256));
  unsigned char* d = static_cast<unsigned char*>(dst);
#define QLAUNCH(ST, BITS) \
  quantize_rows_kernel<ST, BITS><<<grid, 256, 0, st>>>(static_cast<const ST*>(src), ld_src, rows, dim, d, ld_dst)
  if (src_dtype == DLRM_DTYPE_F32) {
    if (dst_dtype == DLRM_DTYPE_Q8) QLAUNCH(float, 8); else QLAUNCH(float, 4);
  } else {
    if (dst_dtype == DLRM_DTYPE_Q8) QLAUNCH(__half, 8); else QLAUNCH(__half, 4);
  }
#undef QLAUNCH
  DLRM_CHECK_LAUNCH("quantize_rows_kernel");
  return 0;
}
