// Operand preparation for the wgmma GEMMs.
//   split_bf16       : fp32 [M,N] -> (hi, lo) bf16 pairs, hi = bf16(x), lo = bf16(x - hi)
//   dense_update_pack: dense branch of optimizer.step() (torch.optim.SGD / optim/rwsadagrad.py:145-148)
//                      fused with the split-K slab reduction of the weight gradients and with the
//                      refresh of the (hi, lo) bf16 operand copy [N, K+1] = [W | bias] of every layer.
#include <cuda_bf16.h>

#include "common.cuh"

namespace dlrm {

__global__ void __launch_bounds__(256) split_bf16_kernel(const float* __restrict__ X, long long ldx,
                                                         long long M, long long N,
                                                         __nv_bfloat16* __restrict__ hi,
                                                         __nv_bfloat16* __restrict__ lo, long long ldo) {
  pdl_launch_dependents();
  pdl_wait();
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= M * N) return;
  const long long m = e / N, n = e - m * N;
  const float x = X[m * ldx + n];
  const __nv_bfloat16 h = __float2bfloat16_rn(x);
  hi[m * ldo + n] = h;
  if (lo) lo[m * ldo + n] = __float2bfloat16_rn(x - __bfloat162float(h));
}

struct DenseLayer {
  float* W; float* b;          // masters [N,K], [N]
  float* sW; float* sb;        // Adagrad sums (null for SGD)
  const float* dW; const float* db;  // slab 0 of the gradients
  __nv_bfloat16* hi; __nv_bfloat16* lo;  // [N, ldp] operand copy, column K = bias (may be null)
  long long slab_stride;
  int N, K, ldp, nslabs;
};
struct DenseLayers {
  DenseLayer l[16];
  int cta_begin[17];
  int num_layers;
  int optimizer;
  float lr, eps;
  const float* lr_dev;         // learning rate in device memory; NULL: lr above
};

__global__ void __launch_bounds__(256) dense_update_pack_kernel(const __grid_constant__ DenseLayers P) {
  pdl_launch_dependents();
  pdl_wait();
  // flattened grid: CTAs [cta_begin[i], cta_begin[i+1]) belong to layer i, 256 elements each
  int li = 0;
  while (li + 1 < P.num_layers && (int)blockIdx.x >= P.cta_begin[li + 1]) ++li;
  const DenseLayer& L = P.l[li];
  const unsigned total = (unsigned)L.N * (unsigned)(L.K + 1);
  const unsigned K1 = (unsigned)(L.K + 1);
  {
    const unsigned e = (unsigned)((int)blockIdx.x - P.cta_begin[li]) * 256u + threadIdx.x;
    if (e >= total) return;
    const int n = (int)(e / K1), k = (int)(e - (unsigned)n * K1);
    const bool is_b = k == L.K;
    const long long o = is_b ? n : (long long)n * L.K + k;
    float g = 0.f;
    if (P.optimizer >= 0 || P.optimizer == -2) {  // pack only (-1) reads no gradient: dW / db may be NULL
      const float* gp = is_b ? L.db : L.dW;
      g = gp[o];
      for (int s = 1; s < L.nslabs; ++s) g += gp[o + s * L.slab_stride];  // fixed order: deterministic
      if (P.optimizer == -2) {  // fold the slabs only (the caller all-reduces slab 0 next)
        const_cast<float*>(gp)[o] = g;
        return;
      }
    }
    float* pp = is_b ? L.b : L.W;
    float p = pp[o];
    const float lr = P.lr_dev ? *P.lr_dev : P.lr;
    if (P.optimizer == DLRM_OPT_RWSADAGRAD) {
      float* sp = is_b ? L.sb : L.sW;
      const float s2 = fmaf(g, g, sp[o]);
      sp[o] = s2;
      p = fmaf(-lr, g / (sqrtf(s2) + P.eps), p);
    } else if (P.optimizer == DLRM_OPT_SGD) {
      p = fmaf(-lr, g, p);
    }  // optimizer < 0: pack only
    pp[o] = p;
    if (L.hi) {
      const __nv_bfloat16 h = __float2bfloat16_rn(p);
      L.hi[(long long)n * L.ldp + k] = h;
      if (L.lo) L.lo[(long long)n * L.ldp + k] = __float2bfloat16_rn(p - __bfloat162float(h));
    }
  }
}

}  // namespace dlrm

extern "C" int dlrm_b200_split_bf16(const float* X, int64_t ldx, int64_t M, int64_t N, void* hi, void* lo,
                                    int64_t ld_out, void* stream) {
  using namespace dlrm;
  if (M <= 0 || N <= 0) return 0;
  if (!X || !hi) return set_error("split_bf16: NULL pointer");
  const long long n = M * N;
  (void)launch_chain(split_bf16_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0,
                     static_cast<cudaStream_t>(stream), X, (long long)ldx, (long long)M, (long long)N,
                     static_cast<__nv_bfloat16*>(hi), static_cast<__nv_bfloat16*>(lo), (long long)ld_out);
  DLRM_CHECK_LAUNCH("split_bf16_kernel");
  return 0;
}

static int dense_update_pack_impl(const dlrm_dense_layer_t* layers, int num_layers, int optimizer, float lr,
                                  const float* lr_dev, float eps, void* stream) {
  using namespace dlrm;
  if (num_layers <= 0) return 0;
  if (num_layers > 16) return set_error("dense_update_pack: at most 16 layers per call (got %d)", num_layers);
  if (optimizer == DLRM_OPT_ADAGRAD) optimizer = DLRM_OPT_RWSADAGRAD;   // the dense branches are the same algorithm
  if (optimizer < -2 || optimizer > DLRM_OPT_RWSADAGRAD) return set_error("dense_update_pack: optimizer=%d", optimizer);
  DenseLayers P;
  long long ctas = 0;
  for (int i = 0; i < num_layers; ++i) {
    const dlrm_dense_layer_t& s = layers[i];
    if (!s.W || !s.b) return set_error("dense_update_pack: layer %d NULL master", i);
    if ((optimizer >= 0 || optimizer == -2) && (!s.dW || !s.db))
      return set_error("dense_update_pack: layer %d NULL grad", i);
    if (optimizer == DLRM_OPT_RWSADAGRAD && (!s.sW || !s.sb))
      return set_error("dense_update_pack: layer %d NULL Adagrad state", i);
    DenseLayer& d = P.l[i];
    d.W = s.W; d.b = s.b; d.sW = s.sW; d.sb = s.sb; d.dW = s.dW; d.db = s.db;
    d.hi = static_cast<__nv_bfloat16*>(s.pack_hi); d.lo = static_cast<__nv_bfloat16*>(s.pack_lo);
    d.slab_stride = s.slab_stride; d.N = (int)s.N; d.K = (int)s.K; d.ldp = (int)s.ld_pack;
    d.nslabs = s.num_slabs < 1 ? 1 : (int)s.num_slabs;
    const long long t = (long long)s.N * (s.K + 1);
    if (t <= 0 || t >= (1ll << 31)) return set_error("dense_update_pack: layer %d has %lld parameters", i, t);
    P.cta_begin[i] = (int)ctas;
    ctas += (t + 255) / 256;
  }
  if (ctas >= (1ll << 31)) return set_error("dense_update_pack: too many parameters");
  for (int i = num_layers; i <= 16; ++i) P.cta_begin[i] = (int)ctas;
  P.num_layers = num_layers;
  P.optimizer = optimizer; P.lr = lr; P.eps = eps; P.lr_dev = lr_dev;
  (void)launch_chain(dense_update_pack_kernel, dim3((unsigned)ctas), dim3(256), 0, static_cast<cudaStream_t>(stream), P);
  DLRM_CHECK_LAUNCH("dense_update_pack_kernel");
  return 0;
}

extern "C" int dlrm_b200_dense_update_pack(const dlrm_dense_layer_t* layers, int num_layers, int optimizer,
                                           float lr, float eps, void* stream) {
  return dense_update_pack_impl(layers, num_layers, optimizer, lr, nullptr, eps, stream);
}

extern "C" int dlrm_b200_dense_update_pack_lr_dev(const dlrm_dense_layer_t* layers, int num_layers, int optimizer,
                                                  float lr, const float* lr_dev, float eps, void* stream) {
  return dense_update_pack_impl(layers, num_layers, optimizer, lr, lr_dev, eps, stream);
}
