// Fused "head" of the top MLP when its last layer has ONE output (the click probability):
//   p = act(h . w + b)                      last nn.Linear + Sigmoid   (dlrm_s_pytorch.py:208-246)
//   z = clamp(p, thr, 1-thr)                 sequential_forward :607-610
//   loss = mean l(z, t)                      loss_fn_wrap :148-156 (MSE / BCE / wBCE)
//   gz   = dloss/d(pre-activation)           autograd through loss, clamp and the activation
//   dW = sum_b gz[b] h[b,:],  db = sum_b gz[b]                     (wgrad + bias grad)
//   gprev[b,:] = gz[b] * w * act_prev'(h[b,:])                      (dgrad + previous act')
// One launch replaces addmm + sigmoid + loss + their three backward GEMV-shaped GEMMs, which are
// pathological for a tiled GEMM (M = 1 or N = 1).  The gradient needs no cross-sample reduction
// (1/n is known on the host); loss, dW and db are reduced deterministically: per-CTA partials,
// then the last CTA to finish sums them in block order.
#include <cuda_bf16.h>

#include "common.cuh"

namespace dlrm {

struct HeadArgs {
  const float* h; long long ldh;
  const float* w; const float* bias;
  const float* target; const float* ws;
  float* p; float* loss; float* gz;
  float* dW; float* db;
  float* gprev; long long ld_gprev;
  __nv_bfloat16* gprev_hi; __nv_bfloat16* gprev_lo; long long ld_gb;
  float* partial; unsigned* counter;
  long long B; int K;
  int act_last, act_prev, loss_kind;
  float thr;
};

constexpr int HEAD_ROWS_MIN = 16;   // scratch is sized for the smaller tile

template <int HEAD_ROWS>
__global__ void __launch_bounds__(256) head_kernel(const HeadArgs a) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float s_gz[HEAD_ROWS], s_loss[HEAD_ROWS];
  __shared__ bool s_last;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long r0 = (long long)blockIdx.x * HEAD_ROWS;
  const int nrows = (int)min((long long)HEAD_ROWS, a.B - r0);
  const bool clampd = a.thr > 0.f && a.thr < 1.f;
  const float inv_n = 1.0f / (float)a.B;
  // ---- phase 1: one warp per sample (4 samples per warp)
  for (int rl = warp; rl < HEAD_ROWS; rl += 8) {
    float per = 0.f, g = 0.f;
    if (rl < nrows) {
      const float* hr = a.h + (r0 + rl) * a.ldh;
      float s = 0.f;
      for (int k = lane; k < a.K; k += 32) s = fmaf(hr[k], a.w[k], s);
      s = warp_sum(s);
      const float zpre = s + a.bias[0];
      float pi = zpre;
      if (a.act_last == DLRM_ACT_SIGMOID) pi = 1.0f / (1.0f + expf(-zpre));
      else if (a.act_last == DLRM_ACT_RELU) pi = fmaxf(zpre, 0.f);
      if (lane == 0) a.p[r0 + rl] = pi;
      if (a.target) {
        const float t = a.target[r0 + rl];
        const float z = clampd ? fminf(fmaxf(pi, a.thr), 1.0f - a.thr) : pi;
        if (a.loss_kind == DLRM_LOSS_MSE) {
          const float d = z - t;
          per = d * d;
          g = 2.0f * d * inv_n;
        } else {
          const float lz = fmaxf(logf(z), -100.0f);
          const float l1z = fmaxf(logf(1.0f - z), -100.0f);
          per = (t - 1.0f) * l1z - t * lz;
          g = (z - t) / fmaxf((1.0f - z) * z, 1e-12f);
          if (a.loss_kind == DLRM_LOSS_WBCE) {
            const float wgt = a.ws[(int)t];
            per *= wgt;
            g *= wgt;
          }
          g *= inv_n;
        }
        if (clampd && !(pi >= a.thr && pi <= 1.0f - a.thr)) g = 0.f;
        if (a.act_last == DLRM_ACT_SIGMOID) g *= (1.0f - pi) * pi;
        else if (a.act_last == DLRM_ACT_RELU) g = pi > 0.f ? g : 0.f;
        if (lane == 0 && a.gz) a.gz[r0 + rl] = g;
      }
    }
    if (lane == 0) { s_gz[rl] = g; s_loss[rl] = per; }
  }
  if (!a.target) return;
  __syncthreads();
  // ---- phase 2: thread = column; partial dW, and the gradient w.r.t. the layer input
  float* part = a.partial + (long long)blockIdx.x * (a.K + 2);
  const bool train = a.dW != nullptr;
  if (train) {
    for (int k = threadIdx.x; k < a.K; k += blockDim.x) {
      const float wk = a.w[k];
      float acc = 0.f;
      for (int rl0 = 0; rl0 < nrows; rl0 += 8) {
        float hv8[8];
#pragma unroll
        for (int u = 0; u < 8; ++u)   // 8 independent loads in flight before the dependent math / stores
          hv8[u] = (rl0 + u < nrows) ? a.h[(r0 + rl0 + u) * a.ldh + k] : 0.f;
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const int rl = rl0 + u;
          if (rl >= nrows) break;
          const float hv = hv8[u];
          const float g = s_gz[rl];
          acc = fmaf(g, hv, acc);
          float gp = g * wk;
          if (a.act_prev == DLRM_ACT_RELU) gp = hv > 0.f ? gp : 0.f;
          else if (a.act_prev == DLRM_ACT_SIGMOID) gp *= (1.0f - hv) * hv;
          if (a.gprev) a.gprev[(r0 + rl) * a.ld_gprev + k] = gp;
          if (a.gprev_hi) {
            const __nv_bfloat16 hb = __float2bfloat16_rn(gp);
            a.gprev_hi[(r0 + rl) * a.ld_gb + k] = hb;
            if (a.gprev_lo) a.gprev_lo[(r0 + rl) * a.ld_gb + k] = __float2bfloat16_rn(gp - __bfloat162float(hb));
          }
        }
      }
      part[k] = acc;
    }
  }
  if (threadIdx.x == 0) {
    float sg = 0.f, sl = 0.f;
    for (int rl = 0; rl < nrows; ++rl) { sg += s_gz[rl]; sl += s_loss[rl]; }
    part[a.K] = sg;
    part[a.K + 1] = sl;
  }
  // ---- deterministic grid reduction by the last CTA
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned ticket = atomicAdd(a.counter, 1u);
    s_last = ticket == gridDim.x - 1;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  const int nb = gridDim.x;
  for (int k = threadIdx.x; k < a.K + 2; k += blockDim.x) {
    if (!train && k < a.K) continue;
    float acc = 0.f;
    for (int b = 0; b < nb; ++b) acc += a.partial[(long long)b * (a.K + 2) + k];
    if (k < a.K) a.dW[k] = acc;
    else if (k == a.K) { if (a.db) a.db[0] = acc; }
    else a.loss[0] = acc * inv_n;
  }
  if (threadIdx.x == 0) *a.counter = 0u;
}

}  // namespace dlrm

extern "C" int64_t dlrm_b200_head_scratch_bytes(int64_t batch, int64_t K) {
  const int64_t nb = (batch + dlrm::HEAD_ROWS_MIN - 1) / dlrm::HEAD_ROWS_MIN;
  return 16 + nb * (K + 2) * 4;
}

extern "C" int dlrm_b200_head_fused(const float* h, int64_t ldh, const float* w, const float* bias,
                                    const float* target, const float* loss_ws, int64_t batch, int64_t K,
                                    int act_last, int act_prev, int loss_kind, float loss_threshold,
                                    float* p, float* loss_out, float* gz, float* dW, float* db,
                                    float* gprev, int64_t ld_gprev, void* gprev_hi, void* gprev_lo,
                                    int64_t ld_gprev_bf16, void* scratch, void* stream) {
  using namespace dlrm;
  if (batch <= 0 || K <= 0) return set_error("head_fused: batch=%lld K=%lld", (long long)batch, (long long)K);
  if (!h || !w || !bias || !p) return set_error("head_fused: NULL pointer");
  if (target && (!loss_out || !scratch)) return set_error("head_fused: loss_out/scratch required with a target");
  if (target && loss_kind == DLRM_LOSS_WBCE && !loss_ws) return set_error("head_fused: wbce needs loss_ws");
  if (dW && !target) return set_error("head_fused: backward requested without a target");
  HeadArgs a;
  a.h = h; a.ldh = ldh; a.w = w; a.bias = bias; a.target = target; a.ws = loss_ws;
  a.p = p; a.loss = loss_out; a.gz = gz; a.dW = dW; a.db = db;
  a.gprev = gprev; a.ld_gprev = ld_gprev;
  a.gprev_hi = static_cast<__nv_bfloat16*>(gprev_hi); a.gprev_lo = static_cast<__nv_bfloat16*>(gprev_lo);
  a.ld_gb = ld_gprev_bf16;
  a.counter = static_cast<unsigned*>(scratch);
  a.partial = scratch ? reinterpret_cast<float*>(static_cast<char*>(scratch) + 16) : nullptr;
  a.B = batch; a.K = (int)K; a.act_last = act_last; a.act_prev = act_prev; a.loss_kind = loss_kind;
  a.thr = loss_threshold;
  // 16 samples per CTA: 128 CTAs at batch 2048 (about one wave of the 132 SMs) instead of 64
  const int rows = get_tunable(TUNE_HEAD_ROWS) == 32 ? 32 : 16;
  const long long nb = (batch + rows - 1) / rows;
  if (rows == 32) (void)launch_chain(head_kernel<32>, dim3((unsigned)nb), dim3(256), 0, static_cast<cudaStream_t>(stream), a);
  else (void)launch_chain(head_kernel<16>, dim3((unsigned)nb), dim3(256), 0, static_cast<cudaStream_t>(stream), a);
  DLRM_CHECK_LAUNCH("head_kernel");
  return 0;
}
