// Loss forward + backward through (loss, clamp, last activation), and the dense-parameter
// optimizer.  Replaces loss_fn_wrap (dlrm_s_pytorch.py:148-156; nn.MSELoss / nn.BCELoss(mean),
// wbce), the clamp of sequential_forward (:607-610), their autograd, and the dense branch of
// optimizer.step() (torch.optim.SGD / optim/rwsadagrad.py:145-148).
#include "common.cuh"

namespace dlrm {

__global__ void __launch_bounds__(1024) loss_kernel(const float* __restrict__ p,
                                                    const float* __restrict__ target,
                                                    const float* __restrict__ ws, long long n,
                                                    int kind, float thr, int last_act,
                                                    float* __restrict__ loss_out,
                                                    float* __restrict__ gz) {
  __shared__ float red[32];
  const bool clampd = thr > 0.f && thr < 1.f;
  const float inv_n = 1.0f / (float)n;
  float sum = 0.f;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) {
    const float pi = p[i], t = target[i];
    const float z = clampd ? fminf(fmaxf(pi, thr), 1.0f - thr) : pi;
    float per, g;
    if (kind == DLRM_LOSS_MSE) {
      const float d = z - t;
      per = d * d;
      g = 2.0f * d * inv_n;
    } else {
      // ATen binary_cross_entropy: log terms clamped at -100; backward divides by max((1-z)z, 1e-12)
      const float lz = fmaxf(logf(z), -100.0f);
      const float l1z = fmaxf(logf(1.0f - z), -100.0f);
      per = (t - 1.0f) * l1z - t * lz;
      g = (z - t) / fmaxf((1.0f - z) * z, 1e-12f);
      if (kind == DLRM_LOSS_WBCE) {
        const float w = ws[(int)t];
        per *= w;
        g *= w;
      }
      g *= inv_n;
    }
    sum += per;
    if (gz) {
      if (clampd && !(pi >= thr && pi <= 1.0f - thr)) g = 0.f;
      if (last_act == DLRM_ACT_SIGMOID) g *= (1.0f - pi) * pi;
      else if (last_act == DLRM_ACT_RELU) g = pi > 0.f ? g : 0.f;
      gz[i] = g;
    }
  }
  sum = warp_sum(sum);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = (threadIdx.x < (blockDim.x >> 5)) ? red[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0) *loss_out = v * inv_n;
  }
}

__global__ void __launch_bounds__(256) dense_update_kernel(float* __restrict__ p,
                                                           const float* __restrict__ g,
                                                           float* __restrict__ s, long long n,
                                                           int opt, float lr, const float* lr_dev,
                                                           float eps) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (lr_dev) lr = *lr_dev;
  const float gi = g[i];
  if (opt == DLRM_OPT_RWSADAGRAD) {
    const float si = fmaf(gi, gi, s[i]);
    s[i] = si;
    p[i] = fmaf(-lr, gi / (sqrtf(si) + eps), p[i]);
  } else {
    p[i] = fmaf(-lr, gi, p[i]);
  }
}

__global__ void __launch_bounds__(256) act_bwd_kernel(const float* __restrict__ gy,
                                                      const float* __restrict__ y,
                                                      float* __restrict__ gz, long long n, int act,
                                                      float thr) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float g = gy[i];
  const float yi = y[i];
  if (thr > 0.f && thr < 1.f && !(yi >= thr && yi <= 1.0f - thr)) g = 0.f;  // clamp backward
  if (act == DLRM_ACT_SIGMOID) g *= (1.0f - yi) * yi;
  else if (act == DLRM_ACT_RELU) g = yi > 0.f ? g : 0.f;
  gz[i] = g;
}

}  // namespace dlrm

extern "C" int dlrm_b200_act_bwd(const float* gy, const float* y, float* gz, int64_t n, int act,
                                 float clamp_threshold, void* stream) {
  using namespace dlrm;
  if (n <= 0) return 0;
  if (!gy || !y || !gz) return set_error("act_bwd: NULL pointer");
  act_bwd_kernel<<<(unsigned)((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(gy, y, gz, n, act, clamp_threshold);
  DLRM_CHECK_LAUNCH("act_bwd_kernel");
  return 0;
}

extern "C" int dlrm_b200_loss_fwd_bwd(const float* p, const float* target, const float* loss_ws,
                                      int64_t n, int loss_kind, float loss_threshold, int last_act,
                                      float* loss_out, float* gz, float* scratch, void* stream) {
  using namespace dlrm;
  (void)scratch;
  if (n <= 0) return set_error("loss_fwd_bwd: n=%lld", (long long)n);
  if (loss_kind < DLRM_LOSS_MSE || loss_kind > DLRM_LOSS_WBCE)
    return set_error("loss_fwd_bwd: loss_kind=%d", loss_kind);
  if (loss_kind == DLRM_LOSS_WBCE && !loss_ws) return set_error("loss_fwd_bwd: wbce needs loss_ws");
  if (!p || !target || !loss_out) return set_error("loss_fwd_bwd: NULL pointer");
  loss_kernel<<<1, 1024, 0, static_cast<cudaStream_t>(stream)>>>(p, target, loss_ws, n, loss_kind,
                                                                 loss_threshold, last_act, loss_out, gz);
  DLRM_CHECK_LAUNCH("loss_kernel");
  return 0;
}

static int dense_update_impl(float* param, const float* grad, float* state, int64_t n, int optimizer, float lr,
                             const float* lr_dev, float eps, void* stream) {
  using namespace dlrm;
  if (n == 0) return 0;
  if (optimizer == DLRM_OPT_ADAGRAD) optimizer = DLRM_OPT_RWSADAGRAD;   // the dense branches are the same algorithm
  if (optimizer != DLRM_OPT_SGD && optimizer != DLRM_OPT_RWSADAGRAD)
    return set_error("dense_update: optimizer=%d", optimizer);
  if (!param || !grad || (optimizer == DLRM_OPT_RWSADAGRAD && !state))
    return set_error("dense_update: NULL pointer");
  dense_update_kernel<<<(unsigned)((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      param, grad, state, n, optimizer, lr, lr_dev, eps);
  DLRM_CHECK_LAUNCH("dense_update_kernel");
  return 0;
}

extern "C" int dlrm_b200_dense_update(float* param, const float* grad, float* state, int64_t n,
                                      int optimizer, float lr, float eps, void* stream) {
  return dense_update_impl(param, grad, state, n, optimizer, lr, nullptr, eps, stream);
}

extern "C" int dlrm_b200_dense_update_lr_dev(float* param, const float* grad, float* state, int64_t n,
                                             int optimizer, float lr, const float* lr_dev, float eps, void* stream) {
  return dense_update_impl(param, grad, state, n, optimizer, lr, lr_dev, eps, stream);
}
