// Fused multi-tensor Adam / AdamW (SURVEY.md 8f row 3): the reference steps torch.optim.AdamW over five parameter
// groups (gaustudio/pipelines/optimizers/base.py:19-20, configs/vanilla.yaml:30-46).  One launch updates every
// group: per element 16 B read (param, grad, exp_avg, exp_avg_sq) and 12-16 B written (the three states, plus the
// zeroed gradient when zero_grad is fused in) -- a pure HBM stream, float4 wide where the tensors allow it.
// Arithmetic follows torch's single-tensor Adam: p *= 1 - lr*wd (AdamW) | g += wd*p (Adam); m = m + (g-m)(1-b1);
// v = v*b2 + (1-b2) g g; p -= (lr/bc1) * m / (sqrt(v)/sqrt(bc2) + eps).
#include "../../include/gsr.h"
#include "gsr_internal.cuh"
#include <cmath>

namespace gsr {

struct AdamTable {
  float* p[GSR_ADAM_MAX_GROUPS]; float* g[GSR_ADAM_MAX_GROUPS]; float* m[GSR_ADAM_MAX_GROUPS]; float* v[GSR_ADAM_MAX_GROUPS];
  float* g2[GSR_ADAM_MAX_GROUPS];  // optional second gradient tensor per group (nullptr: none)
  long long n[GSR_ADAM_MAX_GROUPS];
  float step_size[GSR_ADAM_MAX_GROUPS], decay[GSR_ADAM_MAX_GROUPS];  // lr / bc1; AdamW: 1 - lr*wd, Adam: wd
  unsigned first_block[GSR_ADAM_MAX_GROUPS + 1];
  unsigned char vec4[GSR_ADAM_MAX_GROUPS];
  int groups;
};
constexpr int ADAM_THREADS = 256, ADAM_PER_BLOCK = ADAM_THREADS * 4;

__device__ __forceinline__ void adam_one(float& p, float& g, float& m, float& v, float step_size, float decay, float b1c,
                                         float b2, float b2c, float inv_bc2s, float eps, float gscale, int decoupled) {
  float grad = g * gscale;
  if (decoupled) p = p * decay; else grad = grad + decay * p;
  m = m + (grad - m) * b1c;
  v = v * b2 + b2c * grad * grad;
  const float denom = sqrtf(v) * inv_bc2s + eps;
  p = p - step_size * (m / denom);
}

__global__ void __launch_bounds__(ADAM_THREADS) k_adam(const __grid_constant__ AdamTable t, float b1c, float b2, float b2c,
                                                       float inv_bc2s, float eps, float gscale, int decoupled, int zero_grad) {
  int gi = 0;
  while (gi + 1 < t.groups && blockIdx.x >= t.first_block[gi + 1]) gi++;
  const long long base = (long long)(blockIdx.x - t.first_block[gi]) * ADAM_PER_BLOCK;
  float* __restrict__ P = t.p[gi]; float* __restrict__ G = t.g[gi]; float* __restrict__ M = t.m[gi]; float* __restrict__ V = t.v[gi];
  float* __restrict__ G2 = t.g2[gi];
  const long long n = t.n[gi];
  const float ss = t.step_size[gi], dc = t.decay[gi];
  const long long i = base + threadIdx.x * 4;
  if (t.vec4[gi] && i + 3 < n) {
    float4 p = *reinterpret_cast<float4*>(P + i), g = *reinterpret_cast<float4*>(G + i);
    float4 m = *reinterpret_cast<float4*>(M + i), v = *reinterpret_cast<float4*>(V + i);
    if (G2) {
      const float4 h = *reinterpret_cast<float4*>(G2 + i);
      g.x += h.x; g.y += h.y; g.z += h.z; g.w += h.w;
      if (zero_grad) *reinterpret_cast<float4*>(G2 + i) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    adam_one(p.x, g.x, m.x, v.x, ss, dc, b1c, b2, b2c, inv_bc2s, eps, gscale, decoupled);
    adam_one(p.y, g.y, m.y, v.y, ss, dc, b1c, b2, b2c, inv_bc2s, eps, gscale, decoupled);
    adam_one(p.z, g.z, m.z, v.z, ss, dc, b1c, b2, b2c, inv_bc2s, eps, gscale, decoupled);
    adam_one(p.w, g.w, m.w, v.w, ss, dc, b1c, b2, b2c, inv_bc2s, eps, gscale, decoupled);
    *reinterpret_cast<float4*>(P + i) = p; *reinterpret_cast<float4*>(M + i) = m; *reinterpret_cast<float4*>(V + i) = v;
    if (zero_grad) *reinterpret_cast<float4*>(G + i) = make_float4(0.f, 0.f, 0.f, 0.f);
  } else {
    for (long long k = i; k < n && k < i + 4; k++) {
      float p = P[k], g = G[k], m = M[k], v = V[k];
      if (G2) { g += G2[k]; if (zero_grad) G2[k] = 0.f; }
      adam_one(p, g, m, v, ss, dc, b1c, b2, b2c, inv_bc2s, eps, gscale, decoupled);
      P[k] = p; M[k] = m; V[k] = v;
      if (zero_grad) G[k] = 0.f;
    }
  }
}

}  // namespace gsr

using namespace gsr;

extern "C" int gsr_adam_step(int n_groups, const gsr_adam_group* groups, double beta1, double beta2, double eps,
                             int64_t step, int decoupled, float grad_scale, int zero_grad, void* stream) {
  if (n_groups <= 0) return 0;
  if (!groups || n_groups > GSR_ADAM_MAX_GROUPS) return fail("gsr_adam_step", "1..16 groups");
  if (step < 1) return fail("gsr_adam_step", "step counts from 1");
  for (int i = 0; i < n_groups; i++)
    if (groups[i].numel > 0 && (!groups[i].param || !groups[i].grad || !groups[i].exp_avg || !groups[i].exp_avg_sq))
      return fail("gsr_adam_step", "null tensor in a group");
  AdamTable t;
  const double bc1 = 1.0 - std::pow(beta1, (double)step), bc2 = 1.0 - std::pow(beta2, (double)step);
  unsigned nb = 0;
  int k = 0;
  for (int i = 0; i < n_groups; i++) {
    const gsr_adam_group& q = groups[i];
    if (q.numel <= 0) continue;
    t.p[k] = q.param; t.g[k] = q.grad; t.m[k] = q.exp_avg; t.v[k] = q.exp_avg_sq; t.n[k] = q.numel;
    t.step_size[k] = (float)((double)q.lr / bc1);
    t.decay[k] = decoupled ? (float)(1.0 - (double)q.lr * (double)q.weight_decay) : q.weight_decay;
    t.g2[k] = q.grad2;
    t.vec4[k] = ((reinterpret_cast<size_t>(q.param) | reinterpret_cast<size_t>(q.grad) | reinterpret_cast<size_t>(q.exp_avg) |
                  reinterpret_cast<size_t>(q.exp_avg_sq) | reinterpret_cast<size_t>(q.grad2)) & 15) == 0;
    t.first_block[k] = nb;
    nb += (unsigned)((q.numel + ADAM_PER_BLOCK - 1) / ADAM_PER_BLOCK);
    k++;
  }
  t.first_block[k] = nb;
  t.groups = k;
  if (k)  // every group empty: nothing to launch
    k_adam<<<nb, ADAM_THREADS, 0, (cudaStream_t)stream>>>(t, (float)(1.0 - beta1), (float)beta2, (float)(1.0 - beta2),
                                                           (float)(1.0 / std::sqrt(bc2)), (float)eps, grad_scale,
                                                           decoupled, zero_grad);
  return launched("gsr_adam_step");
}
