// Kernels and GEMM helpers shared by the distributional (C51) twin-critic updates: fastsac.cu and fasttd3.cu.  Dual build like them
// (dual_build.cuh): one thread = one row / element, no shared memory, warp primitives or barriers.
//   [s | a] concatenation and the action-column gather of the critics' input gradients, row pitch `ld` >= obs + act (a padded pitch
//   lets the layer-1 products take a TMA descriptor on the tensor engine);
//   C51 projection of the target distributions, cross-entropy rows, expected values and their gradients, min / max of a row vector;
//   torch.optim.AdamW with the gradient sum of squares (clip_grad_norm_), polyak averaging;
//   torch Linear forward / input gradient / weight gradient through aux_gemm (SIMT, or the wgmma engine where it covers the product).
#pragma once
#include "flat_ops.cuh"

namespace rlx {
namespace c51 {
using namespace rlx::flat;

constexpr int kWgradRows = 1024;   // rows per split of the weight-gradient GEMMs (the splits are summed by reduce_parts_kernel)

#define C51_TRY(expr) do { int _rc = (expr); if (_rc) return _rc; } while (0)

// XA[r, :O+Ad] = [X | A] with row pitch ld (columns >= O + Ad are not written).  thread = element
static __global__ void concat_kernel(const float* __restrict__ X, const float* __restrict__ A, long long n, int O, int Ad, int ld, float* __restrict__ XA) {
  const long long id = gtid();
  const int W = O + Ad;
  if (id >= n * W) return;
  const long long r = id / W;
  const int k = (int)(id % W);
  XA[r * ld + k] = k < O ? X[r * O + k] : A[r * Ad + (k - O)];
}
// dAct[r, a] = dXA0[r, O + a] + dXA1[r, O + a]: the action columns of the two critics' input gradients (row pitch ld).  thread = element
static __global__ void action_grad_kernel(const float* __restrict__ dXA0, const float* __restrict__ dXA1, long long n, int O, int A, int ld,
                                          float* __restrict__ dAct) {
  const long long id = gtid();
  if (id >= n * A) return;
  const long long r = id / A;
  const int a = (int)(id % A);
  dAct[id] = dXA0[r * ld + O + a] + dXA1[r * ld + O + a];
}
// expected value of softmax(logits) on the support; optionally the gradient of (-coef * value) wrt the logits.  thread = row
static __global__ void expect_rows_kernel(const float* __restrict__ logits, long long n, int K, float v_min, float v_max, float* __restrict__ value,
                                          float coef, float* __restrict__ dlogits) {
  const long long r = gtid();
  if (r >= n) return;
  const float* l = logits + r * K;
  float mx = l[0];
  for (int k = 1; k < K; ++k) mx = fmaxf(mx, l[k]);
  float den = 0.f;
  for (int k = 0; k < K; ++k) den += expf(l[k] - mx);
  const float dz = (v_max - v_min) / (float)(K - 1);
  float v = 0.f;
  for (int k = 0; k < K; ++k) v += expf(l[k] - mx) / den * (v_min + dz * (float)k);
  value[r] = v;
  if (dlogits)
    for (int k = 0; k < K; ++k) {
      const float p = expf(l[k] - mx) / den;
      dlogits[r * K + k] = coef * p * ((v_min + dz * (float)k) - v);
    }
}
// gradient of -mean(q) wrt one critic's logits, q = (v1 + v2) / 2 or min(v1, v2) (ties split evenly like torch.minimum).  thread = row
static __global__ void value_grad_rows_kernel(const float* __restrict__ logits, const float* __restrict__ v_self, const float* __restrict__ v_other,
                                              long long n, int K, float v_min, float v_max, int clipped, float inv_n, float* __restrict__ dlogits) {
  const long long r = gtid();
  if (r >= n) return;
  const float vs = v_self[r], vo = v_other[r];
  const float coef = clipped ? (vs < vo ? 1.f : (vs == vo ? 0.5f : 0.f)) : 0.5f;
  const float* l = logits + r * K;
  float mx = l[0];
  for (int k = 1; k < K; ++k) mx = fmaxf(mx, l[k]);
  float den = 0.f;
  for (int k = 0; k < K; ++k) den += expf(l[k] - mx);
  const float dz = (v_max - v_min) / (float)(K - 1);
  for (int k = 0; k < K; ++k) dlogits[r * K + k] = -coef * inv_n * (expf(l[k] - mx) / den) * ((v_min + dz * (float)k) - vs);
}
static __global__ void combine_values_kernel(const float* __restrict__ v1, const float* __restrict__ v2, long long n, int clipped, float* __restrict__ out) {
  const long long r = gtid();
  if (r >= n) return;
  out[r] = clipped ? fminf(v1[r], v2[r]) : (v1[r] + v2[r]) / 2.f;
}
// C51 target of one row (fastsac.py:146-186, fasttd3.py:145-197): both target distributions are projected with the same bins.  The return is
// r - discount * exp(log_alpha) * next_logp, the entropy-adjusted one of FastSAC; a zero next_logp row gives FastTD3's plain r exactly.
// thread = row
static __global__ void c51_project_kernel(const float* __restrict__ tl1, const float* __restrict__ tl2, const float* __restrict__ rewards,
                                          const float* __restrict__ dones, const float* __restrict__ truncs, const float* __restrict__ eff,
                                          const float* __restrict__ next_logp, const float* __restrict__ log_alpha, long long n, int K, float gamma,
                                          float v_min, float v_max, int clipped, float* __restrict__ proj1, float* __restrict__ proj2,
                                          float* __restrict__ q1_next_value) {
  const long long r = gtid();
  if (r >= n) return;
  const float dz = (v_max - v_min) / (float)(K - 1);
  const float bootstrap = 1.f - dones[r] * (1.f - truncs[r]);
  const float discount = powf(gamma, eff[r]) * bootstrap;
  const float adj = rewards[r] - discount * expf(log_alpha[0]) * next_logp[r];
  float m1 = tl1[r * K], m2 = tl2[r * K];
  for (int k = 1; k < K; ++k) { m1 = fmaxf(m1, tl1[r * K + k]); m2 = fmaxf(m2, tl2[r * K + k]); }
  float d1 = 0.f, d2 = 0.f;
  for (int k = 0; k < K; ++k) { d1 += expf(tl1[r * K + k] - m1); d2 += expf(tl2[r * K + k] - m2); }
  for (int k = 0; k < K; ++k) { proj1[r * K + k] = 0.f; proj2[r * K + k] = 0.f; }
  for (int k = 0; k < K; ++k) {
    const float z = fminf(fmaxf(adj + discount * (v_min + dz * (float)k), v_min), v_max);
    const float b = (z - v_min) / dz;
    int lo = (int)floorf(b), up = (int)ceilf(b);
    if (lo == up) {  // b on a bin: move one neighbour so that the two weights still sum to 1 (:155-160)
      if (lo > 0) lo -= 1; else up += 1;
    }
    const float wl = (float)up - b, wu = b - (float)lo;
    const float p1 = expf(tl1[r * K + k] - m1) / d1, p2 = expf(tl2[r * K + k] - m2) / d2;
    proj1[r * K + lo] += p1 * wl; proj1[r * K + up] += p1 * wu;
    proj2[r * K + lo] += p2 * wl; proj2[r * K + up] += p2 * wu;
  }
  float v = 0.f, v2 = 0.f;
  for (int k = 0; k < K; ++k) { v += proj1[r * K + k] * (v_min + dz * (float)k); v2 += proj2[r * K + k] * (v_min + dz * (float)k); }
  q1_next_value[r] = v;
  if (clipped) {  // torch.where(q1_next < q2_next, proj1, proj2) for BOTH critics (fastsac.py:179-182)
    for (int k = 0; k < K; ++k) {
      const float sel = (v < v2) ? proj1[r * K + k] : proj2[r * K + k];
      proj1[r * K + k] = sel;
      proj2[r * K + k] = sel;
    }
  }
}
// cross-entropy of one row against its projected target: loss = -sum_k proj_k log_softmax(logits)_k; dlogits = (softmax * sum(proj) - proj) / n
static __global__ void ce_rows_kernel(const float* __restrict__ logits, const float* __restrict__ proj, long long n, int K, float inv_n,
                                      float* __restrict__ loss_row, float* __restrict__ dlogits) {
  const long long r = gtid();
  if (r >= n) return;
  const float* l = logits + r * K;
  float mx = l[0];
  for (int k = 1; k < K; ++k) mx = fmaxf(mx, l[k]);
  float den = 0.f;
  for (int k = 0; k < K; ++k) den += expf(l[k] - mx);
  const float lse = mx + logf(den);
  float loss = 0.f, ps = 0.f;
  for (int k = 0; k < K; ++k) { loss -= proj[r * K + k] * (l[k] - lse); ps += proj[r * K + k]; }
  for (int k = 0; k < K; ++k) dlogits[r * K + k] = (expf(l[k] - lse) * ps - proj[r * K + k]) * inv_n;
  loss_row[r] = loss;
}
// rows -> (min, max) per chunk, then one thread finishes.
static __global__ void minmax_partial_kernel(const float* __restrict__ x, long long n, float* __restrict__ part) {
  const long long c = gtid();
  const long long nchunk = (n + kColChunk - 1) / kColChunk;
  if (c >= nchunk) return;
  const long long r1 = c * kColChunk + kColChunk < n ? c * kColChunk + kColChunk : n;
  float lo = x[c * kColChunk], hi = lo;
  for (long long r = c * kColChunk + 1; r < r1; ++r) { lo = fminf(lo, x[r]); hi = fmaxf(hi, x[r]); }
  part[2 * c] = lo;
  part[2 * c + 1] = hi;
}
// torch.optim.AdamW (single tensor): p *= 1 - lr wd; m, v updates; p -= lr / bc1 * m / (sqrt(v) / sqrt(bc2) + eps).  Optional clip_grad_norm_.
static __global__ void adamw_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, long long n,
                                    const float* __restrict__ lr, const long long* __restrict__ step, const float* __restrict__ norm, float max_norm,
                                    float wd, float b1, float b2, float eps) {
  const long long i = gtid();
  if (i >= n) return;
  float gi = g[i];
  if (max_norm >= 0.f) gi *= fminf(1.f, max_norm / (norm[0] + 1e-6f));
  const float t = (float)step[0];
  float pi = p[i] * (1.f - lr[0] * wd);
  const float mi = b1 * m[i] + (1.f - b1) * gi;
  const float vi = b2 * v[i] + (1.f - b2) * gi * gi;
  m[i] = mi;
  v[i] = vi;
  const float bc1 = 1.f - powf(b1, t), bc2 = 1.f - powf(b2, t);
  pi -= lr[0] / bc1 * mi / (sqrtf(vi) / sqrtf(bc2) + eps);
  p[i] = pi;
}
static __global__ void polyak_kernel(float* __restrict__ tgt, const float* __restrict__ src, long long n, float tau) {
  const long long i = gtid();
  if (i >= n) return;
  tgt[i] = tgt[i] * (1.f - tau) + tau * src[i];
}

// gradient norm (metrics / clipping), step counter += 1, then AdamW over n parameters.  max_norm < 0: no clipping
static int adamw_step(float* p, const float* g, float* m, float* v, long long n, const float* lr, long long* step, float max_norm, float wd, float b1,
                      float b2, float eps, float* norm_out, float* scratch, cudaStream_t st) {
  const long long nchunk = ceil_div(n, 1024);
  RLX_FLAT_LAUNCH(sumsq_partial_kernel, nchunk, st, g, n, scratch);
  RLX_FLAT_LAUNCH(sumsq_final_kernel, 1, st, scratch, nchunk, norm_out, step);
  RLX_FLAT_LAUNCH(adamw_kernel, n, st, p, g, m, v, n, lr, (const long long*)step, norm_out, max_norm, wd, b1, b2, eps);
  return RLX_OK;
}

// ------------------------------------------------------------------------------------------------------- GEMM helpers
static __global__ void copy_kernel(const float* __restrict__ src, long long n, float* __restrict__ dst) {
  const long long i = gtid();
  if (i < n) dst[i] = src[i];
}
// *out = a network's parameter block as the GEMMs read it: P itself when its base is 16-byte aligned, else a copy of its n floats in `slot`
// (16-byte aligned workspace).  The critics sit back to back in q_params, critic 2 at q_params + nq, and every segment is a multiple of 4
// floats except the last bias (nr_atoms): with 101 atoms nq % 4 == 1, no weight of critic 2 can be a TMA operand in place, and aux_gemm would
// run every GEMM that reads one on the SIMT engine.  The copy holds the same values, so the results do not depend on which one is read.
static int aligned_params(const float* P, long long n, float* slot, const float** out, cudaStream_t st) {
  *out = P;
  if (((uintptr_t)P & 15) == 0) return RLX_OK;
  RLX_FLAT_LAUNCH(copy_kernel, n, st, P, n, slot);
  *out = slot;
  return RLX_OK;
}
// torch Linear: Y[r, o] = epi(sum_i X[r, i] W[o, i] + b[o]), W row pitch ldw (= in unless a padded copy)
template <int EPI = EPI_BIAS>
static int lin_fwd(const float* X, int ldx, const float* W, int in, int out, const float* b, float* Y, int ldy, long long n, cudaStream_t st,
                   int ldw = 0) {
  GemmP g{};
  g.A = X; g.B = W; g.C = Y; g.bias = b;
  g.M = (int)n; g.N = out; g.K = in; g.lda = ldx; g.ldb = ldw > 0 ? ldw : in; g.ldc = ldy;
  g.splits = 1; g.kchunk = (int)(ceil_div(in, 8) * 8);
  return aux_gemm<true, true, EPI>(g, 1, st, KC_GEMM_FWD, n, out);
}
// dX[r, i] = sum_o dY[r, o] W[o, i]; EPI_DRELU: times (H[r, i] > 0), H the input activation (row pitch ldx) of the layer
template <int EPI = EPI_NONE>
static int lin_bwd_input(const float* dY, int ldy, const float* W, int in, int out, float* dX, int ldx, long long n, cudaStream_t st,
                         const float* H = nullptr, int ldw = 0) {
  GemmP g{};
  g.A = dY; g.B = W; g.C = dX; g.aux = H; g.ldaux = ldx;
  g.M = (int)n; g.N = in; g.K = out; g.lda = ldy; g.ldb = ldw > 0 ? ldw : in; g.ldc = ldx;
  g.splits = 1; g.kchunk = (int)(ceil_div(out, 8) * 8);
  return aux_gemm<true, false, EPI>(g, 1, st, KC_GEMM_DX, n, out);
}
// dW[o, i] = sum_r dY[r, o] X[r, i], split over rows
static int lin_bwd_weight(const float* dY, int ldy, const float* X, int ldx, int in, int out, long long n, float* part, float* dW, cudaStream_t st) {
  const int splits = (int)ceil_div(n, kWgradRows);
  GemmP g{};
  g.A = dY; g.B = X; g.C = part;
  g.M = out; g.N = in; g.K = (int)n; g.lda = ldy; g.ldb = ldx; g.ldc = in;
  g.splits = splits; g.kchunk = kWgradRows; g.sSplitC = (long long)in * out;
  int rc = aux_gemm<false, false, EPI_NONE>(g, 1, st, KC_GEMM_DW, n, n);
  if (rc) return rc;
  RLX_FLAT_LAUNCH(reduce_parts_kernel, (long long)in * out, st, part, (long long)splits, (long long)in * out, 1.f, 0.f, dW);
  return RLX_OK;
}

}  // namespace c51
}  // namespace rlx
