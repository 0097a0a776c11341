// FastSAC update (SURVEY.md §8 f4; rl_x/algorithms/fastsac/pytorch): distributional (C51) twin critics, tanh-Gaussian actor, entropy
// coefficient, AdamW, polyak targets, observation normaliser.  Entry points and flat layouts: include/rlx_b200.h.
// Dual build (dual_build.cuh): the host emulation of this file is checked against oracle/fastsac_oracle.py (pinned to the executed
// reference) in tests/test_fastsac_emulation.py.  v1: exact-fp32 SIMT GEMMs, flat one-thread-per-row / per-element kernels.
#include "c51_ops.cuh"

namespace rlx {
namespace fsac {
using namespace rlx::flat;
using namespace rlx::c51;

constexpr int kPW[3] = {512, 256, 128};   // policy torso widths (policy.py:36-46)
constexpr int kQW[3] = {768, 384, 192};   // Q torso widths (q_network.py:24-34)
constexpr float kLnEps = 1e-5f;           // torch.nn.LayerNorm default
constexpr float kHalfLog2Pi = 0.9189385332046727f;

struct Layout {
  long long p[RLX_FASTSAC_POLICY_NSEG + 1], q[RLX_FASTSAC_Q_NSEG + 1];
};
static Layout make_layout(const rlx_fastsac_dims& d) {
  Layout l;
  long long o = 0;
  int in = d.obs_dim, s = 0;
  for (int k = 0; k < 3; ++k) {
    const long long sz[4] = {(long long)kPW[k] * in, kPW[k], kPW[k], kPW[k]};
    for (int j = 0; j < 4; ++j) { l.p[s++] = o; o += sz[j]; }
    in = kPW[k];
  }
  const long long hs[4] = {(long long)d.act_dim * 128, d.act_dim, (long long)d.act_dim * 128, d.act_dim};
  for (int j = 0; j < 4; ++j) { l.p[s++] = o; o += hs[j]; }
  l.p[s] = o;
  o = 0; s = 0; in = d.obs_dim + d.act_dim;
  for (int k = 0; k < 3; ++k) {
    const long long sz[4] = {(long long)kQW[k] * in, kQW[k], kQW[k], kQW[k]};
    for (int j = 0; j < 4; ++j) { l.q[s++] = o; o += sz[j]; }
    in = kQW[k];
  }
  l.q[s++] = o; o += (long long)d.nr_atoms * 192;
  l.q[s++] = o; o += d.nr_atoms;
  l.q[s] = o;
  return l;
}
static bool dims_ok(const rlx_fastsac_dims& d) { return d.obs_dim > 0 && d.act_dim > 0 && d.act_dim <= 64 && d.nr_atoms >= 2 && d.nr_atoms <= 1024; }

// one torso's activations: pre-LayerNorm Z, post-SiLU Y, per-row (mean, rstd)
struct Acts { float *Z[3], *Y[3], *S[3]; };
struct Ws {
  size_t pZ[3], pY[3], pS[3], qZ[2][3], qY[2][3], qS[2][3], XA, Mean, LsRaw, Act, Logp, Logits[2], Proj[2], dLogits, dZ, dY, dXA, dXA2, dAct, dMean, dLs,
      RowA, RowB, Small, QP[2], Part, Col, total;
};
static Ws plan(const rlx_fastsac_dims& d, long long n_) {
  const size_t n = (size_t)n_, O = d.obs_dim, A = d.act_dim, K = d.nr_atoms;
  Ws w;
  size_t o = 0;
  auto take = [&](size_t& f, size_t cnt) { f = o; o += align_up(cnt, 64); };
  for (int k = 0; k < 3; ++k) { take(w.pZ[k], n * kPW[k]); take(w.pY[k], n * kPW[k]); take(w.pS[k], n * 2); }
  for (int q = 0; q < 2; ++q)
    for (int k = 0; k < 3; ++k) { take(w.qZ[q][k], n * kQW[k]); take(w.qY[q][k], n * kQW[k]); take(w.qS[q][k], n * 2); }
  take(w.XA, n * (O + A)); take(w.Mean, n * A); take(w.LsRaw, n * A); take(w.Act, n * A); take(w.Logp, n);
  for (int q = 0; q < 2; ++q) { take(w.Logits[q], n * K); take(w.Proj[q], n * K); }
  take(w.dLogits, n * K); take(w.dZ, n * 768); take(w.dY, n * 768); take(w.dXA, n * (O + A)); take(w.dXA2, n * (O + A)); take(w.dAct, n * A); take(w.dMean, n * A);
  take(w.dLs, n * A); take(w.RowA, n * 4); take(w.RowB, n * 4); take(w.Small, 64);
  const size_t nq = (size_t)make_layout(d).q[RLX_FASTSAC_Q_NSEG];
  take(w.QP[0], nq); take(w.QP[1], nq);   // aligned_params: a critic's parameter block when its base is not 16-byte aligned
  const size_t splits = (size_t)ceil_div((long long)n, kWgradRows);
  size_t biggest = std::max<size_t>((size_t)768 * (O + A), (size_t)768 * 384);
  biggest = std::max<size_t>(biggest, std::max<size_t>((size_t)512 * O, (size_t)K * 192));
  biggest = std::max<size_t>(biggest, (size_t)512 * 256);
  take(w.Part, splits * biggest);
  const size_t chunks = (size_t)ceil_div((long long)n, kColChunk);
  take(w.Col, chunks * 2 * std::max<size_t>(768, std::max<size_t>(K, 8)));
  w.total = o * sizeof(float);
  return w;
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

// ---------------------------------------------------------------------------------------------------------- kernels
// y = SiLU(LayerNorm(z) * g + b), torch LayerNorm (biased variance around the mean, eps 1e-5).  thread = row
__global__ void ln_silu_fwd_kernel(const float* __restrict__ Z, long long R, int W, const float* __restrict__ g, const float* __restrict__ b,
                                   float* __restrict__ Y, float* __restrict__ stats) {
  const long long r = gtid();
  if (r >= R) return;
  const float* z = Z + r * W;
  float s = 0.f;
  for (int j = 0; j < W; ++j) s += z[j];
  const float mean = s / (float)W;
  float q = 0.f;
  for (int j = 0; j < W; ++j) { const float d = z[j] - mean; q += d * d; }
  const float rstd = 1.f / sqrtf(q / (float)W + kLnEps);
  for (int j = 0; j < W; ++j) {
    const float y = (z[j] - mean) * rstd * g[j] + b[j];
    Y[r * W + j] = y * sigmoidf_(y);
  }
  stats[2 * r] = mean;
  stats[2 * r + 1] = rstd;
}
__device__ __forceinline__ float dsilu(float y) { const float s = sigmoidf_(y); return s * (1.f + y * (1.f - s)); }

// dZ for Y = SiLU(LN(z)); dOut = dL/dY.  thread = row
__global__ void ln_silu_bwd_kernel(const float* __restrict__ dOut, const float* __restrict__ Z, long long R, int W, const float* __restrict__ g,
                                   const float* __restrict__ b, const float* __restrict__ stats, float* __restrict__ dZ) {
  const long long r = gtid();
  if (r >= R) return;
  const float mean = stats[2 * r], rstd = stats[2 * r + 1];
  float s1 = 0.f, s2 = 0.f;
  for (int j = 0; j < W; ++j) {
    const float xh = (Z[r * W + j] - mean) * rstd;
    const float dx = dOut[r * W + j] * dsilu(xh * g[j] + b[j]) * g[j];
    s1 += dx;
    s2 += dx * xh;
  }
  s1 /= (float)W;
  s2 /= (float)W;
  for (int j = 0; j < W; ++j) {
    const float xh = (Z[r * W + j] - mean) * rstd;
    const float dx = dOut[r * W + j] * dsilu(xh * g[j] + b[j]) * g[j];
    dZ[r * W + j] = rstd * (dx - s1 - xh * s2);
  }
}
// LayerNorm weight / bias gradient partials: thread = (row chunk, column)
__global__ void ln_silu_param_partial_kernel(const float* __restrict__ dOut, const float* __restrict__ Z, long long R, int W,
                                             const float* __restrict__ g, const float* __restrict__ b, const float* __restrict__ stats,
                                             float* __restrict__ part_g, float* __restrict__ part_b) {
  const long long id = gtid();
  const long long nchunk = (R + kColChunk - 1) / kColChunk;
  if (id >= nchunk * W) return;
  const long long ch = id / W;
  const int j = (int)(id % W);
  const long long r1 = ch * kColChunk + kColChunk < R ? ch * kColChunk + kColChunk : R;
  float sg = 0.f, sb = 0.f;
  for (long long r = ch * kColChunk; r < r1; ++r) {
    const float xh = (Z[r * W + j] - stats[2 * r]) * stats[2 * r + 1];
    const float dy = dOut[r * W + j] * dsilu(xh * g[j] + b[j]);
    sg += dy * xh;
    sb += dy;
  }
  part_g[id] = sg;
  part_b[id] = sb;
}
// policy head: tanh log-std squash, reparameterised sample, tanh action, log-prob with the squash / scale corrections (policy.py:55-75).
// noise == null: deterministic action tanh(mean) * scale.  thread = row
__global__ void squash_sample_kernel(const float* __restrict__ Mean, const float* __restrict__ LsRaw, const float* __restrict__ noise,
                                     const float* __restrict__ scale, long long n, int A, float lsmin, float lsmax, float* __restrict__ action,
                                     float* __restrict__ logp) {
  const long long r = gtid();
  if (r >= n) return;
  float lp = 0.f;
  for (int a = 0; a < A; ++a) {
    const float m = Mean[r * A + a];
    if (noise == nullptr) { action[r * A + a] = tanhf(m) * scale[a]; continue; }
    const float ls = lsmin + 0.5f * (lsmax - lsmin) * (tanhf(LsRaw[r * A + a]) + 1.f);
    const float sd = expf(ls);
    const float raw = m + sd * noise[r * A + a];
    const float th = tanhf(raw);
    action[r * A + a] = th * scale[a];
    const float dd = raw - m;
    lp += -(dd * dd) / (2.f * sd * sd) - ls - kHalfLog2Pi - logf((1.f - th * th) + 1e-6f) - logf(scale[a] + 1e-6f);
  }
  if (logp) logp[r] = lp;
}
// backward of the policy head for L = mean(alpha * logp - q): dAct = dL/d action (already scaled by 1/n), dlogp = alpha / n.  thread = row
__global__ void squash_sample_bwd_kernel(const float* __restrict__ Mean, const float* __restrict__ LsRaw, const float* __restrict__ noise,
                                         const float* __restrict__ scale, const float* __restrict__ dAct, const float* __restrict__ log_alpha,
                                         long long n, int A, float lsmin, float lsmax, float inv_n, float* __restrict__ dMean,
                                         float* __restrict__ dLs) {
  const long long r = gtid();
  if (r >= n) return;
  const float dlogp = expf(log_alpha[0]) * inv_n;
  for (int a = 0; a < A; ++a) {
    const float tl = tanhf(LsRaw[r * A + a]);
    const float ls = lsmin + 0.5f * (lsmax - lsmin) * (tl + 1.f);
    const float sd = expf(ls);
    const float eps = noise[r * A + a];
    const float th = tanhf(Mean[r * A + a] + sd * eps);
    const float one = 1.f - th * th;
    const float g_raw = dAct[r * A + a] * scale[a] * one + dlogp * (2.f * th * one / (one + 1e-6f));
    dMean[r * A + a] = g_raw;
    const float dls = g_raw * sd * eps - dlogp;
    dLs[r * A + a] = dls * 0.5f * (lsmax - lsmin) * (1.f - tl * tl);
  }
}
__global__ void add_inplace_kernel(float* __restrict__ x, const float* __restrict__ y, long long n) {
  const long long i = gtid();
  if (i < n) x[i] += y[i];
}
// critic metrics + the entropy-coefficient gradient (fastsac.py:228-236).  sums: [sum loss1, sum loss2, sum next_logp]
__global__ void critic_finish_kernel(const float* __restrict__ sums, const float* __restrict__ mm_part, long long nchunk, float n,
                                     const float* __restrict__ log_alpha, float target_entropy, float* __restrict__ alpha_grad,
                                     float* __restrict__ metrics) {
  if (gtid() != 0) return;
  float lo = mm_part[0], hi = mm_part[1];
  for (long long c = 1; c < nchunk; ++c) { lo = fminf(lo, mm_part[2 * c]); hi = fmaxf(hi, mm_part[2 * c + 1]); }
  const float ent_mean = -sums[2] / n;
  const float al = expf(log_alpha[0]);
  metrics[0] = sums[0] / n + sums[1] / n;             // q_loss
  metrics[1] = al * (ent_mean - target_entropy);       // entropy_loss = mean(alpha * (entropy - target))
  metrics[2] = lo;
  metrics[3] = hi;
  metrics[4] = ent_mean;
  alpha_grad[0] = al * (ent_mean - target_entropy);    // d/d log_alpha of the mean above
  metrics[6] = alpha_grad[0] * alpha_grad[0];           // entropy_grad_norm as the reference logs it (norm(2) ** 2)
}
__global__ void policy_finish_kernel(const float* __restrict__ sums, float n, const float* __restrict__ log_alpha, float* __restrict__ metrics) {
  if (gtid() != 0) return;
  const float al = expf(log_alpha[0]);
  metrics[0] = al * sums[0] / n - sums[1] / n;  // mean(alpha * logp - q), q = (q1 + q2) / 2 or min(q1, q2)
  metrics[1] = al;
}
// observation normaliser: batch column mean / biased variance from partials, Chan's update (observation_normalizer.py:28-47).  thread = column
__global__ void normalizer_update_kernel(const float* __restrict__ col_sum, const float* __restrict__ col_sq, long long n, int O,
                                         float* __restrict__ mean, float* __restrict__ var, float* __restrict__ stdv,
                                         const long long* __restrict__ count) {
  const long long j = gtid();
  if (j >= O) return;
  const float bc = (float)n, c0 = (float)count[0], c1 = c0 + bc;
  const float bm = col_sum[j] / bc;
  const float bv = col_sq[j] / bc;  // sum of squared deviations from the batch mean / n
  const float delta = bm - mean[j];
  const float nm = mean[j] + delta * bc / c1;
  const float delta2 = bm - nm;
  const float m2 = var[j] * c0 + bv * bc + delta2 * delta2 * c0 * bc / c1;
  mean[j] = nm;
  var[j] = m2 / c1;
  stdv[j] = sqrtf(m2 / c1);
}
__global__ void centered_sq_cols_kernel(const float* __restrict__ x, long long n, int O, const float* __restrict__ col_sum, float* __restrict__ out) {
  const long long id = gtid();
  if (id >= n * O) return;
  const float d = x[id] - col_sum[id % O] / (float)n;
  out[id] = d * d;
}
__global__ void count_add_kernel(long long* __restrict__ count, long long n) {
  if (gtid() == 0) count[0] += n;
}
__global__ void normalize_kernel(const float* __restrict__ x, long long n, int O, const float* __restrict__ mean, const float* __restrict__ stdv,
                                 float eps, float* __restrict__ out) {
  const long long id = gtid();
  if (id >= n * O) return;
  const int j = (int)(id % O);
  out[id] = (x[id] - mean[j]) / (stdv[j] + eps);
}

#define FS_TRY(expr) do { int _rc = (expr); if (_rc) return _rc; } while (0)

// Linear-LayerNorm-SiLU x3.  P: the network's parameter block, off: its segment offsets (first 12 segments)
static int torso_fwd(const float* P, const long long* off, const int* widths, const float* X, int in, long long n, const Acts& a, cudaStream_t st) {
  const float* x = X;
  for (int k = 0; k < 3; ++k) {
    FS_TRY(lin_fwd(x, in, P + off[4 * k], in, widths[k], P + off[4 * k + 1], a.Z[k], widths[k], n, st));
    RLX_FLAT_LAUNCH(ln_silu_fwd_kernel, n, st, a.Z[k], n, widths[k], P + off[4 * k + 2], P + off[4 * k + 3], a.Y[k], a.S[k]);
    x = a.Y[k];
    in = widths[k];
  }
  return RLX_OK;
}
// dOut3: gradient wrt the torso output Y[2] (overwritten).  Writes parameter gradients into G (same offsets); dX (may be null): gradient wrt X.
static int torso_bwd(const float* P, float* G, const long long* off, const int* widths, const float* X, int in0, long long n, const Acts& a,
                     float* dOut3, float* dZ, float* dY, float* dX, float* part, float* col, cudaStream_t st) {
  float* dout = dOut3;
  for (int k = 2; k >= 0; --k) {
    const int W = widths[k], in = k == 0 ? in0 : widths[k - 1];
    const float* xin = k == 0 ? X : a.Y[k - 1];
    const long long nchunk = ceil_div(n, kColChunk);
    RLX_FLAT_LAUNCH(ln_silu_param_partial_kernel, nchunk * W, st, dout, a.Z[k], n, W, P + off[4 * k + 2], P + off[4 * k + 3], a.S[k], col, col + nchunk * W);
    RLX_FLAT_LAUNCH(reduce_parts_kernel, (long long)W, st, col, nchunk, (long long)W, 1.f, 0.f, G + off[4 * k + 2]);
    RLX_FLAT_LAUNCH(reduce_parts_kernel, (long long)W, st, col + nchunk * W, nchunk, (long long)W, 1.f, 0.f, G + off[4 * k + 3]);
    RLX_FLAT_LAUNCH(ln_silu_bwd_kernel, n, st, dout, a.Z[k], n, W, P + off[4 * k + 2], P + off[4 * k + 3], a.S[k], dZ);
    FS_TRY(lin_bwd_weight(dZ, W, xin, in, in, W, n, part, G + off[4 * k], st));
    FS_TRY(colsum(dZ, W, n, W, col, 1.f, 0.f, G + off[4 * k + 1], st));
    if (k > 0) {
      FS_TRY(lin_bwd_input(dZ, W, P + off[4 * k], in, W, dY, in, n, st));
      dout = dY;
    } else if (dX) {
      FS_TRY(lin_bwd_input(dZ, W, P + off[4 * k], in, W, dX, in, n, st));
    }
  }
  return RLX_OK;
}
static Acts acts_p(float* ws, const Ws& w) { Acts a; for (int k = 0; k < 3; ++k) { a.Z[k] = ws + w.pZ[k]; a.Y[k] = ws + w.pY[k]; a.S[k] = ws + w.pS[k]; } return a; }
static Acts acts_q(float* ws, const Ws& w, int q) { Acts a; for (int k = 0; k < 3; ++k) { a.Z[k] = ws + w.qZ[q][k]; a.Y[k] = ws + w.qY[q][k]; a.S[k] = ws + w.qS[q][k]; } return a; }

// policy forward + head on rows X; leaves Mean / LsRaw in the workspace; action (+ logp) out
static int policy_fwd(const rlx_fastsac_dims& d, const Layout& l, const Ws& w, float* ws, const float* P, const float* X, const float* noise,
                      const float* scale, float lsmin, float lsmax, long long n, float* action, float* logp, cudaStream_t st) {
  const Acts a = acts_p(ws, w);
  FS_TRY(torso_fwd(P, l.p, kPW, X, d.obs_dim, n, a, st));
  FS_TRY(lin_fwd(a.Y[2], 128, P + l.p[12], 128, d.act_dim, P + l.p[13], ws + w.Mean, d.act_dim, n, st));
  FS_TRY(lin_fwd(a.Y[2], 128, P + l.p[14], 128, d.act_dim, P + l.p[15], ws + w.LsRaw, d.act_dim, n, st));
  RLX_FLAT_LAUNCH(squash_sample_kernel, n, st, ws + w.Mean, ws + w.LsRaw, noise, scale, n, d.act_dim, lsmin, lsmax, action, logp);
  return RLX_OK;
}
// Q network forward on [X | A] (XA already built): logits out
static int q_fwd(const rlx_fastsac_dims& d, const Layout& l, const float* Q, const float* XA, long long n, const Acts& a, float* logits, cudaStream_t st) {
  FS_TRY(torso_fwd(Q, l.q, kQW, XA, d.obs_dim + d.act_dim, n, a, st));
  return lin_fwd(a.Y[2], 192, Q + l.q[12], 192, d.nr_atoms, Q + l.q[13], logits, d.nr_atoms, n, st);
}
// backward of one Q network from dlogits: parameter gradients into G; dXA optional
static int q_bwd(const rlx_fastsac_dims& d, const Layout& l, const Ws& w, float* ws, const float* Q, float* G, const float* XA, long long n,
                 const Acts& a, float* dlogits, float* dXA, cudaStream_t st) {
  const int K = d.nr_atoms;
  FS_TRY(lin_bwd_weight(dlogits, K, a.Y[2], 192, 192, K, n, ws + w.Part, G + l.q[12], st));
  FS_TRY(colsum(dlogits, K, n, K, ws + w.Col, 1.f, 0.f, G + l.q[13], st));
  FS_TRY(lin_bwd_input(dlogits, K, Q + l.q[12], 192, K, ws + w.dY, 192, n, st));
  // torso_bwd overwrites its dOut3 argument only through dZ / dY ping-pong: dY holds dL/dY[2] here and is re-used below block 2
  return torso_bwd(Q, G, l.q, kQW, XA, d.obs_dim + d.act_dim, n, a, ws + w.dY, ws + w.dZ, ws + w.dY, dXA, ws + w.Part, ws + w.Col, st);
}
static int adamw(float* p, const float* g, float* m, float* v, long long n, const float* lr, long long* step, const rlx_fastsac_hparams& hp,
                 float* norm_out, float* scratch, cudaStream_t st) {
  return adamw_step(p, g, m, v, n, lr, step, hp.max_grad_norm, hp.weight_decay, hp.adam_beta1, hp.adam_beta2, hp.adam_eps, norm_out, scratch, st);
}

}  // namespace fsac
}  // namespace rlx

using namespace rlx;
using namespace rlx::fsac;

extern "C" int rlx_fastsac_param_layout(const rlx_fastsac_dims* d, int64_t* policy_offsets, int64_t* q_offsets) {
  RLX_CHECK_ARG(d != nullptr && dims_ok(*d), "unsupported dims");
  const Layout l = make_layout(*d);
  if (policy_offsets) for (int i = 0; i <= RLX_FASTSAC_POLICY_NSEG; ++i) policy_offsets[i] = l.p[i];
  if (q_offsets) for (int i = 0; i <= RLX_FASTSAC_Q_NSEG; ++i) q_offsets[i] = l.q[i];
  return RLX_OK;
}
extern "C" size_t rlx_fastsac_workspace_bytes(const rlx_fastsac_dims* d, int64_t n) {
  if (d == nullptr || !dims_ok(*d) || n <= 0) return 0;
  return plan(*d, n).total;
}

static int check_update(const rlx_fastsac_update_args* a, bool critic, const Ws& w) {
  RLX_CHECK_ARG(a != nullptr && dims_ok(a->dims) && a->n > 0 && a->n < (1LL << 31), "bad arguments");
  RLX_CHECK_ARG(a->states && a->noise && a->action_scale && a->policy_params && a->q_params && a->log_alpha && a->lr && a->steps && a->metrics,
                "null pointer");
  if (critic) RLX_CHECK_ARG(a->next_states && a->actions && a->rewards && a->dones && a->truncations && a->effective_n_steps && a->q_grads && a->q_m &&
                            a->q_v && a->q_target_params && a->alpha_state, "null pointer (critic update)");
  else RLX_CHECK_ARG(a->policy_grads && a->policy_m && a->policy_v, "null pointer (policy update)");
  if (a->workspace == nullptr || a->workspace_bytes < w.total) {
    set_error("rlx_fastsac update: workspace too small (%zu < %zu)", a->workspace_bytes, w.total);
    return RLX_ERR_WORKSPACE;
  }
  return RLX_OK;
}

extern "C" int rlx_fastsac_critic_update_f32(const rlx_fastsac_update_args* a, void* stream) {
  RLX_CHECK_ARG(a != nullptr && dims_ok(a->dims) && a->n > 0, "bad arguments");
  const rlx_fastsac_dims& d = a->dims;
  const Ws w = plan(d, a->n);
  FS_TRY(check_update(a, true, w));
  cudaStream_t st = (cudaStream_t)stream;
  const Layout l = make_layout(d);
  const long long n = a->n, nq = l.q[RLX_FASTSAC_Q_NSEG];
  const int O = d.obs_dim, A = d.act_dim, K = d.nr_atoms;
  float* ws = (float*)a->workspace;
  const rlx_fastsac_hparams& hp = a->hp;
  float *XA = ws + w.XA, *Act = ws + w.Act, *Logp = ws + w.Logp, *RowA = ws + w.RowA, *RowB = ws + w.RowB, *Small = ws + w.Small, *Col = ws + w.Col;
  const Acts q0 = acts_q(ws, w, 0), q1 = acts_q(ws, w, 1);
  // ---- target (no gradients): a' ~ pi(s'), both target networks on (s', a'), projection (fastsac.py:143-186)
  FS_TRY(policy_fwd(d, l, w, ws, a->policy_params, a->next_states, a->noise, a->action_scale, hp.log_std_min, hp.log_std_max, n, Act, Logp, st));
  RLX_FLAT_LAUNCH(concat_kernel, n * (O + A), st, a->next_states, Act, n, O, A, O + A, XA);
  for (int q = 0; q < 2; ++q) {
    const float* QT;
    FS_TRY(aligned_params(a->q_target_params + q * nq, nq, ws + w.QP[q], &QT, st));
    FS_TRY(q_fwd(d, l, QT, XA, n, q == 0 ? q0 : q1, ws + w.Logits[q], st));
  }
  RLX_FLAT_LAUNCH(c51_project_kernel, n, st, ws + w.Logits[0], ws + w.Logits[1], a->rewards, a->dones, a->truncations, a->effective_n_steps, Logp,
                  a->log_alpha, n, K, hp.gamma, hp.v_min, hp.v_max, hp.clipped_double_q != 0.f ? 1 : 0, ws + w.Proj[0], ws + w.Proj[1],
                  RowA /*q1_next_value*/);
  const long long nchunk = ceil_div(n, kColChunk);
  RLX_FLAT_LAUNCH(minmax_partial_kernel, nchunk, st, RowA, n, RowB);
  // ---- current critics on (s, a): cross-entropy and its gradient (fastsac.py:188-196)
  RLX_FLAT_LAUNCH(concat_kernel, n * (O + A), st, a->states, a->actions, n, O, A, O + A, XA);
  const float inv_n = 1.f / (float)n;
  for (int q = 0; q < 2; ++q) {
    const Acts& aq = q == 0 ? q0 : q1;
    const float* Q;
    FS_TRY(aligned_params(a->q_params + q * nq, nq, ws + w.QP[q], &Q, st));
    FS_TRY(q_fwd(d, l, Q, XA, n, aq, ws + w.Logits[q], st));
    RLX_FLAT_LAUNCH(ce_rows_kernel, n, st, ws + w.Logits[q], ws + w.Proj[q], n, K, inv_n, RowA + (1 + q) * n, ws + w.dLogits);
    FS_TRY(q_bwd(d, l, w, ws, Q, a->q_grads + q * nq, XA, n, aq, ws + w.dLogits, nullptr, st));
  }
  // sums: loss rows of both critics and the next log-probs (entropy = -next_log_probs)
  FS_TRY(colsum(RowA + n, 1, n, 1, Col, 1.f, 0.f, Small + 0, st));
  FS_TRY(colsum(RowA + 2 * n, 1, n, 1, Col, 1.f, 0.f, Small + 1, st));
  FS_TRY(colsum(Logp, 1, n, 1, Col, 1.f, 0.f, Small + 2, st));
  RLX_FLAT_LAUNCH(critic_finish_kernel, 1, st, Small, RowB, nchunk, (float)n, a->log_alpha, hp.target_entropy, a->alpha_state, a->metrics);
  // ---- optimiser steps: q1 | q2 as one AdamW group, then the entropy coefficient; then the polyak update (fastsac.py:198-236, 316-320)
  FS_TRY(adamw(a->q_params, a->q_grads, a->q_m, a->q_v, 2 * nq, a->lr, (long long*)a->steps + 0, hp, a->metrics + 5, ws + w.Part, st));
  rlx_fastsac_hparams hp_alpha = hp;
  hp_alpha.max_grad_norm = -1.f;  // the reference never clips the entropy coefficient
  FS_TRY(adamw(a->log_alpha, a->alpha_state, a->alpha_state + 1, a->alpha_state + 2, 1, a->lr, (long long*)a->steps + 1, hp_alpha, Small + 8,
               ws + w.Part, st));
  RLX_FLAT_LAUNCH(polyak_kernel, 2 * nq, st, a->q_target_params, a->q_params, 2 * nq, hp.tau);
  return RLX_OK;
}

extern "C" int rlx_fastsac_policy_update_f32(const rlx_fastsac_update_args* a, void* stream) {
  RLX_CHECK_ARG(a != nullptr && dims_ok(a->dims) && a->n > 0, "bad arguments");
  const rlx_fastsac_dims& d = a->dims;
  const Ws w = plan(d, a->n);
  FS_TRY(check_update(a, false, w));
  cudaStream_t st = (cudaStream_t)stream;
  const Layout l = make_layout(d);
  const long long n = a->n, nq = l.q[RLX_FASTSAC_Q_NSEG];
  const int O = d.obs_dim, A = d.act_dim, K = d.nr_atoms;
  float* ws = (float*)a->workspace;
  const rlx_fastsac_hparams& hp = a->hp;
  float *XA = ws + w.XA, *Act = ws + w.Act, *Logp = ws + w.Logp, *RowA = ws + w.RowA, *Small = ws + w.Small, *Col = ws + w.Col, *dXA = ws + w.dXA,
        *dAct = ws + w.dAct;
  const Acts pa = acts_p(ws, w);
  const float inv_n = 1.f / (float)n;
  // a ~ pi(s); q = (E[q1] + E[q2]) / 2 on (s, a); L = mean(alpha logp - q)   (fastsac.py:108-124)
  FS_TRY(policy_fwd(d, l, w, ws, a->policy_params, a->states, a->noise, a->action_scale, hp.log_std_min, hp.log_std_max, n, Act, Logp, st));
  RLX_FLAT_LAUNCH(concat_kernel, n * (O + A), st, a->states, Act, n, O, A, O + A, XA);
  const int clipped = hp.clipped_double_q != 0.f ? 1 : 0;
  const float* Qp[2];
  for (int q = 0; q < 2; ++q) {
    FS_TRY(aligned_params(a->q_params + q * nq, nq, ws + w.QP[q], &Qp[q], st));
    FS_TRY(q_fwd(d, l, Qp[q], XA, n, acts_q(ws, w, q), ws + w.Logits[q], st));
    RLX_FLAT_LAUNCH(expect_rows_kernel, n, st, ws + w.Logits[q], n, K, hp.v_min, hp.v_max, RowA + (1 + q) * n, 0.f, (float*)nullptr);
  }
  for (int q = 0; q < 2; ++q) {
    const Acts aq = acts_q(ws, w, q);
    const float* Q = Qp[q];
    // back through the critic to its input only (its own parameter gradients are not needed: the next critic update zeroes them)
    RLX_FLAT_LAUNCH(value_grad_rows_kernel, n, st, ws + w.Logits[q], RowA + (1 + q) * n, RowA + (2 - q) * n, n, K, hp.v_min, hp.v_max, clipped, inv_n,
                    ws + w.dLogits);
    FS_TRY(lin_bwd_input(ws + w.dLogits, K, Q + l.q[12], 192, K, ws + w.dY, 192, n, st));
    for (int k = 2; k >= 0; --k) {
      const int W = kQW[k], in = k == 0 ? O + A : kQW[k - 1];
      RLX_FLAT_LAUNCH(ln_silu_bwd_kernel, n, st, ws + w.dY, aq.Z[k], n, W, Q + l.q[4 * k + 2], Q + l.q[4 * k + 3],
                      aq.S[k], ws + w.dZ);
      float* dst = k == 0 ? (q == 0 ? dXA : ws + w.dXA2) : ws + w.dY;
      FS_TRY(lin_bwd_input(ws + w.dZ, W, Q + l.q[4 * k], in, W, dst, in, n, st));
    }
  }
  // dAct = action columns of both critics' input gradients; back through the squashed-Gaussian head and the policy torso
  RLX_FLAT_LAUNCH(action_grad_kernel, n * A, st, dXA, ws + w.dXA2, n, O, A, O + A, dAct);
  RLX_FLAT_LAUNCH(squash_sample_bwd_kernel, n, st, ws + w.Mean, ws + w.LsRaw, a->noise, a->action_scale, dAct, a->log_alpha, n, A, hp.log_std_min,
                  hp.log_std_max, inv_n, ws + w.dMean, ws + w.dLs);
  const float* P = a->policy_params;
  float* G = a->policy_grads;
  FS_TRY(lin_bwd_weight(ws + w.dMean, A, pa.Y[2], 128, 128, A, n, ws + w.Part, G + l.p[12], st));
  FS_TRY(colsum(ws + w.dMean, A, n, A, Col, 1.f, 0.f, G + l.p[13], st));
  FS_TRY(lin_bwd_weight(ws + w.dLs, A, pa.Y[2], 128, 128, A, n, ws + w.Part, G + l.p[14], st));
  FS_TRY(colsum(ws + w.dLs, A, n, A, Col, 1.f, 0.f, G + l.p[15], st));
  FS_TRY(lin_bwd_input(ws + w.dMean, A, P + l.p[12], 128, A, ws + w.dY, 128, n, st));
  FS_TRY(lin_bwd_input(ws + w.dLs, A, P + l.p[14], 128, A, ws + w.dZ, 128, n, st));
  RLX_FLAT_LAUNCH(add_inplace_kernel, n * 128, st, ws + w.dY, ws + w.dZ, n * 128);
  FS_TRY(torso_bwd(P, G, l.p, kPW, a->states, O, n, pa, ws + w.dY, ws + w.dZ, ws + w.dY, nullptr, ws + w.Part, Col, st));
  // metrics: policy_loss, alpha; then AdamW (its pre-clip gradient norm is metrics[2])
  FS_TRY(colsum(Logp, 1, n, 1, Col, 1.f, 0.f, Small + 0, st));
  RLX_FLAT_LAUNCH(combine_values_kernel, n, st, RowA + n, RowA + 2 * n, n, clipped, RowA + 3 * n);
  FS_TRY(colsum(RowA + 3 * n, 1, n, 1, Col, 1.f, 0.f, Small + 1, st));
  RLX_FLAT_LAUNCH(policy_finish_kernel, 1, st, Small, (float)n, a->log_alpha, a->metrics);
  FS_TRY(adamw(a->policy_params, a->policy_grads, a->policy_m, a->policy_v, l.p[RLX_FASTSAC_POLICY_NSEG], a->lr, (long long*)a->steps + 2, hp,
               a->metrics + 2, ws + w.Part, st));
  return RLX_OK;
}

extern "C" int rlx_fastsac_act_f32(const rlx_fastsac_dims* d, const float* policy_params, const float* obs, const float* noise,
                                   const float* action_scale, float log_std_min, float log_std_max, int64_t n, float* action, void* workspace,
                                   size_t workspace_bytes, void* stream) {
  RLX_CHECK_ARG(d != nullptr && dims_ok(*d) && n > 0, "bad arguments");
  RLX_CHECK_ARG(policy_params && obs && action_scale && action, "null pointer");
  const Ws w = plan(*d, n);
  if (workspace == nullptr || workspace_bytes < w.total) {
    set_error("rlx_fastsac_act_f32: workspace too small (%zu < %zu)", workspace_bytes, w.total);
    return RLX_ERR_WORKSPACE;
  }
  return policy_fwd(*d, make_layout(*d), w, (float*)workspace, policy_params, obs, noise, action_scale, log_std_min, log_std_max, n, action, nullptr,
                    (cudaStream_t)stream);
}

extern "C" int rlx_fastsac_normalize_f32(const float* x, int64_t n, int64_t obs_dim, float* mean, float* var, float* std, int64_t* count,
                                         int32_t update, float eps, float* out, float* workspace, void* stream) {
  RLX_CHECK_ARG(n > 0 && obs_dim > 0 && x && mean && std && out, "bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  const int O = (int)obs_dim;
  if (update) {
    RLX_CHECK_ARG(var && count && workspace, "update needs var / count / workspace");
    const long long nchunk = ceil_div(n, kColChunk);
    float* col_sum = workspace;                 // [O]
    float* col_sq = workspace + O;              // [O]
    float* part = workspace + 2 * O;            // [nchunk, O]
    FS_TRY(colsum(x, O, n, O, part, 1.f, 0.f, col_sum, st));
    // squared deviations from the batch mean, summed per column in the same two stages (out is used as scratch before it is written)
    RLX_FLAT_LAUNCH(centered_sq_cols_kernel, (long long)n * O, st, x, (long long)n, O, col_sum, out);
    FS_TRY(colsum(out, O, n, O, part, 1.f, 0.f, col_sq, st));
    RLX_FLAT_LAUNCH(normalizer_update_kernel, (long long)O, st, col_sum, col_sq, (long long)n, O, mean, var, std, (const long long*)count);
    RLX_FLAT_LAUNCH(count_add_kernel, 1, st, (long long*)count, (long long)n);
    (void)nchunk;
  }
  RLX_FLAT_LAUNCH(normalize_kernel, (long long)n * O, st, x, (long long)n, O, mean, std, eps, out);
  return RLX_OK;
}
