// FastTD3 update (rl_x/algorithms/fasttd3/pytorch): distributional (C51) twin critics, deterministic tanh actor with target-policy
// smoothing, AdamW, polyak targets.  Entry points and flat layouts: include/rlx_b200.h.  The critic machinery is FastSAC's (c51_ops.cuh);
// the networks are plain Linear-ReLU MLPs whose layers go through aux_gemm with the ReLU folded into the GEMM epilogues (EPI_BIAS_RELU
// forward, EPI_DRELU for the input gradients), so rlx_set_aux_gemm_engine(1) puts them on the wgmma 3xTF32 engine.
// Dual build (dual_build.cuh): the host emulation of this file is checked against oracle/fasttd3_oracle.py (pinned to the executed
// reference) in tests/test_fasttd3_emulation.py.
#include "c51_ops.cuh"

namespace rlx {
namespace ftd3 {
using namespace rlx::flat;
using namespace rlx::c51;

constexpr int kPW[3] = {512, 256, 128};    // policy widths (policy.py:33-42)
constexpr int kQW[3] = {1024, 512, 256};   // Q widths (q_network.py:27-35)

struct Layout {
  long long p[RLX_FASTTD3_POLICY_NSEG + 1], q[RLX_FASTTD3_Q_NSEG + 1];
};
static void mlp_layout(long long* off, int in, const int* widths, int out) {
  long long o = 0;
  int s = 0;
  for (int k = 0; k < 4; ++k) {
    const int w = k < 3 ? widths[k] : out;
    off[s++] = o; o += (long long)w * in;
    off[s++] = o; o += w;
    in = w;
  }
  off[s] = o;
}
static Layout make_layout(const rlx_fasttd3_dims& d) {
  Layout l;
  mlp_layout(l.p, d.obs_dim, kPW, d.act_dim);
  mlp_layout(l.q, d.obs_dim + d.act_dim, kQW, d.nr_atoms);
  return l;
}
static bool dims_ok(const rlx_fasttd3_dims& d) { return d.obs_dim > 0 && d.act_dim > 0 && d.act_dim <= 64 && d.nr_atoms >= 2 && d.nr_atoms <= 1024; }
// row pitch of the [s | a] buffers and of the staged layer-1 Q weights: a multiple of 4 floats (16 B), which a TMA descriptor needs
static int xa_pitch(const rlx_fasttd3_dims& d) { return (int)align_up((size_t)(d.obs_dim + d.act_dim), 4); }

struct Ws {
  size_t pH[3], qH[2][3], XA, Act, Logits[2], Proj[2], dLogits, dA, dB, dXa[2], dAct, RowA, RowB, Zero, Small, W1[2], QP[2], Part, Col, total;
};
static Ws plan(const rlx_fasttd3_dims& d, long long n_) {
  const size_t n = (size_t)n_, O = d.obs_dim, A = d.act_dim, K = d.nr_atoms, P = (size_t)xa_pitch(d);
  Ws w;
  size_t o = 0;
  auto take = [&](size_t& f, size_t cnt) { f = o; o += align_up(cnt, 64); };
  for (int k = 0; k < 3; ++k) take(w.pH[k], n * kPW[k]);
  for (int q = 0; q < 2; ++q)
    for (int k = 0; k < 3; ++k) take(w.qH[q][k], n * kQW[k]);
  take(w.XA, n * P); take(w.Act, n * A);
  for (int q = 0; q < 2; ++q) { take(w.Logits[q], n * K); take(w.Proj[q], n * K); }
  take(w.dLogits, n * K); take(w.dA, n * 1024); take(w.dB, n * 1024); take(w.dXa[0], n * A); take(w.dXa[1], n * A); take(w.dAct, n * A);
  take(w.RowA, n * 4); take(w.RowB, n * 4); take(w.Zero, n); take(w.Small, 64);
  take(w.W1[0], (size_t)kQW[0] * P); take(w.W1[1], (size_t)kQW[0] * P);
  const size_t nq = (size_t)make_layout(d).q[RLX_FASTTD3_Q_NSEG];
  take(w.QP[0], nq); take(w.QP[1], nq);   // aligned_params: a critic's parameter block when its base is not 16-byte aligned
  const size_t splits = (size_t)ceil_div((long long)n, kWgradRows);
  size_t biggest = std::max<size_t>((size_t)kQW[0] * P, (size_t)kQW[1] * kQW[0]);
  biggest = std::max<size_t>(biggest, std::max<size_t>((size_t)kPW[0] * O, (size_t)K * kQW[2]));
  take(w.Part, splits * biggest);
  const size_t chunks = (size_t)ceil_div((long long)n, kColChunk);
  take(w.Col, chunks * std::max<size_t>(1024, std::max<size_t>(K, 8)));
  w.total = o * sizeof(float);
  return w;
}

// ---------------------------------------------------------------------------------------------------------- kernels
static __global__ void fill_kernel(float* __restrict__ x, long long n, float v) {
  const long long i = gtid();
  if (i < n) x[i] = v;
}
// dst[r, :cols] = src[r, :cols] with row pitch ld (the padded copy of a layer-1 weight).  thread = element
static __global__ void pitch_copy_kernel(const float* __restrict__ src, long long rows, int cols, int ld, float* __restrict__ dst) {
  const long long id = gtid();
  if (id >= rows * cols) return;
  dst[(id / cols) * ld + id % cols] = src[id];
}
// out[o, i] = sum_s part[s][o, i] with the partials at row pitch ld, the output unpadded [rows, cols].  thread = element
static __global__ void reduce_parts_pitched_kernel(const float* __restrict__ part, long long nparts, long long rows, int cols, int ld,
                                                   float* __restrict__ out) {
  const long long id = gtid();
  if (id >= rows * cols) return;
  const long long src = (id / cols) * ld + id % cols, len = rows * ld;
  float s = 0.f;
  for (long long k = 0; k < nparts; ++k) s += part[k * len + src];
  out[id] = s;
}
// target-policy smoothing in place (fasttd3.py:143-144): act = clamp(act + clamp(eps * noise, -clip, clip), -1, 1).  thread = element
static __global__ void smooth_target_action_kernel(float* __restrict__ act, const float* __restrict__ noise, long long n, float eps, float clip) {
  const long long i = gtid();
  if (i >= n) return;
  const float z = fminf(fmaxf(rn_mul(noise[i], eps), -clip), clip);
  act[i] = fminf(fmaxf(rn_add(act[i], z), -1.f), 1.f);
}
// exploration noise and the optional clip / rescale to the action bounds (policy.py:57-66).  thread = element
static __global__ void explore_kernel(float* __restrict__ action, const float* __restrict__ noise, const float* __restrict__ scale, long long n, int A,
                                      const float* __restrict__ low, const float* __restrict__ high, int clip_rescale, float* __restrict__ env_action) {
  const long long id = gtid();
  if (id >= n * A) return;
  float a = action[id];
  if (noise) {
    a = rn_add(a, rn_mul(noise[id], scale[id / A]));
    action[id] = a;
  }
  if (env_action == nullptr) return;
  const int j = (int)(id % A);
  if (clip_rescale) a = rn_add(low[j], rn_mul(rn_mul(0.5f, rn_add(fminf(fmaxf(a, -1.f), 1.f), 1.f)), rn_sub(high[j], low[j])));
  env_action[id] = a;
}
// tanh backward: dPre = dAct (1 - a^2), a the tanh output.  thread = element
static __global__ void tanh_bwd_kernel(const float* __restrict__ dAct, const float* __restrict__ a, long long n, float* __restrict__ dPre) {
  const long long i = gtid();
  if (i >= n) return;
  dPre[i] = dAct[i] * (1.f - a[i] * a[i]);
}
// critic metrics (fasttd3.py:205-209).  sums: [sum loss1, sum loss2]
static __global__ void critic_finish_kernel(const float* __restrict__ sums, const float* __restrict__ mm_part, long long nchunk, float n,
                                            float* __restrict__ metrics) {
  if (gtid() != 0) return;
  float lo = mm_part[0], hi = mm_part[1];
  for (long long c = 1; c < nchunk; ++c) { lo = fminf(lo, mm_part[2 * c]); hi = fmaxf(hi, mm_part[2 * c + 1]); }
  metrics[0] = sums[0] / n + sums[1] / n;   // q_loss = q1_loss + q2_loss
  metrics[1] = lo;                          // q_min, q_max of the projected q1 next value
  metrics[2] = hi;
}
static __global__ void policy_finish_kernel(const float* __restrict__ sums, float n, float* __restrict__ metrics) {
  if (gtid() == 0) metrics[0] = -(sums[0] / n);   // -mean(q)
}

// ------------------------------------------------------------------------------------------------------- networks
#define TD_TRY(expr) C51_TRY(expr)

// Linear-ReLU x3 + head on X (row pitch ldx, `in` columns).  W1 / ldw1: the first layer's weight as used (a padded copy or the parameter
// block itself); tanh_head: policy (tanh) or Q network (plain logits).  H: the three post-ReLU activations, kept for the backward.
static int mlp_fwd(const float* P, const long long* off, const int* widths, const float* X, int ldx, int in, const float* W1, int ldw1, float* const* H,
                   int out, bool tanh_head, float* Y, long long n, cudaStream_t st) {
  TD_TRY(lin_fwd<EPI_BIAS_RELU>(X, ldx, W1, in, widths[0], P + off[1], H[0], widths[0], n, st, ldw1));
  TD_TRY(lin_fwd<EPI_BIAS_RELU>(H[0], widths[0], P + off[2], widths[0], widths[1], P + off[3], H[1], widths[1], n, st));
  TD_TRY(lin_fwd<EPI_BIAS_RELU>(H[1], widths[1], P + off[4], widths[1], widths[2], P + off[5], H[2], widths[2], n, st));
  if (tanh_head) return lin_fwd<EPI_BIAS_TANH>(H[2], widths[2], P + off[6], widths[2], out, P + off[7], Y, out, n, st);
  return lin_fwd<EPI_BIAS>(H[2], widths[2], P + off[6], widths[2], out, P + off[7], Y, out, n, st);
}
// Parameter gradients of the MLP above into G (same offsets) from dOut [n, out] (the gradient wrt the head's pre-activation).  The first
// layer's weight gradient is computed at the row pitch of X (ldx, a multiple of 4 where X is the padded [s | a]) and written back unpadded.
static int mlp_bwd(const float* P, float* G, const long long* off, const int* widths, const float* X, int ldx, int in, float* const* H, int out,
                   const float* dOut, long long n, float* dA, float* dB, float* part, float* col, cudaStream_t st) {
  TD_TRY(lin_bwd_weight(dOut, out, H[2], widths[2], widths[2], out, n, part, G + off[6], st));
  TD_TRY(colsum(dOut, out, n, out, col, 1.f, 0.f, G + off[7], st));
  TD_TRY(lin_bwd_input<EPI_DRELU>(dOut, out, P + off[6], widths[2], out, dA, widths[2], n, st, H[2]));
  for (int k = 2; k >= 0; --k) {
    const int W = widths[k];
    if (k > 0) {
      TD_TRY(lin_bwd_weight(dA, W, H[k - 1], widths[k - 1], widths[k - 1], W, n, part, G + off[2 * k], st));
    } else {
      const int splits = (int)ceil_div(n, kWgradRows);
      GemmP g{};
      g.A = dA; g.B = X; g.C = part;
      g.M = W; g.N = in; g.K = (int)n; g.lda = W; g.ldb = ldx; g.ldc = ldx;
      g.splits = splits; g.kchunk = kWgradRows; g.sSplitC = (long long)ldx * W;
      TD_TRY((aux_gemm<false, false, EPI_NONE>(g, 1, st, KC_GEMM_DW, n, n)));
      RLX_FLAT_LAUNCH(reduce_parts_pitched_kernel, (long long)W * in, st, part, (long long)splits, (long long)W, in, ldx, G + off[0]);
    }
    TD_TRY(colsum(dA, W, n, W, col, 1.f, 0.f, G + off[2 * k + 1], st));
    if (k > 0) {
      TD_TRY(lin_bwd_input<EPI_DRELU>(dA, W, P + off[2 * k], widths[k - 1], W, dB, widths[k - 1], n, st, H[k - 1]));
      std::swap(dA, dB);
    }
  }
  return RLX_OK;
}
struct Hs { float* h[3]; };
static Hs hs_p(float* ws, const Ws& w) { return {{ws + w.pH[0], ws + w.pH[1], ws + w.pH[2]}}; }
static Hs hs_q(float* ws, const Ws& w, int q) { return {{ws + w.qH[q][0], ws + w.qH[q][1], ws + w.qH[q][2]}}; }

static int policy_fwd(const rlx_fasttd3_dims& d, const Layout& l, const Ws& w, float* ws, const float* P, const float* X, long long n, float* action,
                      cudaStream_t st) {
  const Hs h = hs_p(ws, w);
  return mlp_fwd(P, l.p, kPW, X, d.obs_dim, d.obs_dim, P + l.p[0], d.obs_dim, h.h, d.act_dim, true, action, n, st);
}
// Q network on the padded [s | a] rows: stages the layer-1 weight at the padded pitch into slot `slot`, then the forward
static int q_fwd(const rlx_fasttd3_dims& d, const Layout& l, const Ws& w, float* ws, const float* Q, int slot, const float* XA, long long n, const Hs& h,
                 float* logits, cudaStream_t st) {
  const int in = d.obs_dim + d.act_dim, ldx = xa_pitch(d);
  RLX_FLAT_LAUNCH(pitch_copy_kernel, (long long)kQW[0] * in, st, Q + l.q[0], (long long)kQW[0], in, ldx, ws + w.W1[slot]);
  return mlp_fwd(Q, l.q, kQW, XA, ldx, in, ws + w.W1[slot], ldx, h.h, d.nr_atoms, false, logits, n, st);
}

}  // namespace ftd3
}  // namespace rlx

using namespace rlx;
using namespace rlx::ftd3;

extern "C" int rlx_fasttd3_param_layout(const rlx_fasttd3_dims* d, int64_t* policy_offsets, int64_t* q_offsets) {
  RLX_CHECK_ARG(d != nullptr && dims_ok(*d), "unsupported dims");
  const Layout l = make_layout(*d);
  if (policy_offsets) for (int i = 0; i <= RLX_FASTTD3_POLICY_NSEG; ++i) policy_offsets[i] = l.p[i];
  if (q_offsets) for (int i = 0; i <= RLX_FASTTD3_Q_NSEG; ++i) q_offsets[i] = l.q[i];
  return RLX_OK;
}
extern "C" size_t rlx_fasttd3_workspace_bytes(const rlx_fasttd3_dims* d, int64_t n) {
  if (d == nullptr || !dims_ok(*d) || n <= 0) return 0;
  return plan(*d, n).total;
}

static int check_update(const rlx_fasttd3_update_args* a, bool critic, const Ws& w) {
  RLX_CHECK_ARG(a != nullptr && dims_ok(a->dims) && a->n > 0 && a->n < (1LL << 31), "bad arguments");
  RLX_CHECK_ARG(a->states && a->policy_params && a->q_params && a->lr && a->steps && a->metrics, "null pointer");
  if (critic) RLX_CHECK_ARG(a->next_states && a->actions && a->rewards && a->dones && a->truncations && a->effective_n_steps && a->smoothing_noise &&
                            a->q_grads && a->q_m && a->q_v && a->q_target_params, "null pointer (critic update)");
  else RLX_CHECK_ARG(a->policy_grads && a->policy_m && a->policy_v, "null pointer (policy update)");
  if (a->workspace == nullptr || a->workspace_bytes < w.total) {
    set_error("rlx_fasttd3 update: workspace too small (%zu < %zu)", a->workspace_bytes, w.total);
    return RLX_ERR_WORKSPACE;
  }
  return RLX_OK;
}

extern "C" int rlx_fasttd3_critic_update_f32(const rlx_fasttd3_update_args* a, void* stream) {
  RLX_CHECK_ARG(a != nullptr && dims_ok(a->dims) && a->n > 0, "bad arguments");
  const rlx_fasttd3_dims& d = a->dims;
  const Ws w = plan(d, a->n);
  TD_TRY(check_update(a, true, w));
  cudaStream_t st = (cudaStream_t)stream;
  const Layout l = make_layout(d);
  const long long n = a->n, nq = l.q[RLX_FASTTD3_Q_NSEG];
  const int O = d.obs_dim, A = d.act_dim, K = d.nr_atoms, ldx = xa_pitch(d);
  float* ws = (float*)a->workspace;
  const rlx_fasttd3_hparams& hp = a->hp;
  float *XA = ws + w.XA, *Act = ws + w.Act, *RowA = ws + w.RowA, *RowB = ws + w.RowB, *Small = ws + w.Small, *Zero = ws + w.Zero;
  const Hs q0 = hs_q(ws, w, 0), q1 = hs_q(ws, w, 1);
  // ---- target (no gradients): smoothed a' from the online policy, both target networks on (s', a'), projection (fasttd3.py:142-197)
  TD_TRY(policy_fwd(d, l, w, ws, a->policy_params, a->next_states, n, Act, st));
  RLX_FLAT_LAUNCH(smooth_target_action_kernel, n * A, st, Act, a->smoothing_noise, n * A, hp.smoothing_epsilon, hp.smoothing_clip_value);
  RLX_FLAT_LAUNCH(concat_kernel, n * (O + A), st, a->next_states, Act, n, O, A, ldx, XA);
  for (int q = 0; q < 2; ++q) {
    const float* QT;
    TD_TRY(aligned_params(a->q_target_params + q * nq, nq, ws + w.QP[q], &QT, st));
    TD_TRY(q_fwd(d, l, w, ws, QT, q, XA, n, q == 0 ? q0 : q1, ws + w.Logits[q], st));
  }
  // FastSAC's projection with a zero entropy term: r - discount * exp(0) * 0 == r
  RLX_FLAT_LAUNCH(fill_kernel, n, st, Zero, n, 0.f);
  RLX_FLAT_LAUNCH(fill_kernel, 1, st, Small + 8, 1LL, 0.f);
  RLX_FLAT_LAUNCH(c51_project_kernel, n, st, ws + w.Logits[0], ws + w.Logits[1], a->rewards, a->dones, a->truncations, a->effective_n_steps, Zero,
                  Small + 8, n, K, hp.gamma, hp.v_min, hp.v_max, hp.clipped_double_q != 0.f ? 1 : 0, ws + w.Proj[0], ws + w.Proj[1], RowA /*q1_next_value*/);
  const long long nchunk = ceil_div(n, kColChunk);
  RLX_FLAT_LAUNCH(minmax_partial_kernel, nchunk, st, RowA, n, RowB);
  // ---- current critics on (s, a): cross-entropy and its gradient (fasttd3.py:199-212)
  RLX_FLAT_LAUNCH(concat_kernel, n * (O + A), st, a->states, a->actions, n, O, A, ldx, XA);
  const float inv_n = 1.f / (float)n;
  for (int q = 0; q < 2; ++q) {
    const Hs& h = q == 0 ? q0 : q1;
    const float* Q;
    TD_TRY(aligned_params(a->q_params + q * nq, nq, ws + w.QP[q], &Q, st));
    TD_TRY(q_fwd(d, l, w, ws, Q, q, XA, n, h, ws + w.Logits[q], st));
    RLX_FLAT_LAUNCH(ce_rows_kernel, n, st, ws + w.Logits[q], ws + w.Proj[q], n, K, inv_n, RowA + (1 + q) * n, ws + w.dLogits);
    TD_TRY(mlp_bwd(Q, a->q_grads + q * nq, l.q, kQW, XA, ldx, O + A, h.h, K, ws + w.dLogits, n, ws + w.dA, ws + w.dB, ws + w.Part, ws + w.Col, st));
  }
  TD_TRY(colsum(RowA + n, 1, n, 1, ws + w.Col, 1.f, 0.f, Small + 0, st));
  TD_TRY(colsum(RowA + 2 * n, 1, n, 1, ws + w.Col, 1.f, 0.f, Small + 1, st));
  RLX_FLAT_LAUNCH(critic_finish_kernel, 1, st, Small, RowB, nchunk, (float)n, a->metrics);
  // ---- q1 | q2 as one AdamW group (its pre-clip gradient norm is metrics[3]), then the polyak update (fasttd3.py:211-223, 316-320)
  TD_TRY(adamw_step(a->q_params, a->q_grads, a->q_m, a->q_v, 2 * nq, a->lr, (long long*)a->steps + 0, hp.max_grad_norm, hp.weight_decay, hp.adam_beta1,
                    hp.adam_beta2, hp.adam_eps, a->metrics + 3, ws + w.Part, st));
  RLX_FLAT_LAUNCH(polyak_kernel, 2 * nq, st, a->q_target_params, a->q_params, 2 * nq, hp.tau);
  return RLX_OK;
}

extern "C" int rlx_fasttd3_policy_update_f32(const rlx_fasttd3_update_args* a, void* stream) {
  RLX_CHECK_ARG(a != nullptr && dims_ok(a->dims) && a->n > 0, "bad arguments");
  const rlx_fasttd3_dims& d = a->dims;
  const Ws w = plan(d, a->n);
  TD_TRY(check_update(a, false, w));
  cudaStream_t st = (cudaStream_t)stream;
  const Layout l = make_layout(d);
  const long long n = a->n, nq = l.q[RLX_FASTTD3_Q_NSEG];
  const int O = d.obs_dim, A = d.act_dim, K = d.nr_atoms, ldx = xa_pitch(d);
  float* ws = (float*)a->workspace;
  const rlx_fasttd3_hparams& hp = a->hp;
  float *XA = ws + w.XA, *Act = ws + w.Act, *RowA = ws + w.RowA, *Small = ws + w.Small, *dAct = ws + w.dAct;
  const Hs ph = hs_p(ws, w);
  const float inv_n = 1.f / (float)n;
  const int clipped = hp.clipped_double_q != 0.f ? 1 : 0;
  // a = pi(s); q = min / mean of E[q1], E[q2] on (s, a); L = -mean(q)   (fasttd3.py:106-120)
  TD_TRY(policy_fwd(d, l, w, ws, a->policy_params, a->states, n, Act, st));
  RLX_FLAT_LAUNCH(concat_kernel, n * (O + A), st, a->states, Act, n, O, A, ldx, XA);
  const float* Qp[2];
  for (int q = 0; q < 2; ++q) {
    TD_TRY(aligned_params(a->q_params + q * nq, nq, ws + w.QP[q], &Qp[q], st));
    TD_TRY(q_fwd(d, l, w, ws, Qp[q], q, XA, n, hs_q(ws, w, q), ws + w.Logits[q], st));
    RLX_FLAT_LAUNCH(expect_rows_kernel, n, st, ws + w.Logits[q], n, K, hp.v_min, hp.v_max, RowA + (1 + q) * n, 0.f, (float*)nullptr);
  }
  // back through each critic to its action columns only (its parameter gradients are not needed: the next critic update zeroes them)
  for (int q = 0; q < 2; ++q) {
    const Hs h = hs_q(ws, w, q);
    const float* Q = Qp[q];
    RLX_FLAT_LAUNCH(value_grad_rows_kernel, n, st, ws + w.Logits[q], RowA + (1 + q) * n, RowA + (2 - q) * n, n, K, hp.v_min, hp.v_max, clipped, inv_n,
                    ws + w.dLogits);
    float *dA = ws + w.dA, *dB = ws + w.dB;
    TD_TRY(lin_bwd_input<EPI_DRELU>(ws + w.dLogits, K, Q + l.q[6], kQW[2], K, dA, kQW[2], n, st, h.h[2]));
    for (int k = 2; k > 0; --k) {
      TD_TRY(lin_bwd_input<EPI_DRELU>(dA, kQW[k], Q + l.q[2 * k], kQW[k - 1], kQW[k], dB, kQW[k - 1], n, st, h.h[k - 1]));
      std::swap(dA, dB);
    }
    // dAct_q[r, j] = sum_o dA[r, o] W1[o, O + j]: the action block of the first layer's weight, read in place
    TD_TRY(lin_bwd_input(dA, kQW[0], Q + l.q[0] + O, A, kQW[0], ws + w.dXa[q], A, n, st, nullptr, O + A));
  }
  RLX_FLAT_LAUNCH(action_grad_kernel, n * A, st, ws + w.dXa[0], ws + w.dXa[1], n, 0, A, A, dAct);
  RLX_FLAT_LAUNCH(tanh_bwd_kernel, n * A, st, dAct, Act, n * A, ws + w.dXa[0]);   // dXa[0] is free again: the gradient wrt the pre-tanh head
  TD_TRY(mlp_bwd(a->policy_params, a->policy_grads, l.p, kPW, a->states, O, O, ph.h, A, ws + w.dXa[0], n, ws + w.dA, ws + w.dB, ws + w.Part, ws + w.Col,
                 st));
  // metrics: policy_loss; then AdamW (its pre-clip gradient norm is metrics[1])
  RLX_FLAT_LAUNCH(combine_values_kernel, n, st, RowA + n, RowA + 2 * n, n, clipped, RowA + 3 * n);
  TD_TRY(colsum(RowA + 3 * n, 1, n, 1, ws + w.Col, 1.f, 0.f, Small + 0, st));
  RLX_FLAT_LAUNCH(policy_finish_kernel, 1, st, Small, (float)n, a->metrics);
  return adamw_step(a->policy_params, a->policy_grads, a->policy_m, a->policy_v, l.p[RLX_FASTTD3_POLICY_NSEG], a->lr, (long long*)a->steps + 1,
                    hp.max_grad_norm, hp.weight_decay, hp.adam_beta1, hp.adam_beta2, hp.adam_eps, a->metrics + 1, ws + w.Part, st);
}

extern "C" int rlx_fasttd3_act_f32(const rlx_fasttd3_dims* d, const float* policy_params, const float* obs, const float* noise, const float* noise_scale,
                                   const float* act_low, const float* act_high, int32_t clip_rescale, int64_t n, float* action, float* env_action,
                                   void* workspace, size_t workspace_bytes, void* stream) {
  RLX_CHECK_ARG(d != nullptr && dims_ok(*d) && n > 0, "bad arguments");
  RLX_CHECK_ARG(policy_params && obs && action, "null pointer");
  RLX_CHECK_ARG(noise == nullptr || noise_scale != nullptr, "noise needs noise_scale");
  RLX_CHECK_ARG(!(clip_rescale && env_action) || (act_low && act_high), "clip_rescale needs the action bounds");
  const Ws w = plan(*d, n);
  if (workspace == nullptr || workspace_bytes < w.total) {
    set_error("rlx_fasttd3_act_f32: workspace too small (%zu < %zu)", workspace_bytes, w.total);
    return RLX_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  TD_TRY(policy_fwd(*d, make_layout(*d), w, (float*)workspace, policy_params, obs, n, action, st));
  if (noise || env_action)
    RLX_FLAT_LAUNCH(explore_kernel, n * d->act_dim, st, action, noise, noise_scale, (long long)n, d->act_dim, act_low, act_high, clip_rescale, env_action);
  return RLX_OK;
}
