// Alternative PPO loss head built from GEMMs (opt-in: rlx_set_head_engine(1)); the default stays the fused ppo_head_train3_kernel.
//
// Why: the fused head is latency-bound (ncu: 80 µs per 32 768-row minibatch, 26 % of HBM peak, 128 registers).  The same work split into
//   (1) logits   Mean[m, A] = H2p W3p^T + b3p,  V[m] = H2c W3c^T + b3c                       two GEMMs with tiny N
//   (2) one flat loss kernel over rows: ratio, clipped surrogate, value error -> dMean | dV (the `dhead` operand of the dW3 GEMM)
//   (3) dZ2      [policy | critic halves] = (dhead . W3) * (1 - H2^2)                         two GEMMs with tiny K, tanh' epilogue
//   (4) column sums (layer-2 / head bias gradients, log-std gradient, metric sums) written as ONE partial block in the fused kernel's
//       layout, so the rest of rlx_ppo_minibatch_fwdbwd_f32 (dW3 / dW2 / dX / dW1 GEMMs, grad_reduce) is unchanged
// moves the heavy parts onto the GEMM engines.  This file is dual-build (dual_build.cuh): its host emulation is checked against the
// PPO oracle's autograd in tests/test_lstm_emulation.py::test_emulated_ppo_head_gemm_path.  It stays an opt-in
// (DESIGN.md 4c); the fused kernel is the default.
#include "flat_ops.cuh"
#include "ppo_head_gemm.cuh"

namespace rlx {


namespace headgemm {
using namespace rlx::flat;
constexpr float kHalfLog2Pi = 0.9189385332046727f;

// same arithmetic as the fused kernel (ppo_head.cuh): unbiased-std advantage normalisation is done by the caller (adv_stats),
// torch.maximum splits ties evenly, the clamp passes gradient on the closed interval.  thread = row
__global__ void loss_rows_kernel(const float* __restrict__ Mean, const float* __restrict__ V, const float* __restrict__ actions,
                                 const float* __restrict__ logp_old, const float* __restrict__ adv, const float* __restrict__ ret,
                                 const float* __restrict__ logstd, const float* __restrict__ adv_stats, long long m, int A, int dh_ld,
                                 float clip_range, float critic_coef, float inv_mg, int ratio_delta_metric, float* __restrict__ dhead,
                                 float* __restrict__ dLs, float* __restrict__ terms, float* __restrict__ ratio_abs) {
  const long long r = gtid();
  if (r >= m) return;
  float lp = 0.f;
  for (int a = 0; a < A; ++a) {
    const float sd = expf(logstd[a]);
    const float d = actions[r * A + a] - Mean[r * A + a];
    lp += -(d * d) / (2.f * sd * sd) - logf(sd) - kHalfLog2Pi;
  }
  const float logratio = lp - logp_old[r];
  const float ratio = expf(logratio);
  const float An = (adv[r] - adv_stats[0]) / (adv_stats[1] + 1e-8f);
  const float lo = 1.f - clip_range, hi = 1.f + clip_range;
  const float pg1 = -An * ratio, pg2 = -An * fminf(fmaxf(ratio, lo), hi);
  const float w1 = (pg1 > pg2) ? 1.f : ((pg1 == pg2) ? 0.5f : 0.f);
  const float inr = (ratio >= lo && ratio <= hi) ? 1.f : 0.f;
  const float dlogp = -An * (w1 + (1.f - w1) * inr) * ratio * inv_mg;
  for (int a = 0; a < A; ++a) {
    const float sd = expf(logstd[a]);
    const float var = sd * sd;
    const float d = actions[r * A + a] - Mean[r * A + a];
    dhead[r * dh_ld + a] = dlogp * (d / var);
    dLs[r * A + a] = dlogp * (d * d / var - 1.f);
  }
  const float verr = V[r] - ret[r];
  dhead[r * dh_ld + A] = critic_coef * verr * inv_mg;
  for (int a = A + 1; a < dh_ld; ++a) dhead[r * dh_ld + a] = 0.f;
  terms[4 * r + 0] = fmaxf(pg1, pg2);
  terms[4 * r + 1] = 0.5f * verr * verr;
  terms[4 * r + 2] = (ratio - 1.f) - logratio;
  terms[4 * r + 3] = ratio_delta_metric ? fabsf(ratio - 1.f) : ((fabsf(ratio - 1.f) > clip_range) ? 1.f : 0.f);
  if (ratio_abs != nullptr) ratio_abs[r] = fabsf(ratio - 1.f);
}

}  // namespace headgemm

#define HG_TRY(expr) do { int _rc = (expr); if (_rc) return _rc; } while (0)

int ppo_head_gemm_path(const HeadGemmArgs& a, cudaStream_t st) {
  using namespace headgemm;
  const long long m = a.m;
  const int H = a.H, A = a.A, dh = a.dh_ld;
  float* Mean = a.scratch;                  // [m, A]
  float* V = Mean + m * A;                  // [m]
  float* dLs = V + m;                       // [m, A]
  float* terms = dLs + m * A;               // [m, 4]
  float* col = terms + 4 * m;               // column-sum partials
  // (1) logits: A k-major (H2 halves, row pitch 2H), B k-major (torch [out, in] weights)
  GemmP g{};
  g.A = a.H2; g.B = a.W3p; g.C = Mean; g.bias = a.b3p;
  g.M = (int)m; g.N = A; g.K = H; g.lda = 2 * H; g.ldb = H; g.ldc = A; g.splits = 1; g.kchunk = (int)(ceil_div(H, 8) * 8);
  HG_TRY((launch_sgemm<true, true, EPI_BIAS>(g, 1, st, KC_GEMM_FWD)));
  GemmP gv{};
  gv.A = a.H2 + H; gv.B = a.W3c; gv.C = V; gv.bias = a.b3c;
  gv.M = (int)m; gv.N = 1; gv.K = H; gv.lda = 2 * H; gv.ldb = H; gv.ldc = 1; gv.splits = 1; gv.kchunk = g.kchunk;
  HG_TRY((launch_sgemm<true, true, EPI_BIAS>(gv, 1, st, KC_GEMM_FWD)));
  // (2) per-row loss and head gradients
  RLX_FLAT_LAUNCH(loss_rows_kernel, m, st, Mean, V, a.actions, a.logp_old, a.adv, a.ret, a.logstd, a.adv_stats, m, A, dh, a.clip_range, a.critic_coef,
                  a.inv_mg, a.ratio_delta_metric, a.dhead, dLs, terms, a.ratio_abs);
  // (3) dZ2 = (dhead . W3) * (1 - H2^2): A k-major (dhead), B n-major (W3p[a, h] read as B[k = a][n = h]), tanh' epilogue on the matching half
  GemmP gp{};
  gp.A = a.dhead; gp.B = a.W3p; gp.C = a.dZ2; gp.aux = a.H2;
  gp.M = (int)m; gp.N = H; gp.K = A; gp.lda = dh; gp.ldb = H; gp.ldc = 2 * H; gp.ldaux = 2 * H; gp.splits = 1; gp.kchunk = (int)(ceil_div(A, 8) * 8);
  HG_TRY((launch_sgemm<true, false, EPI_DTANH>(gp, 1, st, KC_GEMM_DX)));
  GemmP gc{};
  gc.A = a.dhead + A; gc.B = a.W3c; gc.C = a.dZ2 + H; gc.aux = a.H2 + H;
  gc.M = (int)m; gc.N = H; gc.K = 1; gc.lda = dh; gc.ldb = H; gc.ldc = 2 * H; gc.ldaux = 2 * H; gc.splits = 1; gc.kchunk = 8;
  HG_TRY((launch_sgemm<true, false, EPI_DTANH>(gc, 1, st, KC_GEMM_DX)));
  // (4) the partial block: db3p | db3c | dlogstd | pg vl kl cf | db2p | db2c
  float* hp = a.headpart;
  HG_TRY(colsum(a.dhead, dh, m, A + 1, col, 1.f, 0.f, hp, st));            // db3p[A], db3c
  HG_TRY(colsum(dLs, A, m, A, col, 1.f, 0.f, hp + A + 1, st));              // dlogstd[A]
  HG_TRY(colsum(terms, 4, m, 4, col, 1.f, 0.f, hp + 2 * A + 1, st));        // pg, vl, kl, cf
  HG_TRY(colsum(a.dZ2, 2 * H, m, 2 * H, col, 1.f, 0.f, hp + 2 * A + 5, st)); // db2p[H] | db2c[H]
  return RLX_OK;
}

}  // namespace rlx

// test / bring-up entries: the path on caller-provided buffers.  The _ratio_ form also takes the optional per-row |ratio - 1| output
// (ratio_abs); the original signature stays as it was for its existing callers and passes none.
using namespace rlx;
extern "C" int rlx_debug_ppo_head_gemm_ratio_f32(int64_t m, int32_t hidden, int32_t act_dim, const float* H2, const float* W3p, const float* W3c,
                                                 const float* b3p, const float* b3c, const float* logstd, const float* actions, const float* logp_old,
                                                 const float* adv, const float* ret, const float* adv_stats, float inv_mg, float clip_range,
                                                 float critic_coef, int32_t ratio_delta_metric, float* dZ2, float* dhead, float* headpart,
                                                 float* ratio_abs, float* scratch, void* stream) {
  RLX_CHECK_ARG(m > 0 && hidden > 0 && act_dim > 0 && act_dim <= 64, "bad sizes");
  RLX_CHECK_ARG(H2 && W3p && W3c && b3p && b3c && logstd && actions && logp_old && adv && ret && adv_stats && dZ2 && dhead && headpart && scratch,
                "null pointer");
  rlx::HeadGemmArgs a{m, hidden, act_dim, (int)(rlx::ceil_div(act_dim + 1, 4) * 4), H2, W3p, W3c, b3p, b3c, logstd, actions, logp_old, adv, ret,
                      adv_stats, inv_mg, clip_range, critic_coef, ratio_delta_metric, dZ2, dhead, headpart, ratio_abs, scratch};
  return rlx::ppo_head_gemm_path(a, (cudaStream_t)stream);
}

extern "C" int rlx_debug_ppo_head_gemm_f32(int64_t m, int32_t hidden, int32_t act_dim, const float* H2, const float* W3p, const float* W3c,
                                           const float* b3p, const float* b3c, const float* logstd, const float* actions, const float* logp_old,
                                           const float* adv, const float* ret, const float* adv_stats, float inv_mg, float clip_range,
                                           float critic_coef, int32_t ratio_delta_metric, float* dZ2, float* dhead, float* headpart, float* scratch,
                                           void* stream) {
  return rlx_debug_ppo_head_gemm_ratio_f32(m, hidden, act_dim, H2, W3p, W3c, b3p, b3c, logstd, actions, logp_old, adv, ret, adv_stats, inv_mg,
                                           clip_range, critic_coef, ratio_delta_metric, dZ2, dhead, headpart, nullptr, scratch, stream);
}
