// Interface of the GEMM-formulated PPO loss head (ppo_head_gemm.cu); plain types only, usable from the dual-build sources and from ppo.cu.
#pragma once

namespace rlx {

struct HeadGemmArgs {
  long long m;
  int H, A, dh_ld;
  const float* H2;        // [m, 2H] post-tanh activations, policy half | critic half
  const float *W3p, *W3c, *b3p, *b3c, *logstd;
  const float *actions, *logp_old, *adv, *ret, *adv_stats;
  float inv_mg, clip_range, critic_coef;
  int ratio_delta_metric;
  float* dZ2;             // [m, 2H] out
  float* dhead;           // [m, dh_ld] out: dMean | dV | zero padding
  float* headpart;        // [2A + 5 + 2H] out: db3p | db3c | dlogstd | pg | vl | kl | cf | db2p | db2c  (one block)
  float* ratio_abs;       // optional [m] out: |ratio - 1| of every row (ESPO's delta_calc_operator = median), or null
  float* scratch;        // >= m * (2A + 8) + (m / 256 + 2) * max(2H, 8) floats
};

// floats of `scratch` the path needs for m rows
inline long long head_gemm_scratch_floats(long long m, int H, int A) {
  const long long widest = 2LL * H > 8 ? 2LL * H : 8;
  return m * (2LL * A + 8) + (m / 256 + 2) * widest;
}

}  // namespace rlx
