// Output-layer ("head") kernels of the PPO policy/critic MLP pair.
//
// The last layers are skinny (hidden -> act and hidden -> 1), i.e. HBM-bound row reductions, so they are not run as
// GEMMs: one warp owns one row of the second hidden activation H2 = [H2p | H2c] ([M, 2H]), computes the act+1 dot
// products with warp-shuffle reductions and then everything that hangs off them in registers:
//   rollout head : action sampling, log-prob, action clip/rescale, value         (ref: policy.py:61-73, critic.py:44-46)
//   train head   : log-prob, ratio, clipped surrogate, value loss, their gradients wrt mean / logstd / value, the
//                  back-propagated dZ2 = dH2 * (1 - H2^2) and the metric sums   (ref: ppo.py:121-141,153-157)
#pragma once
#include "common.cuh"

namespace rlx {

constexpr float kLogSqrt2Pi = 0.91893853320467274178f;  // log(sqrt(2*pi)), torch/distributions/normal.py:101

// ---------------------------------------------------------------------------- counter-based normal generator
__device__ __forceinline__ void philox4x32_10(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c[0]), lo0 = 0xD2511F53u * c[0];
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c[2]), lo1 = 0xCD9E8D57u * c[2];
    const uint32_t n0 = hi1 ^ c[1] ^ k0, n1 = lo1, n2 = hi0 ^ c[3] ^ k1, n3 = lo0;
    c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
}
// Standard normal number `j` of row `row` for call `offset` under `seed` (Box-Muller on Philox output).
__device__ __forceinline__ float philox_normal(uint64_t seed, uint64_t offset, uint32_t row, uint32_t j) {
  uint32_t c[4] = {row, j >> 2, (uint32_t)offset, (uint32_t)(offset >> 32)};
  philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32));
  const uint32_t a = (j & 2) ? c[2] : c[0], b = (j & 2) ? c[3] : c[1];
  const float u1 = ((float)a + 0.5f) * 2.3283064365386963e-10f;  // (0, 1]
  const float u2 = ((float)b + 0.5f) * 2.3283064365386963e-10f;
  const float r = sqrtf(-2.f * logf(fminf(u1, 1.f)));
  float s, co;
  sincospif(2.f * u2, &s, &co);
  return (j & 1) ? r * s : r * co;
}

struct HeadP {
  int M, H, act;
  const float* H2;      // [M, 2H]
  const float* W3p;     // [act, H]
  const float* W3c;     // [H]
  const float* b3p;     // [act]
  const float* b3c;     // [1]
  const float* logstd;  // [act]
  // rollout
  const float* noise;   // [M, act] or null
  unsigned long long seed, offset;
  const float* act_low;
  const float* act_high;
  int clip_rescale, deterministic;
  float* action;        // [M, act]
  float* env_action;    // [M, act]
  float* logp_out;      // [M]
  float* value_out;     // [M]
  // train
  const float* actions; // [M, act]
  const float* logp_old;
  const float* adv;
  const float* ret;
  const float* adv_stats;  // [2]
  float inv_mg;            // 1 / m_global
  float clip_range, critic_coef;
  int ratio_delta_metric;  // != 0: the clip-fraction slot accumulates |ratio - 1| instead (ESPO, espo.py:133)
  float* ratio_abs;        // optional [M]: |ratio - 1| of every row (ESPO's delta_calc_operator = median needs the individual values)
  float* dZ2;              // [M, 2H]
  float* dhead;            // [M, act+1]   (dmean | dv)
  float* block_partials;   // [gridDim.x, 2*act+5+2H]  (db3p | db3c | dlogstd | pg | vloss | kl | clipfrac | db2p[H] | db2c[H])
  int bf16;                // (informational; the kernels are compiled per mode) bf16-autocast mode: the mean / value (outputs of the last Linear) are bf16 tensors, and so are the gradients that
                           // flow back into them and through them (d mean, d value, the linear-backward output and tanh_backward's output)
};

// Loads the row's H2 slices and returns the act means (lane a holds mean a; a+32 in mean_hi) and the value (all lanes).
template <int NCH, bool BF16>
__device__ __forceinline__ void head_row_forward(const HeadP& p, const float* __restrict__ sW3p, const float* __restrict__ sW3c,
                                                 long long row, int lane, float (&hp)[NCH], float (&hc)[NCH], float& mean_lo,
                                                 float& mean_hi, float& value) {
  const float* __restrict__ h = p.H2 + row * (2LL * p.H);
#pragma unroll
  for (int c = 0; c < NCH; ++c) {
    const int j = lane + 32 * c;
    hp[c] = (j < p.H) ? h[j] : 0.f;
    hc[c] = (j < p.H) ? h[p.H + j] : 0.f;
  }
  mean_lo = 0.f;
  mean_hi = 0.f;
  for (int a = 0; a < p.act; ++a) {
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      const int j = lane + 32 * c;
      if (j < p.H) s = fmaf(hp[c], sW3p[a * p.H + j], s);
    }
    s = bf16r_if(warp_sum(s) + p.b3p[a], BF16);
    if (lane == (a & 31)) {
      if (a < 32) mean_lo = s; else mean_hi = s;
    }
  }
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < NCH; ++c) {
    const int j = lane + 32 * c;
    if (j < p.H) s = fmaf(hc[c], sW3c[j], s);
  }
  value = bf16r_if(warp_sum(s) + p.b3c[0], BF16);
}

__device__ __forceinline__ void head_stage_weights(const HeadP& p, float* sW3p, float* sW3c) {
  for (int i = threadIdx.x; i < p.act * p.H; i += blockDim.x) sW3p[i] = p.W3p[i];
  for (int i = threadIdx.x; i < p.H; i += blockDim.x) sW3c[i] = p.W3c[i];
  __syncthreads();
}

// ------------------------------------------------------------------------------------------------ rollout head
template <int NCH, bool BF16 = false>
__global__ void __launch_bounds__(256) ppo_head_rollout_kernel(const HeadP p) {
  extern __shared__ float smem[];
  float* sW3p = smem;
  float* sW3c = smem + p.act * p.H;
  head_stage_weights(p, sW3p, sW3c);
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (long long row = (long long)blockIdx.x * nw + wib; row < p.M; row += (long long)gridDim.x * nw) {
    float hp[NCH], hc[NCH], mean_lo, mean_hi, value;
    head_row_forward<NCH, BF16>(p, sW3p, sW3c, row, lane, hp, hc, mean_lo, mean_hi, value);
    if (p.value_out && lane == 0) p.value_out[row] = value;
    float lp_sum = 0.f;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int a = lane + 32 * half;
      if (a < p.act) {
        const float mean = half ? mean_hi : mean_lo;
        float x = mean;
        if (!p.deterministic) {
          const float ls = p.logstd[a];
          const float sd = expf(ls);
          const float eps = p.noise ? p.noise[row * p.act + a] : philox_normal(p.seed, p.offset, (uint32_t)row, (uint32_t)a);
          const float var = sd * sd;
          if (BF16) {
            // Normal(bf16 loc, fp32 scale).sample() = at::normal(loc, scale): a tensor of loc's dtype filled with N(0,1) draws, then
            // .mul_(scale).add_(loc) in place - three bf16 roundings; log_prob sees (value - loc) and its square as bf16 tensors
            x = bf16r(__fadd_rn(bf16r(__fmul_rn(bf16r(eps), sd)), mean));
            const float d2 = bf16r(bf16r(x - mean) * bf16r(x - mean));
            lp_sum += -d2 / (2.f * var) - logf(sd) - kLogSqrt2Pi;
          } else {
            x = __fadd_rn(mean, __fmul_rn(sd, eps));  // Normal.sample(): loc + scale * eps  (no FMA contraction)
            // Normal.log_prob (torch/distributions/normal.py:87-103)
            const float d = x - mean;
            lp_sum += -(d * d) / (2.f * var) - logf(sd) - kLogSqrt2Pi;
          }
        }
        if (p.action) p.action[row * p.act + a] = x;
        if (p.env_action) {
          float e = x;
          if (p.clip_rescale) {  // policy.py:68-70
            const float c = fminf(fmaxf(x, -1.f), 1.f);
            const float lo = p.act_low[a], hi = p.act_high[a];
            e = lo + bf16r_if(0.5f * bf16r_if(c + 1.f, BF16), BF16) * (hi - lo);  // bf16 mode: clipped + 1.0 and 0.5 * (...) stay bf16 tensors
          }
          p.env_action[row * p.act + a] = e;
        }
      }
    }
    if (!p.deterministic && p.logp_out) {
      lp_sum = warp_sum(lp_sum);
      if (lane == 0) p.logp_out[row] = lp_sum;
    }
  }
}

// -------------------------------------------------------------------------------------------------- train head
template <int NCH, bool BF16 = false>
__global__ void __launch_bounds__(256) ppo_head_train_kernel(const HeadP p) {
  extern __shared__ float smem[];
  float* sW3p = smem;
  float* sW3c = smem + p.act * p.H;
  float* sred = sW3c + p.H;  // [nw][2*act+5+2H]
  head_stage_weights(p, sW3p, sW3c);
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int npart = 2 * p.act + 5 + 2 * p.H;
  float acc_db2p[NCH], acc_db2c[NCH];  // column sums of dZ2 = layer-2 bias gradients (lane owns columns lane + 32c)
#pragma unroll
  for (int c = 0; c < NCH; ++c) acc_db2p[c] = acc_db2c[c] = 0.f;

  const float adv_mean = p.adv_stats[0];
  const float adv_den = p.adv_stats[1] + 1e-8f;  // ppo.py:134
  const float clip_lo = 1.f - p.clip_range, clip_hi = 1.f + p.clip_range;

  // per-lane accumulators: lane a holds component a (and a+32)
  float acc_db3p[2] = {0.f, 0.f}, acc_dls[2] = {0.f, 0.f};
  float acc_db3c = 0.f, acc_pg = 0.f, acc_vl = 0.f, acc_kl = 0.f, acc_cf = 0.f;

  for (long long row = (long long)blockIdx.x * nw + wib; row < p.M; row += (long long)gridDim.x * nw) {
    float hp[NCH], hc[NCH], mean_lo, mean_hi, value;
    head_row_forward<NCH, BF16>(p, sW3p, sW3c, row, lane, hp, hc, mean_lo, mean_hi, value);

    // new log-prob (policy.py:76-82)
    float dmu[2] = {0.f, 0.f}, zz[2] = {0.f, 0.f};  // (x-mean)/var and (x-mean)^2/var per owned component
    float lp = 0.f;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int a = lane + 32 * half;
      if (a < p.act) {
        const float mean = half ? mean_hi : mean_lo;
        const float sd = expf(p.logstd[a]);
        const float var = sd * sd;
        const float d = p.actions[row * p.act + a] - mean;
        lp += -(d * d) / (2.f * var) - logf(sd) - kLogSqrt2Pi;
        dmu[half] = d / var;
        zz[half] = d * d / var;
      }
    }
    const float logp_new = warp_sum(lp);
    const float logratio = logp_new - p.logp_old[row];
    const float ratio = expf(logratio);
    const float A = (p.adv[row] - adv_mean) / adv_den;
    const float pg1 = -A * ratio;
    const float pg2 = -A * fminf(fmaxf(ratio, clip_lo), clip_hi);
    const float pg = fmaxf(pg1, pg2);
    // d pg / d ratio: torch.maximum splits ties evenly, clamp passes gradient on the closed interval.
    const float w1 = (pg1 > pg2) ? 1.f : ((pg1 == pg2) ? 0.5f : 0.f);
    const float inr = (ratio >= clip_lo && ratio <= clip_hi) ? 1.f : 0.f;
    const float dratio = -A * (w1 + (1.f - w1) * inr);
    const float dlogp = dratio * ratio * p.inv_mg;
    const float verr = value - p.ret[row];
    const float dv = bf16r_if(p.critic_coef * verr * p.inv_mg, BF16);

    acc_pg += pg;
    acc_vl += 0.5f * verr * verr;
    acc_kl += (ratio - 1.f) - logratio;
    acc_cf += p.ratio_delta_metric ? fabsf(ratio - 1.f) : ((fabsf(ratio - 1.f) > p.clip_range) ? 1.f : 0.f);
    if (p.ratio_abs != nullptr && lane == 0) p.ratio_abs[row] = fabsf(ratio - 1.f);
    acc_db3c += dv;

    float dmean[2];
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      dmean[half] = bf16r_if(dlogp * dmu[half], BF16);
      acc_db3p[half] += dmean[half];
      acc_dls[half] += dlogp * (zz[half] - 1.f);  // d logp / d logstd = (x-mean)^2/var - 1
      const int a = lane + 32 * half;
      if (a < p.act) p.dhead[row * (p.act + 1) + a] = dmean[half];
    }
    if (lane == 0) p.dhead[row * (p.act + 1) + p.act] = dv;

    // dZ2 = (dhead @ W3) * (1 - H2^2)
    float dz[NCH];
#pragma unroll
    for (int c = 0; c < NCH; ++c) dz[c] = 0.f;
    for (int a = 0; a < p.act; ++a) {
      const float g = __shfl_sync(0xffffffffu, (a < 32) ? dmean[0] : dmean[1], a & 31);
#pragma unroll
      for (int c = 0; c < NCH; ++c) {
        const int j = lane + 32 * c;
        if (j < p.H) dz[c] = fmaf(g, sW3p[a * p.H + j], dz[c]);
      }
    }
    float* __restrict__ out = p.dZ2 + row * (2LL * p.H);
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      const int j = lane + 32 * c;
      if (j < p.H) {
        const float zp = bf16r_if(bf16r_if(dz[c], BF16) * (1.f - hp[c] * hp[c]), BF16);
        const float zc = bf16r_if(bf16r_if(dv * sW3c[j], BF16) * (1.f - hc[c] * hc[c]), BF16);
        out[j] = zp;
        out[p.H + j] = zc;
        acc_db2p[c] += zp;
        acc_db2c[c] += zc;
      }
    }
  }

  // ---- block reduction of the per-warp accumulators (fixed order => deterministic)
  float* my = sred + wib * npart;
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const int a = lane + 32 * half;
    if (a < p.act) {
      my[a] = acc_db3p[half];
      my[p.act + 1 + a] = acc_dls[half];
    }
  }
  if (lane == 0) {
    my[p.act] = acc_db3c;
    my[2 * p.act + 1] = acc_pg;
    my[2 * p.act + 2] = acc_vl;
    my[2 * p.act + 3] = acc_kl;
    my[2 * p.act + 4] = acc_cf;
  }
#pragma unroll
  for (int c = 0; c < NCH; ++c) {
    const int j = lane + 32 * c;
    if (j < p.H) {
      my[2 * p.act + 5 + j] = acc_db2p[c];
      my[2 * p.act + 5 + p.H + j] = acc_db2c[c];
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < npart; i += blockDim.x) {
    float s = 0.f;
    for (int w = 0; w < nw; ++w) s += sred[w * npart + i];
    p.block_partials[(long long)blockIdx.x * npart + i] = s;
  }
}

// ------------------------------------------------------------------------------------- train head, fast variant
// Same math as ppo_head_train_kernel, restructured for throughput (act <= 31, i.e. act+1 outputs fit one warp):
//   * two rows per warp iteration: every W3 element fetched from shared memory feeds two FMAs (the kernel is LDS-bound otherwise)
//   * the act+1 dot products are reduced with a halving butterfly (31 shuffles instead of 5 per output); it leaves output a in
//     lane a, which is exactly the ownership the loss code wants
//   * everything is unrolled at compile time (ACT_MAX) so the independent chains overlap
// dhead is written with a 16-byte-aligned pitch dh_ld = round_up(act+1, 4) for the vectorised weight-gradient kernel below.
template <int NV>
__device__ __forceinline__ void butterfly_step(float (&v)[32], int lane) {
  constexpr int HALF = NV / 2;
  const bool up = (lane & HALF) != 0;
#pragma unroll
  for (int j = 0; j < HALF; ++j) {
    const float a = v[j], b = v[j + HALF];
    const float send = up ? a : b, keep = up ? b : a;
    v[j] = keep + __shfl_xor_sync(0xffffffffu, send, HALF);
  }
}
// v[i] (i < 32) summed over the warp; on return lane l holds the total of index l in v[0].
__device__ __forceinline__ float butterfly_reduce32(float (&v)[32], int lane) {
  butterfly_step<32>(v, lane);
  butterfly_step<16>(v, lane);
  butterfly_step<8>(v, lane);
  butterfly_step<4>(v, lane);
  butterfly_step<2>(v, lane);
  return v[0];
}

struct HeadTrain2Extra {
  int dh_ld;  // pitch of dhead rows
};

template <int NCH, int ACT_MAX, bool BF16 = false>
__global__ void __launch_bounds__(256, 2) ppo_head_train2_kernel(const HeadP p, const HeadTrain2Extra ex) {
  extern __shared__ float smem[];
  float* sW3p = smem;
  float* sW3c = smem + p.act * p.H;
  float* sred = sW3c + p.H;
  head_stage_weights(p, sW3p, sW3c);
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int npart = 2 * p.act + 5 + 2 * p.H;
  const int act = p.act, H = p.H;
  const float adv_mean = p.adv_stats[0];
  const float adv_den = p.adv_stats[1] + 1e-8f;
  const float clip_lo = 1.f - p.clip_range, clip_hi = 1.f + p.clip_range;
  // per-lane constants of the component this lane owns
  const bool own = lane < act;
  const float my_b3 = own ? p.b3p[lane] : ((lane == act) ? p.b3c[0] : 0.f);
  const float my_sd = own ? expf(p.logstd[lane]) : 1.f;
  const float my_var = my_sd * my_sd;
  const float my_logsd = logf(my_sd);

  float acc_db2p[NCH], acc_db2c[NCH];
#pragma unroll
  for (int c = 0; c < NCH; ++c) acc_db2p[c] = acc_db2c[c] = 0.f;
  float acc_db3 = 0.f, acc_dls = 0.f;  // lane a: db3p[a] / dlogstd[a]; lane act: db3c
  float acc_pg = 0.f, acc_vl = 0.f, acc_kl = 0.f, acc_cf = 0.f;

  const long long npairs = ((long long)p.M + 1) / 2;
  for (long long pr = (long long)blockIdx.x * nw + wib; pr < npairs; pr += (long long)gridDim.x * nw) {
    const long long row0 = 2 * pr;
    const bool has1 = row0 + 1 < p.M;
    float hp[2][NCH], hc[2][NCH];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float* __restrict__ h = p.H2 + (row0 + ((r == 1 && !has1) ? 0 : r)) * (2LL * H);
#pragma unroll
      for (int c = 0; c < NCH; ++c) {
        const int j = lane + 32 * c;
        hp[r][c] = (j < H) ? h[j] : 0.f;
        hc[r][c] = (j < H) ? h[H + j] : 0.f;
      }
    }
    // ---- act+1 partial dot products per row, W3 fetched once for both rows
    float v0[32], v1[32];
#pragma unroll
    for (int a = 0; a < 32; ++a) v0[a] = v1[a] = 0.f;
#pragma unroll
    for (int a = 0; a < ACT_MAX; ++a) {
      if (a < act) {
        float s0 = 0.f, s1 = 0.f;
#pragma unroll
        for (int c = 0; c < NCH; ++c) {
          const int j = lane + 32 * c;
          const float w = (j < H) ? sW3p[a * H + j] : 0.f;
          s0 = fmaf(hp[0][c], w, s0);
          s1 = fmaf(hp[1][c], w, s1);
        }
        v0[a] = s0;
        v1[a] = s1;
      }
    }
    {
      float s0 = 0.f, s1 = 0.f;
#pragma unroll
      for (int c = 0; c < NCH; ++c) {
        const int j = lane + 32 * c;
        const float w = (j < H) ? sW3c[j] : 0.f;
        s0 = fmaf(hc[0][c], w, s0);
        s1 = fmaf(hc[1][c], w, s1);
      }
      // the value head rides in slot `act` (act <= 31)
#pragma unroll
      for (int a = 0; a < 32; ++a)
        if (a == act) { v0[a] = s0; v1[a] = s1; }
    }
    const float out0 = bf16r_if(butterfly_reduce32(v0, lane) + my_b3, BF16);  // lane a < act: mean_a; lane act: value (bf16 tensors in bf16 mode)
    const float out1 = bf16r_if(butterfly_reduce32(v1, lane) + my_b3, BF16);

    float dmean[2], dvv[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const long long row = row0 + r;
      const bool valid = (r == 0) || has1;  // warp-uniform
      const float out = r ? out1 : out0;
      const float value = __shfl_sync(0xffffffffu, out, act);
      float lp = 0.f, dmu = 0.f, zz = 0.f;
      if (own && valid) {
        const float d = p.actions[row * act + lane] - out;
        lp = -(d * d) / (2.f * my_var) - my_logsd - kLogSqrt2Pi;
        dmu = d / my_var;
        zz = d * d / my_var;
      }
      const float logp_new = warp_sum(lp);
      float dm = 0.f, dv = 0.f;
      if (valid) {
        const float logratio = logp_new - p.logp_old[row];
        const float ratio = expf(logratio);
        const float A = (p.adv[row] - adv_mean) / adv_den;
        const float pg1 = -A * ratio;
        const float pg2 = -A * fminf(fmaxf(ratio, clip_lo), clip_hi);
        const float w1 = (pg1 > pg2) ? 1.f : ((pg1 == pg2) ? 0.5f : 0.f);
        const float inr = (ratio >= clip_lo && ratio <= clip_hi) ? 1.f : 0.f;
        const float dlogp = (-A * (w1 + (1.f - w1) * inr)) * ratio * p.inv_mg;
        const float verr = value - p.ret[row];
        dv = bf16r_if(p.critic_coef * verr * p.inv_mg, BF16);  // gradient of a bf16 tensor is a bf16 tensor
        acc_pg += fmaxf(pg1, pg2);
        acc_vl += 0.5f * verr * verr;
        acc_kl += (ratio - 1.f) - logratio;
        acc_cf += p.ratio_delta_metric ? fabsf(ratio - 1.f) : ((fabsf(ratio - 1.f) > p.clip_range) ? 1.f : 0.f);
        if (p.ratio_abs != nullptr && lane == 0) p.ratio_abs[row] = fabsf(ratio - 1.f);
        dm = bf16r_if(dlogp * dmu, BF16);
        if (own) {
          acc_db3 += dm;
          acc_dls += dlogp * (zz - 1.f);
          p.dhead[row * ex.dh_ld + lane] = dm;
        } else if (lane == act) {
          acc_db3 += dv;
          p.dhead[row * ex.dh_ld + act] = dv;
        } else if (lane < ex.dh_ld) {
          p.dhead[row * ex.dh_ld + lane] = 0.f;
        }
      }
      dmean[r] = dm;
      dvv[r] = dv;
    }
    // ---- dZ2 = (dhead @ W3) * (1 - H2^2) for both rows, W3 fetched once
    float dz0[NCH], dz1[NCH];
#pragma unroll
    for (int c = 0; c < NCH; ++c) dz0[c] = dz1[c] = 0.f;
#pragma unroll
    for (int a = 0; a < ACT_MAX; ++a) {
      if (a < act) {
        const float g0 = __shfl_sync(0xffffffffu, dmean[0], a);
        const float g1 = __shfl_sync(0xffffffffu, dmean[1], a);
#pragma unroll
        for (int c = 0; c < NCH; ++c) {
          const int j = lane + 32 * c;
          const float w = (j < H) ? sW3p[a * H + j] : 0.f;
          dz0[c] = fmaf(g0, w, dz0[c]);
          dz1[c] = fmaf(g1, w, dz1[c]);
        }
      }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      if (r == 1 && !has1) break;
      float* __restrict__ out = p.dZ2 + (row0 + r) * (2LL * H);
#pragma unroll
      for (int c = 0; c < NCH; ++c) {
        const int j = lane + 32 * c;
        if (j < H) {
          const float hpv = hp[r][c], hcv = hc[r][c];
          const float zp = bf16r_if(bf16r_if(r ? dz1[c] : dz0[c], BF16) * (1.f - hpv * hpv), BF16);  // linear-backward output, then tanh_backward
          const float zc = bf16r_if(bf16r_if(dvv[r] * sW3c[j], BF16) * (1.f - hcv * hcv), BF16);
          out[j] = zp;
          out[H + j] = zc;
          acc_db2p[c] += zp;
          acc_db2c[c] += zc;
        }
      }
    }
  }

  // ---- block reduction (fixed order => deterministic); partial layout as in ppo_head_train_kernel
  float* my = sred + wib * npart;
  if (own) {
    my[lane] = acc_db3;
    my[act + 1 + lane] = acc_dls;
  } else if (lane == act) {
    my[act] = acc_db3;
  }
  if (lane == 0) {
    my[2 * act + 1] = acc_pg;
    my[2 * act + 2] = acc_vl;
    my[2 * act + 3] = acc_kl;
    my[2 * act + 4] = acc_cf;
  }
#pragma unroll
  for (int c = 0; c < NCH; ++c) {
    const int j = lane + 32 * c;
    if (j < H) {
      my[2 * act + 5 + j] = acc_db2p[c];
      my[2 * act + 5 + H + j] = acc_db2c[c];
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < npart; i += blockDim.x) {
    float s = 0.f;
    for (int w = 0; w < nw; ++w) s += sred[w * npart + i];
    p.block_partials[(long long)blockIdx.x * npart + i] = s;
  }
}

// ------------------------------------------------------- weight gradient of the head, fast variant (register tiled)
// dW3 = dhead^T [act+1, M] . H2 [M, 2H].  Thread t owns policy columns {2t, 2t+1} and critic columns {H+2t, H+2t+1}
// (64-bit coalesced loads); the act+1 gradient scalars of a row are broadcast from shared memory as float4.
// part[chunk][(act+1)*H]: rows 0..act-1 = dW3p, row act = dW3c.
struct HeadWgrad2P {
  int M, H, act, dh_ld, rows_per_chunk;
  const float* H2;
  const float* dhead;  // [M, dh_ld]
  float* part;
};

template <int ACT_MAX>  // multiple of 4, >= act + 1
__global__ void __launch_bounds__(512) ppo_head_wgrad2_kernel(const HeadWgrad2P p) {
  extern __shared__ __align__(16) float sd[];  // [rows_per_chunk][dh_ld]
  const int chunk = blockIdx.x;
  const long long r0 = (long long)chunk * p.rows_per_chunk;
  const int nrows = (int)min((long long)p.rows_per_chunk, (long long)p.M - r0);
  for (int i = threadIdx.x; i < nrows * p.dh_ld; i += blockDim.x) sd[i] = p.dhead[r0 * p.dh_ld + i];
  __syncthreads();
  const int t = threadIdx.x;
  if (2 * t >= p.H) return;
  float accp[ACT_MAX][2], accc[2] = {0.f, 0.f};
#pragma unroll
  for (int a = 0; a < ACT_MAX; ++a) accp[a][0] = accp[a][1] = 0.f;
  const float* __restrict__ base = p.H2 + r0 * (2LL * p.H) + 2 * t;
#pragma unroll 2
  for (int r = 0; r < nrows; ++r) {
    const float2 hpv = *reinterpret_cast<const float2*>(base + (long long)r * 2 * p.H);
    const float2 hcv = *reinterpret_cast<const float2*>(base + (long long)r * 2 * p.H + p.H);
    const float4* dr = reinterpret_cast<const float4*>(sd + r * p.dh_ld);
    float d[ACT_MAX];
#pragma unroll
    for (int q = 0; q < ACT_MAX / 4; ++q) {
      if (4 * q < p.dh_ld) {
        const float4 v = dr[q];
        d[4 * q] = v.x; d[4 * q + 1] = v.y; d[4 * q + 2] = v.z; d[4 * q + 3] = v.w;
      } else {
        d[4 * q] = d[4 * q + 1] = d[4 * q + 2] = d[4 * q + 3] = 0.f;
      }
    }
    float dv = 0.f;
#pragma unroll
    for (int a = 0; a < ACT_MAX; ++a) {
      if (a < p.act) {
        accp[a][0] = fmaf(d[a], hpv.x, accp[a][0]);
        accp[a][1] = fmaf(d[a], hpv.y, accp[a][1]);
      } else if (a == p.act) {
        dv = d[a];
      }
    }
    accc[0] = fmaf(dv, hcv.x, accc[0]);
    accc[1] = fmaf(dv, hcv.y, accc[1]);
  }
  float* out = p.part + (long long)chunk * (p.act + 1) * p.H + 2 * t;
#pragma unroll
  for (int a = 0; a < ACT_MAX; ++a)
    if (a < p.act) *reinterpret_cast<float2*>(out + (long long)a * p.H) = make_float2(accp[a][0], accp[a][1]);
  *reinterpret_cast<float2*>(out + (long long)p.act * p.H) = make_float2(accc[0], accc[1]);
}

// ------------------------------------------------------------ train head, vectorised variant (H multiple of 128)
// Lane l owns the 4-column groups {g*128 + 4l .. +3}: H2 / dZ2 rows move as coalesced 128-bit accesses and every W3 fetch is
// one conflict-free LDS.128 that feeds 8 FMAs (2 rows x 4 columns).  ~1.3k warp instructions per row pair (the scalar variant
// above needs ~7k: it is issue-bound).
__device__ __forceinline__ float dot4(const float4& a, const float4& b, float s) {
  s = fmaf(a.x, b.x, s); s = fmaf(a.y, b.y, s); s = fmaf(a.z, b.z, s); return fmaf(a.w, b.w, s);
}
__device__ __forceinline__ void axpy4(float g, const float4& w, float4& d) {
  d.x = fmaf(g, w.x, d.x); d.y = fmaf(g, w.y, d.y); d.z = fmaf(g, w.z, d.z); d.w = fmaf(g, w.w, d.w);
}

template <int H_, int ACT_MAX, bool BF16 = false>
__global__ void __launch_bounds__(256, 2) ppo_head_train3_kernel(const HeadP p, const HeadTrain2Extra ex) {
  constexpr int NG = H_ / 128;
  constexpr int H4 = H_ / 4;
  extern __shared__ __align__(16) float smem[];
  float* sW3p = smem;
  float* sW3c = smem + p.act * H_;
  float* sred = sW3c + H_;
  head_stage_weights(p, sW3p, sW3c);
  const float4* sW3p4 = reinterpret_cast<const float4*>(sW3p);
  const float4* sW3c4 = reinterpret_cast<const float4*>(sW3c);
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int act = p.act;
  const int npart = 2 * act + 5 + 2 * H_;
  const float adv_mean = p.adv_stats[0];
  const float adv_den = p.adv_stats[1] + 1e-8f;
  const float clip_lo = 1.f - p.clip_range, clip_hi = 1.f + p.clip_range;
  const bool own = lane < act;
  const float my_b3 = own ? p.b3p[lane] : ((lane == act) ? p.b3c[0] : 0.f);
  const float my_sd = own ? expf(p.logstd[lane]) : 1.f;
  const float my_var = my_sd * my_sd;
  const float my_logsd = logf(my_sd);

  float4 acc_db2p[NG], acc_db2c[NG];
#pragma unroll
  for (int g = 0; g < NG; ++g) acc_db2p[g] = acc_db2c[g] = make_float4(0.f, 0.f, 0.f, 0.f);
  float acc_db3 = 0.f, acc_dls = 0.f, acc_pg = 0.f, acc_vl = 0.f, acc_kl = 0.f, acc_cf = 0.f;

  const long long npairs = ((long long)p.M + 1) / 2;
  for (long long pr = (long long)blockIdx.x * nw + wib; pr < npairs; pr += (long long)gridDim.x * nw) {
    const long long row0 = 2 * pr;
    const bool has1 = row0 + 1 < p.M;
    float4 hp[2][NG], hc[2][NG];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float4* __restrict__ h = reinterpret_cast<const float4*>(p.H2 + (row0 + ((r == 1 && !has1) ? 0 : r)) * (2LL * H_));
#pragma unroll
      for (int g = 0; g < NG; ++g) {
        hp[r][g] = h[g * 32 + lane];
        hc[r][g] = h[H4 + g * 32 + lane];
      }
    }
    float v0[32], v1[32];
#pragma unroll
    for (int a = 0; a < 32; ++a) v0[a] = v1[a] = 0.f;
#pragma unroll
    for (int a = 0; a < ACT_MAX; ++a) {
      if (a < act) {
        float s0 = 0.f, s1 = 0.f;
#pragma unroll
        for (int g = 0; g < NG; ++g) {
          const float4 w = sW3p4[a * H4 + g * 32 + lane];
          s0 = dot4(hp[0][g], w, s0);
          s1 = dot4(hp[1][g], w, s1);
        }
        v0[a] = s0;
        v1[a] = s1;
      }
    }
    {
      float s0 = 0.f, s1 = 0.f;
#pragma unroll
      for (int g = 0; g < NG; ++g) {
        const float4 w = sW3c4[g * 32 + lane];
        s0 = dot4(hc[0][g], w, s0);
        s1 = dot4(hc[1][g], w, s1);
      }
#pragma unroll
      for (int a = 0; a < 32; ++a)
        if (a == act) { v0[a] = s0; v1[a] = s1; }
    }
    const float out0 = bf16r_if(butterfly_reduce32(v0, lane) + my_b3, BF16);  // lane a < act: mean_a; lane act: value (bf16 tensors in bf16 mode)
    const float out1 = bf16r_if(butterfly_reduce32(v1, lane) + my_b3, BF16);

    float dmean[2], dvv[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const long long row = row0 + r;
      const bool valid = (r == 0) || has1;  // warp-uniform
      const float out = r ? out1 : out0;
      const float value = __shfl_sync(0xffffffffu, out, act);
      float lp = 0.f, dmu = 0.f, zz = 0.f;
      if (own && valid) {
        const float d = p.actions[row * act + lane] - out;
        lp = -(d * d) / (2.f * my_var) - my_logsd - kLogSqrt2Pi;
        dmu = d / my_var;
        zz = d * d / my_var;
      }
      const float logp_new = warp_sum(lp);
      float dm = 0.f, dv = 0.f;
      if (valid) {
        const float logratio = logp_new - p.logp_old[row];
        const float ratio = expf(logratio);
        const float A = (p.adv[row] - adv_mean) / adv_den;
        const float pg1 = -A * ratio;
        const float pg2 = -A * fminf(fmaxf(ratio, clip_lo), clip_hi);
        const float w1 = (pg1 > pg2) ? 1.f : ((pg1 == pg2) ? 0.5f : 0.f);
        const float inr = (ratio >= clip_lo && ratio <= clip_hi) ? 1.f : 0.f;
        const float dlogp = (-A * (w1 + (1.f - w1) * inr)) * ratio * p.inv_mg;
        const float verr = value - p.ret[row];
        dv = bf16r_if(p.critic_coef * verr * p.inv_mg, BF16);  // gradient of a bf16 tensor is a bf16 tensor
        acc_pg += fmaxf(pg1, pg2);
        acc_vl += 0.5f * verr * verr;
        acc_kl += (ratio - 1.f) - logratio;
        acc_cf += p.ratio_delta_metric ? fabsf(ratio - 1.f) : ((fabsf(ratio - 1.f) > p.clip_range) ? 1.f : 0.f);
        if (p.ratio_abs != nullptr && lane == 0) p.ratio_abs[row] = fabsf(ratio - 1.f);
        dm = bf16r_if(dlogp * dmu, BF16);
        if (own) {
          acc_db3 += dm;
          acc_dls += dlogp * (zz - 1.f);
          p.dhead[row * ex.dh_ld + lane] = dm;
        } else if (lane == act) {
          acc_db3 += dv;
          p.dhead[row * ex.dh_ld + act] = dv;
        } else if (lane < ex.dh_ld) {
          p.dhead[row * ex.dh_ld + lane] = 0.f;
        }
      }
      dmean[r] = dm;
      dvv[r] = dv;
    }
    // ---- dZ2 = (dhead @ W3) * (1 - H2^2)
    float4 dz0[NG], dz1[NG];
#pragma unroll
    for (int g = 0; g < NG; ++g) dz0[g] = dz1[g] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int a = 0; a < ACT_MAX; ++a) {
      if (a < act) {
        const float g0 = __shfl_sync(0xffffffffu, dmean[0], a);
        const float g1 = __shfl_sync(0xffffffffu, dmean[1], a);
#pragma unroll
        for (int g = 0; g < NG; ++g) {
          const float4 w = sW3p4[a * H4 + g * 32 + lane];
          axpy4(g0, w, dz0[g]);
          axpy4(g1, w, dz1[g]);
        }
      }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      if (r == 1 && !has1) break;
      float4* __restrict__ out = reinterpret_cast<float4*>(p.dZ2 + (row0 + r) * (2LL * H_));
#pragma unroll
      for (int g = 0; g < NG; ++g) {
        const float4 a4 = hp[r][g], c4 = hc[r][g], d4 = r ? dz1[g] : dz0[g], wc = sW3c4[g * 32 + lane];
        float4 zp, zc;
        constexpr int bf = BF16 ? 1 : 0;  // bf16 mode: the linear-backward output and tanh_backward's output are bf16 tensors
        zp.x = bf16r_if(bf16r_if(d4.x, bf) * (1.f - a4.x * a4.x), bf); zp.y = bf16r_if(bf16r_if(d4.y, bf) * (1.f - a4.y * a4.y), bf);
        zp.z = bf16r_if(bf16r_if(d4.z, bf) * (1.f - a4.z * a4.z), bf); zp.w = bf16r_if(bf16r_if(d4.w, bf) * (1.f - a4.w * a4.w), bf);
        zc.x = bf16r_if(bf16r_if(dvv[r] * wc.x, bf) * (1.f - c4.x * c4.x), bf); zc.y = bf16r_if(bf16r_if(dvv[r] * wc.y, bf) * (1.f - c4.y * c4.y), bf);
        zc.z = bf16r_if(bf16r_if(dvv[r] * wc.z, bf) * (1.f - c4.z * c4.z), bf); zc.w = bf16r_if(bf16r_if(dvv[r] * wc.w, bf) * (1.f - c4.w * c4.w), bf);
        out[g * 32 + lane] = zp;
        out[H4 + g * 32 + lane] = zc;
        acc_db2p[g].x += zp.x; acc_db2p[g].y += zp.y; acc_db2p[g].z += zp.z; acc_db2p[g].w += zp.w;
        acc_db2c[g].x += zc.x; acc_db2c[g].y += zc.y; acc_db2c[g].z += zc.z; acc_db2c[g].w += zc.w;
      }
    }
  }

  float* my = sred + wib * npart;
  if (own) {
    my[lane] = acc_db3;
    my[act + 1 + lane] = acc_dls;
  } else if (lane == act) {
    my[act] = acc_db3;
  }
  if (lane == 0) {
    my[2 * act + 1] = acc_pg;
    my[2 * act + 2] = acc_vl;
    my[2 * act + 3] = acc_kl;
    my[2 * act + 4] = acc_cf;
  }
#pragma unroll
  for (int g = 0; g < NG; ++g) {
    float* q = my + 2 * act + 5 + g * 128 + 4 * lane;
    q[0] = acc_db2p[g].x; q[1] = acc_db2p[g].y; q[2] = acc_db2p[g].z; q[3] = acc_db2p[g].w;
    q[H_] = acc_db2c[g].x; q[H_ + 1] = acc_db2c[g].y; q[H_ + 2] = acc_db2c[g].z; q[H_ + 3] = acc_db2c[g].w;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < npart; i += blockDim.x) {
    float s = 0.f;
    for (int w = 0; w < nw; ++w) s += sred[w * npart + i];
    p.block_partials[(long long)blockIdx.x * npart + i] = s;
  }
}

// ------------------------------------------ weight gradient of the head, one thread per (policy, critic) column pair
template <int ACT_MAX>  // multiple of 4, >= act + 1
__global__ void __launch_bounds__(1024) ppo_head_wgrad3_kernel(const HeadWgrad2P p) {
  extern __shared__ __align__(16) float sd[];  // [rows_per_chunk][dh_ld]
  const int chunk = blockIdx.x;
  const long long r0 = (long long)chunk * p.rows_per_chunk;
  const int nrows = (int)min((long long)p.rows_per_chunk, (long long)p.M - r0);
  for (int i = threadIdx.x; i < nrows * p.dh_ld; i += blockDim.x) sd[i] = p.dhead[r0 * p.dh_ld + i];
  __syncthreads();
  const int t = threadIdx.x;
  if (t >= p.H) return;
  float accp[ACT_MAX], accc = 0.f;
#pragma unroll
  for (int a = 0; a < ACT_MAX; ++a) accp[a] = 0.f;
  const float* __restrict__ base = p.H2 + r0 * (2LL * p.H) + t;
  const long long pitch = 2LL * p.H;
  int r = 0;
  for (; r + 4 <= nrows; r += 4) {
    float hpv[4], hcv[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      hpv[u] = base[(long long)(r + u) * pitch];
      hcv[u] = base[(long long)(r + u) * pitch + p.H];
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const float4* dr = reinterpret_cast<const float4*>(sd + (r + u) * p.dh_ld);
#pragma unroll
      for (int q = 0; q < ACT_MAX / 4; ++q) {
        if (4 * q < p.dh_ld) {
          const float4 v = dr[q];
          const float d[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int a = 4 * q + e;
            if (a < p.act) accp[a] = fmaf(d[e], hpv[u], accp[a]);
            else if (a == p.act) accc = fmaf(d[e], hcv[u], accc);
          }
        }
      }
    }
  }
  for (; r < nrows; ++r) {
    const float hpv = base[(long long)r * pitch], hcv = base[(long long)r * pitch + p.H];
#pragma unroll
    for (int a = 0; a < ACT_MAX; ++a) {
      if (a < p.act) accp[a] = fmaf(sd[r * p.dh_ld + a], hpv, accp[a]);
      else if (a == p.act) accc = fmaf(sd[r * p.dh_ld + a], hcv, accc);
    }
  }
  float* out = p.part + (long long)chunk * (p.act + 1) * p.H + t;
#pragma unroll
  for (int a = 0; a < ACT_MAX; ++a)
    if (a < p.act) out[(long long)a * p.H] = accp[a];
  out[(long long)p.act * p.H] = accc;
}

// ------------------------------------------------------------------ weight gradient of the head (thread per column)
// part[chunk][(act+1)*H]: rows 0..act-1 = dW3p, row act = dW3c, summed over the chunk's rows.
struct HeadWgradP {
  int M, H, act, rows_per_chunk;
  const float* H2;     // [M, 2H]
  const float* dhead;  // [M, act+1]
  float* part;         // [nchunk, (act+1)*H]
};

template <int ACTMAX>
__global__ void __launch_bounds__(256) ppo_head_wgrad_kernel(const HeadWgradP p) {
  extern __shared__ float sd[];  // [rows_per_chunk][act+1]
  const int chunk = blockIdx.x;
  const long long r0 = (long long)chunk * p.rows_per_chunk;
  const int nrows = (int)min((long long)p.rows_per_chunk, (long long)p.M - r0);
  const int w = p.act + 1;
  for (int i = threadIdx.x; i < nrows * w; i += blockDim.x) sd[i] = p.dhead[r0 * w + i];
  __syncthreads();
  const int jj = blockIdx.y * blockDim.x + threadIdx.x;  // column of H2 in [0, 2H)
  if (jj >= 2 * p.H) return;
  const bool is_pol = jj < p.H;
  float acc[ACTMAX];
#pragma unroll
  for (int a = 0; a < ACTMAX; ++a) acc[a] = 0.f;
  const float* __restrict__ col = p.H2 + r0 * (2LL * p.H) + jj;
  if (is_pol) {
#pragma unroll 4
    for (int r = 0; r < nrows; ++r) {
      const float h = col[(long long)r * 2 * p.H];
#pragma unroll
      for (int a = 0; a < ACTMAX; ++a)
        if (a < p.act) acc[a] = fmaf(sd[r * w + a], h, acc[a]);
    }
    float* out = p.part + (long long)chunk * w * p.H + jj;
#pragma unroll
    for (int a = 0; a < ACTMAX; ++a)
      if (a < p.act) out[(long long)a * p.H] = acc[a];
  } else {
    float s = 0.f;
#pragma unroll 4
    for (int r = 0; r < nrows; ++r) s = fmaf(sd[r * w + p.act], col[(long long)r * 2 * p.H], s);
    p.part[(long long)chunk * w * p.H + (long long)p.act * p.H + (jj - p.H)] = s;
  }
}

}  // namespace rlx
