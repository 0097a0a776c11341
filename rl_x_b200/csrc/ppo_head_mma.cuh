// Train head on the legacy tensor path (mma.sync m16n8k8, 3xTF32): rlx_set_head_engine(2).
//
// The fused SIMT head (ppo_head_train3_kernel) is issue-bound: ~1.1k warp instructions per row for 2 x 256 x 18 FMAs, several
// times the HBM time of a 32768-row minibatch.  Here the two skinny products
//     mean[M, act] = H2p[M, H] . W3p^T          and          dH2p[M, H] = dmean[M, act] . W3p
// run as warp-level MMAs on 16-row tiles, everything else (log-prob, ratio, surrogate, value loss, tanh', bias-gradient and metric
// partial sums) stays in the registers of the same kernel, in the same arithmetic as the SIMT head (ref: ppo.py:121-141,153-157).
//
// Fragment bookkeeping (lane = 4g + t).  The MMA's k and n indices are only summation / output labels, so they are permuted such
// that every global access is a 128-bit one and no register shuffles are needed:
//   forward, column block b (16 columns of H2), k-step e: logical k = t   <-> column 16b + 4t + 2e
//                                                          logical k = t+4 <-> column 16b + 4t + 2e + 1
//       => lane loads H2[row g | g+8][16b + 4t .. +3] as one float4 each and owns a0..a3 of both k-steps;
//          the B fragment of n-tile j is W3p[8j + g][16b + 4t .. +3], one LDS.128 from a row-padded table.
//   the C fragment of n-tile j holds mean[g | g+8][8j + 2t, 8j + 2t + 1]; with logical k = t <-> action 8j + 2t and
//   k = t+4 <-> action 8j + 2t + 1 the d-mean values sit exactly where the backward MMA's A fragment wants them.
//   backward, column block b, n-tile e: logical n = 2t' + f <-> column 16b + 4t' + 2e + f, so that the lane ends up with
//       dH2p[g | g+8][16b + 4t .. +3] (two n-tiles side by side) - again one float4 per row.
//
// A CTA works on 128-row super tiles.  Phase 1: warp w runs the forward + loss for rows 16w..16w+15 and leaves its d-mean fragments
// and dv in shared memory.  Phase 2: warp w owns the columns [w*H/8, (w+1)*H/8) of BOTH nets for all 128 rows, so that the
// column sums of dZ2 (= db2) need H/32 float4 accumulators per net instead of H/4.
#pragma once
#include "ppo_head.cuh"

namespace rlx {

__device__ __forceinline__ uint32_t to_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
  hi = to_tf32(x);
  lo = to_tf32(x - __uint_as_float(hi));
}
// D += A(16x8, row) . B(8x8, col), tf32 operands, fp32 accumulation
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

constexpr int kHead4RowTiles = 8;  // 16-row tiles per super tile = warps per CTA

// shared-memory floats of ppo_head_train4_kernel<H, NT>
static inline size_t head4_smem_floats(int H, int act, int NT) {
  const size_t tables = 2ull * act * (H + 16) + H;
  const size_t work = (size_t)(H / 16) * 2 * NT * 32 * 4 + (size_t)kHead4RowTiles * NT * 32 * 4 + kHead4RowTiles * 16;
  const size_t red = 8ull * (2 * act + 5 + 2 * H);
  return tables + (work > red ? work : red);
}

template <int H_, int NT>
__global__ void __launch_bounds__(256, 2) ppo_head_train4_kernel(const HeadP p, const HeadTrain2Extra ex) {
  constexpr int NB = H_ / 16;         // 16-column blocks per net
  constexpr int H4 = H_ / 4;
  constexpr int LDW4 = H4 + 4;        // float4 pitch of one W3p row in the forward tables (conflict-free LDS.128 across g)
  constexpr int RT = kHead4RowTiles;
  constexpr int BPW = NB / 8;         // column blocks per warp in phase 2
  static_assert(H_ % 128 == 0, "H must be a multiple of 128");
  extern __shared__ __align__(16) float smem[];
  const int act = p.act;
  float4* sWh4 = reinterpret_cast<float4*>(smem);                 // [act][LDW4]  tf32 "hi" part of W3p
  float4* sWl4 = sWh4 + act * LDW4;                               // [act][LDW4]  tf32 "lo" part
  float4* sWc4 = sWl4 + act * LDW4;                               // [H4]         W3c
  float4* sBb = sWc4 + H4;                                        // [NB*2][NT][32] backward B fragments (b0hi, b1hi, b0lo, b1lo)
  float4* sDm = sBb + NB * 2 * NT * 32;                           // [RT][NT][32] d-mean in A-fragment order
  float* sDv = reinterpret_cast<float*>(sDm + RT * NT * 32);      // [RT*16]      d-value per row
  float* sred = reinterpret_cast<float*>(sBb);                    // [8][npart]   (aliases the work area after the last tile)

  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
  // ---- tables
  for (int i = threadIdx.x; i < act * H_; i += blockDim.x) {
    const int a = i / H_, c = i - a * H_;
    uint32_t hi, lo;
    split_tf32(p.W3p[i], hi, lo);
    reinterpret_cast<float*>(sWh4)[a * (4 * LDW4) + c] = __uint_as_float(hi);
    reinterpret_cast<float*>(sWl4)[a * (4 * LDW4) + c] = __uint_as_float(lo);
  }
  for (int i = threadIdx.x; i < H_; i += blockDim.x) reinterpret_cast<float*>(sWc4)[i] = p.W3c[i];
  for (int i = threadIdx.x; i < NB * 2 * NT * 32; i += blockDim.x) {
    const int ln = i & 31, q = i >> 5, j = q % NT, be = q / NT, e = be & 1, b = be >> 1;
    const int gg = ln >> 2, tt = ln & 3;
    const int col = 16 * b + 4 * (gg >> 1) + 2 * e + (gg & 1);
    const int a0 = 8 * j + 2 * tt, a1 = a0 + 1;
    const float w0 = (a0 < act) ? p.W3p[a0 * H_ + col] : 0.f;
    const float w1 = (a1 < act) ? p.W3p[a1 * H_ + col] : 0.f;
    uint32_t h0, l0, h1, l1;
    split_tf32(w0, h0, l0);
    split_tf32(w1, h1, l1);
    sBb[i] = make_float4(__uint_as_float(h0), __uint_as_float(h1), __uint_as_float(l0), __uint_as_float(l1));
  }
  __syncthreads();

  // ---- per-lane constants of the actions a = 8j + 2t + f this lane owns in the C fragments
  float c_b3[NT][2], c_var[NT][2], c_logsd[NT][2];
#pragma unroll
  for (int j = 0; j < NT; ++j)
#pragma unroll
    for (int f = 0; f < 2; ++f) {
      const int a = 8 * j + 2 * t + f;
      if (a < act) {
        const float sd = expf(p.logstd[a]);
        c_b3[j][f] = p.b3p[a];
        c_var[j][f] = sd * sd;
        c_logsd[j][f] = logf(sd);
      } else {
        c_b3[j][f] = 0.f;
        c_var[j][f] = 1.f;
        c_logsd[j][f] = 0.f;
      }
    }
  const float b3c = p.b3c[0];
  const float adv_mean = p.adv_stats[0];
  const float adv_den = p.adv_stats[1] + 1e-8f;
  const float clip_lo = 1.f - p.clip_range, clip_hi = 1.f + p.clip_range;
  const int dh_ld = ex.dh_ld;
  const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);

  float acc_db3[NT][2], acc_dls[NT][2];
#pragma unroll
  for (int j = 0; j < NT; ++j) acc_db3[j][0] = acc_db3[j][1] = acc_dls[j][0] = acc_dls[j][1] = 0.f;
  float acc_db3c = 0.f, acc_pg = 0.f, acc_vl = 0.f, acc_kl = 0.f, acc_cf = 0.f;
  float4 acc_db2p[BPW], acc_db2c[BPW];
#pragma unroll
  for (int bb = 0; bb < BPW; ++bb) acc_db2p[bb] = acc_db2c[bb] = zero4;

  const long long M = p.M;
  const long long ntiles = (M + 16 * RT - 1) / (16 * RT);
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    // ================================================================ phase 1: forward + loss of rows R0 .. R0+15
    {
      const long long R0 = tile * (16 * RT) + 16 * wib;
      const long long r2[2] = {R0 + g, R0 + g + 8};
      const bool v2[2] = {r2[0] < M, r2[1] < M};
      const float4* __restrict__ hlo = reinterpret_cast<const float4*>(p.H2 + (v2[0] ? r2[0] : M - 1) * (2LL * H_));
      const float4* __restrict__ hhi = reinterpret_cast<const float4*>(p.H2 + (v2[1] ? r2[1] : M - 1) * (2LL * H_));
      float acc[NT][4], cor[NT][4];
#pragma unroll
      for (int j = 0; j < NT; ++j)
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[j][i] = cor[j][i] = 0.f;
      float sc0 = 0.f, sc1 = 0.f;
#pragma unroll 2
      for (int b = 0; b < NB; ++b) {
        const float4 xl = hlo[4 * b + t], xh = hhi[4 * b + t];
        const float4 cl = hlo[H4 + 4 * b + t], ch = hhi[H4 + 4 * b + t];
        const float4 wc = sWc4[4 * b + t];
        sc0 = dot4(cl, wc, sc0);
        sc1 = dot4(ch, wc, sc1);
        uint32_t ah0[4], al0[4], ah1[4], al1[4];
        split_tf32(xl.x, ah0[0], al0[0]); split_tf32(xh.x, ah0[1], al0[1]); split_tf32(xl.y, ah0[2], al0[2]); split_tf32(xh.y, ah0[3], al0[3]);
        split_tf32(xl.z, ah1[0], al1[0]); split_tf32(xh.z, ah1[1], al1[1]); split_tf32(xl.w, ah1[2], al1[2]); split_tf32(xh.w, ah1[3], al1[3]);
#pragma unroll
        for (int j = 0; j < NT; ++j) {
          const bool brow = (8 * j + g) < act;
          const float4 bh = brow ? sWh4[(8 * j + g) * LDW4 + 4 * b + t] : zero4;
          const float4 bl = brow ? sWl4[(8 * j + g) * LDW4 + 4 * b + t] : zero4;
          mma_tf32(cor[j], al0, __float_as_uint(bh.x), __float_as_uint(bh.y));
          mma_tf32(cor[j], ah0, __float_as_uint(bl.x), __float_as_uint(bl.y));
          mma_tf32(acc[j], ah0, __float_as_uint(bh.x), __float_as_uint(bh.y));
          mma_tf32(cor[j], al1, __float_as_uint(bh.z), __float_as_uint(bh.w));
          mma_tf32(cor[j], ah1, __float_as_uint(bl.z), __float_as_uint(bl.w));
          mma_tf32(acc[j], ah1, __float_as_uint(bh.z), __float_as_uint(bh.w));
        }
      }
      sc0 += __shfl_xor_sync(0xffffffffu, sc0, 1);
      sc0 += __shfl_xor_sync(0xffffffffu, sc0, 2);
      sc1 += __shfl_xor_sync(0xffffffffu, sc1, 1);
      sc1 += __shfl_xor_sync(0xffffffffu, sc1, 2);
      float dmv[2][NT][2], dvv[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const long long row = r2[r];
        const bool valid = v2[r];
        const float value = (r ? sc1 : sc0) + b3c;
        float lp = 0.f, dmu[NT][2], zz[NT][2];
#pragma unroll
        for (int j = 0; j < NT; ++j)
#pragma unroll
          for (int f = 0; f < 2; ++f) {
            const int a = 8 * j + 2 * t + f;
            dmu[j][f] = zz[j][f] = 0.f;
            if (a < act && valid) {
              const float mean = (acc[j][2 * r + f] + cor[j][2 * r + f]) + c_b3[j][f];
              const float d = p.actions[row * act + a] - mean;
              lp += -(d * d) / (2.f * c_var[j][f]) - c_logsd[j][f] - kLogSqrt2Pi;
              dmu[j][f] = d / c_var[j][f];
              zz[j][f] = d * d / c_var[j][f];
            }
          }
        lp += __shfl_xor_sync(0xffffffffu, lp, 1);
        lp += __shfl_xor_sync(0xffffffffu, lp, 2);
        float dv = 0.f, dlogp = 0.f;
        if (valid) {
          const float logratio = lp - p.logp_old[row];
          const float ratio = expf(logratio);
          const float A = (p.adv[row] - adv_mean) / adv_den;
          const float pg1 = -A * ratio;
          const float pg2 = -A * fminf(fmaxf(ratio, clip_lo), clip_hi);
          const float w1 = (pg1 > pg2) ? 1.f : ((pg1 == pg2) ? 0.5f : 0.f);
          const float inr = (ratio >= clip_lo && ratio <= clip_hi) ? 1.f : 0.f;
          dlogp = (-A * (w1 + (1.f - w1) * inr)) * ratio * p.inv_mg;
          const float verr = value - p.ret[row];
          dv = p.critic_coef * verr * p.inv_mg;
          if (t == 0) {  // one lane of the quad books the row's scalars
            acc_pg += fmaxf(pg1, pg2);
            acc_vl += 0.5f * verr * verr;
            acc_kl += (ratio - 1.f) - logratio;
            acc_cf += p.ratio_delta_metric ? fabsf(ratio - 1.f) : ((fabsf(ratio - 1.f) > p.clip_range) ? 1.f : 0.f);
            if (p.ratio_abs != nullptr) p.ratio_abs[row] = fabsf(ratio - 1.f);
          }
        }
        dvv[r] = dv;
#pragma unroll
        for (int j = 0; j < NT; ++j) {
          float o[2];
#pragma unroll
          for (int f = 0; f < 2; ++f) {
            const int a = 8 * j + 2 * t + f;
            const float dm = dlogp * dmu[j][f];  // 0 for a >= act and for rows past the end
            dmv[r][j][f] = dm;
            o[f] = dm;
            if (valid) {
              if (a < act) {
                acc_db3[j][f] += dm;
                acc_dls[j][f] += dlogp * (zz[j][f] - 1.f);
              } else if (a == act) {
                acc_db3c += dv;
                o[f] = dv;
              }
            }
          }
          if (valid && 8 * j + 2 * t < dh_ld) *reinterpret_cast<float2*>(p.dhead + row * dh_ld + 8 * j + 2 * t) = make_float2(o[0], o[1]);
        }
      }
#pragma unroll
      for (int j = 0; j < NT; ++j) sDm[(wib * NT + j) * 32 + lane] = make_float4(dmv[0][j][0], dmv[1][j][0], dmv[0][j][1], dmv[1][j][1]);
      if (t == 0) {
        sDv[wib * 16 + g] = dvv[0];
        sDv[wib * 16 + g + 8] = dvv[1];
      }
    }
    __syncthreads();
    // ================================================================ phase 2: dZ2 of this warp's columns for all row tiles
#pragma unroll 1
    for (int rt = 0; rt < RT; ++rt) {
      const long long S0 = tile * (16 * RT) + 16 * rt;
      if (S0 >= M) break;  // uniform over the CTA
      const long long s2[2] = {S0 + g, S0 + g + 8};
      const bool w2[2] = {s2[0] < M, s2[1] < M};
      const long long q2[2] = {w2[0] ? s2[0] : M - 1, w2[1] ? s2[1] : M - 1};
      uint32_t ah[NT][4], al[NT][4];
#pragma unroll
      for (int j = 0; j < NT; ++j) {
        const float4 a = sDm[(rt * NT + j) * 32 + lane];
        split_tf32(a.x, ah[j][0], al[j][0]);
        split_tf32(a.y, ah[j][1], al[j][1]);
        split_tf32(a.z, ah[j][2], al[j][2]);
        split_tf32(a.w, ah[j][3], al[j][3]);
      }
      const float dv2[2] = {sDv[rt * 16 + g], sDv[rt * 16 + g + 8]};
#pragma unroll
      for (int bb = 0; bb < BPW; ++bb) {
        const int b = wib * BPW + bb;
        float m0[4] = {0.f, 0.f, 0.f, 0.f}, k0[4] = {0.f, 0.f, 0.f, 0.f}, m1[4] = {0.f, 0.f, 0.f, 0.f}, k1[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int j = 0; j < NT; ++j) {
          const float4 B0 = sBb[((b * 2 + 0) * NT + j) * 32 + lane];
          const float4 B1 = sBb[((b * 2 + 1) * NT + j) * 32 + lane];
          mma_tf32(k0, al[j], __float_as_uint(B0.x), __float_as_uint(B0.y));
          mma_tf32(k0, ah[j], __float_as_uint(B0.z), __float_as_uint(B0.w));
          mma_tf32(m0, ah[j], __float_as_uint(B0.x), __float_as_uint(B0.y));
          mma_tf32(k1, al[j], __float_as_uint(B1.x), __float_as_uint(B1.y));
          mma_tf32(k1, ah[j], __float_as_uint(B1.z), __float_as_uint(B1.w));
          mma_tf32(m1, ah[j], __float_as_uint(B1.x), __float_as_uint(B1.y));
        }
        const float4 wc = sWc4[4 * b + t];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const float4* __restrict__ h = reinterpret_cast<const float4*>(p.H2 + q2[r] * (2LL * H_));
          const float4 a4 = h[4 * b + t], c4 = h[H4 + 4 * b + t];
          const float4 d4 = make_float4(m0[2 * r] + k0[2 * r], m0[2 * r + 1] + k0[2 * r + 1], m1[2 * r] + k1[2 * r], m1[2 * r + 1] + k1[2 * r + 1]);
          float4 zp, zc;
          zp.x = d4.x * (1.f - a4.x * a4.x); zp.y = d4.y * (1.f - a4.y * a4.y);
          zp.z = d4.z * (1.f - a4.z * a4.z); zp.w = d4.w * (1.f - a4.w * a4.w);
          zc.x = (dv2[r] * wc.x) * (1.f - c4.x * c4.x); zc.y = (dv2[r] * wc.y) * (1.f - c4.y * c4.y);
          zc.z = (dv2[r] * wc.z) * (1.f - c4.z * c4.z); zc.w = (dv2[r] * wc.w) * (1.f - c4.w * c4.w);
          if (w2[r]) {
            float4* __restrict__ out = reinterpret_cast<float4*>(p.dZ2 + s2[r] * (2LL * H_));
            out[4 * b + t] = zp;
            out[H4 + 4 * b + t] = zc;
            acc_db2p[bb].x += zp.x; acc_db2p[bb].y += zp.y; acc_db2p[bb].z += zp.z; acc_db2p[bb].w += zp.w;
            acc_db2c[bb].x += zc.x; acc_db2c[bb].y += zc.y; acc_db2c[bb].z += zc.z; acc_db2c[bb].w += zc.w;
          }
        }
      }
    }
    __syncthreads();  // sDm / sDv are rewritten by the next tile
  }

  // ---- block partials in the SIMT head's layout: db3p | db3c | dlogstd | pg | vloss | kl | clipfrac | db2p[H] | db2c[H]
  const int npart = 2 * act + 5 + 2 * H_;
  __syncthreads();
  for (int i = threadIdx.x; i < 8 * npart; i += blockDim.x) sred[i] = 0.f;
  __syncthreads();
  float* my = sred + wib * npart;
  // lanes with equal t hold the same actions / columns for different rows: fold over g
#pragma unroll
  for (int j = 0; j < NT; ++j)
#pragma unroll
    for (int f = 0; f < 2; ++f) {
      float x = acc_db3[j][f], y = acc_dls[j][f];
#pragma unroll
      for (int o = 4; o < 32; o <<= 1) {
        x += __shfl_xor_sync(0xffffffffu, x, o);
        y += __shfl_xor_sync(0xffffffffu, y, o);
      }
      const int a = 8 * j + 2 * t + f;
      if (g == 0 && a < act) {
        my[a] = x;
        my[act + 1 + a] = y;
      }
    }
  {
    const float s_db3c = warp_sum(acc_db3c), s_pg = warp_sum(acc_pg), s_vl = warp_sum(acc_vl), s_kl = warp_sum(acc_kl), s_cf = warp_sum(acc_cf);
    if (lane == 0) {
      my[act] = s_db3c;
      my[2 * act + 1] = s_pg;
      my[2 * act + 2] = s_vl;
      my[2 * act + 3] = s_kl;
      my[2 * act + 4] = s_cf;
    }
  }
#pragma unroll
  for (int bb = 0; bb < BPW; ++bb) {
    float v[8] = {acc_db2p[bb].x, acc_db2p[bb].y, acc_db2p[bb].z, acc_db2p[bb].w, acc_db2c[bb].x, acc_db2c[bb].y, acc_db2c[bb].z, acc_db2c[bb].w};
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int o = 4; o < 32; o <<= 1) v[i] += __shfl_xor_sync(0xffffffffu, v[i], o);
    if (g == 0) {
      float* q = my + 2 * act + 5 + 16 * (wib * BPW + bb) + 4 * t;
      q[0] = v[0]; q[1] = v[1]; q[2] = v[2]; q[3] = v[3];
      q[H_] = v[4]; q[H_ + 1] = v[5]; q[H_ + 2] = v[6]; q[H_ + 3] = v[7];
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < npart; i += blockDim.x) {
    float s = 0.f;
    for (int w = 0; w < 8; ++w) s += sred[w * npart + i];
    p.block_partials[(long long)blockIdx.x * npart + i] = s;
  }
}

}  // namespace rlx
