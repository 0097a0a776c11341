// PPO + LSTM update path (SURVEY.md §8 a18; rl_x/algorithms/ppo_lstm/flax): sequence forward with carry reset, combined PPO loss,
// back-propagation through time, Optax clip + Adam.  See include/rlx_b200.h for the entry points and the flat parameter layout.
//
// Written so that the SAME source compiles twice:
//   * nvcc (default): kernels + exact-fp32 SIMT GEMMs (gemm_simt.cuh), part of librlx_b200.so;
//   * g++ -x c++ -DRLX_EMU (tests/test_lstm_emulation.py only): every kernel here is "one thread = one row or one element, no shared
//     memory, no warp primitives, no barriers", so a launch is emulated exactly by loops over (block, thread), and a GEMM by an
//     interpreter of the GemmP contract.  That build checks indexing / strides / gradients against the oracle without a GPU.
// The emulation build is test scaffolding; nothing in the product loads it.
#include "flat_ops.cuh"
#define LSTM_LAUNCH RLX_FLAT_LAUNCH

namespace rlx {
namespace lstm {
using namespace rlx::flat;

constexpr float kLnEps = 1e-6f;             // flax.linen.LayerNorm default
constexpr float kHalfLog2Pi = 0.9189385332046727f;
constexpr int kWgradRows = 1024;            // rows per split of the weight-gradient GEMMs

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

// ---------------------------------------------------------------------------------------------------------- layouts
enum PSeg { WE1 = 0, BE1, G1, N1, WE2, BE2, G2, N2, WI, WH, BH, GL, NL, WT1, BT1, WT2, BT2, WM, BM, P_LOGSTD, WF, BF };
enum CSeg { WC1 = 0, BC1, WC2, BC2, WC3, BC3 };
static inline bool is_film(const rlx_lstm_dims& d) { return (d.options & RLX_LSTM_OPT_FILM) != 0; }
static inline bool is_shared(const rlx_lstm_dims& d) { return (d.options & RLX_LSTM_OPT_SHARED_ENCODER) != 0; }
struct Layout {
  long long p[RLX_LSTM_POLICY_NSEG + 1], c[RLX_LSTM_CRITIC_NSEG + 1];
};
static Layout make_layout(const rlx_lstm_dims& d) {
  const long long O = d.obs_dim, A = d.act_dim, H = d.hidden, E = d.enc_dim, L = d.lstm_dim;
  // options (policy.py:51-59): a shared encoder has no obs_encoder segments; FiLM adds [gamma | beta] dense blocks and narrows the torso input
  const long long E2 = is_shared(d) ? 0 : E, TIW = is_film(d) ? E : E + L, F = is_film(d) ? 2 * E : 0;
  const long long ps[RLX_LSTM_POLICY_NSEG] = {O * E, E, E, E, O * E2, E2, E2, E2, E * 4 * L, L * 4 * L, 4 * L, L, L, TIW * H, H, H * H, H, H * A, A, A,
                                              L * F, F};
  const long long cs[RLX_LSTM_CRITIC_NSEG] = {O * H, H, H * H, H, H, 1};
  Layout l;
  long long o = 0;
  for (int i = 0; i < RLX_LSTM_POLICY_NSEG; ++i) { l.p[i] = o; o += ps[i]; }
  l.p[RLX_LSTM_POLICY_NSEG] = o;
  o = 0;
  for (int i = 0; i < RLX_LSTM_CRITIC_NSEG; ++i) { l.c[i] = o; o += cs[i]; }
  l.c[RLX_LSTM_CRITIC_NSEG] = o;
  return l;
}
// Offsets of the K-major copies PT / TC (rlx_lstm_ppo_minibatch_fwdbwd_f32): the segments of `l` in the same order, each starting on a
// 16-byte boundary, so that a copy is a tensor-engine operand whatever the widths before it (with FiLM and an odd act, Wf itself is not).
static Layout kmajor_layout(const Layout& l) {
  Layout k;
  long long o = 0;
  for (int i = 0; i < RLX_LSTM_POLICY_NSEG; ++i) { o = (o + 3) / 4 * 4; k.p[i] = o; o += l.p[i + 1] - l.p[i]; }
  k.p[RLX_LSTM_POLICY_NSEG] = o;
  o = 0;
  for (int i = 0; i < RLX_LSTM_CRITIC_NSEG; ++i) { o = (o + 3) / 4 * 4; k.c[i] = o; o += l.c[i + 1] - l.c[i]; }
  k.c[RLX_LSTM_CRITIC_NSEG] = o;
  return k;
}
static bool dims_ok(const rlx_lstm_dims& d) {
  return d.obs_dim > 0 && d.act_dim > 0 && d.act_dim <= 64 && d.hidden > 0 && d.enc_dim > 0 && d.enc_dim <= 1024 && d.lstm_dim > 0 && d.lstm_dim <= 1024 &&
         (d.options & ~(RLX_LSTM_OPT_FILM | RLX_LSTM_OPT_SHARED_ENCODER)) == 0;
}

// workspace carve-up (floats); R = T * n_env rows, time-major (row = t * n_env + e)
struct Ws {
  size_t Z1, E1, Z2, TI, Gi, Gates, Call, Hall, Hm, Cm, T1, T2, C1, C2, Mean, V, dMean, dV, Terms, dLs, dT2, dT1, dTI, dHall, dG, dE1, dZ1, dZ2,
      dC2, dC1, Gh, dHn, dCn, Small, Stats1, Stats2, StatsL, Part, Col, WhT, E2, LL, GB, dGB, dOL, dLL, TP, TC, total;
};
static Ws plan(const rlx_lstm_dims& d, long long T, long long n) {
  const size_t R = (size_t)(T * n), O = d.obs_dim, A = d.act_dim, H = d.hidden, E = d.enc_dim, L = d.lstm_dim;
  (void)O;
  Ws w;
  size_t o = 0;
  auto take = [&](size_t& f, size_t cnt) { f = o; o += align_up(cnt, 64); };
  take(w.Z1, R * E); take(w.E1, R * E); take(w.Z2, R * E); take(w.TI, R * (E + L)); take(w.Gi, R * 4 * L); take(w.Gates, R * 4 * L);
  take(w.Call, R * L); take(w.Hall, R * L); take(w.Hm, R * L); take(w.Cm, R * L); take(w.T1, R * H); take(w.T2, R * H); take(w.C1, R * H);
  take(w.C2, R * H); take(w.Mean, R * A); take(w.V, R); take(w.dMean, R * A); take(w.dV, R); take(w.Terms, R * 4); take(w.dLs, R * A);
  take(w.dT2, R * H); take(w.dT1, R * H); take(w.dTI, R * (E + L)); take(w.dHall, R * L); take(w.dG, R * 4 * L); take(w.dE1, R * E);
  take(w.dZ1, R * E); take(w.dZ2, R * E); take(w.dC2, R * H); take(w.dC1, R * H);
  take(w.Gh, (size_t)n * 4 * L); take(w.dHn, (size_t)n * L); take(w.dCn, (size_t)n * L); take(w.Small, 64);
  take(w.Stats1, R * 2); take(w.Stats2, R * 2); take(w.StatsL, R * 2);
  const size_t splits = (size_t)ceil_div((long long)R, kWgradRows);
  size_t biggest = 0;  // largest weight matrix: one partial of it per row split
  for (size_t v : {(size_t)d.obs_dim * E, E * 4 * L, L * 4 * L, (E + L) * H, H * H, H * A, (size_t)d.obs_dim * H, H, L * 2 * E}) biggest = std::max(biggest, v);
  take(w.Part, splits * biggest);
  const size_t chunks = (size_t)ceil_div((long long)R, kColChunk);
  size_t widest = 8;   // widest column reduction; the LayerNorm parameter gradients keep two partial sets side by side
  for (size_t v : {H, 4 * L, 2 * E, 2 * L, A}) widest = std::max(widest, v);
  take(w.Col, chunks * widest);
  take(w.WhT, 4 * L * L);  // recurrent kernel transposed, [4L, L]: coalesced reads in the fused BPTT step
  const size_t film = is_film(d) ? 1 : 0;  // FiLM buffers (policy.py:102-105); zero-sized otherwise
  take(w.E2, film * R * E); take(w.LL, film * R * L); take(w.GB, film * R * 2 * E); take(w.dGB, film * R * 2 * E); take(w.dOL, film * R * E);
  take(w.dLL, film * R * L);
  // K-major ([out, in]) copies of the dense kernels, at the offsets of kmajor_layout (rlx_lstm_ppo_minibatch_fwdbwd_f32 only)
  const Layout lay = kmajor_layout(make_layout(d));
  take(w.TP, (size_t)lay.p[RLX_LSTM_POLICY_NSEG]); take(w.TC, (size_t)lay.c[RLX_LSTM_CRITIC_NSEG]);
  w.total = o * sizeof(float);
  return w;
}

// ---------------------------------------------------------------------------------------------------------- kernels
// (one thread = one row unless stated; all comm-free)

// y = tanh(LayerNorm(z) * g + b) per row; flax fast variance: var = max(0, E[z^2] - E[z]^2); stats = (mean, rstd)
__global__ void ln_tanh_fwd_kernel(const float* __restrict__ Z, int ldz, long long R, int W, const float* __restrict__ g,
                                   const float* __restrict__ b, float* __restrict__ out, int ldo, float* __restrict__ stats) {
  const long long r = gtid();
  if (r >= R) return;
  const float* z = Z + r * ldz;
  float s = 0.f, q = 0.f;
  for (int j = 0; j < W; ++j) { s += z[j]; q += z[j] * z[j]; }
  const float mean = s / (float)W;
  const float var = fmaxf(q / (float)W - mean * mean, 0.f);
  const float rstd = 1.f / sqrtf(var + kLnEps);
  for (int j = 0; j < W; ++j) out[r * ldo + j] = tanhf((z[j] - mean) * (rstd * g[j]) + b[j]);
  stats[2 * r] = mean;
  stats[2 * r + 1] = rstd;
}

// dZ for y = tanh(LN(z)); dOut = dL/dy, Y = y.  dxhat = dOut (1 - y^2) g;  dz = rstd (dxhat - mean(dxhat) - xhat mean(dxhat xhat))
__global__ void ln_tanh_bwd_kernel(const float* __restrict__ dOut, int ldd, const float* __restrict__ Y, int ldy, const float* __restrict__ Z,
                                   int ldz, long long R, int W, const float* __restrict__ g, const float* __restrict__ stats,
                                   float* __restrict__ dZ, int lddz) {
  const long long r = gtid();
  if (r >= R) return;
  const float mean = stats[2 * r], rstd = stats[2 * r + 1];
  float s1 = 0.f, s2 = 0.f;
  for (int j = 0; j < W; ++j) {
    const float y = Y[r * ldy + j];
    const float dx = dOut[r * ldd + j] * (1.f - y * y) * g[j];
    const float xh = (Z[r * ldz + j] - mean) * rstd;
    s1 += dx;
    s2 += dx * xh;
  }
  s1 /= (float)W;
  s2 /= (float)W;
  for (int j = 0; j < W; ++j) {
    const float y = Y[r * ldy + j];
    const float dx = dOut[r * ldd + j] * (1.f - y * y) * g[j];
    const float xh = (Z[r * ldz + j] - mean) * rstd;
    dZ[r * lddz + j] = rstd * (dx - s1 - xh * s2);
  }
}

// partial column sums of the LayerNorm parameter gradients: thread = (row chunk, column).  part_g / part_b: [nchunk, W]
__global__ void ln_param_partial_kernel(const float* __restrict__ dOut, int ldd, const float* __restrict__ Y, int ldy, const float* __restrict__ Z,
                                        int ldz, long long R, int W, const float* __restrict__ stats, float* __restrict__ part_g,
                                        float* __restrict__ part_b) {
  const long long id = gtid();
  const long long nchunk = (R + kColChunk - 1) / kColChunk;
  if (id >= nchunk * W) return;
  const long long ch = id / W;
  const int j = (int)(id % W);
  const long long r1 = ch * kColChunk + kColChunk < R ? ch * kColChunk + kColChunk : R;
  float sg = 0.f, sb = 0.f;
  for (long long r = ch * kColChunk; r < r1; ++r) {
    const float y = Y[r * ldy + j];
    const float dy = dOut[r * ldd + j] * (1.f - y * y);
    sg += dy * ((Z[r * ldz + j] - stats[2 * r]) * stats[2 * r + 1]);
    sb += dy;
  }
  part_g[id] = sg;
  part_b[id] = sb;
}

// One launch per time step of forward_sequence (policy.py:127-146): carry reset, recurrent product and cell update fused.
//   keep = 1 - done[t-1] (1 at t = 0);  hm = hprev * keep, cm = cprev * keep  (stored: the backward pass needs both)
//   z_g = Gi_t[e, gL + j] + bh[gL + j] + sum_k hm[e, k] Wh[k, gL + j];  c = f cm + i g;  h = o tanh(c)
// thread = (env, unit).  Hprev / Cprev are step t-1's rows of Hall / Call (or the initial carry), never the rows written here.
__global__ void lstm_step_fwd_kernel(const float* __restrict__ Gi, const float* __restrict__ Wh, const float* __restrict__ bh,
                                     const float* __restrict__ Hprev, const float* __restrict__ Cprev, const float* __restrict__ done_prev,
                                     long long n, int L, float* __restrict__ Hm, float* __restrict__ Cm, float* __restrict__ gates,
                                     float* __restrict__ C, float* __restrict__ Hh) {
  const long long id = gtid();
  if (id >= n * L) return;
  const long long e = id / L;
  const int j = (int)(id % L);
  const long long base = e * 4 * L;
  const float keep = done_prev ? 1.f - done_prev[e] : 1.f;
  float zi = Gi[base + j] + bh[j], zf = Gi[base + L + j] + bh[L + j], zg = Gi[base + 2 * L + j] + bh[2 * L + j], zo = Gi[base + 3 * L + j] + bh[3 * L + j];
  const float* hp = Hprev + e * L;
  for (int k = 0; k < L; ++k) {
    const float hk = hp[k] * keep;
    const float* w = Wh + (long long)k * 4 * L + j;
    zi = fmaf(hk, w[0], zi);
    zf = fmaf(hk, w[L], zf);
    zg = fmaf(hk, w[2 * L], zg);
    zo = fmaf(hk, w[3 * L], zo);
  }
  const float cm = Cprev[id] * keep;
  Hm[id] = hp[j] * keep;
  Cm[id] = cm;
  const float i = sigmoidf_(zi), f = sigmoidf_(zf), g = tanhf(zg), o = sigmoidf_(zo);
  const float c = f * cm + i * g;
  gates[base + j] = i;
  gates[base + L + j] = f;
  gates[base + 2 * L + j] = g;
  gates[base + 3 * L + j] = o;
  C[id] = c;
  Hh[id] = o * tanhf(c);
}

// gates = act(Gi_t + Gh + bh), c = f * cm + i * g, h = o * tanh(c).  thread = (env, unit)
// (Cm and C may be the same buffer — the rollout step updates the carry in place — so neither is __restrict__)
__global__ void lstm_cell_fwd_kernel(const float* __restrict__ Gi, const float* __restrict__ Gh, const float* __restrict__ bh,
                                     const float* Cm, long long n, int L, float* __restrict__ gates, float* C, float* __restrict__ Hh) {
  const long long id = gtid();
  if (id >= n * L) return;
  const long long e = id / L;
  const int j = (int)(id % L);
  const long long base = e * 4 * L;
  const float zi = Gi[base + j] + Gh[base + j] + bh[j];
  const float zf = Gi[base + L + j] + Gh[base + L + j] + bh[L + j];
  const float zg = Gi[base + 2 * L + j] + Gh[base + 2 * L + j] + bh[2 * L + j];
  const float zo = Gi[base + 3 * L + j] + Gh[base + 3 * L + j] + bh[3 * L + j];
  const float i = sigmoidf_(zi), f = sigmoidf_(zf), g = tanhf(zg), o = sigmoidf_(zo);
  const float c = f * Cm[id] + i * g;
  gates[base + j] = i;
  gates[base + L + j] = f;
  gates[base + 2 * L + j] = g;
  gates[base + 3 * L + j] = o;
  C[id] = c;
  Hh[id] = o * tanhf(c);
}

// out[c, r] = in[r, c]      thread = element of `in` [rows, cols]
__global__ void transpose_kernel(const float* __restrict__ in, int rows, int cols, float* __restrict__ out) {
  const long long id = gtid();
  if (id >= (long long)rows * cols) return;
  const long long r = id / cols, c = id % cols;
  out[c * rows + r] = in[id];
}

// One launch per BPTT step t: the product with the recurrent kernel and the cell backward fused.
//   dHm_{t+1}[e, j] = sum_q dG_{t+1}[e, q] Wh[j, q]  (gradient wrt the MASKED carry of step t+1; WhT is Wh transposed, [4L, L])
//   dH = dHall_t + dHm_{t+1} (1 - done[t]);  dC = dCnext (already masked) + dH o (1 - tanh(c)^2)
//   writes the pre-activation gate gradients dG_t and dCprev = (dC f) keep_t, keep_t = 1 - done[t-1].
// thread = (env, unit).  dGnext (step t+1's rows) and dG (step t's rows) do not overlap; dCnext / dCprev are ONE buffer updated element-wise.
__global__ void lstm_step_bwd_kernel(const float* __restrict__ dHall, const float* __restrict__ dGnext, const float* __restrict__ WhT,
                                     const float* __restrict__ done_t, const float* dCnext, const float* __restrict__ gates,
                                     const float* __restrict__ C, const float* __restrict__ Cm, const float* __restrict__ done_prev, long long n,
                                     int L, float* __restrict__ dG, float* dCprev) {
  const long long id = gtid();
  if (id >= n * L) return;
  const long long e = id / L;
  const int j = (int)(id % L);
  const long long base = e * 4 * L;
  float dH = dHall[id];
  if (dGnext) {
    const float* dg = dGnext + base;
    float acc = 0.f;
    for (int q = 0; q < 4 * L; ++q) acc = fmaf(dg[q], WhT[(long long)q * L + j], acc);
    dH += acc * (1.f - done_t[e]);
  }
  const float i = gates[base + j], f = gates[base + L + j], g = gates[base + 2 * L + j], o = gates[base + 3 * L + j];
  const float tc = tanhf(C[id]);
  const float dC = (dCnext ? dCnext[id] : 0.f) + dH * o * (1.f - tc * tc);
  dG[base + j] = dC * g * i * (1.f - i);
  dG[base + L + j] = dC * Cm[id] * f * (1.f - f);
  dG[base + 2 * L + j] = dC * i * (1.f - g * g);
  dG[base + 3 * L + j] = dH * tc * o * (1.f - o);
  const float keep = done_prev ? 1.f - done_prev[e] : 1.f;
  dCprev[id] = dC * f * keep;
}

// ---- the whole recurrence in ONE launch per direction (rlx_set_lstm_persistent): a block owns EPB envs for all T steps, thread = (env, unit).
// The recurrent kernel lives in shared memory for the life of the block (Wh: [L, 4L], 64 KB at L = 64), the hidden state / the gate
// gradients of the block's envs are exchanged through shared memory (double-buffered: ONE barrier per step) and the cell state / its
// gradient stay in a register.  Every thread performs exactly the arithmetic of lstm_step_fwd_kernel / lstm_step_bwd_kernel in the same
// order, so the results are bit-identical to the one-launch-per-step path.
// shared: sWh [L * 4L] | sH [2][EPB * L]
__global__ void lstm_seq_fwd_kernel(const float* __restrict__ Gi, const float* __restrict__ Wh, const float* __restrict__ bh,
                                    const float* __restrict__ init_h, const float* __restrict__ init_c, const float* __restrict__ dones,
                                    long long T, long long n, int L, int EPB, float* __restrict__ Hm, float* __restrict__ Cm,
                                    float* __restrict__ gates, float* __restrict__ Call, float* __restrict__ Hall) {
  RLX_DYN_SMEM(sm);
  float* sWh = sm;
  float* sH = sm + (long long)L * 4 * L;
  const int tid = (int)threadIdx.x, el = tid / L, j = tid % L;
  const long long e = (long long)blockIdx.x * EPB + el;
  const bool active = e < n;
  for (int i = tid; i < L * 4 * L; i += (int)blockDim.x) sWh[i] = Wh[i];
  float c = active ? init_c[e * L + j] : 0.f;
  sH[el * L + j] = active ? init_h[e * L + j] : 0.f;
  __syncthreads();
  for (long long t = 0; t < T; ++t) {
    const float* hcur = sH + (t & 1) * EPB * L + el * L;
    float* hnext = sH + ((t + 1) & 1) * EPB * L + el * L;
    if (active) {
      const long long row = t * n + e, base = row * 4 * L, id = row * L + j;
      const float keep = t > 0 ? 1.f - dones[(t - 1) * n + e] : 1.f;
      float zi = Gi[base + j] + bh[j], zf = Gi[base + L + j] + bh[L + j], zg = Gi[base + 2 * L + j] + bh[2 * L + j], zo = Gi[base + 3 * L + j] + bh[3 * L + j];
      for (int k = 0; k < L; ++k) {
        const float hk = hcur[k] * keep;
        const float* w = sWh + (long long)k * 4 * L + j;
        zi = fmaf(hk, w[0], zi);
        zf = fmaf(hk, w[L], zf);
        zg = fmaf(hk, w[2 * L], zg);
        zo = fmaf(hk, w[3 * L], zo);
      }
      const float cm = c * keep;
      Hm[id] = hcur[j] * keep;
      Cm[id] = cm;
      const float i = sigmoidf_(zi), f = sigmoidf_(zf), g = tanhf(zg), o = sigmoidf_(zo);
      c = f * cm + i * g;
      gates[base + j] = i;
      gates[base + L + j] = f;
      gates[base + 2 * L + j] = g;
      gates[base + 3 * L + j] = o;
      Call[id] = c;
      const float h = o * tanhf(c);
      Hall[id] = h;
      hnext[j] = h;
    }
    __syncthreads();
  }
}
// shared: sWhT [4L * L] | sdG [2][EPB * 4L]
__global__ void lstm_seq_bwd_kernel(const float* __restrict__ dHall, const float* __restrict__ WhT, const float* __restrict__ dones,
                                    const float* __restrict__ gates, const float* __restrict__ Call, const float* __restrict__ Cm,
                                    long long T, long long n, int L, int EPB, float* __restrict__ dG) {
  RLX_DYN_SMEM(sm);
  float* sWhT = sm;
  float* sdG = sm + (long long)4 * L * L;
  const int tid = (int)threadIdx.x, el = tid / L, j = tid % L;
  const long long e = (long long)blockIdx.x * EPB + el;
  const bool active = e < n;
  for (int i = tid; i < 4 * L * L; i += (int)blockDim.x) sWhT[i] = WhT[i];
  float dCn = 0.f;
  __syncthreads();
  for (long long t = T - 1; t >= 0; --t) {
    const int cur = (int)((T - 1 - t) & 1);                    // slot holding dG_{t+1} of this block's envs; this step writes the other one
    const float* dgn = sdG + cur * EPB * 4 * L + el * 4 * L;
    float* dgo = sdG + (cur ^ 1) * EPB * 4 * L + el * 4 * L;
    if (active) {
      const long long row = t * n + e, base = row * 4 * L, id = row * L + j;
      float dH = dHall[id];
      if (t < T - 1) {
        float acc = 0.f;
        for (int q = 0; q < 4 * L; ++q) acc = fmaf(dgn[q], sWhT[(long long)q * L + j], acc);
        dH += acc * (1.f - dones[t * n + e]);
      }
      const float i = gates[base + j], f = gates[base + L + j], g = gates[base + 2 * L + j], o = gates[base + 3 * L + j];
      const float tc = tanhf(Call[id]);
      const float dC = (t < T - 1 ? dCn : 0.f) + dH * o * (1.f - tc * tc);
      const float gi = dC * g * i * (1.f - i), gf = dC * Cm[id] * f * (1.f - f), gg = dC * i * (1.f - g * g), go = dH * tc * o * (1.f - o);
      dG[base + j] = gi;
      dG[base + L + j] = gf;
      dG[base + 2 * L + j] = gg;
      dG[base + 3 * L + j] = go;
      dgo[j] = gi;
      dgo[L + j] = gf;
      dgo[2 * L + j] = gg;
      dgo[3 * L + j] = go;
      const float keep = t > 0 ? 1.f - dones[(t - 1) * n + e] : 1.f;
      dCn = dC * f * keep;
    }
    __syncthreads();
  }
}

// FiLM combination (policy.py:102-105): GB = [gamma | beta] ([R, 2W]); out = OL * gamma + beta.  thread = element
__global__ void film_fwd_kernel(const float* __restrict__ OL, int ldo, const float* __restrict__ GB, long long R, int W, float* __restrict__ out) {
  const long long id = gtid();
  if (id >= R * W) return;
  const long long r = id / W;
  const int j = (int)(id % W);
  out[id] = OL[r * ldo + j] * GB[r * 2 * W + j] + GB[r * 2 * W + W + j];
}
// dGB = [dOut * OL | dOut], dOL = dOut * gamma.  thread = element
__global__ void film_bwd_kernel(const float* __restrict__ dOut, const float* __restrict__ OL, int ldo, const float* __restrict__ GB, long long R, int W,
                                float* __restrict__ dGB, float* __restrict__ dOL) {
  const long long id = gtid();
  if (id >= R * W) return;
  const long long r = id / W;
  const int j = (int)(id % W);
  const float d = dOut[id];
  dGB[r * 2 * W + j] = d * OL[r * ldo + j];
  dGB[r * 2 * W + W + j] = d;
  dOL[id] = d * GB[r * 2 * W + j];
}
// dst[r, j] = src[r, j] (ACC = false) or dst[r, j] += src[r, j] (ACC = true) over an [R, W] block with row pitches.  thread = element
template <bool ACC>
__global__ void cols_kernel(const float* __restrict__ src, int lds, long long R, int W, float* __restrict__ dst, int ldd) {
  const long long id = gtid();
  if (id >= R * W) return;
  const long long r = id / W;
  const int j = (int)(id % W);
  if (ACC) dst[r * ldd + j] += src[r * lds + j];
  else dst[r * ldd + j] = src[r * lds + j];
}

// per-row loss terms and the gradients wrt the head outputs.  terms[r] = (pg, 0.5 (v - R)^2, approx_kl, clipped?)   thread = row
__global__ void loss_rows_kernel(const float* __restrict__ Mean, const float* __restrict__ V, const float* __restrict__ actions,
                                 const float* __restrict__ logp_old, const float* __restrict__ adv, const float* __restrict__ ret,
                                 const float* __restrict__ logstd, const float* __restrict__ adv_stats, long long R, int A, float clip_range,
                                 float critic_coef, float inv_R, float* __restrict__ dMean, float* __restrict__ dV, float* __restrict__ dLs,
                                 float* __restrict__ terms) {
  const long long r = gtid();
  if (r >= R) return;
  float lp = 0.f;
  for (int a = 0; a < A; ++a) {
    const float sd = expf(logstd[a]);
    const float zz = (actions[r * A + a] - Mean[r * A + a]) / sd;
    lp += -0.5f * zz * zz - kHalfLog2Pi - logstd[a];
  }
  const float logratio = lp - logp_old[r];
  const float ratio = expf(logratio);
  const float An = (adv[r] - adv_stats[0]) / (adv_stats[1] + 1e-8f);
  const float lo = 1.f - clip_range, hi = 1.f + clip_range;
  const float pg1 = -An * ratio, pg2 = -An * fminf(fmaxf(ratio, lo), hi);
  // d max(pg1, pg2) / d ratio: ties split evenly (jnp.maximum), the clip passes gradient on the closed interval
  const float w1 = (pg1 > pg2) ? 1.f : ((pg1 == pg2) ? 0.5f : 0.f);
  const float inr = (ratio >= lo && ratio <= hi) ? 1.f : 0.f;
  const float dlogp = -An * (w1 + (1.f - w1) * inr) * ratio * inv_R;
  for (int a = 0; a < A; ++a) {
    const float sd = expf(logstd[a]);
    const float d = actions[r * A + a] - Mean[r * A + a];
    dMean[r * A + a] = dlogp * d / (sd * sd);
    dLs[r * A + a] = dlogp * (d * d / (sd * sd) - 1.f);
  }
  const float verr = V[r] - ret[r];
  dV[r] = critic_coef * verr * inv_R;
  terms[4 * r + 0] = fmaxf(pg1, pg2);
  terms[4 * r + 1] = 0.5f * verr * verr;
  terms[4 * r + 2] = (ratio - 1.f) - logratio;
  terms[4 * r + 3] = (fabsf(ratio - 1.f) > clip_range) ? 1.f : 0.f;
}

__global__ void finish_metrics_kernel(const float* __restrict__ sums4, const float* __restrict__ logstd, int A, float rows, float* __restrict__ metrics) {
  if (gtid() != 0) return;
  metrics[0] = sums4[0];
  metrics[1] = sums4[1];
  float ent = 0.f;
  for (int a = 0; a < A; ++a) ent += logstd[a] + 0.5f + kHalfLog2Pi;  // log_std + 0.5 log(2 pi e)
  metrics[2] = ent;
  metrics[3] = sums4[2];
  metrics[4] = sums4[3];
  metrics[5] = 0.f;
  metrics[6] = 0.f;
  metrics[7] = rows;
}

// a = mean + exp(logstd) * noise; logp; env action (policy.py:149-157).  noise == null: a = mean.  thread = row
__global__ void sample_rows_kernel(const float* __restrict__ Mean, const float* __restrict__ logstd, const float* __restrict__ noise, long long n,
                                   int A, const float* __restrict__ low, const float* __restrict__ high, int clip_rescale,
                                   float* __restrict__ action, float* __restrict__ env_action, float* __restrict__ logp) {
  const long long r = gtid();
  if (r >= n) return;
  float lp = 0.f;
  for (int a = 0; a < A; ++a) {
    const float sd = expf(logstd[a]);
    const float m = Mean[r * A + a];
    const float act = noise ? m + sd * noise[r * A + a] : m;
    const float zz = (act - m) / sd;
    lp += -0.5f * zz * zz - kHalfLog2Pi - logstd[a];
    action[r * A + a] = act;
    float ea = act;
    if (clip_rescale) ea = low[a] + 0.5f * (fminf(fmaxf(act, -1.f), 1.f) + 1.f) * (high[a] - low[a]);
    env_action[r * A + a] = ea;
  }
  if (logp) logp[r] = lp;
}
__global__ void carry_mask_kernel(float* __restrict__ c, float* __restrict__ h, const float* __restrict__ done, long long n, int L) {
  const long long id = gtid();
  if (id >= n * L) return;
  const float keep = 1.f - done[id / L];
  c[id] *= keep;
  h[id] *= keep;
}
__global__ void centered_sq_kernel(const float* __restrict__ x, long long n, const float* __restrict__ mean, float* __restrict__ out) {
  const long long i = gtid();
  if (i >= n) return;
  const float d = x[i] - mean[0];
  out[i] = d * d;
}
__global__ void sqrt_inplace_kernel(float* __restrict__ x) {
  if (gtid() == 0) x[0] = sqrtf(x[0]);
}

// out[t, j, :] = src[t, idx[j], :]      thread = one float
__global__ void gather_env_kernel(const float* __restrict__ src, const long long* __restrict__ idx, long long T, long long N, long long n,
                                  long long width, float* __restrict__ out) {
  const long long id = gtid();
  if (id >= T * n * width) return;
  const long long k = id % width, j = (id / width) % n, t = id / (width * n);
  out[id] = src[(t * N + idx[j]) * width + k];
}

// optax: g = ||g|| < max_norm ? g : g / ||g|| * max_norm; Adam with bias correction.  thread = element
__global__ void optax_adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ mu, float* __restrict__ nu, long long n,
                                  const float* __restrict__ lr, const long long* __restrict__ step, const float* __restrict__ norm, float max_norm,
                                  float b1, float b2, float eps) {
  const long long i = gtid();
  if (i >= n) return;
  const float gn = norm[0];
  float gi = g[i];
  if (!(gn < max_norm)) gi = gi / gn * max_norm;
  const float t = (float)step[0];
  const float m = b1 * mu[i] + (1.f - b1) * gi;
  const float v = b2 * nu[i] + (1.f - b2) * gi * gi;
  mu[i] = m;
  nu[i] = v;
  const float mh = m / (1.f - powf(b1, t)), vh = v / (1.f - powf(b2, t));
  p[i] -= lr[0] * mh / (sqrtf(vh) + eps);
}

// ------------------------------------------------------------------------------------------------------- GEMM helpers
// forward dense: C[r, o] = act(sum_i X[r, i] W[i, o] + b[o]);  W stored [in, out]
template <int EPI>
static int dense_fwd(const float* X, int ldx, const float* W, int in, int out, const float* bias, float* C, int ldc, long long R, cudaStream_t st) {
  GemmP g{};
  g.A = X; g.B = W; g.C = C; g.bias = bias;
  g.M = (int)R; g.N = out; g.K = in;
  g.lda = ldx; g.ldb = out; g.ldc = ldc;
  g.splits = 1; g.kchunk = (int)(ceil_div(in, 8) * 8);
  return aux_gemm<true, false, EPI>(g, 1, st, KC_GEMM_FWD, R, in);
}
// The same two products on a K-major copy WT [out, in] of the kernel (torch's Linear layout): these operand layouts are the ones every
// epilogue of the tensor engine covers (bias, bias + tanh, tanh'), which the Flax layout [in, out] is not (gemm_tc.cu: RLX_TC_DISPATCH).
template <int EPI>
static int dense_fwd_t(const float* X, int ldx, const float* WT, int in, int out, const float* bias, float* C, int ldc, long long R, cudaStream_t st) {
  GemmP g{};
  g.A = X; g.B = WT; g.C = C; g.bias = bias;
  g.M = (int)R; g.N = out; g.K = in;
  g.lda = ldx; g.ldb = in; g.ldc = ldc;
  g.splits = 1; g.kchunk = (int)(ceil_div(in, 8) * 8);
  return aux_gemm<true, true, EPI>(g, 1, st, KC_GEMM_FWD, R, out);
}
template <int EPI>
static int dense_bwd_input_t(const float* dY, int ldy, const float* WT, int in, int out, const float* aux, int ldaux, float* C, int ldc, long long R,
                             cudaStream_t st) {
  GemmP g{};
  g.A = dY; g.B = WT; g.C = C; g.aux = aux;
  g.M = (int)R; g.N = in; g.K = out;
  g.lda = ldy; g.ldb = in; g.ldc = ldc; g.ldaux = ldaux;
  g.splits = 1; g.kchunk = (int)(ceil_div(out, 8) * 8);
  return aux_gemm<true, false, EPI>(g, 1, st, KC_GEMM_DX, R, out);
}
// weight gradient: dW[i, o] = sum_r X[r, i] dY[r, o], split over rows in chunks of kWgradRows and summed by reduce_parts_kernel
static int dense_bwd_weight(const float* X, int ldx, const float* dY, int ldy, int in, int out, long long R, float* part, float* dW, cudaStream_t st) {
  const int splits = (int)ceil_div(R, kWgradRows);
  GemmP g{};
  g.A = X; g.B = dY; g.C = part;
  g.M = in; g.N = out; g.K = (int)R;
  g.lda = ldx; g.ldb = ldy; g.ldc = out;
  g.splits = splits; g.kchunk = kWgradRows; g.sSplitC = (long long)in * out;
  int rc = aux_gemm<false, false, EPI_NONE>(g, 1, st, KC_GEMM_DW, R, R);
  if (rc) return rc;
  LSTM_LAUNCH(reduce_parts_kernel, (long long)in * out, st, part, (long long)splits, (long long)in * out, 1.f, 0.f, dW);
  return RLX_OK;
}
// LayerNorm scale / bias gradients
static int ln_param_grads(const float* dOut, int ldd, const float* Y, int ldy, const float* Z, int ldz, long long R, int W, const float* stats,
                          float* col_ws, float* dg, float* db, cudaStream_t st) {
  const long long nchunk = ceil_div(R, kColChunk);
  float* pg = col_ws;
  float* pb = col_ws + nchunk * W;
  LSTM_LAUNCH(ln_param_partial_kernel, nchunk * W, st, dOut, ldd, Y, ldy, Z, ldz, R, W, stats, pg, pb);
  LSTM_LAUNCH(reduce_parts_kernel, (long long)W, st, pg, nchunk, (long long)W, 1.f, 0.f, dg);
  LSTM_LAUNCH(reduce_parts_kernel, (long long)W, st, pb, nchunk, (long long)W, 1.f, 0.f, db);
  return RLX_OK;
}

}  // namespace lstm
}  // namespace rlx

using namespace rlx;
using namespace rlx::lstm;

#define LSTM_TRY(expr) do { int _rc = (expr); if (_rc) return _rc; } while (0)

// recurrence: one launch per direction when asked for and when the recurrent kernel fits in shared memory, else one launch per step
static int g_lstm_persistent = 0;
static unsigned long long g_lstm_persistent_launches = 0;  // evidence for tests / bench records that the one-launch path really ran
extern "C" int rlx_set_lstm_persistent(int on) {
  g_lstm_persistent = on ? 1 : 0;
  return g_lstm_persistent;
}
extern "C" uint64_t rlx_lstm_persistent_launch_count(void) { return g_lstm_persistent_launches; }
struct SeqCfg { int epb, threads; size_t smem_fwd, smem_bwd; bool ok; };
static SeqCfg seq_cfg(int L) {
  SeqCfg c;
  c.epb = std::max(1, 128 / L);
  c.threads = c.epb * L;
  c.smem_fwd = ((size_t)L * 4 * L + 2 * (size_t)c.epb * L) * sizeof(float);
  c.smem_bwd = ((size_t)4 * L * L + 2 * (size_t)c.epb * 4 * L) * sizeof(float);
  c.ok = g_lstm_persistent == 1 && c.threads <= 1024 && std::max(c.smem_fwd, c.smem_bwd) <= 200 * 1024;
  return c;
}

extern "C" int rlx_lstm_param_layout(const rlx_lstm_dims* d, int64_t* policy_offsets, int64_t* critic_offsets) {
  RLX_CHECK_ARG(d != nullptr && dims_ok(*d), "unsupported dims");
  const Layout l = make_layout(*d);
  if (policy_offsets) for (int i = 0; i <= RLX_LSTM_POLICY_NSEG; ++i) policy_offsets[i] = l.p[i];
  if (critic_offsets) for (int i = 0; i <= RLX_LSTM_CRITIC_NSEG; ++i) critic_offsets[i] = l.c[i];
  return RLX_OK;
}

extern "C" size_t rlx_lstm_minibatch_workspace_bytes(const rlx_lstm_dims* d, int64_t T, int64_t n_env) {
  if (d == nullptr || !dims_ok(*d) || T <= 0 || n_env <= 0) return 0;
  return plan(*d, T, n_env).total;
}

extern "C" int rlx_lstm_ppo_minibatch_fwdbwd_f32(const rlx_lstm_minibatch_args* a, void* stream) {
  RLX_CHECK_ARG(a != nullptr && dims_ok(a->dims), "unsupported dims");
  RLX_CHECK_ARG(a->T > 0 && a->n_env > 0 && a->T * a->n_env < (1LL << 31), "bad sequence / minibatch size");
  RLX_CHECK_ARG(a->states && a->actions && a->log_probs && a->advantages && a->returns && a->dones && a->init_c && a->init_h && a->adv_stats,
                "null minibatch tensor");
  RLX_CHECK_ARG(a->policy_params && a->critic_params && a->policy_grads && a->critic_grads && a->metrics, "null parameter / gradient / metrics");
  const rlx_lstm_dims& d = a->dims;
  const long long T = a->T, n = a->n_env, R = T * n;
  const int O = d.obs_dim, A = d.act_dim, H = d.hidden, E = d.enc_dim, L = d.lstm_dim, EL = E + L;
  const Ws w = plan(d, T, n);
  if (a->workspace == nullptr || a->workspace_bytes < w.total) {
    set_error("rlx_lstm_ppo_minibatch_fwdbwd_f32: workspace too small (%zu < %zu)", a->workspace_bytes, w.total);
    return RLX_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const Layout l = make_layout(d);
  float* ws = (float*)a->workspace;
  const float* P = a->policy_params;
  const float* Cp = a->critic_params;
  float* gP = a->policy_grads;
  float* gC = a->critic_grads;
  const float* X = a->states;
  float *Z1 = ws + w.Z1, *E1 = ws + w.E1, *Z2 = ws + w.Z2, *TI = ws + w.TI, *Gi = ws + w.Gi, *Gates = ws + w.Gates, *Call = ws + w.Call,
        *Hall = ws + w.Hall, *Hm = ws + w.Hm, *Cm = ws + w.Cm, *T1 = ws + w.T1, *T2 = ws + w.T2, *C1 = ws + w.C1, *C2 = ws + w.C2,
        *Mean = ws + w.Mean, *V = ws + w.V, *dMean = ws + w.dMean, *dV = ws + w.dV, *Terms = ws + w.Terms, *dLs = ws + w.dLs, *dT2 = ws + w.dT2,
        *dT1 = ws + w.dT1, *dTI = ws + w.dTI, *dHall = ws + w.dHall, *dG = ws + w.dG, *dE1 = ws + w.dE1, *dZ1 = ws + w.dZ1, *dZ2 = ws + w.dZ2,
        *dC2 = ws + w.dC2, *dC1 = ws + w.dC1, *dCn = ws + w.dCn, *Small = ws + w.Small, *S1 = ws + w.Stats1, *S2 = ws + w.Stats2,
        *SL = ws + w.StatsL, *Part = ws + w.Part, *Col = ws + w.Col, *WhT = ws + w.WhT;
  // Options (policy.py:51-59, 99-125).  Where the pieces of the decoder input live:
  //   obs latent OL: own encoder -> left E columns of TI (concat) or the E2 buffer (FiLM); shared encoder -> E1 (the LSTM's input latent)
  //   lstm latent LLp = tanh(LN(h)): right L columns of TI (concat) or the LL buffer (FiLM)
  //   torso input TI: [OL | LLp] (concat, width E + L) or OL * gamma + beta (FiLM, width E)
  const bool film = is_film(d), shared = is_shared(d);
  const int TIW = film ? E : EL;
  // K-major copies of the dense kernels (see dense_fwd_t): PT / CT hold P / Cp segment by segment, at the aligned offsets of kmajor_layout
  const Layout kl = kmajor_layout(l);
  float *PT = ws + w.TP, *CT = ws + w.TC;
  {
    const struct { int seg, in, out; bool on; } pk[] = {{WE1, O, E, true}, {WE2, O, E, !shared}, {WI, E, 4 * L, true}, {WT1, TIW, H, true}, {WT2, H, H, true},
                                                        {WM, H, A, true}, {WF, L, 2 * E, film}};
    for (const auto& k : pk)
      if (k.on) LSTM_LAUNCH(transpose_kernel, (long long)k.in * k.out, st, P + l.p[k.seg], k.in, k.out, PT + kl.p[k.seg]);
    const struct { int seg, in, out; } ck[] = {{WC1, O, H}, {WC2, H, H}, {WC3, H, 1}};
    for (const auto& k : ck) LSTM_LAUNCH(transpose_kernel, (long long)k.in * k.out, st, Cp + l.c[k.seg], k.in, k.out, CT + kl.c[k.seg]);
  }
  float* OL = shared ? E1 : (film ? ws + w.E2 : TI);
  const int ldOL = (shared || film) ? E : EL;
  float* LLp = film ? ws + w.LL : TI + E;
  const int ldLL = film ? L : EL;

  // ================================================================ forward
  // encoders (policy.py:79-92): Z = X We + be; E = tanh(LN(Z))
  LSTM_TRY(dense_fwd_t<EPI_BIAS>(X, O, PT + kl.p[WE1], O, E, P + l.p[BE1], Z1, E, R, st));
  LSTM_LAUNCH(ln_tanh_fwd_kernel, R, st, Z1, E, R, E, P + l.p[G1], P + l.p[N1], E1, E, S1);
  if (!shared) {
    LSTM_TRY(dense_fwd_t<EPI_BIAS>(X, O, PT + kl.p[WE2], O, E, P + l.p[BE2], Z2, E, R, st));
    LSTM_LAUNCH(ln_tanh_fwd_kernel, R, st, Z2, E, R, E, P + l.p[G2], P + l.p[N2], OL, ldOL, S2);
  } else if (!film) {
    LSTM_LAUNCH(cols_kernel<false>, R * E, st, E1, E, R, E, TI, EL);
  }
  // input-side gate pre-activations of all steps at once, then the recurrence, one launch per step (policy.py:115-146)
  LSTM_TRY(dense_fwd_t<EPI_NONE>(E1, E, PT + kl.p[WI], E, 4 * L, nullptr, Gi, 4 * L, R, st));
  const SeqCfg seq = seq_cfg(L);
  if (seq.ok) {
    RLX_BLOCK_LAUNCH(lstm_seq_fwd_kernel, ceil_div(n, seq.epb), seq.threads, seq.smem_fwd, st, Gi, P + l.p[WH], P + l.p[BH], a->init_h, a->init_c, a->dones,
                     T, n, L, seq.epb, Hm, Cm, Gates, Call, Hall);
    ++g_lstm_persistent_launches;
  } else {
    for (long long t = 0; t < T; ++t) {
      const float* hprev = t == 0 ? a->init_h : Hall + (t - 1) * n * L;
      const float* cprev = t == 0 ? a->init_c : Call + (t - 1) * n * L;
      const float* done_prev = t == 0 ? nullptr : a->dones + (t - 1) * n;
      LSTM_LAUNCH(lstm_step_fwd_kernel, n * L, st, Gi + t * n * 4 * L, P + l.p[WH], P + l.p[BH], hprev, cprev, done_prev, n, L, Hm + t * n * L,
                  Cm + t * n * L, Gates + t * n * 4 * L, Call + t * n * L, Hall + t * n * L);
    }
  }
  // decode (policy.py:95-112): lstm latent = tanh(LN(h)); combination; torso; mean head
  LSTM_LAUNCH(ln_tanh_fwd_kernel, R, st, Hall, L, R, L, P + l.p[GL], P + l.p[NL], LLp, ldLL, SL);
  if (film) {
    LSTM_TRY(dense_fwd_t<EPI_BIAS>(LLp, L, PT + kl.p[WF], L, 2 * E, P + l.p[BF], ws + w.GB, 2 * E, R, st));
    LSTM_LAUNCH(film_fwd_kernel, R * E, st, OL, ldOL, ws + w.GB, R, E, TI);
  }
  LSTM_TRY(dense_fwd_t<EPI_BIAS_TANH>(TI, TIW, PT + kl.p[WT1], TIW, H, P + l.p[BT1], T1, H, R, st));
  LSTM_TRY(dense_fwd_t<EPI_BIAS_TANH>(T1, H, PT + kl.p[WT2], H, H, P + l.p[BT2], T2, H, R, st));
  LSTM_TRY(dense_fwd_t<EPI_BIAS>(T2, H, PT + kl.p[WM], H, A, P + l.p[BM], Mean, A, R, st));
  // critic (critic.py:22-30)
  LSTM_TRY(dense_fwd_t<EPI_BIAS_TANH>(X, O, CT + kl.c[WC1], O, H, Cp + l.c[BC1], C1, H, R, st));
  LSTM_TRY(dense_fwd_t<EPI_BIAS_TANH>(C1, H, CT + kl.c[WC2], H, H, Cp + l.c[BC2], C2, H, R, st));
  LSTM_TRY(dense_fwd_t<EPI_BIAS>(C2, H, CT + kl.c[WC3], H, 1, Cp + l.c[BC3], V, 1, R, st));

  // ================================================================ loss (ppo_lstm.py:146-172) and head gradients
  const float inv_R = 1.f / (float)R;
  LSTM_LAUNCH(loss_rows_kernel, R, st, Mean, V, a->actions, a->log_probs, a->advantages, a->returns, P + l.p[P_LOGSTD], a->adv_stats, R, A,
              a->clip_range, a->critic_coef, inv_R, dMean, dV, dLs, Terms);
  LSTM_TRY(colsum(Terms, 4, R, 4, Col, inv_R, 0.f, Small, st));
  LSTM_LAUNCH(finish_metrics_kernel, 1, st, Small, P + l.p[P_LOGSTD], A, (float)R, a->metrics);
  // d/dlogstd: sum_r dlogp (z^2 - 1)  -  entropy_coef  (mean over rows of -c * sum_a (logstd_a + const))
  LSTM_TRY(colsum(dLs, A, R, A, Col, 1.f, -a->entropy_coef, gP + l.p[P_LOGSTD], st));

  // ================================================================ backward: policy head and torso
  LSTM_TRY(dense_bwd_weight(T2, H, dMean, A, H, A, R, Part, gP + l.p[WM], st));
  LSTM_TRY(colsum(dMean, A, R, A, Col, 1.f, 0.f, gP + l.p[BM], st));
  LSTM_TRY(dense_bwd_input_t<EPI_DTANH>(dMean, A, PT + kl.p[WM], H, A, T2, H, dT2, H, R, st));          // dL/d(pre-tanh of torso 2)
  LSTM_TRY(dense_bwd_weight(T1, H, dT2, H, H, H, R, Part, gP + l.p[WT2], st));
  LSTM_TRY(colsum(dT2, H, R, H, Col, 1.f, 0.f, gP + l.p[BT2], st));
  LSTM_TRY(dense_bwd_input_t<EPI_DTANH>(dT2, H, PT + kl.p[WT2], H, H, T1, H, dT1, H, R, st));
  LSTM_TRY(dense_bwd_weight(TI, TIW, dT1, H, TIW, H, R, Part, gP + l.p[WT1], st));
  LSTM_TRY(colsum(dT1, H, R, H, Col, 1.f, 0.f, gP + l.p[BT1], st));
  LSTM_TRY(dense_bwd_input_t<EPI_NONE>(dT1, H, PT + kl.p[WT1], TIW, H, nullptr, 0, dTI, TIW, R, st));   // concat: [dOL | dLL]; FiLM: d(OL * gamma + beta)
  // gradients wrt the two latents
  const float* dOL = dTI;
  int lddOL = EL;
  const float* dLL = dTI + E;
  int lddLL = EL;
  if (film) {
    float *GB = ws + w.GB, *dGB = ws + w.dGB;
    LSTM_LAUNCH(film_bwd_kernel, R * E, st, dTI, OL, ldOL, GB, R, E, dGB, ws + w.dOL);
    LSTM_TRY(dense_bwd_weight(LLp, L, dGB, 2 * E, L, 2 * E, R, Part, gP + l.p[WF], st));
    LSTM_TRY(colsum(dGB, 2 * E, R, 2 * E, Col, 1.f, 0.f, gP + l.p[BF], st));
    LSTM_TRY(dense_bwd_input_t<EPI_NONE>(dGB, 2 * E, PT + kl.p[WF], L, 2 * E, nullptr, 0, ws + w.dLL, L, R, st));
    dOL = ws + w.dOL; lddOL = E;
    dLL = ws + w.dLL; lddLL = L;
  }
  // lstm_ln (+ tanh) backward -> dHall
  LSTM_TRY(ln_param_grads(dLL, lddLL, LLp, ldLL, Hall, L, R, L, SL, Col, gP + l.p[GL], gP + l.p[NL], st));
  LSTM_LAUNCH(ln_tanh_bwd_kernel, R, st, dLL, lddLL, LLp, ldLL, Hall, L, R, L, P + l.p[GL], SL, dHall, L);
  // obs_encoder backward (a shared encoder receives dOL together with the LSTM's input gradient below)
  if (!shared) {
    LSTM_TRY(ln_param_grads(dOL, lddOL, OL, ldOL, Z2, E, R, E, S2, Col, gP + l.p[G2], gP + l.p[N2], st));
    LSTM_LAUNCH(ln_tanh_bwd_kernel, R, st, dOL, lddOL, OL, ldOL, Z2, E, R, E, P + l.p[G2], S2, dZ2, E);
    LSTM_TRY(dense_bwd_weight(X, O, dZ2, E, O, E, R, Part, gP + l.p[WE2], st));
    LSTM_TRY(colsum(dZ2, E, R, E, Col, 1.f, 0.f, gP + l.p[BE2], st));
  }

  // ================================================================ back-propagation through time, one launch per step
  LSTM_LAUNCH(transpose_kernel, (long long)L * 4 * L, st, P + l.p[WH], L, 4 * L, WhT);
  if (seq.ok) {
    RLX_BLOCK_LAUNCH(lstm_seq_bwd_kernel, ceil_div(n, seq.epb), seq.threads, seq.smem_bwd, st, dHall, WhT, a->dones, Gates, Call, Cm, T, n, L, seq.epb, dG);
    ++g_lstm_persistent_launches;
  } else {
    for (long long t = T - 1; t >= 0; --t) {
      const bool last = (t == T - 1);
      LSTM_LAUNCH(lstm_step_bwd_kernel, n * L, st, dHall + t * n * L, last ? nullptr : dG + (t + 1) * n * 4 * L, WhT, last ? nullptr : a->dones + t * n,
                  last ? nullptr : dCn, Gates + t * n * 4 * L, Call + t * n * L, Cm + t * n * L, t == 0 ? nullptr : a->dones + (t - 1) * n, n, L,
                  dG + t * n * 4 * L, dCn);
    }
  }
  LSTM_TRY(dense_bwd_weight(Hm, L, dG, 4 * L, L, 4 * L, R, Part, gP + l.p[WH], st));
  LSTM_TRY(colsum(dG, 4 * L, R, 4 * L, Col, 1.f, 0.f, gP + l.p[BH], st));
  LSTM_TRY(dense_bwd_weight(E1, E, dG, 4 * L, E, 4 * L, R, Part, gP + l.p[WI], st));
  LSTM_TRY(dense_bwd_input_t<EPI_NONE>(dG, 4 * L, PT + kl.p[WI], E, 4 * L, nullptr, 0, dE1, E, R, st));
  if (shared) LSTM_LAUNCH(cols_kernel<true>, R * E, st, dOL, lddOL, R, E, dE1, E);
  // lstm_obs_encoder backward
  LSTM_TRY(ln_param_grads(dE1, E, E1, E, Z1, E, R, E, S1, Col, gP + l.p[G1], gP + l.p[N1], st));
  LSTM_LAUNCH(ln_tanh_bwd_kernel, R, st, dE1, E, E1, E, Z1, E, R, E, P + l.p[G1], S1, dZ1, E);
  LSTM_TRY(dense_bwd_weight(X, O, dZ1, E, O, E, R, Part, gP + l.p[WE1], st));
  LSTM_TRY(colsum(dZ1, E, R, E, Col, 1.f, 0.f, gP + l.p[BE1], st));

  // ================================================================ backward: critic
  LSTM_TRY(dense_bwd_weight(C2, H, dV, 1, H, 1, R, Part, gC + l.c[WC3], st));
  LSTM_TRY(colsum(dV, 1, R, 1, Col, 1.f, 0.f, gC + l.c[BC3], st));
  LSTM_TRY(dense_bwd_input_t<EPI_DTANH>(dV, 1, CT + kl.c[WC3], H, 1, C2, H, dC2, H, R, st));
  LSTM_TRY(dense_bwd_weight(C1, H, dC2, H, H, H, R, Part, gC + l.c[WC2], st));
  LSTM_TRY(colsum(dC2, H, R, H, Col, 1.f, 0.f, gC + l.c[BC2], st));
  LSTM_TRY(dense_bwd_input_t<EPI_DTANH>(dC2, H, CT + kl.c[WC2], H, H, C1, H, dC1, H, R, st));
  LSTM_TRY(dense_bwd_weight(X, O, dC1, H, O, H, R, Part, gC + l.c[WC1], st));
  LSTM_TRY(colsum(dC1, H, R, H, Col, 1.f, 0.f, gC + l.c[BC1], st));
  return RLX_OK;
}


// policy.apply_one_step on n rows (policy.py:115-125): leaves Mean in the workspace, updates c / h in place
static int policy_one_step(const rlx_lstm_dims& d, const Layout& l, const Ws& w, float* ws, const float* P, const float* obs, float* c, float* h,
                           long long n, cudaStream_t st) {
  const int O = d.obs_dim, A = d.act_dim, H = d.hidden, E = d.enc_dim, L = d.lstm_dim, EL = E + L;
  float *Z1 = ws + w.Z1, *E1 = ws + w.E1, *Z2 = ws + w.Z2, *TI = ws + w.TI, *Gi = ws + w.Gi, *Gates = ws + w.Gates, *Gh = ws + w.Gh, *T1 = ws + w.T1,
        *T2 = ws + w.T2, *Mean = ws + w.Mean, *S1 = ws + w.Stats1, *S2 = ws + w.Stats2, *SL = ws + w.StatsL;
  const bool film = is_film(d), shared = is_shared(d);  // same placement of the latents as in rlx_lstm_ppo_minibatch_fwdbwd_f32
  const int TIW = film ? E : EL;
  float* OL = shared ? E1 : (film ? ws + w.E2 : TI);
  const int ldOL = (shared || film) ? E : EL;
  float* LLp = film ? ws + w.LL : TI + E;
  const int ldLL = film ? L : EL;
  LSTM_TRY(dense_fwd<EPI_BIAS>(obs, O, P + l.p[WE1], O, E, P + l.p[BE1], Z1, E, n, st));
  LSTM_LAUNCH(ln_tanh_fwd_kernel, n, st, Z1, E, n, E, P + l.p[G1], P + l.p[N1], E1, E, S1);
  if (!shared) {
    LSTM_TRY(dense_fwd<EPI_BIAS>(obs, O, P + l.p[WE2], O, E, P + l.p[BE2], Z2, E, n, st));
    LSTM_LAUNCH(ln_tanh_fwd_kernel, n, st, Z2, E, n, E, P + l.p[G2], P + l.p[N2], OL, ldOL, S2);
  } else if (!film) {
    LSTM_LAUNCH(cols_kernel<false>, n * E, st, E1, E, n, E, TI, EL);
  }
  LSTM_TRY(dense_fwd<EPI_NONE>(E1, E, P + l.p[WI], E, 4 * L, nullptr, Gi, 4 * L, n, st));
  LSTM_TRY(dense_fwd<EPI_NONE>(h, L, P + l.p[WH], L, 4 * L, nullptr, Gh, 4 * L, n, st));
  LSTM_LAUNCH(lstm_cell_fwd_kernel, n * L, st, Gi, Gh, P + l.p[BH], c, n, L, Gates, c, h);  // element-wise in place: thread (e, j) reads and writes c[e, j] only
  LSTM_LAUNCH(ln_tanh_fwd_kernel, n, st, h, L, n, L, P + l.p[GL], P + l.p[NL], LLp, ldLL, SL);
  if (film) {
    LSTM_TRY(dense_fwd<EPI_BIAS>(LLp, L, P + l.p[WF], L, 2 * E, P + l.p[BF], ws + w.GB, 2 * E, n, st));
    LSTM_LAUNCH(film_fwd_kernel, n * E, st, OL, ldOL, ws + w.GB, n, E, TI);
  }
  LSTM_TRY(dense_fwd<EPI_BIAS_TANH>(TI, TIW, P + l.p[WT1], TIW, H, P + l.p[BT1], T1, H, n, st));
  LSTM_TRY(dense_fwd<EPI_BIAS_TANH>(T1, H, P + l.p[WT2], H, H, P + l.p[BT2], T2, H, n, st));
  LSTM_TRY(dense_fwd<EPI_BIAS>(T2, H, P + l.p[WM], H, A, P + l.p[BM], Mean, A, n, st));
  return RLX_OK;
}
static int critic_rows(const rlx_lstm_dims& d, const Layout& l, const Ws& w, float* ws, const float* Cp, const float* x, long long rows, float* out,
                       cudaStream_t st) {
  const int O = d.obs_dim, H = d.hidden;
  float *C1 = ws + w.C1, *C2 = ws + w.C2;
  LSTM_TRY(dense_fwd<EPI_BIAS_TANH>(x, O, Cp + l.c[WC1], O, H, Cp + l.c[BC1], C1, H, rows, st));
  LSTM_TRY(dense_fwd<EPI_BIAS_TANH>(C1, H, Cp + l.c[WC2], H, H, Cp + l.c[BC2], C2, H, rows, st));
  LSTM_TRY(dense_fwd<EPI_BIAS>(C2, H, Cp + l.c[WC3], H, 1, Cp + l.c[BC3], out, 1, rows, st));
  return RLX_OK;
}

extern "C" int rlx_lstm_step_f32(const rlx_lstm_step_args* a, void* stream) {
  RLX_CHECK_ARG(a != nullptr && dims_ok(a->dims) && a->n > 0, "bad arguments");
  RLX_CHECK_ARG(a->obs && a->c && a->h && a->policy_params && a->action && a->env_action, "null pointer");
  RLX_CHECK_ARG((a->value == nullptr) || a->critic_params, "value requested without critic parameters");
  RLX_CHECK_ARG(!a->clip_rescale || (a->act_low && a->act_high), "action bounds are required for clipping / rescaling");
  const Ws w = plan(a->dims, 1, a->n);
  if (a->workspace == nullptr || a->workspace_bytes < w.total) {
    set_error("rlx_lstm_step_f32: workspace too small (%zu < %zu)", a->workspace_bytes, w.total);
    return RLX_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const Layout l = make_layout(a->dims);
  float* ws = (float*)a->workspace;
  LSTM_TRY(policy_one_step(a->dims, l, w, ws, a->policy_params, a->obs, a->c, a->h, a->n, st));
  LSTM_LAUNCH(sample_rows_kernel, a->n, st, ws + w.Mean, a->policy_params + l.p[P_LOGSTD], a->noise, (long long)a->n, a->dims.act_dim, a->act_low,
              a->act_high, a->clip_rescale, a->action, a->env_action, a->logp);
  if (a->value) LSTM_TRY(critic_rows(a->dims, l, w, ws, a->critic_params, a->obs, a->n, a->value, st));
  return RLX_OK;
}

extern "C" int rlx_lstm_mask_carry_f32(float* c, float* h, const float* done, int64_t n, int64_t lstm_dim, void* stream) {
  RLX_CHECK_ARG(n >= 0 && lstm_dim > 0, "bad sizes");
  if (n == 0) return RLX_OK;
  RLX_CHECK_ARG(c && h && done, "null pointer");
  LSTM_LAUNCH(carry_mask_kernel, (long long)n * lstm_dim, (cudaStream_t)stream, c, h, done, (long long)n, (int)lstm_dim);
  return RLX_OK;
}

extern "C" int rlx_lstm_critic_forward_f32(const rlx_lstm_dims* d, const float* critic_params, const float* x, int64_t rows, float* out,
                                           void* workspace, size_t workspace_bytes, void* stream) {
  RLX_CHECK_ARG(d != nullptr && dims_ok(*d) && rows >= 0, "bad arguments");
  if (rows == 0) return RLX_OK;
  RLX_CHECK_ARG(critic_params && x && out, "null pointer");
  const Ws w = plan(*d, 1, rows);
  if (workspace == nullptr || workspace_bytes < w.total) {
    set_error("rlx_lstm_critic_forward_f32: workspace too small (%zu < %zu)", workspace_bytes, w.total);
    return RLX_ERR_WORKSPACE;
  }
  return critic_rows(*d, make_layout(*d), w, (float*)workspace, critic_params, x, rows, out, (cudaStream_t)stream);
}

extern "C" int rlx_mean_popstd_f32(const float* x, int64_t n, float* out, float* workspace, void* stream) {
  RLX_CHECK_ARG(n > 0 && x && out && workspace, "bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  float* sq = workspace;           // [n]
  float* col = workspace + n;      // column-sum partials
  LSTM_TRY(colsum(x, 1, n, 1, col, 1.f / (float)n, 0.f, out, st));
  LSTM_LAUNCH(centered_sq_kernel, (long long)n, st, x, (long long)n, out, sq);
  LSTM_TRY(colsum(sq, 1, n, 1, col, 1.f / (float)n, 0.f, out + 1, st));
  LSTM_LAUNCH(sqrt_inplace_kernel, 1, st, out + 1);
  return RLX_OK;
}

extern "C" int rlx_optax_clip_adam_f32(float* params, const float* grads, float* mu, float* nu, int64_t n, const float* lr, int64_t* step_count,
                                       float max_norm, float beta1, float beta2, float eps, float* norm_out, float* workspace, void* stream) {
  RLX_CHECK_ARG(n >= 0, "negative size");
  if (n == 0) return RLX_OK;
  RLX_CHECK_ARG(params && grads && mu && nu && lr && step_count && norm_out && workspace, "null pointer");
  const long long nchunk = ceil_div(n, 1024);  // the workspace holds one partial sum of squares per 1024 elements
  cudaStream_t st = (cudaStream_t)stream;
  LSTM_LAUNCH(sumsq_partial_kernel, nchunk, st, grads, (long long)n, workspace);
  LSTM_LAUNCH(sumsq_final_kernel, 1, st, workspace, nchunk, norm_out, (long long*)step_count);
  LSTM_LAUNCH(optax_adam_kernel, (long long)n, st, params, grads, mu, nu, (long long)n, lr, (const long long*)step_count, norm_out, max_norm, beta1,
              beta2, eps);
  return RLX_OK;
}

extern "C" int rlx_gather_env_columns_f32(const float* src, const int64_t* env_idx, int64_t T, int64_t N, int64_t n, int64_t width, float* out,
                                          void* stream) {
  RLX_CHECK_ARG(T >= 0 && N > 0 && n >= 0 && width > 0, "bad sizes");
  if (T == 0 || n == 0) return RLX_OK;
  RLX_CHECK_ARG(src && env_idx && out, "null pointer");
  LSTM_LAUNCH(gather_env_kernel, (long long)T * n * width, (cudaStream_t)stream, src, (const long long*)env_idx, (long long)T, (long long)N,
              (long long)n, (long long)width, out);
  return RLX_OK;
}
