// SAC update path (ref: rl_x/algorithms/sac/pytorch/sac.py:89-159,219-259): replay-sampled batch -> target, twin-Q update, Polyak,
// actor + temperature update, all launched from one C call with no host round trip.
//
// Networks (ref: sac/pytorch/policy.py:34-43, q_network.py:27-33): policy obs -> H -> H -> (mean | log_std), ReLU; Q (obs+act) -> H -> H -> 1,
// ReLU, four copies (q1, q2, q1_target, q2_target).  Flat parameter layouts:
//   policy [Pp]: W1[H,O] b1[H] W2[H,H] b2[H] Wm[A,H] Ws[A,H] bm[A] bs[A]      (Wm|Ws adjacent: the two heads are one [2A,H] GEMM)
//   q      [4][Pq]: W1[H,O+A] b1[H] W2[H,H] b2[H] W3[H] b3[1], order q1, q2, q1_target, q2_target (online nets first: one Adam over 2*Pq)
// At batch 4096 / hidden 256 the update is launch-latency-bound (SURVEY.md §8 a15), so the value here is that the ~45 launches
// are issued back-to-back from C++.  Forward and input-gradient GEMMs go through run_gemm (gemm_dispatch.cuh): the wgmma 3xTF32 engine
// under rlx_set_gemm_engine(1) where it covers the shape, the exact-fp32 SIMT engine otherwise; weight gradients always run SIMT.
#include "common.cuh"
#include "gemm_simt.cuh"
#include "gemm_dispatch.cuh"

namespace rlx {

struct SacLayout {
  int O, A, H;
  // policy offsets
  long long pW1, pb1, pW2, pb2, pWh, pbh, Pp;  // Wh = [Wm; Ws] (2A x H), bh = [bm; bs]
  // q offsets (within one net)
  long long qW1, qb1, qW2, qb2, qW3, qb3, Pq;
};
static SacLayout sac_layout(int O, int A, int H) {
  SacLayout L{};
  L.O = O; L.A = A; L.H = H;
  long long o = 0;
  L.pW1 = o; o += (long long)H * O;
  L.pb1 = o; o += H;
  L.pW2 = o; o += (long long)H * H;
  L.pb2 = o; o += H;
  L.pWh = o; o += 2LL * A * H;
  L.pbh = o; o += 2LL * A;
  L.Pp = o;
  o = 0;
  L.qW1 = o; o += (long long)H * (O + A);
  L.qb1 = o; o += H;
  L.qW2 = o; o += (long long)H * H;
  L.qb2 = o; o += H;
  L.qW3 = o; o += H;
  L.qb3 = o; o += 1;
  L.Pq = (o + 63) / 64 * 64;  // per-net stride padded to 256 bytes: every net's tensors keep the 16-byte alignment TMA needs
  return L;
}

// ----------------------------------------------------------------------------------------------- small kernels
__global__ void __launch_bounds__(256) sac_concat_kernel(const float* __restrict__ s, const float* __restrict__ a, float* __restrict__ out, int B,
                                                         int O, int A) {
  const long long n = (long long)B * (O + A);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / (O + A)), c = (int)(i % (O + A));
    out[i] = (c < O) ? s[(long long)r * O + c] : a[(long long)r * A + (c - O)];
  }
}

// Policy head -> squashed action and its log-prob (ref: policy.py:45-64).  head [B, 2A] = (mean | log_std).
__global__ void __launch_bounds__(256) sac_sample_kernel(const float* __restrict__ head, const float* __restrict__ eps, int B, int A, float ls_min,
                                                         float ls_max, const float* __restrict__ low, const float* __restrict__ high,
                                                         float* __restrict__ a_tanh, float* __restrict__ scaled, float* __restrict__ logp,
                                                         int deterministic) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long r = warp; r < B; r += nwarps) {
    float lp = 0.f;
    for (int j = lane; j < A; j += 32) {
      const float mean = head[r * 2 * A + j];
      float u = mean, t;
      if (!deterministic) {
        const float ls = fminf(fmaxf(head[r * 2 * A + A + j], ls_min), ls_max);
        const float sd = expf(ls);
        u = __fadd_rn(mean, __fmul_rn(sd, eps[r * A + j]));  // normal.rsample()
        t = tanhf(u);
        const float d = u - mean;
        // normal.log_prob(action) - log(1 - tanh^2 + 1e-6)
        lp += -(d * d) / (2.f * (sd * sd)) - logf(sd) - 0.91893853320467274178f - logf((1.f - t * t) + 1e-6f);
      } else {
        t = tanhf(u);
      }
      if (a_tanh) a_tanh[r * A + j] = t;
      if (scaled) scaled[r * A + j] = low[j] + (0.5f * (t + 1.f)) * (high[j] - low[j]);
    }
    if (!deterministic && logp) {
      lp = warp_sum(lp);
      if (lane == 0) logp[r] = lp;
    }
  }
}

// y = r + gamma (1 - d) (min(q1t, q2t) - alpha logp')     (ref: sac.py:131-138)
__global__ void __launch_bounds__(256) sac_target_kernel(const float* __restrict__ qt /*[2][B]*/, const float* __restrict__ logp_next,
                                                         const float* __restrict__ rew, const float* __restrict__ done, const float* __restrict__ log_alpha,
                                                         float gamma, int B, float* __restrict__ y) {
  const float alpha = expf(log_alpha[0]);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < B; i += gridDim.x * blockDim.x) {
    const float mq = fminf(qt[i], qt[B + i]);
    y[i] = rew[i] + gamma * (1.f - done[i]) * (mq - alpha * logp_next[i]);
  }
}

// q_loss = (mse(q1,y) + mse(q2,y)) / 2 and dq_n = (q_n - y) / B        (ref: sac.py:140-144).  Single block.
__global__ void __launch_bounds__(1024) sac_critic_loss_kernel(const float* __restrict__ q /*[2][B]*/, const float* __restrict__ y, int B,
                                                               float* __restrict__ dq /*[2][B]*/, float* __restrict__ metrics) {
  __shared__ float sh[34];
  float s = 0.f;
  const float invB = 1.f / (float)B;
  for (int i = threadIdx.x; i < B; i += blockDim.x) {
    const float e1 = q[i] - y[i], e2 = q[B + i] - y[i];
    dq[i] = e1 * invB;
    dq[B + i] = e2 * invB;
    s += e1 * e1 + e2 * e2;
  }
  s = block_sum(s, sh);
  if (threadIdx.x == 0) metrics[5] = 0.5f * s * invB;  // loss/q_loss
}

// policy_loss = mean(alpha logp - min(q1,q2));  dq_n = -w_n / B (torch.minimum splits ties evenly)   (ref: sac.py:93-101).  Single block.
__global__ void __launch_bounds__(1024) sac_policy_loss_kernel(const float* __restrict__ q, const float* __restrict__ logp, const float* __restrict__ log_alpha,
                                                               float target_entropy, int B, float* __restrict__ dq, float* __restrict__ metrics,
                                                               float* __restrict__ g_log_alpha) {
  __shared__ float sh[34];
  const float alpha = expf(log_alpha[0]);
  const float invB = 1.f / (float)B;
  float s_loss = 0.f, s_minq = 0.f, s_lp = 0.f;
  for (int i = threadIdx.x; i < B; i += blockDim.x) {
    const float q1 = q[i], q2 = q[B + i];
    const float w1 = (q1 < q2) ? 1.f : ((q1 == q2) ? 0.5f : 0.f);
    dq[i] = -w1 * invB;
    dq[B + i] = -(1.f - w1) * invB;
    const float mq = fminf(q1, q2);
    s_loss += alpha * logp[i] - mq;
    s_minq += mq;
    s_lp += logp[i];
  }
  s_loss = block_sum(s_loss, sh);
  s_minq = block_sum(s_minq, sh);
  s_lp = block_sum(s_lp, sh);
  if (threadIdx.x == 0) {
    const float ent_mean = -s_lp * invB;                        // entropy_detach.mean()
    const float ent_loss = alpha * (ent_mean - target_entropy); // (log_alpha.exp() * (entropy - target)).mean()
    metrics[0] = alpha;            // entropy/alpha
    metrics[1] = ent_mean;         // entropy/entropy
    metrics[6] = s_loss * invB;    // loss/policy_loss
    metrics[7] = ent_loss;         // loss/entropy_loss
    metrics[8] = s_minq * invB;    // q_value/q_value
    g_log_alpha[0] = ent_loss;     // d/dlog_alpha of exp(log_alpha) * c  ==  exp(log_alpha) * c
    metrics[4] = ent_loss * ent_loss;  // gradients/entropy_grad_norm (the reference logs the squared norm, sac.py:122)
  }
}

// Gradient of the policy loss wrt the head outputs (mean | log_std), given dL/da_tanh from the Q nets (dxa_n[:, O:O+A]) and
// dL/dlogp = alpha / B.  Reparameterised sample u = mean + std eps:  d logp_normal / d mean = 0, d logp_normal / d log_std = -1,
// tanh correction d/du [-log(1 - t^2 + 1e-6)] = 2 t (1 - t^2) / (1 - t^2 + 1e-6).
__global__ void __launch_bounds__(256) sac_policy_grad_kernel(const float* __restrict__ head, const float* __restrict__ eps, const float* __restrict__ a_tanh,
                                                              const float* __restrict__ dxa /*[2][B, O+A]*/, const float* __restrict__ log_alpha, int B,
                                                              int O, int A, float ls_min, float ls_max, float* __restrict__ dhead /*[B, 2A]*/) {
  const float dlogp = expf(log_alpha[0]) / (float)B;
  const long long n = (long long)B * A;
  const long long xs = (long long)B * (O + A);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / A;
    const int j = (int)(i % A);
    const float t = a_tanh[i];
    const float da = dxa[r * (O + A) + O + j] + dxa[xs + r * (O + A) + O + j];
    const float one_m = 1.f - t * t;
    const float du = da * one_m + dlogp * (2.f * t * one_m / (one_m + 1e-6f));
    const float ls_raw = head[r * 2 * A + A + j];
    const bool in_range = ls_raw >= ls_min && ls_raw <= ls_max;  // clamp passes the gradient on the closed interval
    const float sd = expf(fminf(fmaxf(ls_raw, ls_min), ls_max));
    dhead[r * 2 * A + j] = du;
    dhead[r * 2 * A + A + j] = in_range ? (du * sd * eps[i] - dlogp) : 0.f;
  }
}

// dst[b][i] = sum_s src[s*split_stride + b*src_batch + i]   (+ rowsum variant shares it)
__global__ void __launch_bounds__(256) sac_reduce_partials_kernel(float* __restrict__ dst, long long dst_batch, const float* __restrict__ src,
                                                                  long long src_batch, long long split_stride, int nsplit, long long n, int batch) {
  const long long tot = n * batch;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < tot; t += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(t / n);
    const long long i = t % n;
    const float* q = src + b * src_batch + i;
    float s = 0.f;
    for (int sp = 0; sp < nsplit; ++sp) s += q[sp * split_stride];
    dst[b * dst_batch + i] = s;
  }
}

// Adam without clipping on a flat buffer (ref: optim.Adam defaults, sac.py:75-77); step counter incremented by thread 0 of block 0 of
// the preceding sumsq kernel.  norms_out[seg] = sum of squares of the first `valid` elements of segment seg (for logging only).  The
// elements [valid, seg_len) of each segment are the pad of a per-net stride that no gradient kernel writes: they are set to zero here,
// so that whatever the caller's buffer held there, the norm and the Adam step that follows never see it.
__global__ void __launch_bounds__(256) sac_sumsq_step_kernel(float* __restrict__ g, long long n, long long seg_len, long long valid, int nseg,
                                                             float* __restrict__ out, long long* step) {
  __shared__ float sh[34];
  const int seg = blockIdx.x;
  float s = 0.f;
  if (seg < nseg) {
    float* p = g + seg * seg_len;
    for (long long i = threadIdx.x; i < valid; i += blockDim.x) s = fmaf(p[i], p[i], s);
    for (long long i = valid + threadIdx.x; i < seg_len; i += blockDim.x) p[i] = 0.f;
  }
  s = block_sum(s, sh);
  if (threadIdx.x == 0) {
    out[seg] = s;
    if (seg == 0) step[0] += 1;
  }
}
__global__ void __launch_bounds__(256) sac_adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                                                       long long n, const float* __restrict__ lr, const long long* __restrict__ step, float b1, float b2,
                                                       float eps) {
  __shared__ float sc[2];
  if (threadIdx.x == 0) {
    const double t = (double)step[0];
    sc[0] = (float)((double)lr[0] / (1.0 - pow((double)b1, t)));
    sc[1] = (float)sqrt(1.0 - pow((double)b2, t));
  }
  __syncthreads();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float gi = g[i];
  float mi = m[i], vi = v[i];
  mi = mi + (gi - mi) * (1.f - b1);
  vi = vi * b2 + (1.f - b2) * gi * gi;
  p[i] = p[i] - sc[0] * (mi / (sqrtf(vi) / sc[1] + eps));
  m[i] = mi;
  v[i] = vi;
}
__global__ void sac_finish_metrics_kernel(const float* __restrict__ ss_policy, const float* __restrict__ ss_q, float* __restrict__ metrics) {
  if (threadIdx.x == 0) {
    metrics[2] = sqrtf(ss_policy[0]);                    // gradients/policy_grad_norm
    metrics[3] = sqrtf(ss_q[0]) + sqrtf(ss_q[1]);        // gradients/critic_grad_norm = ||g_q1|| + ||g_q2||   (sac.py:149-155)
  }
}

// ------------------------------------------------------------------------------------------------ GEMM helpers
static unsigned small_grid(long long n) { return (unsigned)std::min<long long>(ceil_div(n, 256), (long long)sm_count() * 4); }

// C = act(A W^T + b), batched over `batch` nets with element strides (sA may be 0 for a shared input)
static int layer_fwd(const float* A, int lda, long long sA, const float* W, long long sW, const float* b, long long sb, float* C, int ldc, long long sC,
                     int M, int N, int K, int batch, bool relu, cudaStream_t st) {
  GemmP g{};
  g.A = A; g.B = W; g.C = C; g.bias = b;
  g.M = M; g.N = N; g.K = K;
  g.lda = lda; g.ldb = K; g.ldc = ldc;
  g.sA = sA; g.sB = sW; g.sC = sC; g.sBias = sb;
  g.splits = 1; g.kchunk = (int)(ceil_div(K, 8) * 8);
  const bool tc = g_gemm_engine == 1;
  const long long a_rows = M, b_rows = N;
  return relu ? run_gemm<true, true, EPI_BIAS_RELU>(tc, g, batch, st, KC_GEMM_FWD, a_rows, b_rows)
              : run_gemm<true, true, EPI_BIAS>(tc, g, batch, st, KC_GEMM_FWD, a_rows, b_rows);
}
// dX = (dZ W) [* relu'(aux)],  W is [N_out, K_in] row-major so that dX[m, k] = sum_n dZ[m, n] W[n, k]
static int layer_bwd_input(const float* dZ, int ldz, long long sZ, const float* W, int ldw, long long sW, const float* aux, int ldaux, long long sAux,
                           float* dX, int ldx, long long sX, int M, int Nout, int Kin, int batch, cudaStream_t st) {
  GemmP g{};
  g.A = dZ; g.B = W; g.C = dX; g.aux = aux;
  g.M = M; g.N = Kin; g.K = Nout;
  g.lda = ldz; g.ldb = ldw; g.ldc = ldx; g.ldaux = ldaux;
  g.sA = sZ; g.sB = sW; g.sC = sX; g.sAux = sAux;
  g.splits = 1; g.kchunk = (int)(ceil_div(Nout, 8) * 8);
  const bool tc = g_gemm_engine == 1;
  const long long a_rows = M, b_rows = Nout;
  return aux ? run_gemm<true, false, EPI_DRELU>(tc, g, batch, st, KC_GEMM_DX, a_rows, b_rows)
             : run_gemm<true, false, EPI_NONE>(tc, g, batch, st, KC_GEMM_DX, a_rows, b_rows);
}
// dW[n, k] = sum_m dZ[m, n] X[m, k], db[n] = sum_m dZ[m, n]; split over rows into `part`/`rs`, then reduced into gW / gb (batched).
static int layer_bwd_weight(const float* dZ, int ldz, long long sZ, const float* X, int ldx, long long sX, int M, int Nout, int Kin, int batch, float* part,
                            float* rs, float* gW, float* gb, long long g_batch, cudaStream_t st) {
  const int splits = (int)std::max<long long>(1, std::min<long long>(16, M / 256));
  const int kchunk = (int)(ceil_div(ceil_div(M, splits), 8) * 8);
  const int nsplit = (int)ceil_div(M, kchunk);
  GemmP g{};
  g.A = dZ; g.B = X; g.C = part; g.rowsum = rs;
  g.M = Nout; g.N = Kin; g.K = M;
  g.lda = ldz; g.ldb = ldx; g.ldc = Kin;
  g.sA = sZ; g.sB = sX; g.sC = (long long)Nout * Kin; g.sRowsum = Nout;
  g.splits = nsplit; g.kchunk = kchunk; g.sSplitC = (long long)batch * Nout * Kin; g.sSplitRowsum = (long long)batch * Nout;
  int rc = launch_sgemm<false, false, EPI_NONE>(g, batch, st, KC_GEMM_DW);
  if (rc) return rc;
  const long long nW = (long long)Nout * Kin;
  RLX_LAUNCH_C(KC_GRAD_REDUCE, 0, 4.0 * nW * batch * nsplit, sac_reduce_partials_kernel, small_grid(nW * batch), 256, 0, st, gW, g_batch, part, nW,
               (long long)batch * nW, nsplit, nW, batch);
  RLX_LAUNCH_C(KC_GRAD_REDUCE, 0, 4.0 * Nout * batch * nsplit, sac_reduce_partials_kernel, small_grid((long long)Nout * batch), 256, 0, st, gb, g_batch, rs,
               (long long)Nout, (long long)batch * Nout, nsplit, (long long)Nout, batch);
  return RLX_OK;
}

struct SacWs {
  float *xa, *ph1, *ph2, *phead, *a_tanh, *logp, *logp_next, *qh1, *qh2, *qout, *y, *dq, *dz2, *dz1, *dxa, *dhead, *pdz2, *pdz1, *part, *rs, *ss;
  size_t total;
};
static SacWs sac_plan(const SacLayout& L, long long B, void* base) {
  SacWs w{};
  size_t o = 0;
  auto take = [&](float*& p, size_t n) {
    p = base ? reinterpret_cast<float*>(reinterpret_cast<char*>(base) + o) : nullptr;
    o += align_up(n * sizeof(float), 256);
  };
  const size_t H = L.H, A = L.A, O = L.O;
  take(w.xa, B * (O + A));
  take(w.ph1, B * H); take(w.ph2, B * H); take(w.phead, B * 2 * A);
  take(w.a_tanh, B * A); take(w.logp, B); take(w.logp_next, B);
  take(w.qh1, 2 * B * H); take(w.qh2, 2 * B * H); take(w.qout, 2 * B);
  take(w.y, B); take(w.dq, 2 * B);
  take(w.dz2, 2 * B * H); take(w.dz1, 2 * B * H); take(w.dxa, 2 * B * (O + A));
  take(w.dhead, B * 2 * A); take(w.pdz2, B * H); take(w.pdz1, B * H);
  const size_t max_w = std::max<size_t>(2 * H * std::max<size_t>(H, O + A), 2 * A * H);
  take(w.part, 16 * 2 * std::max<size_t>(max_w, H * std::max(H, O)));
  take(w.rs, 16 * 2 * std::max<size_t>(H, 2 * A));
  take(w.ss, 8);
  w.total = o;
  return w;
}

// policy forward: X [B, O] -> head [B, 2A] (activations kept in ph1 / ph2)
static int policy_forward(const SacLayout& L, const float* pol, const float* X, long long B, const SacWs& w, cudaStream_t st) {
  int rc = layer_fwd(X, L.O, 0, pol + L.pW1, 0, pol + L.pb1, 0, w.ph1, L.H, 0, (int)B, L.H, L.O, 1, true, st);
  if (rc) return rc;
  rc = layer_fwd(w.ph1, L.H, 0, pol + L.pW2, 0, pol + L.pb2, 0, w.ph2, L.H, 0, (int)B, L.H, L.H, 1, true, st);
  if (rc) return rc;
  return layer_fwd(w.ph2, L.H, 0, pol + L.pWh, 0, pol + L.pbh, 0, w.phead, 2 * L.A, 0, (int)B, 2 * L.A, L.H, 1, false, st);
}
// twin Q forward on xa [B, O+A] with nets q + net0*Pq, q + (net0+1)*Pq  -> qout [2][B]
static int q_forward(const SacLayout& L, const float* q, int net0, long long B, const SacWs& w, cudaStream_t st) {
  const float* base = q + net0 * L.Pq;
  int rc = layer_fwd(w.xa, L.O + L.A, 0, base + L.qW1, L.Pq, base + L.qb1, L.Pq, w.qh1, L.H, B * L.H, (int)B, L.H, L.O + L.A, 2, true, st);
  if (rc) return rc;
  rc = layer_fwd(w.qh1, L.H, B * L.H, base + L.qW2, L.Pq, base + L.qb2, L.Pq, w.qh2, L.H, B * L.H, (int)B, L.H, L.H, 2, true, st);
  if (rc) return rc;
  return layer_fwd(w.qh2, L.H, B * L.H, base + L.qW3, L.Pq, base + L.qb3, L.Pq, w.qout, 1, B, (int)B, 1, L.H, 2, false, st);
}

}  // namespace rlx

using namespace rlx;

extern "C" int64_t rlx_sac_policy_param_count(int32_t obs_dim, int32_t act_dim, int32_t hidden) { return sac_layout(obs_dim, act_dim, hidden).Pp; }
extern "C" int64_t rlx_sac_q_param_count(int32_t obs_dim, int32_t act_dim, int32_t hidden) { return sac_layout(obs_dim, act_dim, hidden).Pq; }
extern "C" size_t rlx_sac_workspace_bytes(int32_t obs_dim, int32_t act_dim, int32_t hidden, int64_t batch) {
  return sac_plan(sac_layout(obs_dim, act_dim, hidden), batch, nullptr).total;
}

extern "C" int rlx_sac_act_f32(const rlx_sac_dims* d, const float* policy_params, const float* obs, const float* eps, int64_t n, const float* act_low,
                               const float* act_high, int32_t deterministic, float* action_tanh, float* env_action, float* logp, void* workspace,
                               size_t workspace_bytes, void* stream) {
  RLX_CHECK_ARG(d && policy_params && obs && n >= 0, "bad arguments");
  RLX_CHECK_ARG(deterministic || eps, "eps required for stochastic actions");
  if (n == 0) return RLX_OK;
  const SacLayout L = sac_layout(d->obs_dim, d->act_dim, d->hidden);
  const SacWs w = sac_plan(L, n, workspace);
  if (!workspace || workspace_bytes < w.total) {
    set_error("rlx_sac_act_f32: workspace too small (%zu < %zu)", workspace_bytes, w.total);
    return RLX_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  int rc = policy_forward(L, policy_params, obs, n, w, st);
  if (rc) return rc;
  RLX_LAUNCH_C(KC_HEAD_ROLLOUT, 0, 0, sac_sample_kernel, small_grid(n * 32), 256, 0, st, w.phead, eps, (int)n, L.A, d->log_std_min, d->log_std_max, act_low,
               act_high, action_tanh, env_action, logp, deterministic);
  return RLX_OK;
}

extern "C" int rlx_sac_update_f32(const rlx_sac_update_args* a, void* stream) {
  RLX_CHECK_ARG(a != nullptr, "args is null");
  RLX_CHECK_ARG(a->batch > 0 && a->batch < (1 << 30), "bad batch size");
  RLX_CHECK_ARG(a->policy && a->q && a->log_alpha && a->states && a->next_states && a->actions && a->rewards && a->terminations && a->eps_next && a->eps_cur,
                "null tensor");
  RLX_CHECK_ARG(a->g_policy && a->g_q && a->g_log_alpha && a->m_policy && a->v_policy && a->m_q && a->v_q && a->m_log_alpha && a->v_log_alpha && a->lr &&
                    a->steps && a->metrics,
                "null optimizer state");
  const SacLayout L = sac_layout(a->dims.obs_dim, a->dims.act_dim, a->dims.hidden);
  const long long B = a->batch;
  const SacWs w = sac_plan(L, B, a->workspace);
  if (!a->workspace || a->workspace_bytes < w.total) {
    set_error("rlx_sac_update_f32: workspace too small (%zu < %zu)", a->workspace_bytes, w.total);
    return RLX_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int O = L.O, A = L.A, H = L.H, OA = O + A;
  const float lsmin = a->dims.log_std_min, lsmax = a->dims.log_std_max;
  int rc;
  // ================================================================ critic step (sac.py:129-159)
  // -- target: a', logp' = pi(s');  y = r + gamma (1-d) (min Q_target(s', a') - alpha logp')
  if ((rc = policy_forward(L, a->policy, a->next_states, B, w, st))) return rc;
  RLX_LAUNCH_C(KC_HEAD_ROLLOUT, 0, 0, sac_sample_kernel, small_grid(B * 32), 256, 0, st, w.phead, a->eps_next, (int)B, A, lsmin, lsmax, a->act_low, a->act_high,
               w.a_tanh, (float*)nullptr, w.logp_next, 0);
  RLX_LAUNCH_C(KC_OTHER, 0, 0, sac_concat_kernel, small_grid(B * OA), 256, 0, st, a->next_states, w.a_tanh, w.xa, (int)B, O, A);
  if ((rc = q_forward(L, a->q, 2, B, w, st))) return rc;
  RLX_LAUNCH_C(KC_OTHER, 0, 0, sac_target_kernel, small_grid(B), 256, 0, st, w.qout, w.logp_next, a->rewards, a->terminations, a->log_alpha, a->gamma, (int)B,
               w.y);
  // -- online Q on (s, a) and the MSE gradient
  RLX_LAUNCH_C(KC_OTHER, 0, 0, sac_concat_kernel, small_grid(B * OA), 256, 0, st, a->states, a->actions, w.xa, (int)B, O, A);
  if ((rc = q_forward(L, a->q, 0, B, w, st))) return rc;
  RLX_LAUNCH_C(KC_OTHER, 0, 0, sac_critic_loss_kernel, 1, 1024, 0, st, w.qout, w.y, (int)B, w.dq, a->metrics);
  // -- backward through both online nets (batched)
  float* gq = a->g_q;
  // layer 3: dW3[n] = sum_b dq[n][b] QH2[n][b,:], db3 = sum_b dq
  if ((rc = layer_bwd_weight(w.dq, 1, B, w.qh2, H, B * H, (int)B, 1, H, 2, w.part, w.rs, gq + L.qW3, gq + L.qb3, L.Pq, st))) return rc;
  if ((rc = layer_bwd_input(w.dq, 1, B, a->q + L.qW3, H, L.Pq, w.qh2, H, B * H, w.dz2, H, B * H, (int)B, 1, H, 2, st))) return rc;
  if ((rc = layer_bwd_weight(w.dz2, H, B * H, w.qh1, H, B * H, (int)B, H, H, 2, w.part, w.rs, gq + L.qW2, gq + L.qb2, L.Pq, st))) return rc;
  if ((rc = layer_bwd_input(w.dz2, H, B * H, a->q + L.qW2, H, L.Pq, w.qh1, H, B * H, w.dz1, H, B * H, (int)B, H, H, 2, st))) return rc;
  if ((rc = layer_bwd_weight(w.dz1, H, B * H, w.xa, OA, 0, (int)B, H, OA, 2, w.part, w.rs, gq + L.qW1, gq + L.qb1, L.Pq, st))) return rc;
  // -- grad norms (logging) + Adam over q1 U q2
  RLX_LAUNCH_C(KC_CLIP_ADAM, 0, 0, sac_sumsq_step_kernel, 2, 256, 0, st, gq, 2 * L.Pq, L.Pq, L.qb3 + 1, 2, w.ss + 1, (long long*)a->steps + 1);
  RLX_LAUNCH_C(KC_CLIP_ADAM, 0, 28.0 * 2 * L.Pq, sac_adam_kernel, (unsigned)ceil_div(2 * L.Pq, 256), 256, 0, st, a->q, gq, a->m_q, a->v_q, 2 * L.Pq, a->lr,
               (const long long*)a->steps + 1, a->adam_beta1, a->adam_beta2, a->adam_eps);
  // ================================================================ Polyak (sac.py:238-242)
  if ((rc = rlx_polyak_f32(a->q + 2 * L.Pq, a->q, 2 * L.Pq, a->tau, stream))) return rc;
  // ================================================================ actor + temperature step (sac.py:91-126)
  if ((rc = policy_forward(L, a->policy, a->states, B, w, st))) return rc;
  RLX_LAUNCH_C(KC_HEAD_ROLLOUT, 0, 0, sac_sample_kernel, small_grid(B * 32), 256, 0, st, w.phead, a->eps_cur, (int)B, A, lsmin, lsmax, a->act_low, a->act_high,
               w.a_tanh, (float*)nullptr, w.logp, 0);
  RLX_LAUNCH_C(KC_OTHER, 0, 0, sac_concat_kernel, small_grid(B * OA), 256, 0, st, a->states, w.a_tanh, w.xa, (int)B, O, A);
  if ((rc = q_forward(L, a->q, 0, B, w, st))) return rc;  // the just-updated online critics
  RLX_LAUNCH_C(KC_OTHER, 0, 0, sac_policy_loss_kernel, 1, 1024, 0, st, w.qout, w.logp, a->log_alpha, a->target_entropy, (int)B, w.dq, a->metrics, a->g_log_alpha);
  // -- through the critics to their action input (critic parameter gradients are not needed: q_optimizer.zero_grad() discards them)
  if ((rc = layer_bwd_input(w.dq, 1, B, a->q + L.qW3, H, L.Pq, w.qh2, H, B * H, w.dz2, H, B * H, (int)B, 1, H, 2, st))) return rc;
  if ((rc = layer_bwd_input(w.dz2, H, B * H, a->q + L.qW2, H, L.Pq, w.qh1, H, B * H, w.dz1, H, B * H, (int)B, H, H, 2, st))) return rc;
  if ((rc = layer_bwd_input(w.dz1, H, B * H, a->q + L.qW1, OA, L.Pq, nullptr, 0, 0, w.dxa, OA, B * OA, (int)B, H, OA, 2, st))) return rc;
  RLX_LAUNCH_C(KC_OTHER, 0, 0, sac_policy_grad_kernel, small_grid(B * A), 256, 0, st, w.phead, a->eps_cur, w.a_tanh, w.dxa, a->log_alpha, (int)B, O, A, lsmin,
               lsmax, w.dhead);
  // -- policy backward
  float* gp = a->g_policy;
  if ((rc = layer_bwd_weight(w.dhead, 2 * A, 0, w.ph2, H, 0, (int)B, 2 * A, H, 1, w.part, w.rs, gp + L.pWh, gp + L.pbh, 0, st))) return rc;
  if ((rc = layer_bwd_input(w.dhead, 2 * A, 0, a->policy + L.pWh, H, 0, w.ph2, H, 0, w.pdz2, H, 0, (int)B, 2 * A, H, 1, st))) return rc;
  if ((rc = layer_bwd_weight(w.pdz2, H, 0, w.ph1, H, 0, (int)B, H, H, 1, w.part, w.rs, gp + L.pW2, gp + L.pb2, 0, st))) return rc;
  if ((rc = layer_bwd_input(w.pdz2, H, 0, a->policy + L.pW2, H, 0, w.ph1, H, 0, w.pdz1, H, 0, (int)B, H, H, 1, st))) return rc;
  if ((rc = layer_bwd_weight(w.pdz1, H, 0, a->states, O, 0, (int)B, H, O, 1, w.part, w.rs, gp + L.pW1, gp + L.pb1, 0, st))) return rc;
  RLX_LAUNCH_C(KC_CLIP_ADAM, 0, 0, sac_sumsq_step_kernel, 1, 256, 0, st, gp, L.Pp, L.Pp, L.Pp, 1, w.ss, (long long*)a->steps);
  RLX_LAUNCH_C(KC_CLIP_ADAM, 0, 28.0 * L.Pp, sac_adam_kernel, (unsigned)ceil_div(L.Pp, 256), 256, 0, st, a->policy, gp, a->m_policy, a->v_policy, L.Pp, a->lr,
               (const long long*)a->steps, a->adam_beta1, a->adam_beta2, a->adam_eps);
  // -- temperature
  RLX_LAUNCH_C(KC_CLIP_ADAM, 0, 0, sac_sumsq_step_kernel, 1, 256, 0, st, a->g_log_alpha, 1, 1, 1, 1, w.ss + 3, (long long*)a->steps + 2);
  RLX_LAUNCH_C(KC_CLIP_ADAM, 0, 0, sac_adam_kernel, 1, 256, 0, st, a->log_alpha, a->g_log_alpha, a->m_log_alpha, a->v_log_alpha, 1, a->lr,
               (const long long*)a->steps + 2, a->adam_beta1, a->adam_beta2, a->adam_eps);
  RLX_LAUNCH(sac_finish_metrics_kernel, 1, 32, 0, st, w.ss, w.ss + 1, a->metrics);
  return RLX_OK;
}
