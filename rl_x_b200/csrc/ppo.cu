// PPO MLP pair: forward (rollout / eval / bootstrap values) and the minibatch forward+backward+optimiser step.
//
// Network (ref: policy.py:45-52, critic.py:29-35): two independent 3-layer tanh MLPs on the same input.  They are
// evaluated as ONE pipeline over a fused activation layout [rows, 2H] = [policy half | critic half]:
//   layer 1   one GEMM  [rows, obs] x [2H, obs]^T          (shared A operand, SURVEY §8 a11)
//   layer 2   one batched GEMM (batch = 2 nets) [rows, H] x [H, H]^T on the two halves
//   layer 3   skinny head kernels (ppo_head.cuh) fused with sampling / loss
// Backward mirrors it: head -> (dW3 | dZ2) -> batched dW2 (split over rows) -> batched dH1*tanh' -> dW1 (split over rows),
// no dX for layer 1.  Bias gradients fall out of the dW GEMMs as row sums of the dZ operand.
#include "common.cuh"
#include "gemm_simt.cuh"
#include "gemm_dispatch.cuh"
#include "ppo_head.cuh"
#include "ppo_head_gemm.cuh"
#include "ppo_head_mma.cuh"
#include "ppo_optim.cuh"

namespace rlx {

static bool use_tc(const rlx_ppo_dims& d) { return g_gemm_engine == 1 && tc_supported(d); }
}  // namespace rlx
// comm.cu: all-reduce of [gradient | metrics]; *nblk_out > 0 when the kernel also wrote that many (policy, critic) sum-of-squares partial pairs
int comm_allreduce_ppo(rlx_comm* c, float* out, int64_t n, const rlx_ppo_dims& d, float* norm_partials, long long* step_count, void* stream, int* nblk_out);
namespace rlx {

struct Splits {
  int splits, kchunk;
};
// choose a split-K factor for a [M' x N'] output reduced over `rows`: ~2 CTAs per SM for the SIMT engine, one persistent
// CTA per SM for the wgmma engine (k-chunks are multiples of 32 there: one 128-byte swizzle row of fp32)
static Splits choose_splits(long long rows, int out_m, int out_n, int batch, bool tc) {
  if (tc) {
    // persistent kernel, one CTA per SM: pick the split count whose tile total fills whole waves of SMs.  The tensor core's
    // accumulation error grows with the chain length, so each accumulation chain is also kept <= 1024 rows (128 MMAs); the long part
    // of the reduction happens in the fp32 grad_reduce kernel.
    const long long tiles = ceil_div(out_m, 128) * ceil_div(out_n, 128) * batch;
    const long long smin = std::max<long long>(1, ceil_div(rows, 1024)), smax = std::max<long long>(smin, std::min<long long>(smin + 64, rows / 64));
    const long long sms = sm_count();
    long long best = smin;
    double best_fill = -1.0;
    for (long long s = smin; s <= smax; ++s) {
      const long long t = tiles * s;
      const double fill = (double)t / (double)(ceil_div(t, sms) * sms);
      if (fill > best_fill + 0.02) { best_fill = fill; best = s; }
    }
    long long kchunk = std::max<long long>(32, ceil_div(ceil_div(rows, best), 32) * 32);
    return Splits{(int)ceil_div(rows, kchunk), (int)kchunk};
  }
  const long long tiles = ceil_div(out_m, GBM) * ceil_div(out_n, GBN) * batch;
  const long long target = (long long)sm_count() * 2;
  long long s = std::max<long long>(1, target / std::max<long long>(tiles, 1));
  s = std::min<long long>(s, std::max<long long>(1, rows / 256));  // at least 256 rows per split
  long long kchunk = std::max<long long>(8, ceil_div(ceil_div(rows, s), 8) * 8);
  return Splits{(int)ceil_div(rows, kchunk), (int)kchunk};
}

// bf16-autocast mode: dst = bf16-rounded copy of src (what `.to(torch.bfloat16)` of autocast's Linear does to the input and to the
// weights), except the [keep_lo, keep_hi) range, which is copied as is (logstd: an fp32 parameter no autocast op touches)
__global__ void __launch_bounds__(256) round_bf16_kernel(const float* __restrict__ src, float* __restrict__ dst, long long n, long long keep_lo,
                                                         long long keep_hi) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const float x = src[i];
    dst[i] = (i >= keep_lo && i < keep_hi) ? x : bf16r(x);
  }
}
static int launch_round_bf16(const float* src, float* dst, long long n, long long keep_lo, long long keep_hi, cudaStream_t st) {
  if (n <= 0) return RLX_OK;
  const unsigned grid = (unsigned)std::min<long long>(ceil_div(n, 256), (long long)sm_count() * 8);
  RLX_LAUNCH_C(KC_OTHER, 0, 8.0 * n, round_bf16_kernel, grid, 256, 0, st, src, dst, n, keep_lo, keep_hi);
  return RLX_OK;
}
// bf16-autocast mode: points `params` and `X` (n_x floats) at rounded copies made in pr / xr (what autocast's casts hand to every Linear)
static int round_inputs_bf16(const PpoLayout& L, const float*& params, const float*& X, long long n_x, float* pr, float* xr, cudaStream_t st) {
  int rc = launch_round_bf16(params, pr, L.total(), L.off[LOGSTD], L.off[LOGSTD + 1], st);
  if (rc) return rc;
  rc = launch_round_bf16(X, xr, n_x, 0, 0, st);
  if (rc) return rc;
  params = pr;
  X = xr;
  return RLX_OK;
}

// Observation index sets: the layer-1 operand W1cat [2H, obs] = zeros, with W1p [H, P] scattered into the policy_idx columns of rows
// 0..H-1 and W1c [H, C] into the critic_idx columns of rows H..2H-1.  For distinct indices every product the reference's index-select
// forms is formed once and the rest are x * 0, so the GEMMs, the tf32 split, the bf16 rounding and the dW1 | db1 GEMM run unchanged at
// the full observation width.  One CTA per row: zero it, then scatter (the barrier orders the two stores).
__global__ void __launch_bounds__(256) ppo_embed_w1_kernel(const float* __restrict__ w1p, const float* __restrict__ w1c, const int32_t* __restrict__ pidx,
                                                           const int32_t* __restrict__ cidx, int H, int obs, int in_p, int in_c, float* __restrict__ out) {
  const int row = blockIdx.x;
  float* dst = out + (long long)row * obs;
  for (int c = threadIdx.x; c < obs; c += blockDim.x) dst[c] = 0.f;
  __syncthreads();
  const bool critic = row >= H;
  const int in = critic ? in_c : in_p;
  const int32_t* idx = critic ? cidx : pidx;
  const float* src = critic ? w1c + (long long)(row - H) * in_c : w1p + (long long)row * in_p;
  for (int j = threadIdx.x; j < in; j += blockDim.x) dst[idx ? idx[j] : j] = src[j];
}

// The layer-1 weight operand [2H, obs] of this call: W1p | W1c of `params` in place, or (index sets) the embedded matrix written into
// `emb` from the current parameters - on every call, so that whatever wrote them last is what the GEMMs see
static int layer1_weights(const PpoLayout& L, const float* params, float* emb, const float*& w1, cudaStream_t st) {
  if (!L.embed) {
    w1 = params + L.off[W1P];
    return RLX_OK;
  }
  const double bytes = 4.0 * L.H * (2.0 * L.obs + 2.0 * L.in_p + 2.0 * L.in_c);
  RLX_LAUNCH_C(KC_OTHER, 0, bytes, ppo_embed_w1_kernel, (unsigned)(2 * L.H), 256, 0, st, params + L.off[W1P], params + L.off[W1C], L.pidx, L.cidx,
               L.H, L.obs, L.in_p, L.in_c, emb);
  w1 = emb;
  return RLX_OK;
}
// workspace floats of the embedded matrix (none without index sets)
static size_t embed_floats(const rlx_ppo_dims& d) {
  return make_layout(d).embed ? (size_t)2 * d.hidden * d.obs_dim : 0;
}

struct FwdPlan {
  size_t off_H1, off_H2, off_P, off_X, off_W1, total;
};
static FwdPlan plan_forward(const rlx_ppo_dims& d, long long n) {
  FwdPlan P;
  size_t o = 0;
  const size_t act_bytes = align_up((size_t)n * 2 * d.hidden * sizeof(float), 256);
  P.off_H1 = o; o += act_bytes;
  P.off_H2 = o; o += act_bytes;
  // bf16-autocast mode: rounded copies of the parameters and of the observations (always planned: the mode is a run-time switch)
  P.off_P = o; o += align_up((size_t)make_layout(d).total() * sizeof(float), 256);
  P.off_X = o; o += align_up((size_t)n * d.obs_dim * sizeof(float), 256);
  P.off_W1 = o; o += align_up(embed_floats(d) * sizeof(float), 256);  // observation index sets: embedded layer-1 matrix
  P.total = o;
  return P;
}

constexpr int kHeadWgradRows = 64;

// tf32 hi / lo copies of the weights the forward and dX GEMMs take as B, at the originals' pitches and per-net offsets
enum { WS_W1_HI, WS_W1_LO, WS_W2_HI, WS_W2_LO, WS_W2T_HI, WS_W2T_LO, WS_COUNT };

struct TrainPlan {
  size_t off_H1, off_H2, off_dZ2, off_dZ1, off_dhead, off_headpart, off_part1, off_rs1, off_part2, off_part3, off_norm, off_barrier, off_P, off_X, off_ratio,
      off_W1, total;
  size_t off_wsplit[WS_COUNT];
  int max_s1, max_s2, max_s3;
  int head_blocks, wgrad_chunks, norm_blocks, head_npart;
};
static int head_grid(long long m) { return (int)std::min<long long>(ceil_div(m, 16), (long long)sm_count() * 2); }

static TrainPlan plan_train(const rlx_ppo_dims& d, long long m) {
  TrainPlan P;
  const long long H = d.hidden, O = d.obs_dim, A = d.act_dim;
  P.max_s1 = std::max(choose_splits(m, (int)(2 * H), (int)O, 1, false).splits, choose_splits(m, (int)O + 1, (int)(2 * H), 1, true).splits);
  P.max_s2 = std::max(choose_splits(m, (int)H, (int)H, 2, false).splits, choose_splits(m, (int)H, (int)H, 2, true).splits);
  P.head_blocks = head_grid(m);
  P.head_npart = (int)(2 * A + 5 + 2 * H);
  P.wgrad_chunks = (int)ceil_div(m, kHeadWgradRows);
  // one (policy, critic) partial pair per CTA of whichever kernel leaves the squared norms behind: the 64 CTAs of the sum-of-squares
  // kernel, the <= SM-count grids of the exchange kernels, or the gradient-assembly grid (one CTA per 256 flat elements + one per 8 "tall"
  // elements)
  P.norm_blocks = (int)std::max<long long>(std::max(64, sm_count()), ceil_div(make_layout(d).total(), 256) + ceil_div(2 * H + 2 * A + 1 + (A + 1) * H, 8) + 8);
  size_t o = 0;
  auto take = [&](size_t& off, size_t nfloats) {
    off = o;
    o += align_up(nfloats * sizeof(float), 256);
  };
  take(P.off_H1, (size_t)m * 2 * H);
  take(P.off_H2, (size_t)m * 2 * H);
  take(P.off_dZ2, (size_t)m * 2 * H);
  take(P.off_dZ1, (size_t)m * 2 * H);
  take(P.off_dhead, (size_t)m * (ceil_div(A + 1, 4) * 4));
  take(P.off_headpart, (size_t)P.head_blocks * P.head_npart);
  take(P.off_part1, (size_t)P.max_s1 * 2 * H * O);
  take(P.off_rs1, (size_t)P.max_s1 * 2 * H);
  take(P.off_part2, (size_t)P.max_s2 * 2 * H * H);
  const size_t dh_ld_plan = (size_t)(ceil_div(A + 1, 4) * 4);
  P.max_s3 = choose_splits(m, (int)dh_ld_plan, (int)H, 2, true).splits;
  take(P.off_part3, std::max<size_t>((size_t)P.wgrad_chunks * (A + 1) * H, (size_t)P.max_s3 * 2 * dh_ld_plan * H));
  take(P.off_norm, (size_t)P.norm_blocks * 2);
  take(P.off_barrier, 64);
  take(P.off_P, (size_t)make_layout(d).total());                          // bf16-autocast mode: rounded parameter copy
  take(P.off_X, (size_t)m * (size_t)(ceil_div(O + 1, 4) * 4));             // ... and rounded copy of the minibatch states (pitch <= obs + 4)
  take(P.off_ratio, (size_t)m);                                           // ESPO median: |ratio - 1| per row
  for (int i = 0; i < WS_COUNT; ++i) take(P.off_wsplit[i], i < WS_W2_HI ? (size_t)(2 * H * O) : (size_t)(2 * H * H));
  take(P.off_W1, embed_floats(d));                                        // observation index sets: embedded layer-1 matrix
  P.total = o;
  return P;
}

template <typename T>
static T* ws_ptr(void* ws, size_t off) {
  return reinterpret_cast<T*>(reinterpret_cast<char*>(ws) + off);
}

static size_t head_smem_bytes(const rlx_ppo_dims& d, bool train) {
  size_t s = ((size_t)d.act_dim * d.hidden + d.hidden) * sizeof(float);
  if (train) s += (size_t)8 * (2 * d.act_dim + 5 + 2 * d.hidden) * sizeof(float);
  return s;
}

// The minibatch update's copies (pointers into the workspace); split_weights refreshes them from the parameters.
struct SplitWeights {
  const float* p[WS_COUNT];
};
static int split_weights(const PpoLayout& L, const float* params, const float* w1, void* ws, const TrainPlan& P, SplitWeights& sw, cudaStream_t st) {
  const int H = L.H;
  float* w[WS_COUNT];
  for (int i = 0; i < WS_COUNT; ++i) sw.p[i] = w[i] = ws_ptr<float>(ws, P.off_wsplit[i]);
  const Tf32SplitJob jobs[3] = {{w1, w[WS_W1_HI], w[WS_W1_LO], 1, 2 * H, L.obs, 0},
                                {params + L.off[W2P], w[WS_W2_HI], w[WS_W2_LO], 1, 2 * H, H, 0},
                                {params + L.off[W2P], w[WS_W2T_HI], w[WS_W2T_LO], 2, H, H, 1}};
  return tf32_split(jobs, 3, KC_GEMM_FWD, st);  // a few microseconds, charged to the forward GEMMs
}

// hidden layers: H1 = tanh(X W1cat^T + b1cat), H2 = tanh(H1 (blockdiag W2)^T + b2cat).  w1 = W1cat [2H, obs] (layer1_weights).  ldx = row
// pitch of X.  sw: tf32 hi / lo copies of W1cat and W2 (wgmma engine, fp32 mode), or null.
static int mlp_hidden_forward(const rlx_ppo_dims& d, const PpoLayout& L, const float* params, const float* w1, const float* X, long long ldx,
                              long long rows, float* H1, float* H2, cudaStream_t stream, int bf16 = 0, const SplitWeights* sw = nullptr) {
  const int H = L.H;
  const bool tc = use_tc(d);
  GemmP g{};
  g.A = X; g.B = w1; g.C = H1; g.bias = params + L.off[B1P];
  g.M = (int)rows; g.N = 2 * H; g.K = L.obs;
  g.lda = (int)ldx; g.ldb = L.obs; g.ldc = 2 * H;
  g.splits = 1; g.kchunk = (int)(ceil_div(L.obs, 8) * 8);
  g.bf16 = bf16;
  if (sw) { g.b_hi = sw->p[WS_W1_HI]; g.b_lo = sw->p[WS_W1_LO]; }
  int rc = run_gemm<true, true, EPI_BIAS_TANH>(tc, g, 1, stream, KC_GEMM_FWD, rows, 2 * H);
  if (rc) return rc;
  GemmP g2{};
  g2.A = H1; g2.B = params + L.off[W2P]; g2.C = H2; g2.bias = params + L.off[B2P];
  if (sw) { g2.b_hi = sw->p[WS_W2_HI]; g2.b_lo = sw->p[WS_W2_LO]; }
  g2.M = (int)rows; g2.N = H; g2.K = H;
  g2.lda = 2 * H; g2.ldb = H; g2.ldc = 2 * H;
  g2.sA = H; g2.sB = (long long)H * H; g2.sC = H; g2.sBias = H;
  g2.splits = 1; g2.kchunk = (int)(ceil_div(H, 8) * 8);
  g2.bf16 = bf16;
  return run_gemm<true, true, EPI_BIAS_TANH>(tc, g2, 2, stream, KC_GEMM_FWD, rows, H);
}

#define RLX_DISPATCH_NCH_1(CLS, FLOPS, BYTES, KERNEL, NCH_, BF_, grid, block, smem, stream, arg)                                    \
  do {                                                                                                                              \
    RLX_CHECK_CUDA(cudaFuncSetAttribute(KERNEL<NCH_, BF_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(smem)));              \
    RLX_LAUNCH_C(CLS, FLOPS, BYTES, (KERNEL<NCH_, BF_>), grid, block, smem, stream, arg);                                           \
  } while (0)
#define RLX_DISPATCH_NCH_B(CLS, FLOPS, BYTES, H, KERNEL, BF_, grid, block, smem, stream, arg)                                       \
  do {                                                                                                                              \
    const int _nch = (int)ceil_div((H), 32);                                                                                        \
    if (_nch <= 2) RLX_DISPATCH_NCH_1(CLS, FLOPS, BYTES, KERNEL, 2, BF_, grid, block, smem, stream, arg);                           \
    else if (_nch <= 4) RLX_DISPATCH_NCH_1(CLS, FLOPS, BYTES, KERNEL, 4, BF_, grid, block, smem, stream, arg);                      \
    else if (_nch <= 8) RLX_DISPATCH_NCH_1(CLS, FLOPS, BYTES, KERNEL, 8, BF_, grid, block, smem, stream, arg);                      \
    else if (_nch <= 16) RLX_DISPATCH_NCH_1(CLS, FLOPS, BYTES, KERNEL, 16, BF_, grid, block, smem, stream, arg);                    \
    else RLX_DISPATCH_NCH_1(CLS, FLOPS, BYTES, KERNEL, 32, BF_, grid, block, smem, stream, arg);                                    \
  } while (0)
// bf16-autocast mode selects the kernels compiled with the bf16 roundings (h.bf16 is set by the callers)
#define RLX_DISPATCH_NCH(CLS, FLOPS, BYTES, H, KERNEL, grid, block, smem, stream, arg)                                              \
  do {                                                                                                                              \
    if ((arg).bf16) RLX_DISPATCH_NCH_B(CLS, FLOPS, BYTES, H, KERNEL, true, grid, block, smem, stream, arg);                         \
    else RLX_DISPATCH_NCH_B(CLS, FLOPS, BYTES, H, KERNEL, false, grid, block, smem, stream, arg);                                   \
  } while (0)

static bool head_dims_ok(const rlx_ppo_dims& d) {
  return dims_ok(d) && d.hidden <= 1024 && head_smem_bytes(d, true) <= 200 * 1024;
}

int ppo_head_gemm_path(const HeadGemmArgs& a, cudaStream_t st);  // ppo_head_gemm.cu
static int g_head_engine = 0;                                       // 0 fused SIMT kernel, 1 GEMM formulation, 2 fused mma.sync kernel (rlx_set_head_engine)

static void fill_head_common(HeadP& h, const PpoLayout& L, const float* params, const float* H2, long long rows) {
  h.M = (int)rows; h.H = L.H; h.act = L.act;
  h.H2 = H2;
  h.W3p = params + L.off[W3P]; h.W3c = params + L.off[W3C];
  h.b3p = params + L.off[B3P]; h.b3c = params + L.off[B3C];
  h.logstd = params + L.off[LOGSTD];
}

}  // namespace rlx

using namespace rlx;

// ------------------------------------------------------------------------------------------------ forward API
extern "C" size_t rlx_ppo_forward_workspace_bytes(const rlx_ppo_dims* d, int64_t n) {
  if (d == nullptr || !head_dims_ok(*d) || n < 0) return 0;
  return plan_forward(*d, n).total;
}

extern "C" int rlx_ppo_forward_f32(const rlx_ppo_forward_args* a, void* stream) {
  RLX_CHECK_ARG(a != nullptr, "args is null");
  const char* ip = ppo_index_problem(a->dims);
  RLX_CHECK_ARG(ip == nullptr, ip);
  RLX_CHECK_ARG(head_dims_ok(a->dims), "unsupported dims (act <= 64, hidden <= 1024)");
  RLX_CHECK_ARG(a->n >= 0 && a->n < (1LL << 31), "bad row count");
  if (a->n == 0) return RLX_OK;
  RLX_CHECK_ARG(a->params && a->obs, "params / obs is null");
  RLX_CHECK_ARG(!a->env_action || !a->clip_rescale || (a->act_low && a->act_high), "action bounds required for clip_rescale");
  const FwdPlan P = plan_forward(a->dims, a->n);
  if (a->workspace == nullptr || a->workspace_bytes < P.total) {
    set_error("rlx_ppo_forward_f32: workspace too small (%zu < %zu)", a->workspace_bytes, P.total);
    return RLX_ERR_WORKSPACE;
  }
  const PpoLayout L = make_layout(a->dims);
  float* H1 = ws_ptr<float>(a->workspace, P.off_H1);
  float* H2 = ws_ptr<float>(a->workspace, P.off_H2);
  cudaStream_t st = (cudaStream_t)stream;
  const int bf16 = g_autocast_bf16;
  const float* params = a->params;
  const float* obs = a->obs;
  int rc;
  if (bf16) {
    rc = round_inputs_bf16(L, params, obs, a->n * (long long)L.obs, ws_ptr<float>(a->workspace, P.off_P), ws_ptr<float>(a->workspace, P.off_X), st);
    if (rc) return rc;
  }
  const float* w1 = nullptr;
  rc = layer1_weights(L, params, ws_ptr<float>(a->workspace, P.off_W1), w1, st);
  if (rc) return rc;
  rc = mlp_hidden_forward(a->dims, L, params, w1, obs, a->dims.obs_dim, a->n, H1, H2, st, bf16);
  if (rc) return rc;
  HeadP h{};
  fill_head_common(h, L, params, H2, a->n);
  h.bf16 = bf16;
  h.noise = a->noise; h.seed = a->rng_seed; h.offset = a->rng_offset;
  h.act_low = a->act_low; h.act_high = a->act_high;
  h.clip_rescale = a->clip_rescale; h.deterministic = a->deterministic;
  h.action = a->action; h.env_action = a->env_action; h.logp_out = a->logp; h.value_out = a->value;
  const size_t smem = head_smem_bytes(a->dims, false);
  const int grid = head_grid(a->n);
  RLX_DISPATCH_NCH(KC_HEAD_ROLLOUT, 2.0 * a->n * L.H * (L.act + 1), 4.0 * a->n * (2.0 * L.H + 3.0 * L.act + 2), L.H, ppo_head_rollout_kernel, grid, 256, smem, st, h);
  return RLX_OK;
}

extern "C" int rlx_critic_forward_f32(const rlx_ppo_dims* d, const float* params, const float* obs, int64_t n, float* value,
                                      void* workspace, size_t workspace_bytes, void* stream) {
  RLX_CHECK_ARG(d != nullptr, "dims is null");
  rlx_ppo_forward_args a{};
  a.dims = *d; a.n = n; a.params = params; a.obs = obs; a.deterministic = 1; a.value = value;
  a.workspace = workspace; a.workspace_bytes = workspace_bytes;
  return rlx_ppo_forward_f32(&a, stream);
}

// ---------------------------------------------------------------------------------------- minibatch update API
extern "C" size_t rlx_ppo_minibatch_workspace_bytes(const rlx_ppo_dims* d, int64_t m) {
  if (d == nullptr || !head_dims_ok(*d) || m < 0) return 0;
  return plan_train(*d, std::max<int64_t>(m, 1)).total;
}

static int check_mb_args(const rlx_ppo_minibatch_args* a, bool need_data, TrainPlan& P) {
  RLX_CHECK_ARG(a != nullptr, "args is null");
  const char* ip = ppo_index_problem(a->dims);
  RLX_CHECK_ARG(ip == nullptr, ip);
  RLX_CHECK_ARG(head_dims_ok(a->dims), "unsupported dims (act <= 64, hidden <= 1024)");
  RLX_CHECK_ARG(a->m >= 0 && a->m < (1LL << 31) && a->m_global >= 1, "bad minibatch size");
  RLX_CHECK_ARG(a->params && a->grads, "params / grads is null");
  if (need_data && a->m > 0) {
    RLX_CHECK_ARG(a->states && a->actions && a->log_probs && a->advantages && a->returns && a->adv_stats, "null minibatch tensor");
  }
  P = plan_train(a->dims, std::max<int64_t>(a->m, 1));
  if (a->workspace == nullptr || a->workspace_bytes < P.total) {
    set_error("rlx_ppo_minibatch: workspace too small (%zu < %zu)", a->workspace_bytes, P.total);
    return RLX_ERR_WORKSPACE;
  }
  return RLX_OK;
}

static long long tall_elements(const GradReduceP& r) {
  long long tall = 0;
  for (int gi = 0; gi < kNumGroups; ++gi)
    if (r.g[gi].nsplit > kTallSplit) tall += r.g[gi].len;
  return tall;
}
static double partial_bytes(const GradReduceP& r) {
  double b = 0;
  for (int gi = 0; gi < kNumGroups; ++gi) b += 4.0 * r.g[gi].nsplit * r.g[gi].len;
  return b;
}
static int launch_grad_reduce(const GradReduceP& r, cudaStream_t st) {
  const int flat_blocks = (int)ceil_div(r.total, 256);
  const int tall_blocks = (int)ceil_div(tall_elements(r), 8);  // 8 warps per CTA, one element per warp
  RLX_LAUNCH_C(KC_GRAD_REDUCE, 0, partial_bytes(r) + 4.0 * r.total, ppo_grad_reduce_kernel, (unsigned)(flat_blocks + tall_blocks), 256, 0, st, r, flat_blocks);
  return RLX_OK;
}

// ---- stages of minibatch_fwdbwd, in launch order
// the head kernels with the act <= 31 specialisations (and their dW3 kernels) cover the shape
static bool fast_head_ok(const PpoLayout& L) { return (L.act <= 31) && (L.H % 2 == 0) && (L.H <= 1024); }

// loss head: loss + dZ2 + dhead + block partials (incl. db2 = column sums of dZ2).  Returns the number of partial blocks written, < 0 on error.
static int launch_train_head(const rlx_ppo_minibatch_args* a, const PpoLayout& L, const TrainPlan& P, const float* params, int bf16, cudaStream_t st) {
  const long long m = a->m;
  const int H = L.H, A = L.act;
  void* ws = a->workspace;
  float* H2 = ws_ptr<float>(ws, P.off_H2);
  float* dZ2 = ws_ptr<float>(ws, P.off_dZ2);
  float* dhead = ws_ptr<float>(ws, P.off_dhead);
  float* headpart = ws_ptr<float>(ws, P.off_headpart);
  const float inv_mg = 1.f / (float)a->m_global;
  HeadP h{};
  fill_head_common(h, L, params, H2, m);
  h.bf16 = bf16;
  h.actions = a->actions; h.logp_old = a->log_probs; h.adv = a->advantages; h.ret = a->returns; h.adv_stats = a->adv_stats;
  h.inv_mg = inv_mg; h.clip_range = a->hp.clip_range; h.critic_coef = a->hp.critic_coef;
  h.ratio_delta_metric = a->hp.ratio_delta_metric != 0.f ? 1 : 0;
  const bool want_median = a->hp.ratio_delta_metric == 2.f;  // ESPO delta_calc_operator = median (espo.py:59-60)
  h.ratio_abs = want_median ? ws_ptr<float>(ws, P.off_ratio) : nullptr;
  h.dZ2 = dZ2; h.dhead = dhead; h.block_partials = headpart;
  int head_blocks = P.head_blocks;
  const size_t smem = head_smem_bytes(a->dims, true);
  const int dh_ld = (int)(ceil_div(A + 1, 4) * 4);
  const bool fast_head = fast_head_ok(L);
  const double head_flops = 4.0 * m * H * (A + 1), head_bytes = 4.0 * m * (4.0 * H + 2.0 * A + 5);
  // opt-in GEMM formulation of the head (ppo_head_gemm.cu); dZ1 is free until the dX GEMM and serves as its scratch
  const bool gemm_head = fast_head && g_head_engine == 1 && !bf16 && head_gemm_scratch_floats(m, H, A) <= m * 2LL * H;
  if (gemm_head) {
    HeadGemmArgs ha{m, H, A, dh_ld, H2, a->params + L.off[W3P], a->params + L.off[W3C], a->params + L.off[B3P], a->params + L.off[B3C],
                    a->params + L.off[LOGSTD], a->actions, a->log_probs, a->advantages, a->returns, a->adv_stats, inv_mg, a->hp.clip_range,
                    a->hp.critic_coef, a->hp.ratio_delta_metric != 0.f ? 1 : 0, dZ2, dhead, headpart, ws_ptr<float>(ws, P.off_dZ1)};
    const int rc = ppo_head_gemm_path(ha, st);
    if (rc) return rc;
    return 1;  // the path writes ONE partial block in the fused kernel's layout
  }
  if (!fast_head) {
    RLX_DISPATCH_NCH(KC_HEAD_TRAIN, head_flops, head_bytes, H, ppo_head_train_kernel, head_blocks, 256, smem, st, h);
    return head_blocks;
  }
  HeadTrain2Extra ex{dh_ld};
  const bool vec_head = (H == 128 || H == 256 || H == 512);
  // fused head on the warp-level tensor path (ppo_head_mma.cuh): fp32 mode, <= 4 n-tiles of 8 head columns
  const int nt4 = (int)ceil_div(dh_ld, 8);
  const size_t smem4 = head4_smem_floats(H, A, nt4) * sizeof(float);
  const bool mma_head = vec_head && g_head_engine == 2 && !bf16 && nt4 <= 4 && smem4 <= 220 * 1024;
  if (mma_head) {
    head_blocks = (int)std::min<long long>(ceil_div(m, 16 * kHead4RowTiles), (long long)P.head_blocks);
#define RLX_HEAD4(H_, NT_)                                                                                                          \
  do {                                                                                                                              \
    RLX_CHECK_CUDA(cudaFuncSetAttribute(ppo_head_train4_kernel<H_, NT_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem4)); \
    RLX_LAUNCH_C(KC_HEAD_TRAIN, head_flops, head_bytes, (ppo_head_train4_kernel<H_, NT_>), head_blocks, 256, smem4, st, h, ex);     \
  } while (0)
#define RLX_HEAD4_NT(H_)              \
  do {                                \
    if (nt4 == 1) RLX_HEAD4(H_, 1);   \
    else if (nt4 == 2) RLX_HEAD4(H_, 2); \
    else if (nt4 == 3) RLX_HEAD4(H_, 3); \
    else RLX_HEAD4(H_, 4);            \
  } while (0)
    if (H == 128) RLX_HEAD4_NT(128);
    else if (H == 256) RLX_HEAD4_NT(256);
    else RLX_HEAD4_NT(512);
#undef RLX_HEAD4_NT
#undef RLX_HEAD4
  } else if (vec_head) {
#define RLX_HEAD3_B(H_, AM_, BF_)                                                                                                     \
  do {                                                                                                                                \
    RLX_CHECK_CUDA(cudaFuncSetAttribute(ppo_head_train3_kernel<H_, AM_, BF_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    RLX_LAUNCH_C(KC_HEAD_TRAIN, head_flops, head_bytes, (ppo_head_train3_kernel<H_, AM_, BF_>), head_blocks, 256, smem, st, h, ex);    \
  } while (0)
#define RLX_HEAD3(H_, AM_)                          \
  do {                                              \
    if (bf16) RLX_HEAD3_B(H_, AM_, true);           \
    else RLX_HEAD3_B(H_, AM_, false);               \
  } while (0)
#define RLX_HEAD3_ACT(H_)                      \
  do {                                         \
    if (A <= 8) RLX_HEAD3(H_, 8);              \
    else if (A <= 16) RLX_HEAD3(H_, 16);       \
    else if (A <= 24) RLX_HEAD3(H_, 24);       \
    else RLX_HEAD3(H_, 31);                    \
  } while (0)
    if (H == 128) RLX_HEAD3_ACT(128);
    else if (H == 256) RLX_HEAD3_ACT(256);
    else RLX_HEAD3_ACT(512);
#undef RLX_HEAD3_ACT
#undef RLX_HEAD3
#undef RLX_HEAD3_B
  } else {
    const int nch = (int)ceil_div(H, 32);
#define RLX_HEAD2_B(NCH_, AM_, BF_)                                                                                                   \
  do {                                                                                                                                \
    RLX_CHECK_CUDA(cudaFuncSetAttribute(ppo_head_train2_kernel<NCH_, AM_, BF_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    RLX_LAUNCH_C(KC_HEAD_TRAIN, head_flops, head_bytes, (ppo_head_train2_kernel<NCH_, AM_, BF_>), head_blocks, 256, smem, st, h, ex);  \
  } while (0)
#define RLX_HEAD2(NCH_, AM_)                        \
  do {                                              \
    if (bf16) RLX_HEAD2_B(NCH_, AM_, true);         \
    else RLX_HEAD2_B(NCH_, AM_, false);             \
  } while (0)
#define RLX_HEAD2_ACT(NCH_)                         \
  do {                                              \
    if (A <= 8) RLX_HEAD2(NCH_, 8);                 \
    else if (A <= 16) RLX_HEAD2(NCH_, 16);          \
    else if (A <= 24) RLX_HEAD2(NCH_, 24);          \
    else RLX_HEAD2(NCH_, 31);                       \
  } while (0)
    if (nch <= 2) RLX_HEAD2_ACT(2);
    else if (nch <= 4) RLX_HEAD2_ACT(4);
    else if (nch <= 8) RLX_HEAD2_ACT(8);
    else if (nch <= 16) RLX_HEAD2_ACT(16);
    else RLX_HEAD2_ACT(32);
#undef RLX_HEAD2_ACT
#undef RLX_HEAD2
#undef RLX_HEAD2_B
  }
  return head_blocks;
}

// Where the dW3 partials are: split s of dW3p [act, H] at src + s * stride, of dW3c [H] at src + critic_off + s * stride.
struct W3Partials {
  float* src;
  int nsplit;
  long long stride, critic_off;
};
// the layout of the SIMT kernels: part[chunk][(act+1)*H], rows 0..act-1 = dW3p, row act = dW3c
static W3Partials chunked_w3(const PpoLayout& L, float* part3, int nchunks) {
  return W3Partials{part3, nchunks, (long long)(L.act + 1) * L.H, (long long)L.act * L.H};
}

// dW3 = dhead^T [act+1, m] . H2 [m, 2H]
static int launch_head_wgrad(const PpoLayout& L, const TrainPlan& P, long long m, bool tc, int bf16, void* ws, cudaStream_t st, W3Partials& w3) {
  const int H = L.H, A = L.act;
  float* H2 = ws_ptr<float>(ws, P.off_H2);
  float* dhead = ws_ptr<float>(ws, P.off_dhead);
  float* part3 = ws_ptr<float>(ws, P.off_part3);
  const int wgrad_chunks = (int)ceil_div(m, kHeadWgradRows);
  const double wflops = 2.0 * m * H * (A + 1), wbytes = 4.0 * m * (2.0 * H + A + 1);
  if (!fast_head_ok(L)) {
    // thread per column, chunked over rows
    HeadWgradP w{(int)m, H, A, kHeadWgradRows, H2, dhead, part3};
    dim3 wg((unsigned)wgrad_chunks, (unsigned)ceil_div(2 * H, 256));
    const size_t wsmem = (size_t)kHeadWgradRows * (A + 1) * sizeof(float);
    if (A <= 8) RLX_LAUNCH_C(KC_HEAD_WGRAD, wflops, wbytes, ppo_head_wgrad_kernel<8>, wg, 256, wsmem, st, w);
    else if (A <= 32) RLX_LAUNCH_C(KC_HEAD_WGRAD, wflops, wbytes, ppo_head_wgrad_kernel<32>, wg, 256, wsmem, st, w);
    else {
      RLX_CHECK_CUDA(cudaFuncSetAttribute(ppo_head_wgrad_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wsmem));
      RLX_LAUNCH_C(KC_HEAD_WGRAD, wflops, wbytes, ppo_head_wgrad_kernel<64>, wg, 256, wsmem, st, w);
    }
    count_gemm_path(GP_HEAD_WGRAD_SIMT);
    w3 = chunked_w3(L, part3, wgrad_chunks);
    return RLX_OK;
  }
  const int dh_ld = (int)(ceil_div(A + 1, 4) * 4);
  if (tc) {
    // tensor cores: one MN-major GEMM per net half (batch 2); the act+1 (padded to dh_ld) gradient columns are the M side
    const Splits S3 = choose_splits(m, dh_ld, H, 2, true);
    GemmP g3{};
    g3.A = dhead; g3.B = H2; g3.C = part3;
    g3.M = dh_ld; g3.N = H; g3.K = (int)m;
    g3.lda = dh_ld; g3.ldb = 2 * H; g3.ldc = H;
    g3.sA = 0; g3.sB = H; g3.sC = (long long)dh_ld * H;
    g3.splits = S3.splits; g3.kchunk = S3.kchunk; g3.sSplitC = 2LL * dh_ld * H;
    g3.bf16 = bf16;
    const int rc = tc_gemm(g3, false, false, TC_NONE, 2, KC_HEAD_WGRAD, m, m, st);
    if (rc == RLX_OK) {
      // net 1 (critic half of H2), row `act` of its [dh_ld, H] block
      w3 = W3Partials{part3, S3.splits, 2LL * dh_ld * H, (long long)dh_ld * H + (long long)A * H};
      return RLX_OK;
    }
    if (rc != RLX_ERR_UNSUPPORTED) return rc;
  }
  // SIMT: one thread per (policy, critic) column pair, 64 rows per CTA
  HeadWgrad2P w{(int)m, H, A, dh_ld, kHeadWgradRows, H2, dhead, part3};
  const unsigned wthreads = (unsigned)(ceil_div(H, 32) * 32);
  const size_t wsmem = (size_t)kHeadWgradRows * dh_ld * sizeof(float);
  if (A + 1 <= 4) RLX_LAUNCH_C(KC_HEAD_WGRAD, wflops, wbytes, ppo_head_wgrad3_kernel<4>, wgrad_chunks, wthreads, wsmem, st, w);
  else if (A + 1 <= 8) RLX_LAUNCH_C(KC_HEAD_WGRAD, wflops, wbytes, ppo_head_wgrad3_kernel<8>, wgrad_chunks, wthreads, wsmem, st, w);
  else if (A + 1 <= 12) RLX_LAUNCH_C(KC_HEAD_WGRAD, wflops, wbytes, ppo_head_wgrad3_kernel<12>, wgrad_chunks, wthreads, wsmem, st, w);
  else if (A + 1 <= 16) RLX_LAUNCH_C(KC_HEAD_WGRAD, wflops, wbytes, ppo_head_wgrad3_kernel<16>, wgrad_chunks, wthreads, wsmem, st, w);
  else if (A + 1 <= 20) RLX_LAUNCH_C(KC_HEAD_WGRAD, wflops, wbytes, ppo_head_wgrad3_kernel<20>, wgrad_chunks, wthreads, wsmem, st, w);
  else if (A + 1 <= 24) RLX_LAUNCH_C(KC_HEAD_WGRAD, wflops, wbytes, ppo_head_wgrad3_kernel<24>, wgrad_chunks, wthreads, wsmem, st, w);
  else RLX_LAUNCH_C(KC_HEAD_WGRAD, wflops, wbytes, ppo_head_wgrad3_kernel<32>, wgrad_chunks, wthreads, wsmem, st, w);
  count_gemm_path(GP_HEAD_WGRAD_SIMT);
  w3 = chunked_w3(L, part3, wgrad_chunks);
  return RLX_OK;
}

// hidden layers backward: dW2, dZ1, dW1 | db1 (split over rows; s1 / s2 = split counts of the dW1 | db1 / dW2 partials).  sw: as in
// mlp_hidden_forward (dZ1 takes W2^T)
static int launch_hidden_backward(const PpoLayout& L, const TrainPlan& P, const float* params, const float* states, long long ldx, bool ones_col,
                                  long long m, bool tc, int bf16, const SplitWeights* sw, void* ws, cudaStream_t st, int& s1, int& s2) {
  const int H = L.H, O = L.obs;
  float* H1 = ws_ptr<float>(ws, P.off_H1);
  float* dZ2 = ws_ptr<float>(ws, P.off_dZ2);
  float* dZ1 = ws_ptr<float>(ws, P.off_dZ1);
  float* part1 = ws_ptr<float>(ws, P.off_part1);
  float* rs1 = ws_ptr<float>(ws, P.off_rs1);
  float* part2 = ws_ptr<float>(ws, P.off_part2);
  // ---- dW2 : part2[split][net][o][i] = sum_rows dZ2[r, net*H+o] * H1[r, net*H+i]   (db2 comes from the head kernel)
  const Splits S2 = choose_splits(m, H, H, 2, tc);
  s2 = S2.splits;
  GemmP g{};
  g.A = dZ2; g.B = H1; g.C = part2;
  g.M = H; g.N = H; g.K = (int)m;
  g.lda = 2 * H; g.ldb = 2 * H; g.ldc = H;
  g.sA = H; g.sB = H; g.sC = (long long)H * H;
  g.splits = S2.splits; g.kchunk = S2.kchunk; g.sSplitC = 2LL * H * H;
  g.bf16 = bf16;
  int rc = run_gemm<false, false, EPI_NONE>(tc, g, 2, st, KC_GEMM_DW, m, m);
  if (rc) return rc;
  // ---- dZ1 = (dZ2 @ W2) * (1 - H1^2)   per net
  GemmP gd{};
  gd.A = dZ2; gd.B = params + L.off[W2P]; gd.C = dZ1; gd.aux = H1;
  gd.bf16 = bf16;
  gd.M = (int)m; gd.N = H; gd.K = H;
  gd.lda = 2 * H; gd.ldb = H; gd.ldc = 2 * H; gd.ldaux = 2 * H;
  gd.sA = H; gd.sB = (long long)H * H; gd.sC = H; gd.sAux = H;
  gd.splits = 1; gd.kchunk = (int)(ceil_div(H, 8) * 8);
  if (sw) { gd.b_hi = sw->p[WS_W2T_HI]; gd.b_lo = sw->p[WS_W2T_LO]; }  // W2^T [i][o] is the K-major form of W2 here (square: same pitch)
  rc = run_gemm<true, false, EPI_DTANH>(tc, gd, 2, st, KC_GEMM_DX, m, H);
  if (rc) return rc;
  // ---- dW1cat | db1cat : part1[split][o][i] = sum_rows dZ1[r, o] * X[r, i];  db1[o] = sum_rows dZ1[r, o]
  if (tc && ones_col) {
    // tensor-core path, computed TRANSPOSED: C^T[i, o] = sum_r X_aug[r, i] dZ1[r, o] with M = O+1 (the constant-one column of X
    // makes db1 the last output row) and N = 2H = whole 128-wide tiles; the epilogue stores C^T transposed back into [o][i].
    const Splits S1 = choose_splits(m, O + 1, 2 * H, 1, true);
    GemmP gt{};
    gt.A = states; gt.B = dZ1; gt.C = part1;
    gt.bf16 = bf16;
    gt.M = O + 1; gt.N = 2 * H; gt.K = (int)m;
    gt.lda = (int)ldx; gt.ldb = 2 * H; gt.ldc = O;
    gt.splits = S1.splits; gt.kchunk = S1.kchunk; gt.sSplitC = 2LL * H * O;
    rc = tc_gemm_t(gt, false, false, TC_NONE, 1, KC_GEMM_DW, m, m, O, rs1, 0, 2LL * H, st);
    if (rc == RLX_OK) {
      s1 = S1.splits;
      return RLX_OK;
    }
    if (rc != RLX_ERR_UNSUPPORTED) return rc;
  }
  const Splits S1 = choose_splits(m, 2 * H, O, 1, false);
  s1 = S1.splits;
  GemmP g1{};
  g1.A = dZ1; g1.B = states; g1.C = part1;
  g1.bf16 = bf16;
  g1.M = 2 * H; g1.N = O; g1.K = (int)m;
  g1.lda = 2 * H; g1.ldb = (int)ldx; g1.ldc = O;
  g1.rowsum = rs1;
  g1.splits = S1.splits; g1.kchunk = S1.kchunk; g1.sSplitC = 2LL * H * O; g1.sSplitRowsum = 2LL * H;
  return launch_sgemm<false, false, EPI_NONE>(g1, 1, st, KC_GEMM_DW);
}

// assembly of the flat gradient from the partials the stages left (m == 0: a rank that owns no row of this minibatch contributes zeros)
static GradReduceP make_grad_reduce(const rlx_ppo_minibatch_args* a, const PpoLayout& L, const TrainPlan& P, int head_blocks, const W3Partials& w3,
                                    int s1, int s2, bool fuse_norms) {
  const int H = L.H, O = L.obs, A = L.act;
  void* ws = a->workspace;
  const float* headpart = ws_ptr<float>(ws, P.off_headpart);
  const int npart = P.head_npart;
  const float inv_mg = 1.f / (float)a->m_global;
  GradReduceP r{};
  r.g[0] = GradGroup{L.off[W1P], 2LL * H * O, ws_ptr<float>(ws, P.off_part1), s1, 2LL * H * O};
  if (L.embed) {
    // the dW1 partials are [2H, obs] gradients of the embedded matrix: fold them onto W1p [H, P] | W1c [H, C]
    r.g[0].len = (long long)H * (L.in_p + L.in_c);
    r.g[0].map0 = L.pidx; r.g[0].map1 = L.cidx;
    r.g[0].in0 = L.in_p; r.g[0].in1 = L.in_c; r.g[0].rows = H; r.g[0].ld = O;
  }
  r.g[1] = GradGroup{L.off[B1P], 2LL * H, ws_ptr<float>(ws, P.off_rs1), s1, 2LL * H};
  r.g[2] = GradGroup{L.off[W2P], 2LL * H * H, ws_ptr<float>(ws, P.off_part2), s2, 2LL * H * H};
  r.g[3] = GradGroup{L.off[B2P], 2LL * H, headpart + (2 * A + 5), head_blocks, (long long)npart};
  r.g[4] = GradGroup{L.off[W3P], (long long)A * H, w3.src, w3.nsplit, w3.stride};
  r.g[5] = GradGroup{L.off[B3P], 2LL * A + 1, headpart, head_blocks, (long long)npart};
  r.g[6] = GradGroup{L.off[W3C], (long long)H, w3.src + w3.critic_off, w3.nsplit, w3.stride};
  r.total = L.total();
  r.logstd_off = L.off[LOGSTD];
  r.act = A;
  r.entropy_grad = -a->hp.entropy_coef * (float)a->m * inv_mg;
  r.grads = a->grads;
  r.head_partials = headpart; r.nblk = head_blocks; r.npart = npart; r.inv_mg = inv_mg; r.critic_coef = a->hp.critic_coef;
  r.logstd = a->params + L.off[LOGSTD];
  r.metrics = a->metrics; r.m_local = (float)a->m;
  r.bf16 = g_autocast_bf16;
  if (fuse_norms) {
    r.norm_partials = ws_ptr<float>(ws, P.off_norm);
    r.done = ws_ptr<unsigned int>(ws, P.off_barrier);
    r.norm_out = ws_ptr<float>(ws, P.off_barrier) + 4;
    r.step_count = (long long*)a->step_count;
    r.net = make_net_map(L);
  }
  return r;
}

// `fuse_norms`: the assembly kernel also leaves the two squared clip norms in the workspace (off_barrier + 16 bytes) and bumps Adam's
// step counter, so that clip + Adam can follow without the separate sum-of-squares launch.
static int minibatch_fwdbwd(const rlx_ppo_minibatch_args* a, void* stream, bool fuse_norms = false) {
  TrainPlan P;
  int rc = check_mb_args(a, true, P);
  if (rc) return rc;
  const PpoLayout L = make_layout(a->dims);
  const long long m = a->m;
  const long long ldx = a->states_ld > 0 ? a->states_ld : L.obs;
  RLX_CHECK_ARG(ldx >= L.obs, "states_ld smaller than obs_dim");
  RLX_CHECK_ARG(!a->states_ones_col || ldx > L.obs, "states_ones_col needs states_ld > obs_dim");
  const bool tc = use_tc(a->dims);
  const int bf16 = g_autocast_bf16;
  cudaStream_t st = (cudaStream_t)stream;
  void* ws = a->workspace;
  int head_blocks = 0, s1 = 0, s2 = 0;
  W3Partials w3 = chunked_w3(L, ws_ptr<float>(ws, P.off_part3), 0);
  if (m > 0) {
    const float* params = a->params;
    const float* states = a->states;
    if (bf16) {
      RLX_CHECK_ARG(ldx <= (long long)(ceil_div(L.obs + 1, 4) * 4), "bf16 mode: states_ld larger than the planned rounded copy");
      rc = round_inputs_bf16(L, params, states, m * ldx, ws_ptr<float>(ws, P.off_P), ws_ptr<float>(ws, P.off_X), st);
      if (rc) return rc;
    }
    // wgmma engine, fp32: split the weights once here rather than in every tile of the forward and dX GEMMs.  Made from the current
    // parameters on every call, so whatever wrote them last (Adam, init, a checkpoint load, a broadcast) is what the GEMMs see.
    const float* w1 = nullptr;
    rc = layer1_weights(L, params, ws_ptr<float>(ws, P.off_W1), w1, st);
    if (rc) return rc;
    SplitWeights sw{};
    const bool presplit = tc && !bf16;
    if (presplit) {
      rc = split_weights(L, params, w1, ws, P, sw, st);
      if (rc) return rc;
    }
    rc = mlp_hidden_forward(a->dims, L, params, w1, states, ldx, m, ws_ptr<float>(ws, P.off_H1), ws_ptr<float>(ws, P.off_H2), st, bf16,
                            presplit ? &sw : nullptr);
    if (rc) return rc;
    head_blocks = launch_train_head(a, L, P, params, bf16, st);
    if (head_blocks < 0) return head_blocks;
    rc = launch_head_wgrad(L, P, m, tc, bf16, ws, st, w3);
    if (rc) return rc;
    rc = launch_hidden_backward(L, P, params, states, ldx, a->states_ones_col, m, tc, bf16, presplit ? &sw : nullptr, ws, st, s1, s2);
    if (rc) return rc;
  }
  rc = launch_grad_reduce(make_grad_reduce(a, L, P, head_blocks, w3, s1, s2, fuse_norms), st);
  if (rc) return rc;
  if (a->hp.ratio_delta_metric == 2.f && m > 0 && a->metrics != nullptr) {
    // metrics[4] <- torch.median(|ratio - 1|) of this minibatch, overwriting the mean the assembly kernel has just put there
    RLX_LAUNCH_C(KC_OTHER, 0, 16.0 * m, median_lower_kernel, 1, 1024, 0, st, ws_ptr<float>(ws, P.off_ratio), (long long)m, a->metrics + 4);
  }
  return RLX_OK;
}

extern "C" int rlx_ppo_minibatch_fwdbwd_f32(const rlx_ppo_minibatch_args* a, void* stream) { return minibatch_fwdbwd(a, stream); }

static AdamP make_adam_params(const rlx_ppo_minibatch_args* a, const PpoLayout& L, float* norm_partials, int nblk_norm) {
  AdamP p{};
  p.total = L.total();
  p.net = make_net_map(L);
  p.params = a->params; p.grads = a->grads; p.m = a->exp_avg; p.v = a->exp_avg_sq;
  p.lr = a->lr; p.step_count = (long long*)a->step_count;
  p.max_norm = a->hp.max_grad_norm; p.beta1 = a->hp.adam_beta1; p.beta2 = a->hp.adam_beta2; p.eps = a->hp.adam_eps;
  p.norm_partials = norm_partials;
  p.nblk_norm = nblk_norm;
  p.metrics = a->metrics;
  return p;
}

// clip + Adam, the two squared norms summed from `nblk` (policy, critic) partial pairs at `norm_partials`
static int launch_clip_adam(const rlx_ppo_minibatch_args* a, const PpoLayout& L, float* norm_partials, int nblk, cudaStream_t st) {
  const AdamP p = make_adam_params(a, L, norm_partials, nblk);
  RLX_LAUNCH_C(KC_CLIP_ADAM, 0, 28.0 * L.total(), ppo_clip_adam_kernel, (unsigned)ceil_div(L.total(), 256), 256, 0, st, p);
  return RLX_OK;
}

extern "C" int rlx_gradnorm_clip_adam_f32(const rlx_ppo_minibatch_args* a, void* stream) {
  TrainPlan P;
  int rc = check_mb_args(a, false, P);
  if (rc) return rc;
  RLX_CHECK_ARG(a->exp_avg && a->exp_avg_sq && a->lr && a->step_count, "optimizer state is null");
  const PpoLayout L = make_layout(a->dims);
  cudaStream_t st = (cudaStream_t)stream;
  const int nblk = 64;
  float* partials = ws_ptr<float>(a->workspace, P.off_norm);
  const AdamP p = make_adam_params(a, L, partials, nblk);
  RLX_LAUNCH_C(KC_CLIP_ADAM, 0, 4.0 * L.total(), ppo_grad_sumsq_kernel, (unsigned)nblk, 256, 0, st, p);
  return launch_clip_adam(a, L, partials, nblk, st);
}

// minibatch k of an epoch: m gathered rows from row r0 on, and row k of the advantage statistics
static rlx_ppo_minibatch_args minibatch_slice(const rlx_ppo_minibatch_args* first, int64_t k, int64_t r0, int64_t m) {
  const int64_t ld = first->states_ld > 0 ? first->states_ld : first->dims.obs_dim;  // row pitch of the gathered states
  rlx_ppo_minibatch_args a = *first;
  a.m = m;
  a.states = first->states + r0 * ld;
  a.actions = first->actions + r0 * first->dims.act_dim;
  a.log_probs = first->log_probs + r0;
  a.advantages = first->advantages + r0;
  a.returns = first->returns + r0;
  a.adv_stats = first->adv_stats + 2 * k;
  return a;
}

extern "C" int rlx_ppo_update_epoch_f32(const rlx_ppo_minibatch_args* first, int64_t count, int64_t mb, void* stream) {
  RLX_CHECK_ARG(first != nullptr && count >= 0 && mb > 0, "bad arguments");
  const int64_t nmb = ceil_div(count, mb), full = std::min<int64_t>(mb, count);
  cudaStream_t st = (cudaStream_t)stream;
  // clip norms fused into the gradient-assembly kernel (needs the optimiser state and the ticket word in the workspace zeroed once)
  bool norms_in_reduce = dims_ok(first->dims) && first->exp_avg && first->exp_avg_sq && first->lr && first->step_count && first->workspace;
  TrainPlan P{};
  if (norms_in_reduce) {
    P = plan_train(first->dims, std::max<int64_t>(full, 1));
    if (first->workspace_bytes < P.total) norms_in_reduce = false;
    else RLX_CHECK_CUDA(cudaMemsetAsync(ws_ptr<unsigned int>(first->workspace, P.off_barrier), 0, 64, st));
  }
  for (int64_t k = 0; k < nmb; ++k) {
    rlx_ppo_minibatch_args a = minibatch_slice(first, k, k * mb, std::min<int64_t>(mb, count - k * mb));
    a.m_global = a.m;
    a.metrics = first->metrics ? first->metrics + RLX_PPO_NMETRIC * k : nullptr;
    int rc;
    if (norms_in_reduce && a.m == full) {
      // the assembly kernel leaves the clip norms behind; clip + Adam read them (no separate sum-of-squares launch)
      rc = minibatch_fwdbwd(&a, stream, true);
      if (rc) return rc;
      rc = launch_clip_adam(&a, make_layout(a.dims), ws_ptr<float>(a.workspace, P.off_barrier) + 4, 1, st);
    } else {
      // no optimiser state, or the short last minibatch (its workspace plan puts the ticket word elsewhere, not zeroed above):
      // separate sum-of-squares launch
      rc = minibatch_fwdbwd(&a, stream);
      if (rc) return rc;
      rc = rlx_gradnorm_clip_adam_f32(&a, stream);
    }
    if (rc) return rc;
  }
  return RLX_OK;
}

extern "C" int rlx_ppo_update_epoch_sharded_f32(const rlx_ppo_minibatch_args* first, int64_t num_mb, const int64_t* counts,
                                                const int64_t* global_counts, rlx_comm* comm, void* stream) {
  RLX_CHECK_ARG(first != nullptr && num_mb >= 0 && counts && global_counts && comm, "bad arguments");
  RLX_CHECK_ARG(first->metrics != nullptr, "metrics rows are required");
  const PpoLayout L = make_layout(first->dims);
  const int64_t P = L.total();
  cudaStream_t st = (cudaStream_t)stream;
  int64_t r0 = 0;
  for (int64_t k = 0; k < num_mb; ++k) {
    RLX_CHECK_ARG(counts[k] >= 0 && global_counts[k] >= 1, "bad minibatch sizes");
    rlx_ppo_minibatch_args a = minibatch_slice(first, k, r0, counts[k]);
    a.m_global = global_counts[k];
    float* send = rlx_comm_send_buffer(comm);  // partial gradient [P] followed by the partial metric sums
    a.grads = send;
    a.metrics = send + P;
    int rc = minibatch_fwdbwd(&a, stream);
    if (rc) return rc;
    // the two-shot exchange kernel leaves the per-net squared norms of the reduced gradient behind (and bumps Adam's step counter):
    // clip + Adam follow directly, without a separate pass over the gradient
    float* norm_partials = ws_ptr<float>(a.workspace, plan_train(a.dims, std::max<int64_t>(a.m, 1)).off_norm);
    int nblk = 0;
    rc = comm_allreduce_ppo(comm, first->grads, P + RLX_PPO_NMETRIC, a.dims, norm_partials, (long long*)a.step_count, stream, &nblk);
    if (rc) return rc;
    a.grads = first->grads;
    a.metrics = first->grads + P;
    if (nblk > 0) {
      RLX_CHECK_ARG(a.exp_avg && a.exp_avg_sq && a.lr && a.step_count, "optimizer state is null");
      rc = launch_clip_adam(&a, L, norm_partials, nblk, st);
    } else {
      rc = rlx_gradnorm_clip_adam_f32(&a, stream);  // writes the two pre-clip norms next to the summed metrics
    }
    if (rc) return rc;
    RLX_CHECK_CUDA(cudaMemcpyAsync(first->metrics + RLX_PPO_NMETRIC * k, first->grads + P, RLX_PPO_NMETRIC * sizeof(float),
                                   cudaMemcpyDeviceToDevice, st));
    r0 += counts[k];
  }
  return RLX_OK;
}

// Test hook: one plain GEMM through either engine (single batch, no split): layout 0 = A k-major, B k-major (C = A B^T);
// 1 = A k-major, B n-major (C = A B); 2 = A m-major, B n-major (C = A^T B, A is [K, M]).  Epilogue 0 none, 1 bias+tanh, 3 bias+relu,
// 5 bias (layout 0), 2 tanh', 4 relu' (layout 1, aux [M, ldaux]); 6 (layout 2, wgmma engine only) the transposed store with an extra row:
// rows 0 .. M-2 of the product go transposed into C [N, ldc], row M-1 into row N of C.  Pre-split B (wgmma engine only): layout 3 = layout 0
// with epilogue 1, B [N, ldb] split by tf32_split into a scratch copy first; 4 = layout 1 with epilogue 2, B [K, ldb] split and transposed
// into a [ldb, K] copy first (K a multiple of 4) - the forward and dX GEMMs of the PPO update.
extern "C" int rlx_debug_gemm_f32(int engine, int layout, int epilogue, int64_t M, int64_t N, int64_t K, const float* A, int64_t lda,
                                  const float* B, int64_t ldb, float* C, int64_t ldc, const float* bias, const float* aux, int64_t ldaux,
                                  void* stream) {
  RLX_CHECK_ARG(A && B && C && M > 0 && N > 0 && K > 0, "bad arguments");
  RLX_CHECK_ARG(engine == 0 || engine == 1, "unknown engine (0 = SIMT, 1 = wgmma tensor cores)");
  const bool bias_epi = epilogue == 1 || epilogue == 3 || epilogue == 5, aux_epi = epilogue == 2 || epilogue == 4;
  const bool presplit = layout == 3 || layout == 4;
  RLX_CHECK_ARG((epilogue == 0 && !presplit) || (bias_epi && layout == 0 && bias) || (aux_epi && layout == 1 && aux) ||
                    (epilogue == 6 && layout == 2 && engine == 1 && M >= 2) ||
                    (engine == 1 && layout == 3 && epilogue == 1 && bias) || (engine == 1 && layout == 4 && epilogue == 2 && aux && K % 4 == 0),
                "unsupported epilogue/layout");
  GemmP g{};
  g.A = A; g.B = B; g.C = C; g.bias = bias; g.aux = aux;
  g.M = (int)M; g.N = (int)N; g.K = (int)K;
  g.lda = (int)lda; g.ldb = (int)ldb; g.ldc = (int)ldc; g.ldaux = (int)ldaux;
  g.splits = 1; g.kchunk = (int)(ceil_div(K, 8) * 8);
  cudaStream_t st = (cudaStream_t)stream;
  if (presplit) {
    const int rows = (int)(layout == 3 ? N : K);
    float* hi = nullptr;
    RLX_CHECK_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&hi), 2 * sizeof(float) * rows * ldb, st));
    const Tf32SplitJob job{B, hi, hi + rows * ldb, 1, rows, (int)ldb, layout == 4};
    int rc = tf32_split(&job, 1, KC_OTHER, st);
    if (rc == RLX_OK) {
      g.b_hi = job.hi; g.b_lo = job.lo;
      if (layout == 4) g.ldb = (int)K;  // pitch of the transposed copy
      rc = tc_gemm(g, true, layout == 3, epilogue, 1, KC_OTHER, M, layout == 3 ? N : K, st);
    }
    RLX_CHECK_CUDA(cudaFreeAsync(hi, st));
    return rc;
  }
  const bool a_k = layout != 2, b_k = layout == 0;
  const long long a_rows = a_k ? M : K, b_rows = b_k ? N : K;
  if (engine == 1) {
    const int rc = epilogue == 6 ? tc_gemm_t(g, a_k, b_k, TC_NONE, 1, KC_OTHER, a_rows, b_rows, (int)M - 1, C + N * ldc, 0, 0, st)
                                 : tc_gemm(g, a_k, b_k, epilogue, 1, KC_OTHER, a_rows, b_rows, st);
    if (rc == RLX_ERR_UNSUPPORTED) set_error("rlx_debug_gemm_f32: shape/alignment not supported by the wgmma engine");
    return rc;
  }
  if (layout == 0 && epilogue == 1) return launch_sgemm<true, true, EPI_BIAS_TANH>(g, 1, st);
  if (layout == 0 && epilogue == 3) return launch_sgemm<true, true, EPI_BIAS_RELU>(g, 1, st);
  if (layout == 0 && epilogue == 5) return launch_sgemm<true, true, EPI_BIAS>(g, 1, st);
  if (layout == 0) return launch_sgemm<true, true, EPI_NONE>(g, 1, st);
  if (layout == 1 && epilogue == 2) return launch_sgemm<true, false, EPI_DTANH>(g, 1, st);
  if (layout == 1 && epilogue == 4) return launch_sgemm<true, false, EPI_DRELU>(g, 1, st);
  if (layout == 1) return launch_sgemm<true, false, EPI_NONE>(g, 1, st);
  return launch_sgemm<false, false, EPI_NONE>(g, 1, st);
}

// Test hook: the tf32 hi / lo split the minibatch update makes of its weights (tf32_split), of src [batch][rows][cols]
extern "C" int rlx_debug_tf32_split_f32(const float* src, int64_t batch, int64_t rows, int64_t cols, int trans, float* hi, float* lo, void* stream) {
  RLX_CHECK_ARG(src && hi && lo && batch > 0 && rows > 0 && cols > 0 && batch * rows * cols < (1LL << 31), "bad arguments");
  const Tf32SplitJob job{src, hi, lo, (int)batch, (int)rows, (int)cols, trans ? 1 : 0};
  return tf32_split(&job, 1, KC_OTHER, (cudaStream_t)stream);
}

extern "C" int rlx_set_head_engine(int engine) {
  if (engine >= 0 && engine <= 2) g_head_engine = engine;
  else set_error("rlx_set_head_engine: unknown engine %d", engine);
  return g_head_engine;
}

extern "C" int rlx_set_gemm_engine(int engine) {
  if (engine != 0 && engine != 1) {
    set_error("rlx_set_gemm_engine: unknown engine %d", engine);
    return g_gemm_engine;
  }
  g_gemm_engine = engine;
  return g_gemm_engine;
}
