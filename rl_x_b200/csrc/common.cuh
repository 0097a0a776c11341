// Shared helpers for the rlx_b200 C-ABI library (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <algorithm>
#include <atomic>

#include "../../include/rlx_b200.h"

namespace rlx {

void set_error(const char* fmt, ...);
extern std::atomic<uint64_t> g_launch_count;
extern int g_gemm_engine;
extern int g_aux_gemm_engine;
extern std::atomic<uint64_t> g_aux_tc_gemms;
// bf16-autocast mode of the PPO path (rlx_set_autocast_bf16; the reference's `bf16_mixed_precision_training`, ppo.py:98-107,123,155,208,253):
// every value torch's autocast would hold in a bf16 tensor is rounded to bf16 (round-to-nearest-even) where torch rounds it, and kept in
// fp32 storage.  bf16 values are exact TF32 operands, so ONE kind::tf32 MMA per product gives exactly the bf16 x bf16 -> fp32 products of a
// bf16 tensor-core GEMM: the 3-way split (and the splitter warps' work) is switched off in this mode.
extern int g_autocast_bf16;

inline void count_launch(uint64_t n = 1) { g_launch_count.fetch_add(n, std::memory_order_relaxed); }

// Launches of each GEMM path (rlx_gemm_path_count): slot tc_path_slot(...) per tc_gemm_kernel instance, then tf32_split, the SIMT GEMM and the
// SIMT head weight-gradient kernels.  Counted on the host right after a successful launch.
enum { GP_TF32_SPLIT = 256, GP_SGEMM, GP_HEAD_WGRAD_SIMT, GP_COUNT };
static_assert(GP_COUNT == RLX_GEMM_PATH_SLOTS, "GEMM path slots out of sync with rlx_b200.h");
extern std::atomic<uint64_t> g_gemm_path[GP_COUNT];
inline void count_gemm_path(int slot) { g_gemm_path[slot].fetch_add(1, std::memory_order_relaxed); }
constexpr int tc_path_slot(bool a_kmaj, bool b_kmaj, int epi, bool bf16, bool trans, bool split_b) {
  return (a_kmaj ? 1 : 0) | (b_kmaj ? 2 : 0) | (epi << 2) | (bf16 ? 32 : 0) | (trans ? 64 : 0) | (split_b ? 128 : 0);
}

#define RLX_CHECK_ARG(cond, msg)                                  \
  do {                                                            \
    if (!(cond)) {                                                \
      rlx::set_error("%s: invalid argument: %s", __func__, msg);  \
      return RLX_ERR_INVALID_ARG;                                 \
    }                                                             \
  } while (0)

#define RLX_CHECK_CUDA(expr)                                                                      \
  do {                                                                                            \
    cudaError_t _e = (expr);                                                                      \
    if (_e != cudaSuccess) {                                                                      \
      rlx::set_error("%s: CUDA error %s at %s:%d", __func__, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return RLX_ERR_CUDA;                                                                        \
    }                                                                                             \
  } while (0)

// Kernel classes for the optional event-timing facility (rlx_timing_begin / rlx_timing_end).
enum KClass { KC_GEMM_FWD = 0, KC_GEMM_DX, KC_GEMM_DW, KC_HEAD_ROLLOUT, KC_HEAD_TRAIN, KC_HEAD_WGRAD, KC_GRAD_REDUCE, KC_CLIP_ADAM,
              KC_GATHER, KC_ADV_STATS, KC_GAE, KC_STORE, KC_ALLREDUCE, KC_OTHER, KC_COUNT };
static_assert(KC_COUNT == RLX_NKCLASS, "kernel class count out of sync with rlx_b200.h");
extern bool g_timing;
void timing_before(int cls, double flops, double bytes, cudaStream_t stream);
void timing_after(cudaStream_t stream);

// Every kernel launch in the library goes through this so that rlx_launch_count() is an honest count.
// cls/flops/bytes: kernel class and ALGORITHMIC work of this launch (only consumed when timing is enabled).
#define RLX_LAUNCH_C(cls, flops, bytes, kernel, grid, block, smem, stream, ...)              \
  do {                                                                                       \
    if (rlx::g_timing) rlx::timing_before((cls), (double)(flops), (double)(bytes), (cudaStream_t)(stream)); \
    kernel<<<(grid), (block), (smem), (cudaStream_t)(stream)>>>(__VA_ARGS__);                \
    if (rlx::g_timing) rlx::timing_after((cudaStream_t)(stream));                            \
    rlx::count_launch();                                                                     \
    RLX_CHECK_CUDA(cudaPeekAtLastError());                                                   \
  } while (0)
#define RLX_LAUNCH(kernel, grid, block, smem, stream, ...) \
  RLX_LAUNCH_C(rlx::KC_OTHER, 0, 0, kernel, grid, block, smem, stream, __VA_ARGS__)

inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }
inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

int sm_count();

// round-to-nearest-even to bfloat16, returned as fp32 (what `x.to(torch.bfloat16).float()` gives; NaN stays NaN)
__device__ __forceinline__ float bf16r(float x) {
  const unsigned u = __float_as_uint(x);
  if ((u & 0x7F800000u) == 0x7F800000u) return x;  // inf / nan
  return __uint_as_float((u + 0x7FFFu + ((u >> 16) & 1u)) & 0xFFFF0000u);
}
__device__ __forceinline__ float bf16r_if(float x, int on) { return on ? bf16r(x) : x; }

// Branch-free tanh for the tensor-engine epilogues: |x| < 0.25: odd Taylor polynomial through x^9 (truncation < 2e-9); otherwise
// 1 - 2 / (exp(2|x|) + 1) on the MUFU units (ex2.approx 2 ulp, rcp.approx 1 ulp), sign restored.  Max relative error 5.5e-7 with
// both approximations at their worst, rms 9e-8 (model in fp32 arithmetic over 3.2 M points incl. the branch point) against tanhf's 1-2 ulp:
// the same accuracy class as the 3xTF32 products feeding it (1e-6), far inside the 1e-5 parity bar.  ~14 instructions and no divergence
// where tanhf executes both of its paths for a warp with mixed magnitudes (~35): the forward GEMMs' epilogue is issue-bound on it.
__device__ __forceinline__ float tanh_fast(float x) {
  const float x2 = x * x;
  float p = fmaf(x2, 62.f / 2835.f, -17.f / 315.f);
  p = fmaf(p, x2, 2.f / 15.f);
  p = fmaf(p, x2, -1.f / 3.f);
  p = fmaf(p, x2, 1.f);
  const float small = x * p;
  const float ax = fminf(fabsf(x), 15.f);
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(ax * 2.885390081777927f));  // exp(2|x|) = 2^(2|x| log2 e)
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(e + 1.f));
  const float big = copysignf(fmaf(-2.f, r, 1.f), x);
  return (fabsf(x) < 0.25f) ? small : big;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Block-wide sum for blockDim.x <= 1024 (multiple of 32); result valid in all threads. `sh` holds >= 33 floats.
__device__ __forceinline__ float block_sum(float v, float* sh) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) sh[w] = v;
  __syncthreads();
  float r = (threadIdx.x < nw) ? sh[threadIdx.x] : 0.f;
  if (w == 0) {
    r = warp_sum(r);
    if (lane == 0) sh[32] = r;
  }
  __syncthreads();
  return sh[32];
}

// ------------------------------------------------------------------ PPO flat parameter layout (see rlx_b200.h)
struct PpoLayout {
  int64_t off[RLX_PPO_NSEG + 1];
  int obs, act, H;
  int in_p, in_c;                 // layer-1 inputs of the policy / critic (= obs without index sets)
  const int32_t* pidx;            // observation index sets (device), null = identity
  const int32_t* cidx;
  bool embed;                     // an index set is present: layer 1 runs on the embedded [2H, obs] matrix
  __host__ __device__ int64_t total() const { return off[RLX_PPO_NSEG]; }
};
enum Seg { W1P = 0, W1C, B1P, B1C, W2P, W2C, B2P, B2C, W3P, W3C, B3P, B3C, LOGSTD };

inline int ppo_in_dim(int32_t in_dim, int32_t obs) { return in_dim > 0 ? in_dim : obs; }

inline PpoLayout make_layout(const rlx_ppo_dims& d) {
  PpoLayout L;
  const int64_t H = d.hidden, A = d.act_dim;
  L.in_p = ppo_in_dim(d.policy_in_dim, d.obs_dim);
  L.in_c = ppo_in_dim(d.critic_in_dim, d.obs_dim);
  L.pidx = d.policy_idx;
  L.cidx = d.critic_idx;
  L.embed = d.policy_idx != nullptr || d.critic_idx != nullptr;
  const int64_t sz[RLX_PPO_NSEG] = {H * L.in_p, H * L.in_c, H, H, H * H, H * H, H, H, A * H, H, A, 1, A};
  int64_t o = 0;
  for (int i = 0; i < RLX_PPO_NSEG; ++i) {
    L.off[i] = o;
    o += sz[i];
  }
  L.off[RLX_PPO_NSEG] = o;
  L.obs = d.obs_dim;
  L.act = d.act_dim;
  L.H = d.hidden;
  return L;
}
inline bool seg_is_critic(int s) { return s == W1C || s == B1C || s == W2C || s == B2C || s == W3C || s == B3C; }

// Which net owns flat element i, in a form kernels can take by value (embedded in the parameter blocks of the norm kernels).
struct PpoNetMap {
  long long seg_off[RLX_PPO_NSEG + 1];
  unsigned critic_mask;  // bit s set => segment s belongs to the critic
};
inline PpoNetMap make_net_map(const PpoLayout& L) {
  PpoNetMap map{};
  for (int i = 0; i <= RLX_PPO_NSEG; ++i) map.seg_off[i] = L.off[i];
  for (int i = 0; i < RLX_PPO_NSEG; ++i)
    if (seg_is_critic(i)) map.critic_mask |= (1u << i);
  return map;
}
// 0 = policy, 1 = critic
__device__ __forceinline__ int net_of(const PpoNetMap& map, long long i) {
  int seg = 0;
#pragma unroll
  for (int s = 1; s < RLX_PPO_NSEG; ++s) seg += (i >= map.seg_off[s]) ? 1 : 0;
  return (map.critic_mask >> seg) & 1u;
}

// What is wrong with the observation index fields of d (include/rlx_b200.h), or null.  The index VALUES live on the device and are
// the caller's to validate.
inline const char* ppo_index_problem(const rlx_ppo_dims& d) {
  const int32_t in[2] = {d.policy_in_dim, d.critic_in_dim};
  const int32_t* idx[2] = {d.policy_idx, d.critic_idx};
  for (int k = 0; k < 2; ++k) {
    if (idx[k] != nullptr && (in[k] < 1 || in[k] > d.obs_dim))
      return k == 0 ? "policy_idx given: policy_in_dim must be in [1, obs_dim]" : "critic_idx given: critic_in_dim must be in [1, obs_dim]";
    if (idx[k] == nullptr && in[k] != 0 && in[k] != d.obs_dim)
      return k == 0 ? "policy_idx is NULL (identity): policy_in_dim must be 0 or obs_dim"
                    : "critic_idx is NULL (identity): critic_in_dim must be 0 or obs_dim";
  }
  return nullptr;
}

inline bool dims_ok(const rlx_ppo_dims& d) {
  return d.obs_dim > 0 && d.act_dim > 0 && d.hidden > 0 && d.act_dim <= 64 && d.hidden <= 4096 && d.obs_dim <= 65536 &&
         ppo_index_problem(d) == nullptr;
}

}  // namespace rlx
