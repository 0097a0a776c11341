// Library-level state: error strings, launch counter, engine selection, device properties.
#include "common.cuh"
#include <vector>

namespace rlx {

static thread_local char g_err[512] = "";
std::atomic<uint64_t> g_launch_count{0};
int g_gemm_engine = 0;
int g_aux_gemm_engine = 0;  // FastSAC / PPO+LSTM dense layers (rlx_set_aux_gemm_engine)
std::atomic<uint64_t> g_aux_tc_gemms{0};
std::atomic<uint64_t> g_gemm_path[GP_COUNT];
int g_autocast_bf16 = 0;

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

// ------------------------------------------------------------------------------------------- event timing
bool g_timing = false;
namespace {
struct TimingRec { int cls; double flops, bytes; cudaEvent_t e0, e1; };
std::vector<TimingRec> g_recs;
std::vector<cudaEvent_t> g_event_pool;
size_t g_event_next = 0;
cudaEvent_t take_event() {
  if (g_event_next == g_event_pool.size()) {
    cudaEvent_t e;
    cudaEventCreate(&e);
    g_event_pool.push_back(e);
  }
  return g_event_pool[g_event_next++];
}
}  // namespace
void timing_before(int cls, double flops, double bytes, cudaStream_t stream) {
  TimingRec r{cls, flops, bytes, take_event(), take_event()};
  cudaEventRecord(r.e0, stream);
  g_recs.push_back(r);
}
void timing_after(cudaStream_t stream) { cudaEventRecord(g_recs.back().e1, stream); }

int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      n = 132;  // H100 SXM
  }
  return n;
}

}  // namespace rlx

extern "C" int rlx_version(void) { return 1; }
extern "C" const char* rlx_last_error_string(void) { return rlx::g_err; }
extern "C" uint64_t rlx_launch_count(void) { return rlx::g_launch_count.load(); }
extern "C" void rlx_reset_launch_count(void) { rlx::g_launch_count.store(0); }
extern "C" void rlx_add_launch_count(uint64_t n) { rlx::g_launch_count.fetch_add(n); }
extern "C" int rlx_get_gemm_engine(void) { return rlx::g_gemm_engine; }
extern "C" uint64_t rlx_aux_tc_gemm_count(void) { return rlx::g_aux_tc_gemms.load(); }
extern "C" uint64_t rlx_gemm_path_count(int slot) { return (slot >= 0 && slot < rlx::GP_COUNT) ? rlx::g_gemm_path[slot].load() : 0; }
extern "C" void rlx_reset_gemm_path_counts(void) {
  for (auto& c : rlx::g_gemm_path) c.store(0);
}
extern "C" int rlx_set_aux_gemm_engine(int engine) {
  if (engine == 0 || engine == 1) rlx::g_aux_gemm_engine = engine;
  else rlx::set_error("rlx_set_aux_gemm_engine: unknown engine %d", engine);
  return rlx::g_aux_gemm_engine;
}
extern "C" int rlx_set_autocast_bf16(int on) {
  rlx::g_autocast_bf16 = on ? 1 : 0;
  return rlx::g_autocast_bf16;
}

extern "C" int64_t rlx_ppo_param_count(const rlx_ppo_dims* d) {
  if (d == nullptr || !rlx::dims_ok(*d)) {
    rlx::set_error("rlx_ppo_param_count: unsupported dims");
    return RLX_ERR_INVALID_ARG;
  }
  return rlx::make_layout(*d).total();
}

extern "C" int rlx_ppo_param_layout(const rlx_ppo_dims* d, int64_t* offsets, int32_t* is_critic) {
  RLX_CHECK_ARG(d != nullptr && rlx::dims_ok(*d), "unsupported dims");
  RLX_CHECK_ARG(offsets != nullptr, "offsets is null");
  const rlx::PpoLayout L = rlx::make_layout(*d);
  for (int i = 0; i <= RLX_PPO_NSEG; ++i) offsets[i] = L.off[i];
  if (is_critic)
    for (int i = 0; i < RLX_PPO_NSEG; ++i) is_critic[i] = rlx::seg_is_critic(i) ? 1 : 0;
  return RLX_OK;
}

extern "C" int rlx_timing_begin(void) {
  rlx::g_recs.clear();
  rlx::g_event_next = 0;
  rlx::g_timing = true;
  return RLX_OK;
}

extern "C" int rlx_timing_end(double* ms, uint64_t* launches, double* flops, double* bytes) {
  rlx::g_timing = false;
  RLX_CHECK_CUDA(cudaDeviceSynchronize());
  for (int i = 0; i < RLX_NKCLASS; ++i) {
    if (ms) ms[i] = 0;
    if (launches) launches[i] = 0;
    if (flops) flops[i] = 0;
    if (bytes) bytes[i] = 0;
  }
  for (const auto& r : rlx::g_recs) {
    float t = 0.f;
    RLX_CHECK_CUDA(cudaEventElapsedTime(&t, r.e0, r.e1));
    if (ms) ms[r.cls] += t;
    if (launches) launches[r.cls] += 1;
    if (flops) flops[r.cls] += r.flops;
    if (bytes) bytes[r.cls] += r.bytes;
  }
  rlx::g_recs.clear();
  rlx::g_event_next = 0;
  return RLX_OK;
}

extern "C" const char* rlx_kernel_class_name(int cls) {
  static const char* names[RLX_NKCLASS] = {"gemm_fwd", "gemm_dx", "gemm_dw", "head_rollout", "head_train", "head_wgrad", "grad_reduce",
                                           "clip_adam", "gather", "adv_stats", "gae", "rollout_store", "peer_allreduce", "other"};
  return (cls >= 0 && cls < RLX_NKCLASS) ? names[cls] : "?";
}
