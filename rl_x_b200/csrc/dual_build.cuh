// Dual-build support for the "one thread = one row / element" sources (lstm.cu, replay_nstep.cu): the same file compiles with nvcc into
// the product library, and with  g++ -x c++ -DRLX_EMU  into a host library for the CPU tests, where a kernel launch is a loop over
// (block, thread) and a GEMM is an interpreter of the GemmP contract of gemm_simt.cuh.  Kernels launched with RLX_FLAT_LAUNCH must not
// use shared memory, warp primitives or barriers.  Block-cooperative kernels (dynamic shared memory + __syncthreads, no warp
// primitives) go through RLX_BLOCK_LAUNCH: the emulation runs one block at a time with one OS thread per CUDA thread and a real
// barrier, so a missing __syncthreads is a real data race there too (and ThreadSanitizer sees it: tests/emu_tsan_lstm.cpp).
// The emulation build is test scaffolding; nothing in the product loads it.
#pragma once
#include <stdint.h>
#include <stddef.h>

#include "../../include/rlx_b200.h"

#ifdef RLX_EMU
#include <math.h>
#include <stdio.h>
#include <stdarg.h>
#include <algorithm>
#include <condition_variable>
#include <mutex>
#include <thread>
#include <vector>
namespace rlx {
struct EmuDim { unsigned x, y, z; };
static thread_local EmuDim threadIdx, blockIdx, blockDim, gridDim;
// one block of a block-cooperative launch: its dynamic shared memory and its barrier
struct EmuBlock {
  std::vector<float> smem;
  std::mutex m;
  std::condition_variable cv;
  unsigned nthreads = 0, waiting = 0, generation = 0;
  void sync() {
    std::unique_lock<std::mutex> lk(m);
    const unsigned gen = generation;
    if (++waiting == nthreads) { waiting = 0; ++generation; cv.notify_all(); }
    else cv.wait(lk, [&] { return generation != gen; });
  }
};
static thread_local EmuBlock* g_emu_block = nullptr;
// Order in which the emulated threads of a launch run: 0 = ascending (block, thread), 1 = descending.  A kernel whose threads only
// touch their own outputs gives bit-identical results either way; one thread reading what another thread of the SAME launch writes
// (a data race on the device) does not.  tests/test_*_emulation.py run every entry point both ways.
static int g_emu_reverse = 0;
typedef void* cudaStream_t;
static char g_emu_err[512];
static void set_error(const char* fmt, ...) { va_list ap; va_start(ap, fmt); vsnprintf(g_emu_err, sizeof(g_emu_err), fmt, ap); va_end(ap); }
inline long long ceil_div(long long a, long long b) { return (a + b - 1) / b; }
inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }
enum Epi { EPI_NONE = 0, EPI_BIAS = 1, EPI_BIAS_TANH = 2, EPI_DTANH = 3, EPI_BIAS_RELU = 4, EPI_DRELU = 5 };
enum { KC_OTHER = 0, KC_GEMM_FWD = 0, KC_GEMM_DX = 0, KC_GEMM_DW = 0 };
struct GemmP {
  const float* A; const float* B; float* C; const float* bias; const float* aux; float* rowsum;
  int M, N, K; int lda, ldb, ldc, ldaux;
  long long sA, sB, sC, sBias, sAux, sRowsum;
  int splits; int kchunk; long long sSplitC, sSplitRowsum;
};
// interpreter of the GemmP contract of gemm_simt.cuh (same fp32 fmaf accumulation in k order within a split).
// a_rows / b_rows >= 0: the operands are read the way the tensor engine reads them, through a descriptor of that many rows in memory with
// zeros beyond (TMA out-of-bounds fill) - a caller that passes a wrong extent to aux_gemm gets wrong numbers here too.
template <bool A_KMAJ, bool B_KMAJ, int EPI>
int launch_sgemm(const GemmP& p, int batch, cudaStream_t, int = 0, long long a_rows = -1, long long b_rows = -1) {
  for (int z = 0; z < batch * p.splits; ++z) {
    const int b = z / p.splits, sp = z % p.splits;
    const int kbeg = sp * p.kchunk, kend = std::min(p.K, kbeg + p.kchunk);
    const float* A = p.A + b * p.sA; const float* B = p.B + b * p.sB;
    float* C = p.C + b * p.sC + sp * p.sSplitC;
    for (int m = 0; m < p.M; ++m)
      for (int n = 0; n < p.N; ++n) {
        float acc = 0.f;
        for (int k = kbeg; k < kend; ++k) {
          const bool a_in = a_rows < 0 || (A_KMAJ ? m : k) < a_rows, b_in = b_rows < 0 || (B_KMAJ ? n : k) < b_rows;
          const float a = !a_in ? 0.f : A_KMAJ ? A[(long long)m * p.lda + k] : A[(long long)k * p.lda + m];
          const float w = !b_in ? 0.f : B_KMAJ ? B[(long long)n * p.ldb + k] : B[(long long)k * p.ldb + n];
          acc = fmaf(a, w, acc);
        }
        if (EPI == EPI_BIAS) acc += p.bias[b * p.sBias + n];
        if (EPI == EPI_BIAS_TANH) acc = tanhf(acc + p.bias[b * p.sBias + n]);
        if (EPI == EPI_DTANH) { const float h = p.aux[b * p.sAux + (long long)m * p.ldaux + n]; acc = acc * (1.f - h * h); }
        if (EPI == EPI_BIAS_RELU) acc = fmaxf(acc + p.bias[b * p.sBias + n], 0.f);
        if (EPI == EPI_DRELU) { const float h = p.aux[b * p.sAux + (long long)m * p.ldaux + n]; acc = h > 0.f ? acc : 0.f; }
        C[(long long)m * p.ldc + n] = acc;
      }
  }
  return RLX_OK;
}
}  // namespace rlx
namespace rlx {
// dense layer of a dual-build source; the host build interprets the GemmP contract (a_rows / b_rows only matter to the tensor engine)
template <bool A_KMAJ, bool B_KMAJ, int EPI>
int aux_gemm(const GemmP& p, int batch, cudaStream_t st, int kclass, long long a_rows, long long b_rows) {
  if (a_rows <= 0 || b_rows <= 0) return RLX_ERR_INVALID_ARG;
  // Too small an extent turns operand rows into zeros (wrong numbers in the parity tests); too large a one makes the descriptor cover
  // memory the operand does not own: touch the last element each descriptor declares, so that an AddressSanitizer build of the
  // emulation (tests/conftest.py::emu_build_cmd) sees it.
  volatile float touch = p.A[(a_rows - 1) * p.lda + ((A_KMAJ ? p.K : p.M) - 1)] + p.B[(b_rows - 1) * p.ldb + ((B_KMAJ ? p.K : p.N) - 1)];
  (void)touch;
  return launch_sgemm<A_KMAJ, B_KMAJ, EPI>(p, batch, st, kclass, a_rows, b_rows);
}
}  // namespace rlx
extern "C" void rlx_emu_set_thread_order(int reverse) { rlx::g_emu_reverse = reverse; }
#define __syncthreads() rlx::g_emu_block->sync()
#define RLX_DYN_SMEM(name) float* name = rlx::g_emu_block->smem.data()
// block-cooperative launch: blocks one after the other, the threads of a block concurrently (they meet at __syncthreads)
#define RLX_BLOCK_LAUNCH(kernel, nb_, nt_, smem_, stream, ...)                            \
  do {                                                                                            \
    const unsigned _nb = (unsigned)(nb_), _nt = (unsigned)(nt_);                         \
    for (unsigned _b = 0; _b < _nb; ++_b) {                                                       \
      rlx::EmuBlock _blk;                                                                         \
      _blk.smem.assign(((size_t)(smem_) + 3) / 4, nanf(""));                                 \
      _blk.nthreads = _nt;                                                                        \
      std::vector<std::thread> _ths;                                                              \
      for (unsigned _t = 0; _t < _nt; ++_t)                                                       \
        _ths.emplace_back([=, &_blk] {                                                            \
          rlx::g_emu_block = &_blk;                                                               \
          rlx::blockDim = {_nt, 1, 1};                                                            \
          rlx::gridDim = {_nb, 1, 1};                                                             \
          rlx::blockIdx = {_b, 0, 0};                                                             \
          rlx::threadIdx = {_t, 0, 0};                                                            \
          kernel(__VA_ARGS__);                                                                    \
        });                                                                                       \
      for (auto& _th : _ths) _th.join();                                                          \
    }                                                                                             \
  } while (0)
#define __global__
#define __device__
#define __forceinline__ inline
#define __restrict__
#define __launch_bounds__(...)
#define RLX_CHECK_ARG(cond, msg) do { if (!(cond)) { rlx::set_error("%s: invalid argument: %s", __func__, msg); return RLX_ERR_INVALID_ARG; } } while (0)
#define RLX_FLAT_LAUNCH(kernel, nthreads_total, stream, ...)                                          \
  do {                                                                                            \
    const long long _n = (nthreads_total);                                                        \
    rlx::blockDim = {256, 1, 1};                                                                  \
    rlx::gridDim = {(unsigned)rlx::ceil_div(_n, 256), 1, 1};                                      \
    for (unsigned _bi = 0; _bi < rlx::gridDim.x; ++_bi)                                           \
      for (unsigned _ti = 0; _ti < 256; ++_ti) {                                                  \
        const unsigned _b = rlx::g_emu_reverse ? rlx::gridDim.x - 1 - _bi : _bi;                  \
        const unsigned _t = rlx::g_emu_reverse ? 255 - _ti : _ti;                                 \
        rlx::blockIdx = {_b, 0, 0};                                                               \
        rlx::threadIdx = {_t, 0, 0};                                                              \
        kernel(__VA_ARGS__);                                                                      \
      }                                                                                           \
  } while (0)
#else
#include "common.cuh"
#include "gemm_dispatch.cuh"
namespace rlx {
// dense layer of a dual-build source: exact-fp32 SIMT engine, or (rlx_set_aux_gemm_engine(1)) the wgmma 3xTF32 engine where it covers the
// layout / epilogue / alignment.  a_rows / b_rows: rows of the operand tensors in memory (see run_gemm).  Single-CTA tensor kernels, and
// only for products with at least half a tile in each output dimension: the skinny ones (heads, biases-as-GEMMs) carry no FLOPs worth
// a TMA descriptor and stay on the SIMT engine.
template <bool A_KMAJ, bool B_KMAJ, int EPI>
static int aux_gemm(const GemmP& p, int batch, cudaStream_t st, int kclass, long long a_rows, long long b_rows) {
  if (g_aux_gemm_engine == 1 && p.M >= 64 && p.N >= 64 && p.K >= 32 && p.rowsum == nullptr) {
    const int rc = tc_gemm(p, A_KMAJ, B_KMAJ, tc_epi_of<EPI>(), batch, kclass, a_rows, b_rows, 0, nullptr, 0, 0, st);
    if (rc == RLX_OK) g_aux_tc_gemms.fetch_add(1, std::memory_order_relaxed);   // rlx_aux_tc_gemm_count(): evidence of which engine ran
    if (rc != RLX_ERR_UNSUPPORTED) return rc;
  }
  return launch_sgemm<A_KMAJ, B_KMAJ, EPI>(p, batch, st, kclass);
}
}  // namespace rlx
#define RLX_FLAT_LAUNCH(kernel, nthreads_total, stream, ...)                                                                       \
  do {                                                                                                                         \
    const long long _n = (nthreads_total);                                                                                     \
    if (_n > 0) RLX_LAUNCH_C(rlx::KC_OTHER, 0, 0, kernel, (unsigned)rlx::ceil_div(_n, 256), 256, 0, (cudaStream_t)(stream), __VA_ARGS__); \
  } while (0)
#define RLX_DYN_SMEM(name) extern __shared__ float name[]
// block-cooperative launch with dynamic shared memory (opted in above the 48 KB default once per kernel)
#define RLX_BLOCK_LAUNCH(kernel, nb_, nt_, smem_, stream, ...)                                                                   \
  do {                                                                                                                         \
    static size_t _smem_set = 0;                                                                                               \
    if ((size_t)(smem_) > _smem_set) {                                                                                    \
      RLX_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(smem_)));            \
      _smem_set = (size_t)(smem_);                                                                                        \
    }                                                                                                                          \
    RLX_LAUNCH_C(rlx::KC_OTHER, 0, 0, kernel, (unsigned)(nb_), (unsigned)(nt_), (size_t)(smem_), (cudaStream_t)(stream), __VA_ARGS__); \
  } while (0)
#endif

// fp32 multiply / add that the compiler may not contract into an FMA (results must match a plain float32 restatement bit for bit)
namespace rlx {
#ifdef RLX_EMU
inline float rn_mul(float a, float b) { volatile float r = a * b; return r; }
inline float rn_add(float a, float b) { volatile float r = a + b; return r; }
inline float rn_sub(float a, float b) { volatile float r = a - b; return r; }
#else
__device__ __forceinline__ float rn_mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float rn_add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float rn_sub(float a, float b) { return __fsub_rn(a, b); }
#endif
}  // namespace rlx
