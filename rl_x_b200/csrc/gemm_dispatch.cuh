// One GEMM through the selected engine: wgmma 3xTF32 when it covers the shape / alignment, exact-fp32 SIMT otherwise.
#pragma once
#include "gemm_simt.cuh"

namespace rlx {

// gemm_tc.cu; returns RLX_ERR_UNSUPPORTED when a shape / alignment is not covered
int tc_supported(const rlx_ppo_dims& d);
int tc_gemm(const GemmP& g, bool a_kmaj, bool b_kmaj, int epi, int batch, int kclass, long long a_rows, long long b_rows, cudaStream_t stream);
// C^T stored: element (m, n) at C[n * ldc + m] for m < m_main; row m_main goes to extra_row[n] (+ batch / split offsets).  MN-major A and B,
// no epilogue function.
int tc_gemm_t(const GemmP& g, bool a_kmaj, bool b_kmaj, int epi, int batch, int kclass, long long a_rows, long long b_rows, int m_main, float* extra_row,
              long long extra_batch_off, long long extra_split_off, cudaStream_t stream);
enum { TC_NONE = 0, TC_BIAS_TANH = 1, TC_DTANH = 2, TC_BIAS_RELU = 3, TC_DRELU = 4, TC_BIAS = 5 };

// tf32 hi / lo split of fp32 matrices for GemmP::b_hi / b_lo, the wgmma engine's converter arithmetic: hi = x & 0xFFFFE000, lo = x - hi.
// src is [batch][rows][cols] contiguous; hi / lo get the same layout, or with trans [batch][cols][rows].  One launch for all jobs.
struct Tf32SplitJob {
  const float* src;
  float* hi;
  float* lo;
  int batch, rows, cols, trans;
};
constexpr int kMaxTf32SplitJobs = 3;
int tf32_split(const Tf32SplitJob* jobs, int njobs, int kclass, cudaStream_t stream);

template <int EPI>
constexpr int tc_epi_of() {
  return EPI == EPI_BIAS_TANH ? TC_BIAS_TANH : EPI == EPI_DTANH ? TC_DTANH : EPI == EPI_BIAS_RELU ? TC_BIAS_RELU : EPI == EPI_DRELU ? TC_DRELU
       : EPI == EPI_BIAS ? TC_BIAS : TC_NONE;
}

// a_rows / b_rows: rows of the operand tensors as laid out in memory (TMA needs the true extents for its zero fill).
template <bool A_KMAJ, bool B_KMAJ, int EPI>
static int run_gemm(bool tc, const GemmP& g, int batch, cudaStream_t st, int kclass, long long a_rows, long long b_rows) {
  if (tc && g.rowsum == nullptr && g.K >= 32) {
    const int rc = tc_gemm(g, A_KMAJ, B_KMAJ, tc_epi_of<EPI>(), batch, kclass, a_rows, b_rows, st);
    if (rc != RLX_ERR_UNSUPPORTED) return rc;
  }
  return launch_sgemm<A_KMAJ, B_KMAJ, EPI>(g, batch, st, kclass);
}

}  // namespace rlx
