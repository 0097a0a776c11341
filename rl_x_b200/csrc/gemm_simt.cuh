// fp32 SIMT (FFMA) GEMM engine: 128x128x8 register-tiled kernel, double-buffered shared memory.
// This is the exact-fp32 engine (bitwise fp32 FMA accumulation in k order); the wgmma 3xTF32 engine in gemm_tc.cu
// is validated against it.  One template covers the three operand layouts the MLP needs:
//   forward      C[m,n] = act(sum_k A[m,k] W[n,k] + b[n])           A k-major, B k-major   ("NT")
//   backward dX  C[m,n] = (sum_k dZ[m,k] W[k,n]) * (1 - H[m,n]^2)    A k-major, B n-major   ("NN")
//   backward dW  C[o,i] = sum_m dZ[m,o] X[m,i]  (split over m)       A m-major, B n-major   ("TN")
#pragma once
#include "common.cuh"

namespace rlx {

enum Epi { EPI_NONE = 0, EPI_BIAS = 1, EPI_BIAS_TANH = 2, EPI_DTANH = 3, EPI_BIAS_RELU = 4, EPI_DRELU = 5 };

struct GemmP {
  const float* A;
  const float* B;
  float* C;
  const float* bias;  // [N] (EPI_BIAS*)
  const float* aux;   // [M, ldaux] activation values for EPI_DTANH / EPI_DRELU
  float* rowsum;      // optional (TN only): rowsum[z][m] = sum_k Aop[m,k]  (bias gradients), written by the n-tile-0 CTAs
  int M, N, K;        // C is [M, N]; K = reduction length
  int lda, ldb, ldc, ldaux;
  long long sA, sB, sC, sBias, sAux, sRowsum;  // batch strides (elements)
  int splits;         // split-K factor (grid.z = batch * splits)
  int kchunk;         // rows of K per split (multiple of 8)
  long long sSplitC, sSplitRowsum;             // per-split output strides
  int bf16;           // bf16-autocast mode: operands are bf16 values; Linear outputs / activations / their gradients are rounded to bf16
                      // where torch's autocast rounds them (EPI_NONE outputs - split-K partials of weight gradients - stay fp32: they
                      // are rounded once after the full reduction)
  const float* b_hi;  // optional, wgmma engine only: tf32 hi / lo copies of B (tf32_split), K-major [N, K] with pitch ldb and batch stride sB;
  const float* b_lo;  // the forward (bias+tanh) and dX (tanh') GEMMs then skip the B converter.  The SIMT engine reads B.
};

constexpr int GBM = 128, GBN = 128, GBK = 8, GPAD = 4;

template <bool KMAJ, bool VEC>
__device__ __forceinline__ void gemm_load_tile(const float* __restrict__ X, int ld, int row0, int nrows, int k0, int kend,
                                               int tid, float (&r)[4]) {
  // KMAJ:  element (row, k) at X[row*ld + k]; thread loads 4 consecutive k of one row.
  // !KMAJ: element (row, k) at X[k*ld + row]; thread loads 4 consecutive rows of one k.
  if (KMAJ) {
    const int row = row0 + (tid >> 1), k = k0 + (tid & 1) * 4;
    if (row < nrows) {
      const float* p = X + (long long)row * ld + k;
      if (VEC && k + 3 < kend) {
        const float4 v = *reinterpret_cast<const float4*>(p);
        r[0] = v.x; r[1] = v.y; r[2] = v.z; r[3] = v.w;
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) r[j] = (k + j < kend) ? p[j] : 0.f;
      }
    } else {
      r[0] = r[1] = r[2] = r[3] = 0.f;
    }
  } else {
    const int k = k0 + (tid >> 5), row = row0 + (tid & 31) * 4;
    if (k < kend) {
      const float* p = X + (long long)k * ld + row;
      if (VEC && row + 3 < nrows) {
        const float4 v = *reinterpret_cast<const float4*>(p);
        r[0] = v.x; r[1] = v.y; r[2] = v.z; r[3] = v.w;
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) r[j] = (row + j < nrows) ? p[j] : 0.f;
      }
    } else {
      r[0] = r[1] = r[2] = r[3] = 0.f;
    }
  }
}

template <bool KMAJ>
__device__ __forceinline__ void gemm_store_tile(float (*S)[GBM + GPAD], int tid, const float (&r)[4]) {
  if (KMAJ) {
    const int row = tid >> 1, k = (tid & 1) * 4;
#pragma unroll
    for (int j = 0; j < 4; ++j) S[k + j][row] = r[j];
  } else {
    const int k = tid >> 5, row = (tid & 31) * 4;
    *reinterpret_cast<float4*>(&S[k][row]) = make_float4(r[0], r[1], r[2], r[3]);
  }
}

template <bool A_KMAJ, bool B_KMAJ, int EPI, bool VEC>
__global__ void __launch_bounds__(256, 2) sgemm_kernel(const GemmP p) {
  __shared__ __align__(16) float As[2][GBK][GBM + GPAD];
  __shared__ __align__(16) float Bs[2][GBK][GBN + GPAD];

  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int batch = blockIdx.z / p.splits, split = blockIdx.z % p.splits;
  const int m0 = blockIdx.y * GBM, n0 = blockIdx.x * GBN;
  const int kbeg = split * p.kchunk;
  const int kend = min(p.K, kbeg + p.kchunk);

  const float* __restrict__ A = p.A + batch * p.sA;
  const float* __restrict__ B = p.B + batch * p.sB;

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  float rs[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) rs[i] = 0.f;
  const bool do_rowsum = (p.rowsum != nullptr) && blockIdx.x == 0 && tx == 0;

  float ra[4], rb[4];
  const int nk = (kend - kbeg + GBK - 1) / GBK;
  if (nk > 0) {
    gemm_load_tile<A_KMAJ, VEC>(A, p.lda, m0, p.M, kbeg, kend, tid, ra);
    gemm_load_tile<B_KMAJ, VEC>(B, p.ldb, n0, p.N, kbeg, kend, tid, rb);
    gemm_store_tile<A_KMAJ>(As[0], tid, ra);
    gemm_store_tile<B_KMAJ>(Bs[0], tid, rb);
  }
  __syncthreads();

  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) {
      gemm_load_tile<A_KMAJ, VEC>(A, p.lda, m0, p.M, kbeg + (kt + 1) * GBK, kend, tid, ra);
      gemm_load_tile<B_KMAJ, VEC>(B, p.ldb, n0, p.N, kbeg + (kt + 1) * GBK, kend, tid, rb);
    }
#pragma unroll
    for (int k = 0; k < GBK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4 + 64]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4 + 64]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
      if (do_rowsum) {
#pragma unroll
        for (int i = 0; i < 8; ++i) rs[i] += a[i];
      }
    }
    if (kt + 1 < nk) {
      gemm_store_tile<A_KMAJ>(As[buf ^ 1], tid, ra);
      gemm_store_tile<B_KMAJ>(Bs[buf ^ 1], tid, rb);
    }
    __syncthreads();
  }

  // ---------------------------------------------------------------- epilogue
  float* __restrict__ C = p.C + batch * p.sC + split * p.sSplitC;
  const float* __restrict__ bias = (EPI == EPI_BIAS || EPI == EPI_BIAS_TANH || EPI == EPI_BIAS_RELU) ? p.bias + batch * p.sBias : nullptr;
  const float* __restrict__ aux = (EPI == EPI_DTANH || EPI == EPI_DRELU) ? p.aux + batch * p.sAux : nullptr;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int m = m0 + ((i < 4) ? (ty * 4 + i) : (64 + ty * 4 + (i - 4)));
    if (m >= p.M) continue;
#pragma unroll
    for (int jh = 0; jh < 2; ++jh) {
      const int nb = n0 + jh * 64 + tx * 4;
      float v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int n = nb + j;
        float x = acc[i][jh * 4 + j];
        if (n < p.N) {
          if (EPI == EPI_BIAS) x = bf16r_if(x + bias[n], p.bf16);
          if (EPI == EPI_BIAS_TANH) x = bf16r_if(tanhf(bf16r_if(x + bias[n], p.bf16)), p.bf16);  // Linear output bf16, tanh output bf16
          if (EPI == EPI_BIAS_RELU) x = fmaxf(x + bias[n], 0.f);
          if (EPI == EPI_DTANH) {
            const float h = aux[(long long)m * p.ldaux + n];
            x = bf16r_if(bf16r_if(x, p.bf16) * (1.f - h * h), p.bf16);  // linear-backward output bf16, then tanh_backward in bf16
          }
          if (EPI == EPI_DRELU) {
            const float h = aux[(long long)m * p.ldaux + n];
            x = (h > 0.f) ? x : 0.f;
          }
        }
        v[j] = x;
      }
      float* cp = C + (long long)m * p.ldc + nb;
      if (VEC && nb + 3 < p.N) {
        *reinterpret_cast<float4*>(cp) = make_float4(v[0], v[1], v[2], v[3]);
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (nb + j < p.N) cp[j] = v[j];
      }
    }
  }
  if (do_rowsum) {
    float* rsout = p.rowsum + batch * p.sRowsum + split * p.sSplitRowsum;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int m = m0 + ((i < 4) ? (ty * 4 + i) : (64 + ty * 4 + (i - 4)));
      if (m < p.M) rsout[m] = rs[i];
    }
  }
}

inline bool gemm_vec_ok(const GemmP& p) {
  auto al = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  bool ok = al(p.A) && al(p.B) && al(p.C) && (p.lda % 4 == 0) && (p.ldb % 4 == 0) && (p.ldc % 4 == 0);
  ok = ok && (p.sA % 4 == 0) && (p.sB % 4 == 0) && (p.sC % 4 == 0) && (p.sSplitC % 4 == 0) && (p.kchunk % 4 == 0);
  return ok;
}

template <bool A_KMAJ, bool B_KMAJ, int EPI>
int launch_sgemm(const GemmP& p, int batch, cudaStream_t stream, int kclass = KC_OTHER) {
  if (p.M <= 0 || p.N <= 0) return RLX_OK;
  dim3 grid((unsigned)ceil_div(p.N, GBN), (unsigned)ceil_div(p.M, GBM), (unsigned)(batch * p.splits));
  const double flops = 2.0 * p.M * p.N * (double)p.K * batch;
  const double bytes = 4.0 * batch * ((double)p.M * p.K + (double)p.N * p.K + (double)p.M * p.N * p.splits);
  if (gemm_vec_ok(p)) {
    RLX_LAUNCH_C(kclass, flops, bytes, (sgemm_kernel<A_KMAJ, B_KMAJ, EPI, true>), grid, 256, 0, stream, p);
  } else {
    RLX_LAUNCH_C(kclass, flops, bytes, (sgemm_kernel<A_KMAJ, B_KMAJ, EPI, false>), grid, 256, 0, stream, p);
  }
  return RLX_OK;
}

}  // namespace rlx
