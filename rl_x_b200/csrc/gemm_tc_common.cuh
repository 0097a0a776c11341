// Pieces of the Hopper tensor-core GEMM engine (gemm_tc.cu): tile constants, kernel parameters, PTX wrappers (mbarrier, TMA,
// wgmma), shared-memory matrix descriptors, TMA tensor maps.
#pragma once
#include <cuda.h>

#include "common.cuh"
#include "gemm_simt.cuh"

namespace rlx {
namespace tc {

constexpr int BM = 128;        // two consumer warpgroups, 64 rows each (wgmma M = 64)
constexpr int BN = 128;        // wgmma N
constexpr int BK = 32;         // fp32 elements per k-block = one 128-byte swizzle row
constexpr int WG_K = 8;        // tf32: 32 bytes of K per wgmma
constexpr int NUM_THREADS = 384;  // warpgroup 0: TMA + hi/lo converter; warpgroups 1, 2: wgmma consumers + epilogue

enum TcEpi { TC_EPI_NONE = 0, TC_EPI_BIAS_TANH = 1, TC_EPI_DTANH = 2, TC_EPI_BIAS_RELU = 3, TC_EPI_DRELU = 4, TC_EPI_BIAS = 5 };

struct TcParams {
  int M, N, K;               // per-z output is [M, N]; K = full reduction extent
  int batch, splits, kchunk; // z = batch * splits; kchunk multiple of BK
  int tiles_m, tiles_n;
  // TMA coordinate offsets per batch index (elements)
  int a_mn_off, a_k_off, b_mn_off, b_k_off;
  float* C;
  long long ldc, c_batch_off, c_split_off;
  int n_main;                // columns >= n_main are not stored to C; column == n_main goes to extra_col (bias-gradient trick)
  int transpose_out;         // store C^T: element (m, n) at C[n * ldc + m]; rows >= m_main are not stored, row == m_main goes to extra_col[n]
  int m_main;
  float* extra_col;          // [z][M] or null
  long long extra_batch_off, extra_split_off;
  const float* bias;         // TC_EPI_BIAS_TANH
  long long bias_batch_off;
  const float* aux;          // TC_EPI_DTANH: activation values, same indexing as C
  long long ldaux, aux_batch_off;
  int single;                // bf16-autocast mode: operands are bf16 values = exact TF32 operands -> ONE MMA per k-slice, no lo tiles
  int bf16;                  // round Linear outputs / activations / activation gradients to bf16 in the epilogue (see GemmP::bf16)
};

// ------------------------------------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
      "@P1 bra WAIT_DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t"
      "}" ::"r"(smem_u32(bar)), "r"(parity)
      : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }

__device__ __forceinline__ void tma_load_2d(const CUtensorMap* map, uint64_t* bar, void* smem, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(smem)),
               "l"((uint64_t)map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)map) : "memory");
}

// wgmma shared-memory matrix descriptor (sm_90 layout): [0,14) start address >> 4, [16,30) leading byte offset >> 4,
// [32,46) stride byte offset >> 4, [62,64) layout type (1 = SWIZZLE_128B).  Only K-major operands exist for tf32: a row of
// 32 fp32 k-values is one 128-byte swizzle row, 8 rows form a 1024-byte atom (SBO), LBO is unused.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFFu);
  d |= (uint64_t)1u << 16;
  d |= (uint64_t)(1024u >> 4) << 32;
  d |= 1ull << 62;
  return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accesses of accumulator registers across wgmma issue / wait
__device__ __forceinline__ void fence_acc(float (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x 128] (+)= A[64 x 8] * B[128 x 8]^T, both tf32 K-major in shared memory, fp32 accumulators in registers
__device__ __forceinline__ void wgmma_tf32_m64n128k8(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1;\n\t"
      "}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
        "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
        "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]),
        "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]),
        "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]),
        "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a_desc), "l"(b_desc), "r"(accumulate)
      : "memory");
}


// ------------------------------------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static inline EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(ptr);
  }
  return fn;
}

// 2-D fp32 row-major tensor [rows, cols] with row pitch ld (elements); box = [box_cols (<= 32), box_rows], SWIZZLE_128B.
static inline int make_tmap(CUtensorMap* map, const float* base, long long rows, long long cols, long long ld, int box_cols, int box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) {
    set_error("tensor-core engine: cuTensorMapEncodeTiled is unavailable");
    return RLX_ERR_UNSUPPORTED;
  }
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstride[1] = {(cuuint64_t)ld * 4};
  cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("tensor-core engine: cuTensorMapEncodeTiled failed (%d) rows=%lld cols=%lld ld=%lld box=%dx%d", (int)r, rows, cols, ld, box_cols, box_rows);
    return RLX_ERR_CUDA;
  }
  return RLX_OK;
}

struct TcOperand {
  const float* base;
  long long rows, cols, ld;  // global tensor as allocated: [rows, cols], pitch ld
};


}  // namespace tc
}  // namespace rlx
