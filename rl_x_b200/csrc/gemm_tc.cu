// Hopper tensor-core (wgmma) GEMM engine with fp32-equivalent accuracy: 3xTF32 split.
//
//   C[m,n] = epilogue( sum_k A(m,k) * B(n,k) ),  A, B, C fp32 in global memory, accumulation in fp32 registers.
//
// Each fp32 operand x is used as  x = hi + lo  with hi = x with the low 13 mantissa bits cleared (an exact tf32 value) and
// lo = x - hi (exact in fp32); three MMAs per k-slice accumulate  hi*hi + hi*lo + lo*hi  (the lo*lo term is below fp32
// resolution).  That is the accuracy class of an fp32 FMA loop (SURVEY.md §7a: single-pass TF32 misses the 1e-5 loss-parity bar,
// 3xTF32 does not) at one third of the TF32 tensor rate.
//
// Structure (one persistent CTA per SM, 384 threads = 3 warpgroups, static tile schedule, 128 x 128 output tiles):
//   warpgroup 0   thread 0 issues cp.async.bulk.tensor 2-D tiles (SWIZZLE_128B) of raw fp32 A and B into a 3-stage ring, running ahead
//                 of the conversion; all 128 threads then write the hi and lo tiles of both operands, K-major and 128-byte swizzled
//                 (the only layout wgmma accepts for tf32), into a 2-stage operand ring and fence.proxy.async it for the tensor core
//   warpgroups 1, 2   rows 0-63 / 64-127 of the tile: wgmma.mma_async m64n128k8 tf32 (3 per k-slice of 8), then the epilogue straight
//                 from the accumulator registers: bias+tanh / tanh' / relu / plain, stores to C (or C^T)
// Operand layouts in global memory: K-major (row = m or n, 32 consecutive k = one 128-byte swizzle row) or MN-major (row = k, 32
// consecutive m/n per 128-byte row; used by the weight-gradient GEMMs whose reduction runs over the minibatch rows).  The converter
// transposes MN-major tiles to K-major.  Out-of-bounds parts of a box are zero-filled by TMA, so M / N / K tails need no special code
// in the main loop.
#include "gemm_dispatch.cuh"
#include "gemm_tc_common.cuh"

namespace rlx {
namespace tc {

// The main product and the correction terms go to separate accumulators: tiny correction terms added into the large running sum
// would lose their low bits to the tensor core's accumulation rounding; the epilogue adds the two in fp32 round-to-nearest.
struct Cfg {
  static constexpr int A_BYTES = BM * BK * 4;                   // 16 KB
  static constexpr int B_BYTES = BN * BK * 4;                   // 16 KB
  static constexpr int RAW_BYTES = A_BYTES + B_BYTES;           // raw stage: [A | B] as TMA wrote them
  static constexpr int OP_BYTES = 2 * RAW_BYTES;                // operand stage: [hi A | hi B | lo A | lo B], K-major swizzled
  static constexpr int RAW_STAGES = 3, OP_STAGES = 2;
  static constexpr int SMEM_BYTES = RAW_STAGES * RAW_BYTES + OP_STAGES * OP_BYTES + 1024 /*barriers*/ + 1024 /*alignment slack*/;
};
static_assert(Cfg::SMEM_BYTES <= 227 * 1024, "shared memory of one H100 block");

// One operand tile (ROWS x BK) from its raw stage to K-major swizzled hi / lo tiles.  In the 128-byte swizzle every 16-byte chunk
// (4 k-values) c of row r sits at r * 128 + ((c ^ (r & 7)) << 4).  Thread t of the warpgroup handles chunks t, t + 128, ...
template <bool KMAJ, bool BF16, int ROWS>
__device__ __forceinline__ void convert_tile(const uint8_t* raw, uint8_t* hi, uint8_t* lo, int t) {
  constexpr uint32_t HI = 0xFFFFE000u;
  if (KMAJ) {
    // TMA wrote the tile in exactly the target layout: an element-wise pass
#pragma unroll 4
    for (int i = t; i < ROWS * 8; i += 128) {
      const uint4 v = reinterpret_cast<const uint4*>(raw)[i];
      const uint4 h = make_uint4(v.x & HI, v.y & HI, v.z & HI, v.w & HI);
      reinterpret_cast<uint4*>(hi)[i] = h;
      if (!BF16)
        reinterpret_cast<float4*>(lo)[i] = make_float4(__uint_as_float(v.x) - __uint_as_float(h.x), __uint_as_float(v.y) - __uint_as_float(h.y),
                                                       __uint_as_float(v.z) - __uint_as_float(h.z), __uint_as_float(v.w) - __uint_as_float(h.w));
    }
  } else {
    // ROWS / 32 boxes of [BK k-rows][32 mn] (4 KB each, swizzled the same way with k as the row).  A warp handles 32 consecutive mn of
    // one k-chunk: its reads of one k-row hit 32 different banks, its 16-byte writes are conflict-free per quarter warp.
#pragma unroll 2
    for (int i = t; i < ROWS * 8; i += 128) {
      const int mn = i % ROWS, kc = i / ROWS;
      const uint8_t* box = raw + (mn >> 5) * (BK * 128);
      const int c = (mn & 31) >> 2, e = mn & 3;
      uint32_t v[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int k = kc * 4 + q;
        v[q] = *reinterpret_cast<const uint32_t*>(box + k * 128 + ((c ^ (k & 7)) << 4) + e * 4);
      }
      const int off = mn * 128 + ((kc ^ (mn & 7)) << 4);
      const uint4 h = make_uint4(v[0] & HI, v[1] & HI, v[2] & HI, v[3] & HI);
      *reinterpret_cast<uint4*>(hi + off) = h;
      if (!BF16)
        *reinterpret_cast<float4*>(lo + off) = make_float4(__uint_as_float(v[0]) - __uint_as_float(h.x), __uint_as_float(v[1]) - __uint_as_float(h.y),
                                                           __uint_as_float(v[2]) - __uint_as_float(h.z), __uint_as_float(v[3]) - __uint_as_float(h.w));
    }
  }
}

// BF16: the bf16-autocast variant (single-pass MMAs on bf16-valued operands, bf16 roundings in the epilogue), a compile-time switch so that
// the fp32-equivalent kernels carry none of it
template <bool A_KMAJ, bool B_KMAJ, int EPI, bool BF16>
__global__ void __launch_bounds__(NUM_THREADS, 1) tc_gemm_kernel(const __grid_constant__ CUtensorMap tmap_a,
                                                                 const __grid_constant__ CUtensorMap tmap_b, const TcParams p) {
  constexpr int RAW_STAGES = Cfg::RAW_STAGES, OP_STAGES = Cfg::OP_STAGES;
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment (swizzle atoms) as an OFFSET on the __shared__ pointer: a round trip through uintptr_t makes the compiler lose
  // the shared address space and emit generic loads / stores
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* ops = smem + RAW_STAGES * Cfg::RAW_BYTES;
  uint64_t* raw_full = reinterpret_cast<uint64_t*>(ops + OP_STAGES * Cfg::OP_BYTES);  // [RAW_STAGES]  TMA landed
  uint64_t* op_full = raw_full + RAW_STAGES;                                          // [OP_STAGES]   hi / lo tiles written
  uint64_t* op_empty = op_full + OP_STAGES;                                           // [OP_STAGES]   wgmmas of the slot retired

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_a);
    prefetch_tmap(&tmap_b);
    for (int s = 0; s < RAW_STAGES; ++s) mbar_init(&raw_full[s], 1);
    for (int s = 0; s < OP_STAGES; ++s) {
      mbar_init(&op_full[s], 1);
      mbar_init(&op_empty[s], 8);  // one arrival per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  const int tiles_per_z = p.tiles_m * p.tiles_n;
  const int num_tiles = tiles_per_z * p.batch * p.splits;

  auto tile_coords = [&](int tile, int& zb, int& zs, int& m0, int& n0, int& kbeg, int& nkb) {
    const int z = tile / tiles_per_z, r = tile % tiles_per_z;
    zb = z / p.splits;
    zs = z % p.splits;
    m0 = (r / p.tiles_n) * BM;
    n0 = (r % p.tiles_n) * BN;
    kbeg = zs * p.kchunk;
    const int kend = min(p.K, kbeg + p.kchunk);
    nkb = (kend - kbeg + BK - 1) / BK;
  };

  if (warp < 4) {
    // ===================================================== TMA (thread 0) + hi / lo converter (warpgroup 0)
    const int t = threadIdx.x;
    // load cursor: the k-blocks of this CTA's tiles in consumption order; a raw slot is refilled as soon as the converter is done with it
    int ld_tile = blockIdx.x, ld_kb = 0, ld_count = 0;
    auto load_next = [&]() {
      while (ld_tile < num_tiles) {
        int zb, zs, m0, n0, kbeg, nkb;
        tile_coords(ld_tile, zb, zs, m0, n0, kbeg, nkb);
        if (ld_kb >= nkb) {
          ld_tile += gridDim.x;
          ld_kb = 0;
          continue;
        }
        const int slot = ld_count % RAW_STAGES;
        uint8_t* sa = smem + slot * Cfg::RAW_BYTES;
        uint8_t* sb = sa + Cfg::A_BYTES;
        uint64_t* bar = &raw_full[slot];
        const int k0 = kbeg + ld_kb * BK;
        mbar_arrive_expect_tx(bar, Cfg::RAW_BYTES);
        if (A_KMAJ) {
          tma_load_2d(&tmap_a, bar, sa, p.a_k_off * zb + k0, p.a_mn_off * zb + m0);
        } else {
#pragma unroll
          for (int j = 0; j < BM / 32; ++j) tma_load_2d(&tmap_a, bar, sa + j * (BK * 128), p.a_mn_off * zb + m0 + 32 * j, p.a_k_off * zb + k0);
        }
        if (B_KMAJ) {
          tma_load_2d(&tmap_b, bar, sb, p.b_k_off * zb + k0, p.b_mn_off * zb + n0);
        } else {
#pragma unroll
          for (int j = 0; j < BN / 32; ++j) tma_load_2d(&tmap_b, bar, sb + j * (BK * 128), p.b_mn_off * zb + n0 + 32 * j, p.b_k_off * zb + k0);
        }
        ++ld_kb;
        ++ld_count;
        return;
      }
    };
    if (t == 0)
      for (int i = 0; i < RAW_STAGES; ++i) load_next();
    int rs = 0, os = 0;
    uint32_t rph = 0, oph = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int zb, zs, m0, n0, kbeg, nkb;
      tile_coords(tile, zb, zs, m0, n0, kbeg, nkb);
      for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait(&raw_full[rs], rph);
        mbar_wait(&op_empty[os], oph ^ 1);
        const uint8_t* raw = smem + rs * Cfg::RAW_BYTES;
        uint8_t* op = ops + os * Cfg::OP_BYTES;
        convert_tile<A_KMAJ, BF16, BM>(raw, op, op + Cfg::RAW_BYTES, t);
        convert_tile<B_KMAJ, BF16, BN>(raw + Cfg::A_BYTES, op + Cfg::A_BYTES, op + Cfg::RAW_BYTES + Cfg::A_BYTES, t);
        fence_proxy_async();  // generic-proxy writes -> visible to the tensor core's async-proxy reads
        named_bar_sync(1, 128);  // the whole warpgroup is done with raw slot rs and has written operand slot os
        if (t == 0) {
          mbar_arrive(&op_full[os]);
          load_next();  // refills raw slot rs
        }
        if (++rs == RAW_STAGES) { rs = 0; rph ^= 1; }
        if (++os == OP_STAGES) { os = 0; oph ^= 1; }
      }
    }
  } else {
    // ===================================================== wgmma consumers + epilogue (warpgroups 1, 2)
    const int cw = (warp >> 2) - 1;  // rows 64 * cw .. 64 * cw + 63 of the tile
    float acc[64], cor[64];
    int os = 0;
    uint32_t oph = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int zb, zs, m0, n0, kbeg, nkb;
      tile_coords(tile, zb, zs, m0, n0, kbeg, nkb);
      for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait(&op_full[os], oph);
        const uint32_t op = smem_u32(ops + os * Cfg::OP_BYTES);
        const uint64_t da = make_smem_desc(op + cw * 64 * 128), db = make_smem_desc(op + Cfg::A_BYTES);
        const uint64_t da_lo = make_smem_desc(op + Cfg::RAW_BYTES + cw * 64 * 128), db_lo = make_smem_desc(op + Cfg::RAW_BYTES + Cfg::A_BYTES);
        fence_acc(acc);
        if (!BF16) fence_acc(cor);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < BK / WG_K; ++kk) {
          // advancing along k inside the 128-byte swizzle row: the descriptors differ only in the start address (units of 16 bytes)
          const uint64_t ko = (uint64_t)((kk * WG_K * 4) >> 4);
          const uint32_t accum = (kb | kk) != 0 ? 1u : 0u;
          if (!BF16) {
            wgmma_tf32_m64n128k8(cor, da_lo + ko, db + ko, accum);  // lo * hi   } small terms, own accumulator
            wgmma_tf32_m64n128k8(cor, da + ko, db_lo + ko, 1u);     // hi * lo   }
          }
          wgmma_tf32_m64n128k8(acc, da + ko, db + ko, accum);       // hi * hi  (bf16-valued operands: the whole product)
        }
        wgmma_commit();
        wgmma_wait_all();
        fence_acc(acc);
        if (!BF16) fence_acc(cor);
        __syncwarp();
        if (lane == 0) mbar_arrive(&op_empty[os]);
        if (++os == OP_STAGES) { os = 0; oph ^= 1; }
      }

      // ---- epilogue.  Accumulator layout of wgmma m64nN f32: register j of lane l in warp w (of the warpgroup) holds row
      // 16 w + l / 4 + 8 ((j >> 1) & 1), column 8 (j >> 2) + 2 (l & 3) + (j & 1).
      const int r_base = m0 + cw * 64 + (warp & 3) * 16 + (lane >> 2);
      const int c_base = n0 + 2 * (lane & 3);
      float* cbase = p.C + p.c_batch_off * zb + p.c_split_off * zs;
      float* ebase = p.extra_col != nullptr ? p.extra_col + p.extra_batch_off * zb + p.extra_split_off * zs : nullptr;
      constexpr bool HAS_AUX = (EPI == TC_EPI_DTANH || EPI == TC_EPI_DRELU);
      constexpr bool HAS_BIAS = (EPI == TC_EPI_BIAS_TANH || EPI == TC_EPI_BIAS_RELU || EPI == TC_EPI_BIAS);
      const float* abase = HAS_AUX ? (p.aux + p.aux_batch_off * zb) : nullptr;
      const float* bias = HAS_BIAS ? (p.bias + p.bias_batch_off * zb) : nullptr;
#pragma unroll
      for (int j = 0; j < 64; ++j) {
        const int m = r_base + 8 * ((j >> 1) & 1);
        const int n = c_base + 8 * (j >> 2) + (j & 1);
        if (m >= p.M || n >= p.N) continue;
        float x = BF16 ? acc[j] : acc[j] + cor[j];  // main + correction (fp32 RN)
        if (p.transpose_out) {
          if (m < p.m_main) cbase[(long long)n * p.ldc + m] = x;
          else if (m == p.m_main && ebase != nullptr) ebase[n] = x;
          continue;
        }
        if (HAS_AUX) {
          const float h = abase[(long long)m * p.ldaux + n];
          // bf16 mode: linear-backward output rounded to bf16, then tanh_backward rounded to bf16
          x = (EPI == TC_EPI_DTANH) ? bf16r_if(bf16r_if(x, BF16) * (1.f - h * h), BF16) : ((h > 0.f) ? x : 0.f);
        }
        if (HAS_BIAS) {
          const float z = (EPI == TC_EPI_BIAS_RELU) ? x + bias[n] : bf16r_if(x + bias[n], BF16);  // bf16 mode: Linear output is a bf16 tensor
          x = (EPI == TC_EPI_BIAS_TANH) ? bf16r_if(tanh_fast(z), BF16) : ((EPI == TC_EPI_BIAS_RELU) ? fmaxf(z, 0.f) : z);
        }
        if (n < p.n_main) cbase[(long long)m * p.ldc + n] = x;
        else if (n == p.n_main && ebase != nullptr) ebase[m] = x;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ host side
template <bool A_KMAJ, bool B_KMAJ, int EPI, bool BF16 = false>
static int launch_cfg(const TcOperand& A, const TcOperand& B, TcParams p, int kclass, cudaStream_t stream) {
  CUtensorMap ta, tb;
  int rc = make_tmap(&ta, A.base, A.rows, A.cols, A.ld, 32, A_KMAJ ? BM : BK);
  if (rc) return rc;
  rc = make_tmap(&tb, B.base, B.rows, B.cols, B.ld, 32, B_KMAJ ? BN : BK);
  if (rc) return rc;
  p.tiles_m = (int)ceil_div(p.M, BM);
  p.tiles_n = (int)ceil_div(p.N, BN);
  const long long tiles = (long long)p.tiles_m * p.tiles_n * p.batch * p.splits;
  if (tiles <= 0) return RLX_OK;
  auto kern = tc_gemm_kernel<A_KMAJ, B_KMAJ, EPI, BF16>;
  static bool attr_done = false;
  if (!attr_done) {
    RLX_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    attr_done = true;
  }
  const unsigned grid = (unsigned)std::min<long long>(tiles, sm_count());
  const double flops = 2.0 * p.M * p.N * (double)p.K * p.batch;
  const double bytes = 4.0 * p.batch * ((double)p.M * p.K + (double)p.N * p.K + (double)p.M * p.N * p.splits);
  RLX_LAUNCH_C(kclass, flops, bytes, kern, grid, NUM_THREADS, Cfg::SMEM_BYTES, stream, ta, tb, p);
  return RLX_OK;
}

}  // namespace tc

// ------------------------------------------------------------------------------------------------ engine entry points
using namespace tc;

int tc_supported(const rlx_ppo_dims& d) {
  return (d.hidden % 128 == 0) && d.hidden >= 128 && d.hidden <= 1024 && (d.obs_dim % 4 == 0) && d.obs_dim >= 32;
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// Generic front end over the SIMT engine's GemmP (same meaning of every field).  Supported: all strides multiples of 4 floats,
// 16-byte aligned bases, batch strides that are pure row or column offsets of the operand tensors.
int tc_gemm(const GemmP& g, bool a_kmaj, bool b_kmaj, int epi, int batch, int kclass, long long a_rows, long long b_rows, int n_main,
            float* extra_col, long long extra_batch_off, long long extra_split_off, cudaStream_t stream) {
  return tc_gemm_t(g, a_kmaj, b_kmaj, epi, batch, kclass, a_rows, b_rows, n_main, extra_col, extra_batch_off, extra_split_off, stream, 0, 0);
}

int tc_gemm_t(const GemmP& g, bool a_kmaj, bool b_kmaj, int epi, int batch, int kclass, long long a_rows, long long b_rows, int n_main,
              float* extra_col, long long extra_batch_off, long long extra_split_off, cudaStream_t stream, int transpose_out, int m_main) {
  if (g.M <= 0 || g.N <= 0) return RLX_OK;
  if (!aligned16(g.A) || !aligned16(g.B) || !aligned16(g.C) || g.lda % 4 || g.ldb % 4 || g.ldc % 4) return RLX_ERR_UNSUPPORTED;
  if (g.splits > 1 && g.kchunk % BK) return RLX_ERR_UNSUPPORTED;
  if (batch > 1) {
    // A batch stride must be a pure row offset or a pure column offset of the operand's 2-D tensor to become a TMA coordinate.
    // Otherwise (e.g. parameter blocks of different nets that are not a whole number of rows apart) run the nets one by one.
    auto expressible = [](long long off, int ld) { return off == 0 || off % ld == 0 || off < ld; };
    if (!expressible(g.sA, g.lda) || !expressible(g.sB, g.ldb)) {
      if (g.sA % 4 || g.sB % 4 || g.sC % 4 || g.sAux % 4) return RLX_ERR_UNSUPPORTED;
      for (int b = 0; b < batch; ++b) {
        GemmP gb = g;
        gb.A = g.A + b * g.sA; gb.B = g.B + b * g.sB; gb.C = g.C + b * g.sC;
        if (g.bias) gb.bias = g.bias + b * g.sBias;
        if (g.aux) gb.aux = g.aux + b * g.sAux;
        gb.sA = gb.sB = gb.sC = gb.sBias = gb.sAux = 0;
        const long long ar = a_rows, br = b_kmaj ? (long long)g.N : (long long)g.K;
        const int rc = tc_gemm_t(gb, a_kmaj, b_kmaj, epi, 1, kclass, ar, br, n_main, extra_col ? extra_col + b * extra_batch_off : nullptr, 0, extra_split_off, stream,
                                 transpose_out, m_main);
        if (rc) return rc;
      }
      return RLX_OK;
    }
  }
  TcParams p{};
  p.M = g.M; p.N = g.N; p.K = g.K;
  p.batch = batch; p.splits = g.splits;
  p.kchunk = (g.splits > 1) ? g.kchunk : (int)(ceil_div(g.K, BK) * BK);
  // batch offsets -> TMA coordinates
  auto split_off = [](long long off, int ld, bool kmaj, int& mn_off, int& k_off) {
    const long long r = off / ld, c = off % ld;
    if (kmaj) { mn_off = (int)r; k_off = (int)c; } else { k_off = (int)r; mn_off = (int)c; }
  };
  split_off(g.sA, g.lda, a_kmaj, p.a_mn_off, p.a_k_off);
  split_off(g.sB, g.ldb, b_kmaj, p.b_mn_off, p.b_k_off);
  p.C = g.C; p.ldc = g.ldc; p.c_batch_off = g.sC; p.c_split_off = g.sSplitC;
  p.n_main = n_main > 0 ? n_main : g.N;
  p.transpose_out = transpose_out;
  p.m_main = (transpose_out && m_main > 0) ? m_main : g.M;
  p.extra_col = extra_col; p.extra_batch_off = extra_batch_off; p.extra_split_off = extra_split_off;
  p.bias = g.bias; p.bias_batch_off = g.sBias;
  p.aux = g.aux; p.ldaux = g.ldaux; p.aux_batch_off = g.sAux;
  p.single = g.bf16 ? 1 : 0;
  p.bf16 = g.bf16;
  // global tensors: K-major [mn_rows, k_cols]; MN-major [k_rows, mn_cols].  a_rows / b_rows are the VALID rows of one batch entry
  // (TMA zero-fills beyond them); batch entries that sit at row offsets extend the tensor accordingly.
  TcOperand A{g.A, (a_kmaj ? (long long)p.a_mn_off : (long long)p.a_k_off) * (batch - 1) + a_rows,
              a_kmaj ? (long long)(p.a_k_off * (batch - 1) + g.K) : (long long)(p.a_mn_off * (batch - 1) + g.M), g.lda};
  TcOperand B{g.B, (b_kmaj ? (long long)p.b_mn_off : (long long)p.b_k_off) * (batch - 1) + b_rows,
              b_kmaj ? (long long)(p.b_k_off * (batch - 1) + g.K) : (long long)(p.b_mn_off * (batch - 1) + g.N), g.ldb};
  if (p.bf16 && a_kmaj && b_kmaj && epi == TC_EPI_BIAS_TANH) return launch_cfg<true, true, TC_EPI_BIAS_TANH, true>(A, B, p, kclass, stream);
  if (p.bf16 && a_kmaj && !b_kmaj && epi == TC_EPI_DTANH) return launch_cfg<true, false, TC_EPI_DTANH, true>(A, B, p, kclass, stream);
  if (p.bf16 && !a_kmaj && !b_kmaj && epi == TC_EPI_NONE) return launch_cfg<false, false, TC_EPI_NONE, true>(A, B, p, kclass, stream);
  if (p.bf16) return RLX_ERR_UNSUPPORTED;
  if (a_kmaj && b_kmaj && epi == TC_EPI_BIAS_TANH) return launch_cfg<true, true, TC_EPI_BIAS_TANH>(A, B, p, kclass, stream);
  if (a_kmaj && b_kmaj && epi == TC_EPI_NONE) return launch_cfg<true, true, TC_EPI_NONE>(A, B, p, kclass, stream);
  if (a_kmaj && b_kmaj && epi == TC_EPI_BIAS_RELU) return launch_cfg<true, true, TC_EPI_BIAS_RELU>(A, B, p, kclass, stream);
  if (a_kmaj && b_kmaj && epi == TC_EPI_BIAS) return launch_cfg<true, true, TC_EPI_BIAS>(A, B, p, kclass, stream);
  if (a_kmaj && !b_kmaj && epi == TC_EPI_DRELU) return launch_cfg<true, false, TC_EPI_DRELU>(A, B, p, kclass, stream);
  if (a_kmaj && !b_kmaj && epi == TC_EPI_DTANH) return launch_cfg<true, false, TC_EPI_DTANH>(A, B, p, kclass, stream);
  if (a_kmaj && !b_kmaj && epi == TC_EPI_NONE) return launch_cfg<true, false, TC_EPI_NONE>(A, B, p, kclass, stream);
  if (!a_kmaj && !b_kmaj && epi == TC_EPI_NONE) return launch_cfg<false, false, TC_EPI_NONE>(A, B, p, kclass, stream);
  return RLX_ERR_UNSUPPORTED;
}

}  // namespace rlx
