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
//   warpgroup 0   thread 0 issues cp.async.bulk.tensor 2-D tiles (SWIZZLE_128B) of raw fp32 A and B into a 3-stage ring; all 128 threads
//                 then write the hi and lo tiles of B, K-major and 128-byte swizzled (the only shared-memory layout wgmma accepts for
//                 tf32), into a 4-stage operand ring and fence.proxy.async it for the tensor core
//   warpgroups 1, 2   rows 0-63 / 64-127 of the tile: read their A fragments straight from the raw stage, split them into hi / lo in
//                 registers, and issue wgmma.mma_async m64n128k8 tf32 with A from registers (3 per k-slice of 8), keeping one half k-block
//                 of MMAs in flight while the next half's fragments are loaded; then the epilogue straight from the accumulator registers: bias+tanh / tanh' /
//                 relu / plain, stores to C (or C^T)
// A raw slot is refilled once the converter has used its B and all 8 consumer warps hold its A in registers; an operand slot once the
// wgmmas that read it have retired.
// Pre-split instances (SPLIT_B: B is a weight matrix whose tf32 hi / lo copies tf32_split made in global memory, K-major): thread 0
// TMA-loads A, hi B and lo B into one stage [A | hi B | lo B] of a 4-stage ring, which is exactly the layout the converter would have
// written; warpgroup 0 does no conversion, and a stage is refilled once the wgmmas that read it have retired.
// Operand layouts in global memory: K-major (row = m or n, 32 consecutive k = one 128-byte swizzle row) or MN-major (row = k, 32
// consecutive m/n per 128-byte row; used by the weight-gradient GEMMs whose reduction runs over the minibatch rows).  The converter
// transposes MN-major B tiles to K-major; the consumers' fragment reads transpose MN-major A.  Out-of-bounds parts of a box are
// zero-filled by TMA, so M / N / K tails need no special code in the main loop.
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
  static constexpr int OP_BYTES = 2 * B_BYTES;                  // operand stage: [hi B | lo B], K-major swizzled
  // the consumers hold up to two operand slots (the k-block being issued and the one retiring), so 4 stages let the converter run two ahead
  static constexpr int RAW_STAGES = 3, OP_STAGES = 4;
  static constexpr int SMEM_BYTES = RAW_STAGES * RAW_BYTES + OP_STAGES * OP_BYTES + 1024 /*barriers*/ + 1024 /*alignment slack*/;
  // pre-split B: stage [A | hi B | lo B]; the consumers hold up to two stages, so 4 stages let the TMA run two ahead
  static constexpr int SPLIT_STAGE_BYTES = A_BYTES + 2 * B_BYTES;  // 48 KB
  static constexpr int SPLIT_STAGES = 4;
  static constexpr int SPLIT_SMEM_BYTES = SPLIT_STAGES * SPLIT_STAGE_BYTES + 1024 + 1024;
  // consumers: 2 x 64 accumulators + 2 half k-blocks x 16 A-fragment registers
  static constexpr int PRODUCER_REGS = 56, CONSUMER_REGS = 224;
};
static_assert(Cfg::SMEM_BYTES <= 227 * 1024 && Cfg::SPLIT_SMEM_BYTES <= 227 * 1024, "shared memory of one H100 block");
static_assert(Cfg::PRODUCER_REGS * 128 + Cfg::CONSUMER_REGS * 256 <= 65536, "register file of one SM");

// One B tile (ROWS x BK) from its raw stage to K-major swizzled hi / lo tiles.  In the 128-byte swizzle every 16-byte chunk
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

// A fragments of one half k-block (k-slices 2 half, 2 half + 1) for one consumer thread, from the raw stage, split into hi / lo (the
// same split as convert_tile).  The thread holds rows r0 and r0 + 8 (r0 = row within the tile, r0 % 8 = lane / 4) at
// k = lane % 4 + 4 j, j = 4 half + jj: k-slice of the half jj / 2, fragment register 2 (jj & 1) + row (see wgmma_tf32_m64n128k8).
template <bool KMAJ, bool BF16>
__device__ __forceinline__ void load_a_frags(const uint8_t* raw, int r0, int lane, int half, uint32_t (&hi)[2][4], uint32_t (&lo)[2][4]) {
  constexpr uint32_t HI = 0xFFFFE000u;
  const int t4 = lane & 3;
  uint32_t v[2][4];
  if (KMAJ) {
    // row r is one 128-byte swizzle row; chunk j sits at (j ^ (r & 7)): the 8 row groups of a warp hit 8 different chunks, no conflicts
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const uint8_t* row = raw + (r0 + 8 * r) * 128 + t4 * 4;
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) v[r][jj] = *reinterpret_cast<const uint32_t*>(row + (((4 * half + jj) ^ (r0 & 7)) << 4));
    }
  } else {
    // BM / 32 boxes of [BK k-rows][32 m]: element (m, k) at box m / 32, k * 128 + ((((m & 31) >> 2) ^ (k & 7)) << 4) + (m & 3) * 4.
    // Lanes 16-31 read the pair partner j ^ 1 first: without that, lanes l and l ^ 17 hit the same bank (2-way conflicts).
    const int s = (lane >> 4) & 1;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int m = r0 + 8 * r;
      const uint8_t* box = raw + (m >> 5) * (BK * 128) + (m & 3) * 4;
      const int mc = (m & 31) >> 2;
#pragma unroll
      for (int jj = 0; jj < 4; jj += 2) {
        const int j = 4 * half + jj;
        const int k0 = t4 + 4 * (j + s), k1 = t4 + 4 * (j + 1 - s);
        const uint32_t x0 = *reinterpret_cast<const uint32_t*>(box + k0 * 128 + ((mc ^ (k0 & 7)) << 4));
        const uint32_t x1 = *reinterpret_cast<const uint32_t*>(box + k1 * 128 + ((mc ^ (k1 & 7)) << 4));
        v[r][jj] = s ? x1 : x0;
        v[r][jj + 1] = s ? x0 : x1;
      }
    }
  }
#pragma unroll
  for (int r = 0; r < 2; ++r)
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const uint32_t h = v[r][jj] & HI;
      hi[jj >> 1][2 * (jj & 1) + r] = h;
      if (!BF16) lo[jj >> 1][2 * (jj & 1) + r] = __float_as_uint(__uint_as_float(v[r][jj]) - __uint_as_float(h));
    }
}

// ---- epilogue.  Accumulator layout of wgmma m64nN f32: register j of lane l in warp w (of the warpgroup) holds row
// 16 w + l / 4 + 8 ((j >> 1) & 1), column 8 (j >> 2) + 2 (l & 3) + (j & 1).  So a thread owns two rows (row half h = (j >> 1) & 1) and in
// each the 16 column pairs c = j >> 2; registers 4 c + 2 h and 4 c + 2 h + 1 are the adjacent columns of one pair.

// Epilogue operands (bias, or aux of one row) of a thread's column pairs c0 .. c0 + 7: v[2 c + e] = src[8 c + e].  FULL: the tile lies inside
// the matrix.  Otherwise a column past the last valid one (offset lim) is not loaded: predicated loads, no branch, and the values of those
// columns are never stored.
template <bool FULL>
__device__ __forceinline__ void load_cols(float (&v)[32], const float* src, int lim, int c0) {
#pragma unroll
  for (int i = 2 * c0; i < 2 * c0 + 16; ++i) {
    const int o = 8 * (i >> 1) + (i & 1);
    v[i] = (FULL || o <= lim) ? src[o] : 0.f;
  }
}

template <int EPI, bool BF16>
__device__ __forceinline__ float epilogue_op(float x, float e) {
  if (EPI == TC_EPI_DTANH || EPI == TC_EPI_DRELU)
    // bf16 mode: linear-backward output rounded to bf16, then tanh_backward rounded to bf16
    x = (EPI == TC_EPI_DTANH) ? bf16r_if(bf16r_if(x, BF16) * (1.f - e * e), BF16) : ((e > 0.f) ? x : 0.f);
  if (EPI == TC_EPI_BIAS_TANH || EPI == TC_EPI_BIAS_RELU || EPI == TC_EPI_BIAS) {
    const float z = (EPI == TC_EPI_BIAS_RELU) ? x + e : bf16r_if(x + e, BF16);  // bf16 mode: Linear output is a bf16 tensor
    x = (EPI == TC_EPI_BIAS_TANH) ? bf16r_if(tanh_fast(z), BF16) : ((EPI == TC_EPI_BIAS_RELU) ? fmaxf(z, 0.f) : z);
  }
  return x;
}

// acc, cor: main and correction accumulators (the accumulator registers are only read here: a write to them would make ptxas serialise
// the next tile's wgmmas).  e[h]: the epilogue operand of row half h (the same bias for both); with aux, the thread's 64 values go in four
// chunks of 8 column pairs, and load_aux(q) issues chunk q + 1 before chunk q is used (chunk 0 is loaded before the MMAs drain): the
// consumers have no register room for more.  m: global row of row half 0; ct: global column of pair 0.  FULL: every element of the tile
// is stored, so no bounds tests.
template <int EPI, bool BF16, bool TRANS, bool FULL, class LoadAux>
__device__ __forceinline__ void store_tile(const float (&acc)[64], const float (&cor)[64], float (&e)[2][32], const TcParams& p, float* cbase,
                                           float* ebase, int m, int ct, LoadAux load_aux) {
  auto x = [&](int j) { return BF16 ? acc[j] : acc[j] + cor[j]; };  // main + correction (fp32 RN)
  constexpr bool HAS_AUX = (EPI == TC_EPI_DTANH || EPI == TC_EPI_DRELU);
  if (!TRANS) {
    // one 8-byte store per column pair: a warp instruction writes 8 whole 32-byte sectors
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int mh = m + 8 * h;
      float* row = cbase + (long long)mh * p.ldc + ct;
      const bool row_ok = FULL || mh < p.M;
#pragma unroll
      for (int c = 0; c < 16; ++c) {
        if (HAS_AUX && c % 8 == 0 && 2 * h + c / 8 < 3) load_aux(2 * h + c / 8 + 1);
        const int j = 4 * c + 2 * h;
        const float x0 = epilogue_op<EPI, BF16>(x(j), e[HAS_AUX ? h : 0][2 * c]);
        const float x1 = epilogue_op<EPI, BF16>(x(j + 1), e[HAS_AUX ? h : 0][2 * c + 1]);
        const int n = ct + 8 * c;
        if (FULL || (row_ok && n + 1 < p.N)) *reinterpret_cast<float2*>(row + 8 * c) = make_float2(x0, x1);
        else if (row_ok && n < p.N) row[8 * c] = x0;
      }
    }
  } else {
    // C^T: element (m, n) at C[n * ldc + m]; scalar stores, each warp instruction fills 4 sectors (8 rows of 4 consecutive m)
    float* col = cbase + (long long)ct * p.ldc + m;
    const int ldc = (int)p.ldc;
#pragma unroll
    for (int c = 0; c < 16; ++c)
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int off = (8 * c + q) * ldc;
        const int n = ct + 8 * c + q;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float v = x(4 * c + 2 * h + q);
          const int mh = m + 8 * h;
          if (FULL || (n < p.N && mh < p.m_main)) col[off + 8 * h] = v;
          else if (n < p.N && mh == p.m_main && mh < p.M && ebase != nullptr) ebase[n] = v;
        }
      }
  }
}

// BF16: the bf16-autocast variant (single-pass MMAs on bf16-valued operands, bf16 roundings in the epilogue), a compile-time switch so that
// the fp32-equivalent kernels carry none of it.  TRANS: store C^T (the transposed dW1 | db1 GEMM), an instance of its own.  SPLIT_B: B
// arrives pre-split (tmap_b = hi, tmap_b_lo = lo, both K-major); the other instances do not read tmap_b_lo.
template <bool A_KMAJ, bool B_KMAJ, int EPI, bool BF16, bool TRANS, bool SPLIT_B>
__global__ void __launch_bounds__(NUM_THREADS, 1) tc_gemm_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                                                                 const __grid_constant__ CUtensorMap tmap_b_lo, const TcParams p) {
  static_assert(!SPLIT_B || (B_KMAJ && !BF16), "pre-split B is K-major fp32 hi / lo");
  // SPLIT_B: one ring; a raw stage is the whole stage [A | hi B | lo B], raw_full / op_empty are its full / empty barriers (rs == os)
  constexpr int RAW_STAGES = SPLIT_B ? Cfg::SPLIT_STAGES : Cfg::RAW_STAGES, OP_STAGES = SPLIT_B ? Cfg::SPLIT_STAGES : Cfg::OP_STAGES;
  constexpr int RAW_BYTES = SPLIT_B ? Cfg::SPLIT_STAGE_BYTES : Cfg::RAW_BYTES;
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment (swizzle atoms) as an OFFSET on the __shared__ pointer: a round trip through uintptr_t makes the compiler lose
  // the shared address space and emit generic loads / stores
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* ops = smem + RAW_STAGES * RAW_BYTES;
  uint64_t* raw_full = reinterpret_cast<uint64_t*>(ops + (SPLIT_B ? 0 : OP_STAGES * Cfg::OP_BYTES));  // [RAW_STAGES]  TMA landed
  uint64_t* raw_empty = raw_full + RAW_STAGES;                                        // [RAW_STAGES]  B converted, A in registers
  uint64_t* op_full = raw_empty + RAW_STAGES;                                         // [OP_STAGES]   hi / lo B tiles written
  uint64_t* op_empty = op_full + OP_STAGES;                                           // [OP_STAGES]   wgmmas of the slot retired

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_a);
    prefetch_tmap(&tmap_b);
    if (SPLIT_B) prefetch_tmap(&tmap_b_lo);
    for (int s = 0; s < RAW_STAGES; ++s) {
      mbar_init(&raw_full[s], 1);
      mbar_init(&raw_empty[s], 1 + 8);  // the converter + one arrival per consumer warp
    }
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
    // ===================================================== TMA (thread 0) + B hi / lo converter (warpgroup 0)
    setmaxnreg_dec<Cfg::PRODUCER_REGS>();
    const int t = threadIdx.x;
    // load cursor: the k-blocks of this CTA's tiles in consumption order; a raw slot is refilled once its raw_empty phase completes
    // (SPLIT_B: once its op_empty phase completes).  Returns false past the last k-block.
    uint64_t* ld_empty = SPLIT_B ? op_empty : raw_empty;
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
        mbar_wait(&ld_empty[slot], ((ld_count / RAW_STAGES) & 1) ^ 1);  // the first round passes: a fresh barrier's previous phase
        uint8_t* sa = smem + slot * RAW_BYTES;
        uint8_t* sb = sa + Cfg::A_BYTES;
        uint64_t* bar = &raw_full[slot];
        const int k0 = kbeg + ld_kb * BK;
        mbar_arrive_expect_tx(bar, RAW_BYTES);
        if (A_KMAJ) {
          tma_load_2d(&tmap_a, bar, sa, p.a_k_off * zb + k0, p.a_mn_off * zb + m0);
        } else {
#pragma unroll
          for (int j = 0; j < BM / 32; ++j) tma_load_2d(&tmap_a, bar, sa + j * (BK * 128), p.a_mn_off * zb + m0 + 32 * j, p.a_k_off * zb + k0);
        }
        if (B_KMAJ) {
          tma_load_2d(&tmap_b, bar, sb, p.b_k_off * zb + k0, p.b_mn_off * zb + n0);
          if (SPLIT_B) tma_load_2d(&tmap_b_lo, bar, sb + Cfg::B_BYTES, p.b_k_off * zb + k0, p.b_mn_off * zb + n0);
        } else {
#pragma unroll
          for (int j = 0; j < BN / 32; ++j) tma_load_2d(&tmap_b, bar, sb + j * (BK * 128), p.b_mn_off * zb + n0 + 32 * j, p.b_k_off * zb + k0);
        }
        ++ld_kb;
        ++ld_count;
        return true;
      }
      return false;
    };
    if constexpr (SPLIT_B) {
      // nothing to convert: thread 0 streams the k-blocks through the ring, the rest of the warpgroup is done
      if (t == 0)
        while (load_next()) {
        }
      return;
    }
    if (t == 0)
      for (int i = 0; i < RAW_STAGES; ++i) load_next();
    int rs = 0, os = 0;
    uint32_t rph = 0, oph = 0;
    bool refill = false;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int zb, zs, m0, n0, kbeg, nkb;
      tile_coords(tile, zb, zs, m0, n0, kbeg, nkb);
      for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait(&raw_full[rs], rph);
        mbar_wait(&op_empty[os], oph ^ 1);
        uint8_t* op = ops + os * Cfg::OP_BYTES;
        convert_tile<B_KMAJ, BF16, BN>(smem + rs * Cfg::RAW_BYTES + Cfg::A_BYTES, op, op + Cfg::B_BYTES, t);
        fence_proxy_async();  // generic-proxy writes -> visible to the tensor core's async-proxy reads
        named_bar_sync(1, 128);  // the whole warpgroup is done with raw slot rs and has written operand slot os
        if (t == 0) {
          mbar_arrive(&op_full[os]);
          mbar_arrive(&raw_empty[rs]);
          // refill the PREVIOUS k-block's raw slot: the consumers have usually taken its A by now, so this rarely waits, and the TMA
          // still runs RAW_STAGES - 1 k-blocks ahead of the converter
          if (refill) load_next();
          refill = true;
        }
        if (++rs == RAW_STAGES) { rs = 0; rph ^= 1; }
        if (++os == OP_STAGES) { os = 0; oph ^= 1; }
      }
    }
  } else {
    // ===================================================== wgmma consumers + epilogue (warpgroups 1, 2)
    setmaxnreg_inc<Cfg::CONSUMER_REGS>();
    const int cw = (warp >> 2) - 1;  // rows 64 * cw .. 64 * cw + 63 of the tile
    const int r0 = cw * 64 + (warp & 3) * 16 + (lane >> 2);
    float acc[64], cor[64];
    // A fragments of the two half k-blocks that can be in flight: [half][k-slice of the half][register].  Each half is one commit group
    // with registers of its own: a register operand must keep its value until its wgmma retires.
    uint32_t ah[2][2][4], al[2][2][4];
    int rs = 0, os = 0;
    uint32_t rph = 0, oph = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int zb, zs, m0, n0, kbeg, nkb;
      tile_coords(tile, zb, zs, m0, n0, kbeg, nkb);
      for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait(&raw_full[rs], rph);
        if (!SPLIT_B) mbar_wait(&op_full[os], oph);
        const uint8_t* raw = smem + rs * RAW_BYTES;
        const uint32_t op = SPLIT_B ? smem_u32(raw + Cfg::A_BYTES) : smem_u32(ops + os * Cfg::OP_BYTES);
        const uint64_t db = make_smem_desc(op), db_lo = make_smem_desc(op + Cfg::B_BYTES);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          load_a_frags<A_KMAJ, BF16>(raw, r0, lane, h, ah[h], al[h]);
          if (!SPLIT_B && h == 1) {
            __syncwarp();
            if (lane == 0) mbar_arrive(&raw_empty[rs]);  // this warp holds all of the k-block's A
          }
          fence_frags(ah[h]);
          if (!BF16) fence_frags(al[h]);
          wgmma_fence();  // orders the A-fragment register writes before the wgmmas that read them
#pragma unroll
          for (int q = 0; q < 2; ++q) {
            const int kk = 2 * h + q;
            // advancing along k inside the 128-byte swizzle row: the descriptors differ only in the start address (units of 16 bytes)
            const uint64_t ko = (uint64_t)((kk * WG_K * 4) >> 4);
            const uint32_t accum = (kb | kk) != 0 ? 1u : 0u;
            if (!BF16) {
              wgmma_tf32_m64n128k8(cor, al[h][q], db + ko, accum);  // lo * hi   } small terms, own accumulator
              wgmma_tf32_m64n128k8(cor, ah[h][q], db_lo + ko, 1u);  // hi * lo   }
            }
            wgmma_tf32_m64n128k8(acc, ah[h][q], db + ko, accum);    // hi * hi  (bf16-valued operands: the whole product)
          }
          wgmma_commit();
          // the previous half has retired: its A registers may be rewritten, and after the first half the previous k-block's operand
          // slot is free
          wgmma_wait_1();
          if (h == 0 && kb > 0 && lane == 0) mbar_arrive(&op_empty[os == 0 ? OP_STAGES - 1 : os - 1]);
        }
        if (++rs == RAW_STAGES) { rs = 0; rph ^= 1; }
        if (++os == OP_STAGES) { os = 0; oph ^= 1; }
      }

      // ---- epilogue (layout above).  Its first operands (the bias, or the first aux chunk) are loaded while the last half k-block's MMAs
      // run, into registers the retired half's A fragments left free.
      constexpr bool HAS_AUX = (EPI == TC_EPI_DTANH || EPI == TC_EPI_DRELU);
      constexpr bool HAS_BIAS = (EPI == TC_EPI_BIAS_TANH || EPI == TC_EPI_BIAS_RELU || EPI == TC_EPI_BIAS);
      const int m = m0 + r0, ct = n0 + 2 * (lane & 3);
      const bool full = m0 + BM <= (TRANS ? p.m_main : p.M) && n0 + BN <= p.N;  // one test per tile
      const int clim = p.N - 1 - ct;
      const float* abase = HAS_AUX ? p.aux + p.aux_batch_off * zb + ct : nullptr;
      float e[2][32];
      // aux chunk q: row half q / 2, column pairs 8 (q % 2) .. + 7
      auto load_aux = [&](int q) {
        const float* arow = abase + (long long)min(m + 8 * (q >> 1), p.M - 1) * p.ldaux;
        if (full) load_cols<true>(e[q >> 1], arow, clim, 8 * (q & 1));
        else load_cols<false>(e[q >> 1], arow, clim, 8 * (q & 1));
      };
      if (HAS_BIAS) {
        const float* b = p.bias + p.bias_batch_off * zb + ct;
#pragma unroll
        for (int c0 = 0; c0 < 16; c0 += 8) {
          if (full) load_cols<true>(e[0], b, clim, c0);
          else load_cols<false>(e[0], b, clim, c0);
        }
      }
      if (HAS_AUX) load_aux(0);
      if (nkb > 0) {
        wgmma_wait_all();
        if (lane == 0) mbar_arrive(&op_empty[os == 0 ? OP_STAGES - 1 : os - 1]);
      }
      fence_acc(acc);
      if (!BF16) fence_acc(cor);
      float* cbase = p.C + p.c_batch_off * zb + p.c_split_off * zs;
      float* ebase = (TRANS && p.extra_row != nullptr) ? p.extra_row + p.extra_batch_off * zb + p.extra_split_off * zs : nullptr;
      if (full) store_tile<EPI, BF16, TRANS, true>(acc, cor, e, p, cbase, ebase, m, ct, load_aux);
      else store_tile<EPI, BF16, TRANS, false>(acc, cor, e, p, cbase, ebase, m, ct, load_aux);
    }
  }
}

// ------------------------------------------------------------------------------------------------ host side
// SPLIT_B: B.base is the hi copy, b_lo the lo copy (same extents and pitch)
template <bool A_KMAJ, bool B_KMAJ, int EPI, bool BF16 = false, bool TRANS = false, bool SPLIT_B = false>
static int launch_cfg(const TcOperand& A, const TcOperand& B, TcParams p, int kclass, cudaStream_t stream, const float* b_lo = nullptr) {
  CUtensorMap ta, tb, tb_lo;
  int rc = make_tmap(&ta, A.base, A.rows, A.cols, A.ld, 32, A_KMAJ ? BM : BK);
  if (rc) return rc;
  rc = make_tmap(&tb, B.base, B.rows, B.cols, B.ld, 32, B_KMAJ ? BN : BK);
  if (rc) return rc;
  if (SPLIT_B) {
    rc = make_tmap(&tb_lo, b_lo, B.rows, B.cols, B.ld, 32, BN);
    if (rc) return rc;
  } else {
    tb_lo = tb;  // not read
  }
  p.tiles_m = (int)ceil_div(p.M, BM);
  p.tiles_n = (int)ceil_div(p.N, BN);
  const long long tiles = (long long)p.tiles_m * p.tiles_n * p.batch * p.splits;
  if (tiles <= 0) return RLX_OK;
  static_assert(!TRANS || EPI == TC_EPI_NONE, "the transposed store has no epilogue function");
  auto kern = tc_gemm_kernel<A_KMAJ, B_KMAJ, EPI, BF16, TRANS, SPLIT_B>;
  constexpr int smem = SPLIT_B ? Cfg::SPLIT_SMEM_BYTES : Cfg::SMEM_BYTES;
  static bool attr_done = false;
  if (!attr_done) {
    RLX_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr_done = true;
  }
  const unsigned grid = (unsigned)std::min<long long>(tiles, sm_count());
  const double flops = 2.0 * p.M * p.N * (double)p.K * p.batch;
  const double bytes = 4.0 * p.batch * ((double)p.M * p.K + (SPLIT_B ? 2.0 : 1.0) * p.N * p.K + (double)p.M * p.N * p.splits);
  RLX_LAUNCH_C(kclass, flops, bytes, kern, grid, NUM_THREADS, smem, stream, ta, tb, tb_lo, p);
  count_gemm_path(tc_path_slot(A_KMAJ, B_KMAJ, EPI, BF16, TRANS, SPLIT_B));
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
// 16-byte aligned bases, batch strides that are pure row or column offsets of the operand tensors, and (for the pairwise stores of C) even
// batch and split offsets of C.  trans: the transposed store (tc_gemm_t).
static int tc_gemm_impl(const GemmP& g, bool a_kmaj, bool b_kmaj, int epi, int batch, int kclass, long long a_rows, long long b_rows, bool trans,
                        int m_main, float* extra_row, long long extra_batch_off, long long extra_split_off, cudaStream_t stream) {
  if (g.M <= 0 || g.N <= 0) return RLX_OK;
  // pre-split B (g.b_hi / g.b_lo, K-major [N, K] per batch entry): the instances that exist take it, the rest read g.B through the converter
  const bool split_b = g.b_hi != nullptr && !g.bf16 && !trans && a_kmaj && (epi == TC_EPI_BIAS_TANH || epi == TC_EPI_DTANH);
  if (split_b) {
    if (!aligned16(g.b_hi) || !aligned16(g.b_lo)) return RLX_ERR_UNSUPPORTED;
    b_kmaj = true;
    b_rows = g.N;
  }
  if (!aligned16(g.A) || !aligned16(g.B) || !aligned16(g.C) || g.lda % 4 || g.ldb % 4 || g.ldc % 4) return RLX_ERR_UNSUPPORTED;
  if (g.splits > 1 && g.kchunk % BK) return RLX_ERR_UNSUPPORTED;
  if (!trans && (((batch > 1 ? g.sC : 0) | (g.splits > 1 ? g.sSplitC : 0)) & 1)) return RLX_ERR_UNSUPPORTED;
  if (batch > 1) {
    // A batch stride must be a pure row offset or a pure column offset of the operand's 2-D tensor to become a TMA coordinate.
    // Otherwise (e.g. parameter blocks of different nets that are not a whole number of rows apart) run the nets one by one.
    auto expressible = [](long long off, int ld) { return off == 0 || off % ld == 0 || off < ld; };
    if (!expressible(g.sA, g.lda) || !expressible(g.sB, g.ldb)) {
      if (g.sA % 4 || g.sB % 4 || g.sC % 4 || g.sAux % 4) return RLX_ERR_UNSUPPORTED;
      for (int b = 0; b < batch; ++b) {
        GemmP gb = g;
        gb.A = g.A + b * g.sA; gb.B = g.B + b * g.sB; gb.C = g.C + b * g.sC;
        if (g.b_hi) { gb.b_hi = g.b_hi + b * g.sB; gb.b_lo = g.b_lo + b * g.sB; }
        if (g.bias) gb.bias = g.bias + b * g.sBias;
        if (g.aux) gb.aux = g.aux + b * g.sAux;
        gb.sA = gb.sB = gb.sC = gb.sBias = gb.sAux = 0;
        const long long ar = a_rows, br = b_kmaj ? (long long)g.N : (long long)g.K;
        const int rc = tc_gemm_impl(gb, a_kmaj, b_kmaj, epi, 1, kclass, ar, br, trans, m_main, extra_row ? extra_row + b * extra_batch_off : nullptr, 0,
                                    extra_split_off, stream);
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
  p.m_main = (trans && m_main > 0) ? m_main : g.M;
  p.extra_row = extra_row; p.extra_batch_off = extra_batch_off; p.extra_split_off = extra_split_off;
  p.bias = g.bias; p.bias_batch_off = g.sBias;
  p.aux = g.aux; p.ldaux = g.ldaux; p.aux_batch_off = g.sAux;
  p.single = g.bf16 ? 1 : 0;
  p.bf16 = g.bf16;
  // global tensors: K-major [mn_rows, k_cols]; MN-major [k_rows, mn_cols].  a_rows / b_rows are the VALID rows of one batch entry
  // (TMA zero-fills beyond them); batch entries that sit at row offsets extend the tensor accordingly.
  TcOperand A{g.A, (a_kmaj ? (long long)p.a_mn_off : (long long)p.a_k_off) * (batch - 1) + a_rows,
              a_kmaj ? (long long)(p.a_k_off * (batch - 1) + g.K) : (long long)(p.a_mn_off * (batch - 1) + g.M), g.lda};
  TcOperand B{split_b ? g.b_hi : g.B, (b_kmaj ? (long long)p.b_mn_off : (long long)p.b_k_off) * (batch - 1) + b_rows,
              b_kmaj ? (long long)(p.b_k_off * (batch - 1) + g.K) : (long long)(p.b_mn_off * (batch - 1) + g.N), g.ldb};
  if (trans) {
    if (!a_kmaj && !b_kmaj && epi == TC_EPI_NONE)
      return p.bf16 ? launch_cfg<false, false, TC_EPI_NONE, true, true>(A, B, p, kclass, stream)
                    : launch_cfg<false, false, TC_EPI_NONE, false, true>(A, B, p, kclass, stream);
    return RLX_ERR_UNSUPPORTED;
  }
  if (p.bf16 && a_kmaj && b_kmaj && epi == TC_EPI_BIAS_TANH) return launch_cfg<true, true, TC_EPI_BIAS_TANH, true>(A, B, p, kclass, stream);
  if (p.bf16 && a_kmaj && !b_kmaj && epi == TC_EPI_DTANH) return launch_cfg<true, false, TC_EPI_DTANH, true>(A, B, p, kclass, stream);
  if (p.bf16 && !a_kmaj && !b_kmaj && epi == TC_EPI_NONE) return launch_cfg<false, false, TC_EPI_NONE, true>(A, B, p, kclass, stream);
  if (p.bf16) return RLX_ERR_UNSUPPORTED;
  if (split_b && epi == TC_EPI_BIAS_TANH) return launch_cfg<true, true, TC_EPI_BIAS_TANH, false, false, true>(A, B, p, kclass, stream, g.b_lo);
  if (split_b && epi == TC_EPI_DTANH) return launch_cfg<true, true, TC_EPI_DTANH, false, false, true>(A, B, p, kclass, stream, g.b_lo);
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

int tc_gemm(const GemmP& g, bool a_kmaj, bool b_kmaj, int epi, int batch, int kclass, long long a_rows, long long b_rows, cudaStream_t stream) {
  return tc_gemm_impl(g, a_kmaj, b_kmaj, epi, batch, kclass, a_rows, b_rows, false, 0, nullptr, 0, 0, stream);
}

int tc_gemm_t(const GemmP& g, bool a_kmaj, bool b_kmaj, int epi, int batch, int kclass, long long a_rows, long long b_rows, int m_main, float* extra_row,
              long long extra_batch_off, long long extra_split_off, cudaStream_t stream) {
  return tc_gemm_impl(g, a_kmaj, b_kmaj, epi, batch, kclass, a_rows, b_rows, true, m_main, extra_row, extra_batch_off, extra_split_off, stream);
}

// ------------------------------------------------------------------------------------------------ tf32 hi / lo split
namespace tc {
struct Tf32SplitJobs {
  Tf32SplitJob job[kMaxTf32SplitJobs];
  int first_tile[kMaxTf32SplitJobs + 1];  // CTA range of each job
};

// one 32 x 32 tile of one job per CTA (256 threads), through shared memory so that the transposed writes are coalesced too
__global__ void __launch_bounds__(256) tf32_split_kernel(const __grid_constant__ Tf32SplitJobs J) {
  __shared__ float tile[32][33];
  int j = 0;
  while ((int)blockIdx.x >= J.first_tile[j + 1]) ++j;
  const Tf32SplitJob& s = J.job[j];
  const int tiles_c = (s.cols + 31) / 32, tiles_rc = ((s.rows + 31) / 32) * tiles_c;
  const int b = (int)blockIdx.x - J.first_tile[j];
  const int z = b / tiles_rc, r0 = (b % tiles_rc) / tiles_c * 32, c0 = b % tiles_c * 32;
  const long long zoff = (long long)z * s.rows * s.cols;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
#pragma unroll
  for (int i = ty; i < 32; i += 8)
    if (r0 + i < s.rows && c0 + tx < s.cols) tile[i][tx] = s.src[zoff + (long long)(r0 + i) * s.cols + c0 + tx];
  __syncthreads();
#pragma unroll
  for (int i = ty; i < 32; i += 8) {
    // destination row / column and source tile element of this thread
    const int dr = s.trans ? c0 + i : r0 + i, dc = s.trans ? r0 + tx : c0 + tx, dcols = s.trans ? s.rows : s.cols;
    if (dr < (s.trans ? s.cols : s.rows) && dc < dcols) {
      const float x = s.trans ? tile[tx][i] : tile[i][tx];
      const uint32_t h = __float_as_uint(x) & 0xFFFFE000u;  // convert_tile's split
      const long long o = zoff + (long long)dr * dcols + dc;
      s.hi[o] = __uint_as_float(h);
      s.lo[o] = x - __uint_as_float(h);
    }
  }
}
}  // namespace tc

int tf32_split(const Tf32SplitJob* jobs, int njobs, int kclass, cudaStream_t stream) {
  if (njobs < 1 || njobs > kMaxTf32SplitJobs) return RLX_ERR_INVALID_ARG;
  Tf32SplitJobs J{};
  long long tiles = 0, elems = 0;
  for (int i = 0; i < njobs; ++i) {
    J.job[i] = jobs[i];
    J.first_tile[i] = (int)tiles;
    tiles += (long long)jobs[i].batch * ceil_div(jobs[i].rows, 32) * ceil_div(jobs[i].cols, 32);
    elems += (long long)jobs[i].batch * jobs[i].rows * jobs[i].cols;
  }
  for (int i = njobs; i <= kMaxTf32SplitJobs; ++i) J.first_tile[i] = (int)tiles;
  if (tiles == 0) return RLX_OK;
  RLX_LAUNCH_C(kclass, 0, 12.0 * elems, tf32_split_kernel, (unsigned)tiles, 256, 0, stream, J);
  count_gemm_path(GP_TF32_SPLIT);
  return RLX_OK;
}

}  // namespace rlx
