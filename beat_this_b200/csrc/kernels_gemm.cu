// 16-bit tensor-core GEMM for sm_90a: D = A * W^T over "planes" with shifted slabs (linear layers, the
// k(2,3) frontend convolutions as implicit GEMM, frontend.linear), wgmma with register accumulators,
// TMA (cp.async.bulk.tensor) operand staging through an mbarrier ring, persistent over output tiles,
// warp-specialised roles (one producer warp, two consumer warpgroups), fused epilogues (epilogue.cuh) staged through
// shared memory: the fp32 residual comes in by TMA during the tile's MMAs, the results go out by TMA stores.  Reference
// call sites: every nn.Linear / Conv2d of beat_this/model/roformer.py:53-61,103-111 and beat_tracker.py:77,155-166.
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "tc_common.cuh"

namespace bt {

// --------------------------------------------------------------------------- tensor maps
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                    const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_encodeTiled g_encode = nullptr;
int g_num_sms = 132;

static bool make_tmap_any(CUtensorMap* tm, CUtensorMapDataType dt, const void* base, int rank, const uint64_t* dims,
                          const uint64_t* strides_bytes /* rank-1 */, const uint32_t* box, int swizzle_bytes,
                          char* err, int errlen) {
  cuuint64_t gd[5];
  cuuint64_t gs[4];
  cuuint32_t bx[5];
  cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) { gd[i] = dims[i]; bx[i] = box[i]; es[i] = 1; }
  for (int i = 0; i < rank - 1; ++i) gs[i] = strides_bytes[i];
  CUtensorMapSwizzle sw = swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                          : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                          : swizzle_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B
                                                : CU_TENSOR_MAP_SWIZZLE_NONE;
  CUresult r = g_encode(tm, dt, rank, const_cast<void*>(base), gd, gs, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    snprintf(err, errlen, "cuTensorMapEncodeTiled failed (%d): rank %d dims %llu,%llu,%llu box %u,%u,%u stride0 %llu",
             static_cast<int>(r), rank, (unsigned long long)gd[0], (unsigned long long)(rank > 1 ? gd[1] : 0),
             (unsigned long long)(rank > 2 ? gd[2] : 0), bx[0], rank > 1 ? bx[1] : 0, rank > 2 ? bx[2] : 0,
             (unsigned long long)gs[0]);
    return false;
  }
  return true;
}
bool make_tmap(CUtensorMap* tm, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
               const uint32_t* box, int swizzle_bytes, char* err, int errlen) {
  return make_tmap_any(tm, BT_H16_IS_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, base, rank,
                       dims, strides_bytes, box, swizzle_bytes, err, errlen);
}

// =============================================================================== GEMM
// CTA = 128 output rows x BN columns, persistent over tiles (stride gridDim.x).  Warp 0 (one elected lane) streams
// the A and W k-blocks through a STAGES-deep TMA ring; warpgroups 1 and 2 own rows [0, 64) and [64, 128) of the
// tile and issue one wgmma m64nBNk16 per k16 step, keeping one k-block's MMAs in flight while the next is issued.
// At BN = 256 the producer warpgroup hands registers to the consumers (setmaxnreg 40 / 232), which is what lets the
// 128 fp32 accumulators per thread live in registers.  Narrower tiles fit the 168 registers of 384 threads and skip
// it: with it, the fp32-residual GEMMs at BN = 128 measured 10-15 % slower on H100.
//
// Epilogue of kinds 0 and 1, staged through shared memory: each warpgroup applies the epilogue arithmetic
// (epilogue.cuh) to its accumulators in place, writes the results into staging units in the 128-byte (64-byte for a
// 32-column 16-bit unit) swizzled layout of the output's tensor map, and its leader stores every unit with one TMA
// store.  A unit holds 128 rows x 128 bytes (32 fp32 or 64 16-bit columns; warpgroup w writes rows [64 w, 64 w + 64)),
// and the epilogue uses them in turn: first the BN / 32 fp32 units, then the 16-bit ones.  A unit is rewritten only
// after its last store has read it (cp.async.bulk.wait_group.read).  A GEMM that adds the fp32 residual has it loaded
// into its fp32 units by the producer while the tile's MMAs run (its own full / empty mbarrier pair); the result
// overwrites it in place, so a tile that reads and writes the same rows of X stays correct.  The 3-D output maps clip
// rows >= L of each plane.  The gates GEMM (kind 2, N = 32 into [M, heads]) stores from registers.
constexpr int TG_BM = 128;
constexpr int TG_THREADS = 384;  // warpgroup 0: producer (warp 0), warpgroups 1-2: MMA + epilogue
constexpr int TG_UNIT_BYTES = TG_BM * 128;

template <int BN, int BK>
struct TgCfg {
  static constexpr int A_BYTES = TG_BM * BK * 2;
  static constexpr int W_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + W_BYTES;
  static constexpr int ACT_COLS = BN < 64 ? BN : 64;  // columns of a 16-bit unit
  // staging units: up to BN = 128 a whole tile in fp32 and in 16 bits at once (the residual GEMMs keep their fp32
  // units for the residual); the wider tiles cycle through 4 (BN = 192) or 2 (BN = 256) of them and keep 4 stages
  static constexpr int SLOTS = BN == 256 ? 2 : BN == 192 ? 4 : BN / 32 + BN / ACT_COLS;
  static constexpr int EPI_BYTES = SLOTS * TG_UNIT_BYTES;
  static constexpr int FIXED = 1024 /*align*/ + 256 /*barriers*/;
  static constexpr int STAGES_FIT = (232448 - FIXED - EPI_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = STAGES_FIT > 6 ? 6 : STAGES_FIT;
  static constexpr int SMEM = STAGES * STAGE_BYTES + EPI_BYTES + FIXED;
  static constexpr int SWZ = BK * 2;  // 128 or 64 byte rows
  static_assert(STAGES >= 4, "pipeline too shallow");
};

// byte offset inside a staging unit of rows of RB bytes, in the layout TMA reads with CU_TENSOR_MAP_SWIZZLE_{RB}B: the
// 16-byte chunk index XOR the row (RB = 128) or the row pair (RB = 64) within each group of 1024 bytes
template <int RB>
__device__ __forceinline__ uint32_t swz(uint32_t off) {
  return off ^ (((off >> 7) & (RB / 16 - 1)) << 4);
}

template <int BN, int BK, int KIND>
__global__ void __launch_bounds__(TG_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW,
               const __grid_constant__ CUtensorMap tmR, const __grid_constant__ CUtensorMap tmF,
               const __grid_constant__ CUtensorMap tmH, const GemmShape g, const EpiParams e, int num_tiles, int t_tiles,
               int n_tiles, int m_tiles) {
  using Cfg = TgCfg<BN, BK>;
  constexpr int STAGES = Cfg::STAGES;
  constexpr int SLOTS = Cfg::SLOTS;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sA = sbase;
  const uint32_t sW = sbase + STAGES * Cfg::A_BYTES;
  const uint32_t sE = sbase + STAGES * Cfg::STAGE_BYTES;     // [SLOTS] staging units
  const uint32_t full = sE + Cfg::EPI_BYTES;                  // [STAGES] k-block landed
  const uint32_t empty = full + 8 * STAGES;                   // [STAGES] both consumer warpgroups done with it
  const uint32_t rfull = empty + 8 * STAGES;                  // the tile's residual landed
  const uint32_t rempty = rfull + 8;                          // both consumer warpgroups' stores have read it
  const bool has_resid = KIND == 0 && e.resid != nullptr;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmW);
    if (has_resid) tma_prefetch_desc(&tmR);
    if (KIND == 0 && e.out_f32) tma_prefetch_desc(&tmF);
    if (KIND != 2 && e.out_act) tma_prefetch_desc(&tmH);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(full + 8 * i, 1);
      mbar_init(empty + 8 * i, 2);
    }
    mbar_init(rfull, 1);
    mbar_init(rempty, 2);
    fence_barrier_init();
  }
  __syncthreads();

  const int kb_per_slab = g.Kslab / BK;
  const int num_kb = g.nslab * kb_per_slab;

  if (warp < 4) {
    if constexpr (BN == 256) setmaxnreg_dec<40>();
    if (warp == 0 && lane == 0) {
      // The residual of a tile is requested once its first k-blocks are queued (at most STAGES - 1 of them): its
      // buffer comes free when the consumers start the tile, and the ring stays full meanwhile.
      const int kb_resid = (num_kb < STAGES - 1 ? num_kb : STAGES - 1) - 1;
      int stage = 0;
      uint32_t phase = 0, rphase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int mt = tile / n_tiles, nt = tile % n_tiles;
        const int p_out = mt / t_tiles;
        const int t0 = (mt - p_out * t_tiles) * TG_BM;
        for (int kb = 0; kb < num_kb; ++kb) {
          const int s = kb / kb_per_slab;
          const int k0 = (kb - s * kb_per_slab) * BK;
          mbar_wait(empty + 8 * stage, phase ^ 1);
          const uint32_t fb = full + 8 * stage;
          mbar_expect_tx(fb, Cfg::STAGE_BYTES);
          // A rows outside [0, L) of the plane (conv time shifts, the last tile of a plane) arrive as zeros
          tma_load_3d(sA + stage * Cfg::A_BYTES, &tmA, fb, k0, t0 + g.t_shift[s], p_out * g.plane_mul + g.plane_add[s]);
          tma_load_2d(sW + stage * Cfg::W_BYTES, &tmW, fb, s * g.Kslab + k0, nt * BN);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
          if (has_resid && kb == kb_resid) {
            mbar_wait(rempty, rphase ^ 1);
            mbar_expect_tx(rfull, TG_BM * BN * 4);
            for (int u = 0; u < BN / 32; ++u) tma_load_3d(sE + u * TG_UNIT_BYTES, &tmR, rfull, nt * BN + 32 * u, t0, p_out);
            rphase ^= 1;
          }
        }
      }
    }
  } else {
    if constexpr (BN == 256) setmaxnreg_inc<232>();
    const int wg = (warp >> 2) - 1;   // 0: tile rows [0, 64), 1: [64, 128)
    const int wq = warp & 3;          // warp inside the warpgroup: 16 rows each
    const bool leader = (threadIdx.x & 127) == 0;
    const uint32_t a_off = static_cast<uint32_t>(wg * 64 * BK * 2);
    const int row_q = wq * 16 + (lane >> 2);  // this thread's accumulator rows row_q and row_q + 8 of the warpgroup
    const int c0 = 2 * (lane & 3);            // and columns 8 j + c0, 8 j + c0 + 1
    const uint32_t my_rows = sE + wg * (TG_UNIT_BYTES / 2);
    int stage = 0;
    uint32_t phase = 0, rphase = 0;
    float acc[BN / 2];
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int mt = tile / n_tiles, nt = tile % n_tiles;
      const int p_out = mt / t_tiles;
      const int t0 = (mt - p_out * t_tiles) * TG_BM;
      int prev = -1;  // stage of the k-block whose MMAs are still in flight
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(full + 8 * stage, phase);
        const uint32_t a_base = sA + stage * Cfg::A_BYTES + a_off;
        const uint32_t b_base = sW + stage * Cfg::W_BYTES;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k)
          wgmma_m64k16<BN>(acc, make_wgmma_desc<Cfg::SWZ>(a_base + k * 32), make_wgmma_desc<Cfg::SWZ>(b_base + k * 32),
                           (kb | k) != 0 ? 1u : 0u);
        wgmma_commit();
        if (KIND != 2 && kb == 0 && leader && tile != blockIdx.x) {
          // while the first MMAs run: the previous tile's stores have read the staging units, which frees them and
          // the residual buffer
          bulk_wait_read<0>();
          if (has_resid) mbar_arrive(rempty);
        }
        wgmma_wait<1>();  // the previous k-block's MMAs are done: its stage goes back to the producer
        if (leader && prev >= 0) mbar_arrive(empty + 8 * prev);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      if (leader) mbar_arrive(empty + 8 * prev);
      if constexpr (KIND == 2) {
        const int tr = t0 + wg * 64 + row_q;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int t = tr + 8 * h;
          if (t < g.L && mt < m_tiles) {
            const int64_t m = static_cast<int64_t>(p_out) * g.L + t;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j)
              epi_gates_pair(e, m, nt * BN + 8 * j + c0, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
          }
        }
        continue;
      } else if constexpr (KIND == 0) {
#pragma unroll
        for (int j = 0; j < BN / 8; ++j)
#pragma unroll
          for (int h = 0; h < 2; ++h) epi_bias_gelu<h16>(e, nt * BN + 8 * j + c0, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
      }
      if (has_resid) {
        mbar_wait(rfull, rphase);
        rphase ^= 1;
      }
      named_bar_sync(1 + wg, 128);  // the leader's bulk_wait_read: every unit is free
      int seq = 0;                  // units used in this tile
      if (KIND == 0 && e.out_f32) {
#pragma unroll
        for (int u = 0; u < BN / 32; ++u, ++seq) {
          const uint32_t unit = my_rows + (seq % SLOTS) * TG_UNIT_BYTES;
          if (seq >= SLOTS) {  // wait until the unit's previous store has read it
            if (leader) bulk_wait_read<SLOTS - 1>();
            named_bar_sync(1 + wg, 128);
          }
#pragma unroll
          for (int jj = 0; jj < 4; ++jj)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int j = 4 * u + jj;
              const uint32_t a = unit + swz<128>((row_q + 8 * h) * 128 + jj * 32 + c0 * 4);
              if (has_resid) epi_resid(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], ld_shared_v2_f32(a));
              st_shared_v2_f32(a, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
            }
          fence_proxy_async_smem();
          named_bar_sync(1 + wg, 128);
          if (leader) {
            tma_store_3d(&tmF, unit, nt * BN + 32 * u, t0 + 64 * wg, p_out);
            bulk_commit();
          }
        }
      }
      if (e.out_act) {
        constexpr int AC = Cfg::ACT_COLS, RB = AC * 2;
        // stmatrix: lane l addresses row l % 8 of matrix l / 8; the four matrices are rows 0-7 and 8-15 of column
        // group j, then of j + 1
        const int srow = wq * 16 + (lane & 7) + 8 * ((lane >> 3) & 1);
        const int sbyte = (lane >> 4) * 16;
#pragma unroll
        for (int u = 0; u < BN / AC; ++u, ++seq) {
          const uint32_t unit = my_rows + (seq % SLOTS) * TG_UNIT_BYTES;
          if (seq >= SLOTS) {
            if (leader) bulk_wait_read<SLOTS - 1>();
            named_bar_sync(1 + wg, 128);
          }
          if constexpr (KIND == 1) {
            // RoPE of the unit's columns, one row at a time (cos / sin of one position live at once).  BN and C (heads
            // of 32) are multiples of 32, so column 8j + 2 (lane % 4) of the tile is RoPE pair (lane % 4) + 4 (j % 4)
            // of its head; a unit never straddles the k / v boundary 2C, and v columns are not rotated.
            static_assert(BN % 32 == 0, "RoPE pairs of a column need BN % 32 == 0");
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int t = t0 + wg * 64 + row_q + 8 * h;
              const int pos = e.posmode == 0 ? t : p_out % e.F;
              float co[4] = {}, si[4] = {};
              if (t < g.L && nt * BN + AC * u < 2 * e.C) {
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                  co[q] = __ldg(e.rope_cos + pos * 16 + 4 * q + (lane & 3));
                  si[q] = __ldg(e.rope_sin + pos * 16 + 4 * q + (lane & 3));
                }
              }
#pragma unroll
              for (int j = u * (AC / 8); j < (u + 1) * (AC / 8); ++j)
                epi_rope(e, nt * BN + 8 * j + c0, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], co[j & 3], si[j & 3]);
            }
          }
#pragma unroll
          for (int p = 0; p < AC / 16; ++p) {
            const int j = u * (AC / 8) + 2 * p;
            stmatrix_x4(unit + swz<RB>(srow * RB + p * 32 + sbyte), pack_h16x2(acc[4 * j], acc[4 * j + 1]),
                        pack_h16x2(acc[4 * j + 2], acc[4 * j + 3]), pack_h16x2(acc[4 * j + 4], acc[4 * j + 5]),
                        pack_h16x2(acc[4 * j + 6], acc[4 * j + 7]));
          }
          fence_proxy_async_smem();
          named_bar_sync(1 + wg, 128);
          if (leader) {
            tma_store_3d(&tmH, unit, nt * BN + AC * u, t0 + 64 * wg, p_out);
            bulk_commit();
          }
        }
      }
    }
    if (KIND != 2 && leader) bulk_wait_read<0>();  // shared memory stays until the last stores have read it
  }
}

struct TcGemmPlan {
  CUtensorMap tmA, tmW;
  CUtensorMap tmR, tmF, tmH;  // [planes_out, L, N] views of e.resid, e.out_f32, e.out_act (kinds 0 and 1, when present)
  EpiParams e;
  GemmShape g;
  int kind;  // kernel instantiation: 0 generic, 1 qkv, 2 gates
  int BN, BK;
  int num_tiles, t_tiles, n_tiles, m_tiles, grid;
};

// Widest tile that divides N and is at most max_bn.  BK = 32 tiles stay at BN <= 128.  A GEMM whose epilogue reads the
// fp32 residual stays at BN <= 128 as well: its epilogue keeps the whole fp32 tile (the residual, then the result) in
// shared memory next to a 4-stage ring, which BN = 192 or 256 would not leave room for.
static int pick_bn(int N, int max_bn) {
  const int cands[5] = {256, 192, 128, 64, 32};
  for (int i = 0; i < 5; ++i)
    if (cands[i] <= max_bn && N % cands[i] == 0) return cands[i];
  return 0;
}

// [planes_out, L, N] view of an epilogue operand (leading dimension ld elements of es bytes) in boxes of 64 rows (128
// for the residual, which the producer loads for both warpgroups) and 128 bytes (64 when a 16-bit tile is 32 wide)
static bool make_epi_tmap(CUtensorMap* tm, const void* base, int ld, int es, uint32_t box_cols, uint32_t box_rows,
                          const GemmShape& g, const char* what, char* err, int errlen) {
  if (reinterpret_cast<uintptr_t>(base) % 16 != 0 || (static_cast<int64_t>(ld) * es) % 16 != 0 || ld < g.N) {
    snprintf(err, errlen, "tc gemm: the %s needs a 16-byte aligned base and a 16-byte multiple row stride of at least "
             "N elements (base %p, leading dimension %d, N %d)", what, base, ld, g.N);
    return false;
  }
  const uint64_t dims[3] = {static_cast<uint64_t>(g.N), static_cast<uint64_t>(g.L), static_cast<uint64_t>(g.planes_out)};
  const uint64_t strides[2] = {static_cast<uint64_t>(ld) * es, static_cast<uint64_t>(g.L) * ld * es};
  const uint32_t box[3] = {box_cols, box_rows, 1};
  return make_tmap_any(tm, es == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                               : BT_H16_IS_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16,
                       base, 3, dims, strides, box, static_cast<int>(box_cols) * es, err, errlen);
}

// Every gemm_tc_kernel instantiation (BN, BK, epilogue kind): tc_init sets their shared-memory limits, plan creation
// refuses any other tile and launch_gemm_tc dispatches over the same list.  The gates GEMM (kind 2) is N = 32 wide.
#define BT_GEMM_TC_INSTANCES(X)                                                                                         \
  X(256, 64, 0) X(256, 64, 1) X(192, 64, 0) X(192, 64, 1) X(128, 64, 0) X(128, 64, 1) X(64, 64, 0) X(64, 64, 1)       \
  X(32, 64, 0) X(32, 64, 1) X(128, 32, 0) X(128, 32, 1) X(64, 32, 0) X(64, 32, 1) X(32, 32, 0) X(32, 32, 1)             \
  X(32, 64, 2) X(32, 32, 2)

static bool has_instance(const TcGemmPlan* p) {
#define BT_TG_HAS(bn, bk, kd) if (p->BN == bn && p->BK == bk && p->kind == kd) return true;
  BT_GEMM_TC_INSTANCES(BT_TG_HAS)
#undef BT_TG_HAS
  return false;
}

TcGemmPlan* tc_gemm_plan_create(const void* A, const void* W, const GemmShape& g, int planes_in, bool resid_epilogue,
                                const EpiParams& e, char* err, int errlen) {
  TcGemmPlan* p = new TcGemmPlan();
  p->g = g;
  p->e = e;
  p->kind = e.kind == 1 || e.kind == 2 ? e.kind : 0;
  p->BK = (g.Kslab % 64 == 0) ? 64 : 32;
  p->BN = pick_bn(g.N, p->BK == 32 || resid_epilogue ? 128 : 256);
  if (p->BN == 0 || g.Kslab % 32 != 0) {
    snprintf(err, errlen, "tc gemm: unsupported shape N=%d Kslab=%d", g.N, g.Kslab);
    delete p;
    return nullptr;
  }
  if (!has_instance(p)) {
    snprintf(err, errlen, "tc gemm: no kernel for the tile BN=%d BK=%d of epilogue kind %d", p->BN, p->BK, p->kind);
    delete p;
    return nullptr;
  }
  if (p->kind == 1 && (e.resid || e.out_f32)) {
    snprintf(err, errlen, "tc gemm: the qkv epilogue (kind 1) writes its 16-bit output only: no residual, no fp32 output");
    delete p;
    return nullptr;
  }
  if (p->kind != 2 && e.resid && (p->BN > 128 || !e.out_f32)) {
    snprintf(err, errlen, "tc gemm: a residual epilogue needs BN <= 128 (plan it with resid_epilogue) and an fp32 output");
    delete p;
    return nullptr;
  }
  const int swz = p->BK * 2;
  {
    const uint64_t dims[3] = {static_cast<uint64_t>(g.Kslab), static_cast<uint64_t>(g.L),
                              static_cast<uint64_t>(planes_in)};
    const uint64_t strides[2] = {static_cast<uint64_t>(g.lda) * 2, static_cast<uint64_t>(g.L) * g.lda * 2};
    const uint32_t box[3] = {static_cast<uint32_t>(p->BK), TG_BM, 1};
    if (!make_tmap(&p->tmA, A, 3, dims, strides, box, swz, err, errlen)) { delete p; return nullptr; }
  }
  {
    const uint64_t Ktot = static_cast<uint64_t>(g.Kslab) * g.nslab;
    const uint64_t dims[2] = {Ktot, static_cast<uint64_t>(g.N)};
    const uint64_t strides[1] = {Ktot * 2};
    const uint32_t box[2] = {static_cast<uint32_t>(p->BK), static_cast<uint32_t>(p->BN)};
    if (!make_tmap(&p->tmW, W, 2, dims, strides, box, swz, err, errlen)) { delete p; return nullptr; }
  }
  const uint32_t act_cols = p->BN < 64 ? p->BN : 64;
  if (p->kind != 2 &&  // the gates GEMM stores from registers
      ((e.resid && !make_epi_tmap(&p->tmR, e.resid, e.ldr, 4, 32, TG_BM, g, "residual", err, errlen)) ||
       (e.out_f32 && !make_epi_tmap(&p->tmF, e.out_f32, e.ldo_f32, 4, 32, 64, g, "fp32 output", err, errlen)) ||
       (e.out_act && !make_epi_tmap(&p->tmH, e.out_act, e.ldo_act, 2, act_cols, 64, g, "16-bit output", err, errlen)))) {
    delete p;
    return nullptr;
  }
  p->t_tiles = ceil_div(g.L, TG_BM);
  p->n_tiles = g.N / p->BN;
  p->m_tiles = p->t_tiles * g.planes_out;
  p->num_tiles = p->m_tiles * p->n_tiles;
  p->grid = p->num_tiles < g_num_sms ? p->num_tiles : g_num_sms;
  return p;
}
void tc_gemm_plan_destroy(TcGemmPlan* p) { delete p; }
void tc_gemm_plan_tile(const TcGemmPlan* p, int* bn, int* bk) { *bn = p->BN; *bk = p->BK; }

void launch_gemm_tc(const TcGemmPlan* p, cudaStream_t st) {
#define BT_TG_LAUNCH(bn, bk, kd)                                                                                       \
  if (p->BN == bn && p->BK == bk && p->kind == kd) {                                                                   \
    gemm_tc_kernel<bn, bk, kd><<<p->grid, TG_THREADS, TgCfg<bn, bk>::SMEM, st>>>(                                     \
        p->tmA, p->tmW, p->tmR, p->tmF, p->tmH, p->g, p->e, p->num_tiles, p->t_tiles, p->n_tiles, p->m_tiles);        \
    return;                                                                                                            \
  }
  BT_GEMM_TC_INSTANCES(BT_TG_LAUNCH)
#undef BT_TG_LAUNCH
}

int tc_init(char* err, int errlen) {
  if (!g_encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t r = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
    if (r != cudaSuccess || fn == nullptr || qres != cudaDriverEntryPointSuccess) {
      snprintf(err, errlen, "cudaGetDriverEntryPoint(cuTensorMapEncodeTiled) failed: %s", cudaGetErrorString(r));
      return -1;
    }
    g_encode = reinterpret_cast<PFN_encodeTiled>(fn);
  }
  int dev = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
  cudaError_t r = cudaSuccess;
#define BT_TG_ATTR(bn, bk, kd)                                                                                         \
  if (r == cudaSuccess)                                                                                                \
    r = cudaFuncSetAttribute(gemm_tc_kernel<bn, bk, kd>, cudaFuncAttributeMaxDynamicSharedMemorySize, TgCfg<bn, bk>::SMEM);
  BT_GEMM_TC_INSTANCES(BT_TG_ATTR)
#undef BT_TG_ATTR
  if (r != cudaSuccess) {
    snprintf(err, errlen, "cudaFuncSetAttribute(gemm_tc_kernel) failed: %s", cudaGetErrorString(r));
    return -1;
  }
  if (tc_init_attn(err, errlen) != 0) return -1;
  if (tc_init_attn_freq(err, errlen) != 0) return -1;
  if (tc_init_fused(err, errlen) != 0) return -1;
  return 0;
}

}  // namespace bt
