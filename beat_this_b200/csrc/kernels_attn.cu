// Tensor-core flash attention for head_dim 32 over sequences of any length (a ctx's chunks are at most bt_max_chunk
// frames): the time-direction attention of the three frontend blocks and of the 6 main layers (reference
// roformer.py:73-80 SDPA, called from roformer.py:114-132 / beat_tracker.py:290-301).  Row and tile indices are
// 32-bit (L < 2^31); element offsets are 64-bit.
#include <cstdio>
#include <type_traits>

#include "tc_common.cuh"

namespace bt {

// CTA = 128 queries of one (sequence, head): 4 MMA warps of 32 query rows each.  Thread 0 TMA-loads Q once and the
// K / V tiles of 64 keys through an AT_NST-deep ring of mbarriers (64-byte swizzled rows, the layout ldmatrix reads
// without bank conflicts); it refills a stage once every warp has arrived on its `empty` barrier.  Each MMA warp
// keeps S, P and O in registers (mma.sync m16n8k16, fp32 accumulate): S = Q K^T -> online softmax in log2 units (q carries scale * log2 e) ->
// P packed to 16 bits straight from the S accumulator layout -> O += P V.  With head_dim 32 there are only 128
// tensor FLOPs per exponential: the exponentials (MUFU.EX2, 16 /clk/SM) bound the kernel, so a share of them can
// run as a polynomial on the FMA pipe instead: 3 of every 8 score pairs (AT_POLY_MASK).
// A warp's 32 rows are two m16 row blocks: each K / V fragment it loads feeds the MMAs of both, the two softmax
// chains interleave, and the loop's fixed cost (barrier wait, addresses, branch) is paid once per 32 rows.  Every
// row goes through the same operations in the same order as in a warp of one row block, so the bits do not depend
// on the number of blocks per warp.
constexpr int AT_BQ = 128;
constexpr int AT_BKV = 64;
constexpr int AT_NST = 4;
constexpr int AT_WARPS = 4;
constexpr int AT_RB = 2;  // m16 row blocks per MMA warp: AT_BQ = AT_WARPS * AT_RB * 16
constexpr int AT_THREADS = 32 * AT_WARPS;
constexpr int AT_SQ = AT_BQ * 64;    // 128 query rows x 32 dims x 2 bytes
constexpr int AT_SKV = AT_BKV * 64;  // 64 key rows x 32 dims x 2 bytes
constexpr int AT_SMEM = 1024 + AT_SQ + AT_NST * 2 * AT_SKV + 128;
static_assert(AT_BQ == AT_WARPS * AT_RB * 16, "every query row of the tile belongs to one row block");

// which of every 8 score pairs take the polynomial exp2 (spread out so that MUFU and FMA work interleave)
constexpr uint32_t AT_POLY_MASK = 0x52u;

// byte offset of 16-byte chunk c of row r in a tile of 64-byte rows written by TMA with CU_TENSOR_MAP_SWIZZLE_64B
__device__ __forceinline__ uint32_t sw64_off(int r, int c) {
  return static_cast<uint32_t>(r * 64 + ((c ^ ((r >> 1) & 3)) << 4));
}

// 3 CTAs per SM (12 warps with two softmax chains each) leave 168 registers per thread, which the loop needs without
// spills.  A dedicated producer warp would take a fifth of the register file and force 128 or fewer.
__global__ void __launch_bounds__(AT_THREADS, 3)
attn_time_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmKV,
                 const float* __restrict__ gates, h16* __restrict__ out, int L, int heads,
                 const ChunkSrc* __restrict__ chunks, int seqs_per_chunk) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sQ = sbase;
  const uint32_t sK = sQ + AT_SQ;              // [AT_NST] key tiles
  const uint32_t sV = sK + AT_NST * AT_SKV;    // [AT_NST] value tiles
  const uint32_t bar_q = sV + AT_NST * AT_SKV;
  const uint32_t full = bar_q + 8;             // [AT_NST] K and V of a tile landed
  const uint32_t empty = full + 8 * AT_NST;    // [AT_NST] every MMA warp is done with the stage

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * AT_BQ;
  const int h = blockIdx.y;
  const int seq = blockIdx.z;
  const int C = heads * 32;
  // keys that exist for this sequence: the whole plane, or (waves of chunks of different lengths) its chunk's frames
  const int Lk = chunks ? chunks[seq / seqs_per_chunk].len : L;
  const int nkv = ceil_div(Lk, AT_BKV);

  if (threadIdx.x == 0) {
    mbar_init(bar_q, 1);
    for (int i = 0; i < AT_NST; ++i) {
      mbar_init(full + 8 * i, 1);
      mbar_init(empty + 8 * i, AT_WARPS);
    }
    fence_barrier_init();
  }
  __syncthreads();

  auto load_tile = [&](int t) {  // key / value tile t into stage t % AT_NST
    const int st = t % AT_NST;
    mbar_expect_tx(full + 8 * st, 2 * AT_SKV);
    tma_load_3d(sK + st * AT_SKV, &tmKV, full + 8 * st, C + h * 32, t * AT_BKV, seq);
    tma_load_3d(sV + st * AT_SKV, &tmKV, full + 8 * st, 2 * C + h * 32, t * AT_BKV, seq);
  };
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmKV);
    mbar_expect_tx(bar_q, AT_SQ);
    tma_load_3d(sQ, &tmQ, bar_q, h * 32, q0, seq);
    for (int t = 0; t < nkv && t < AT_NST; ++t) load_tile(t);
  }

  // this warp's query rows [r0, r0 + 32) of the tile; in row block b the thread holds rows r0 + 16 b + lane/4 and +8
  const int r0 = warp * (AT_RB * 16);
  mbar_wait(bar_q, 0);

  uint32_t qa[AT_RB][2][4];
#pragma unroll
  for (int b = 0; b < AT_RB; ++b)
#pragma unroll
    for (int ks = 0; ks < 2; ++ks)
      ldmatrix_x4(sQ + sw64_off(r0 + 16 * b + (lane & 15), 2 * ks + (lane >> 4)), qa[b][ks]);

  // Per-lane ldmatrix addresses in stage 0.  A tile row's swizzle depends only on its row mod 8, which the lane
  // fixes: K fragment nb (keys 8 nb + lane % 8) sits 512 nb bytes further, V fragment kk (keys 16 kk + lane % 16)
  // 1024 kk bytes further, and both offsets become immediates of the ldmatrix.
  const uint32_t k_addr0 = sK + sw64_off(lane & 7, lane >> 3);
  const uint32_t v_addr0[2] = {sV + sw64_off(lane & 15, lane >> 4), sV + sw64_off(lane & 15, 2 + (lane >> 4))};
  const int key_lane = 2 * (lane & 3);  // key of the thread's first S column in a fragment

  float o[AT_RB][4][4];
#pragma unroll
  for (int b = 0; b < AT_RB; ++b)
#pragma unroll
    for (int d = 0; d < 4; ++d) o[b][d][0] = o[b][d][1] = o[b][d][2] = o[b][d][3] = 0.f;
  float m_run[AT_RB][2], l_run[AT_RB][2];
#pragma unroll
  for (int b = 0; b < AT_RB; ++b) m_run[b][0] = m_run[b][1] = -INFINITY, l_run[b][0] = l_run[b][1] = 0.f;
  // One tile j of 64 keys: ring stage `stage` (bytes: (j % AT_NST) * AT_SKV), barrier parity `phase` ((j / AT_NST) & 1).
  // The last tile is a separate instantiation (`last`) that sets keys >= lim to -inf, so the steady loop carries no
  // masking.
  auto kv_step = [&](uint32_t stage, uint32_t phase, auto last, int lim) {
    mbar_wait(full + stage / (AT_SKV / 8), phase);
    const uint32_t ka = k_addr0 + stage, va0 = v_addr0[0] + stage, va1 = v_addr0[1] + stage;
    float s[AT_RB][8][4];
#pragma unroll
    for (int nb = 0; nb < 8; ++nb) {  // keys [8 nb, 8 nb + 8)
      uint32_t kf[4];
      ldmatrix_x4(ka + nb * 512, kf);
#pragma unroll
      for (int b = 0; b < AT_RB; ++b) {
        s[b][nb][0] = s[b][nb][1] = s[b][nb][2] = s[b][nb][3] = 0.f;
        mma_16816(s[b][nb], qa[b][0], kf[0], kf[1]);
        mma_16816(s[b][nb], qa[b][1], kf[2], kf[3]);
      }
    }
    if constexpr (decltype(last)::value) {  // keys >= lim are padding
#pragma unroll
      for (int nb = 0; nb < 8; ++nb) {
        const int key = nb * 8 + key_lane;
#pragma unroll
        for (int b = 0; b < AT_RB; ++b) {
          if (key >= lim) s[b][nb][0] = s[b][nb][2] = -INFINITY;
          if (key + 1 >= lim) s[b][nb][1] = s[b][nb][3] = -INFINITY;
        }
      }
    }
    float mref[AT_RB][2];
#pragma unroll
    for (int b = 0; b < AT_RB; ++b) {
      // row maxima as a tree (depth 4 instead of a chain of 16): a maximum is exact, so any order gives its bits
      float mx[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        float t[8];
#pragma unroll
        for (int nb = 0; nb < 8; ++nb) t[nb] = fmaxf(s[b][nb][2 * r], s[b][nb][2 * r + 1]);
#pragma unroll
        for (int w = 4; w > 0; w >>= 1)
#pragma unroll
          for (int i = 0; i < w; ++i) t[i] = fmaxf(t[i], t[i + w]);
        mx[r] = t[0];
      }
      float alpha[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
        mref[b][r] = fmaxf(m_run[b][r], mx[r]);  // finite: the first tile holds key 0 of every row
        alpha[r] = ex2_approx(m_run[b][r] - mref[b][r]);
        m_run[b][r] = mref[b][r];
        l_run[b][r] *= alpha[r];
      }
#pragma unroll
      for (int d = 0; d < 4; ++d) {
        o[b][d][0] *= alpha[0]; o[b][d][1] *= alpha[0];
        o[b][d][2] *= alpha[1]; o[b][d][3] *= alpha[1];
      }
    }
    uint32_t pa[AT_RB][4][4];  // P as the A operand of P V: 16 keys per k-step
#pragma unroll
    for (int b = 0; b < AT_RB; ++b)
#pragma unroll
      for (int nb = 0; nb < 8; ++nb) {
        float p[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float x = s[b][nb][i] - mref[b][i >> 1];
          p[i] = ((AT_POLY_MASK >> nb) & 1u) ? ex2_poly(x) : ex2_approx(x);
        }
        l_run[b][0] += p[0] + p[1];
        l_run[b][1] += p[2] + p[3];
        pa[b][nb >> 1][(nb & 1) * 2] = pack_h16x2(p[0], p[1]);
        pa[b][nb >> 1][(nb & 1) * 2 + 1] = pack_h16x2(p[2], p[3]);
      }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
      for (int dp = 0; dp < 2; ++dp) {  // dims [16 dp, 16 dp + 16)
        uint32_t vf[4];
        ldmatrix_x4_trans((dp ? va1 : va0) + kk * 1024, vf);
#pragma unroll
        for (int b = 0; b < AT_RB; ++b) {
          mma_16816(o[b][2 * dp], pa[b][kk], vf[0], vf[1]);
          mma_16816(o[b][2 * dp + 1], pa[b][kk], vf[2], vf[3]);
        }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(empty + stage / (AT_SKV / 8));
  };
  uint32_t stage = 0, phase = 0;
  for (int j = 0; j < nkv - 1; ++j) {
    // tile j + AT_NST - 1 goes into the stage of tile j - 1 once every warp is done with that; tiles >= AT_NST are
    // issued by steps 1 .. nkv - AT_NST, so the last tile's step never refills
    if (threadIdx.x == 0 && j > 0 && j + AT_NST - 1 < nkv) {
      mbar_wait(empty + 8 * ((j - 1) % AT_NST), ((j - 1) / AT_NST) & 1);
      load_tile(j + AT_NST - 1);
    }
    kv_step(stage, phase, std::false_type{}, 0);
    stage += AT_SKV;
    if (stage == AT_NST * AT_SKV) stage = 0, phase ^= 1;
  }
  if (nkv > 0) kv_step(stage, phase, std::true_type{}, Lk - (nkv - 1) * AT_BKV);
#pragma unroll
  for (int b = 0; b < AT_RB; ++b)
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      l_run[b][r] += __shfl_xor_sync(0xffffffffu, l_run[b][r], 1);
      l_run[b][r] += __shfl_xor_sync(0xffffffffu, l_run[b][r], 2);
    }
#pragma unroll
  for (int b = 0; b < AT_RB; ++b)
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int q = q0 + r0 + 16 * b + (lane >> 2) + 8 * r;
      if (q < L) {
        const int64_t m = static_cast<int64_t>(seq) * L + q;
        const float gsc = gates[m * heads + h] / l_run[b][r];
        h16* dst = out + m * C + h * 32 + 2 * (lane & 3);
#pragma unroll
        for (int d = 0; d < 4; ++d)
          *reinterpret_cast<uint32_t*>(dst + 8 * d) = pack_h16x2(o[b][d][2 * r] * gsc, o[b][d][2 * r + 1] * gsc);
      }
    }
}

struct TcAttnPlan {
  CUtensorMap tmQ;   // [seqs, L, 3C] 16-bit, boxes of 128 rows x 32 columns (one head's queries)
  CUtensorMap tmKV;  // same tensor, boxes of 64 rows (one key / value tile)
  int seqs, L, heads;
};

TcAttnPlan* tc_attn_plan_create(const void* qkv, int seqs, int L, int heads, char* err, int errlen) {
  TcAttnPlan* p = new TcAttnPlan();
  p->seqs = seqs; p->L = L; p->heads = heads;
  const int C = heads * 32;
  const uint64_t dims[3] = {static_cast<uint64_t>(3 * C), static_cast<uint64_t>(L), static_cast<uint64_t>(seqs)};
  const uint64_t strides[2] = {static_cast<uint64_t>(3 * C) * 2, static_cast<uint64_t>(L) * 3 * C * 2};
  const uint32_t box_q[3] = {32, AT_BQ, 1};
  const uint32_t box_kv[3] = {32, AT_BKV, 1};
  if (!make_tmap(&p->tmQ, qkv, 3, dims, strides, box_q, 64, err, errlen) ||
      !make_tmap(&p->tmKV, qkv, 3, dims, strides, box_kv, 64, err, errlen)) {
    delete p;
    return nullptr;
  }
  return p;
}
void tc_attn_plan_destroy(TcAttnPlan* p) { delete p; }

void launch_attn_time_tc(const TcAttnPlan* p, const float* gates, void* out, cudaStream_t st, const ChunkSrc* chunks,
                         int seqs_per_chunk) {
  dim3 grid(ceil_div(p->L, AT_BQ), p->heads, p->seqs);
  attn_time_kernel<<<grid, AT_THREADS, AT_SMEM, st>>>(p->tmQ, p->tmKV, gates, reinterpret_cast<h16*>(out), p->L, p->heads,
                                                      chunks, seqs_per_chunk);
}

int tc_init_attn(char* err, int errlen) {
  const cudaError_t r = cudaFuncSetAttribute(attn_time_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, AT_SMEM);
  if (r != cudaSuccess) {
    snprintf(err, errlen, "cudaFuncSetAttribute(attn_time_kernel) failed: %s", cudaGetErrorString(r));
    return -1;
  }
  return 0;
}

}  // namespace bt
