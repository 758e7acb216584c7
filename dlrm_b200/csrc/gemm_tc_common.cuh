// Pieces of the wgmma GEMM kernel (gemm_tc.cu): tile constants, the problem description, PTX wrappers
// (mbarrier, TMA, wgmma), the wgmma shared-memory descriptor, the consumer main loop, the epilogue and the
// plan object the C ABI hands out.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>

#include "common.cuh"

namespace dlrm {

constexpr int TC_BM = 128;
constexpr int TC_BK = 64;  // 64 bf16 = 128 bytes = one swizzle row
constexpr int TC_MAX_SMEM = 227 * 1024;   // dynamic shared memory one sm_90 block may opt in to

struct TcArgs {
  long long M, N, K;
  int x3;
  int a_mn, b_mn;  // operand majorness (0 = K-major, 1 = MN-major)
  int kb_per_split, num_kb;
  int act;
  int mask_act;
  const __nv_bfloat16* mask_hi;
  const __nv_bfloat16* mask_lo;
  long long ldmask;
  float* out_f32;
  long long ld_f32, slab_stride;
  __nv_bfloat16* out_hi;
  __nv_bfloat16* out_lo;
  long long ld_out;
  __nv_bfloat16* outT_hi;
  __nv_bfloat16* outT_lo;
  long long ld_outT;
  float* out_col;
  long long col_index, col_slab_stride;
  const float* bias;   // optional fp32 [N], added to the accumulator before the activation
};

// ------------------------------------------------------------------------------------------ PTX
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  // try_wait suspends for a bounded time per call; a protocol bug must trap (after 2 s of wall clock),
  // not hang the GPU
  uint32_t ok = 0;
  unsigned long long t0 = 0;
  while (true) {
    asm volatile(
        "{\n\t.reg .pred P1;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, P1;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    if (ok) break;
    const unsigned long long now = globaltimer_ns();
    if (t0 == 0) t0 = now;
    else if (now - t0 > 2000000000ull) __trap();
  }
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int x, int y) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
      "l"(map), "r"(bar), "r"(x), "r"(y)
      : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}

// wgmma.mma_async m64nNk16, bf16 x bf16 -> f32 accumulated in registers (scale-d = 1: the caller zeroes d).
// TA / TB: operand A / B is MN-major (transposed) in shared memory.  Fragment of thread t of the warpgroup:
// d[4j + 2h + c] = D[16 (t / 32) + (t % 32) / 4 + 8h][8j + 2 (t % 4) + c].
template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16(float (&d)[16], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, %19, %20;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(adesc), "l"(bdesc), "r"(1), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16(float (&d)[32], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(1), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16(float (&d)[64], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, %67, %68;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(1), "n"(TA), "n"(TB));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// wgmma shared-memory descriptor (sm_90): start>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46), base offset 0
// (every tile is 1024-byte aligned), layout [62,64): SWIZZLE_128B = 1, SWIZZLE_64B = 2.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t addr, uint32_t lbo_bytes, uint32_t sbo_bytes,
                                                   uint32_t layout = 1) {
  uint64_t d = 0;
  d |= (uint64_t)((addr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)layout << 62;
  return d;
}

__device__ __forceinline__ float apply_act_tc(float v, int act) {
  if (act == DLRM_ACT_RELU) return fmaxf(v, 0.f);
  if (act == DLRM_ACT_SIGMOID) return 1.0f / (1.0f + expf(-v));
  return v;
}


// ------------------------------------------------------------------------------------------ CTA layout
// Warpgroup 0: warp 0 lane 0 is the TMA producer (warps 1-3 only exist so that the consumers are whole,
// aligned warpgroups).  Warpgroups 1 and 2 are the consumers: consumer warpgroup w issues the wgmmas of
// accumulator rows [BM/2 w, BM/2 w + BM/2) of the BM x BN tile, then all 8 consumer warps run the epilogue.
// BM = 128: one m64 accumulator per consumer warpgroup, k blocks of 64 (128-byte rows, 128-byte swizzle).
// BM = 256: two m64 accumulators per consumer warpgroup (128 fp32 registers per thread), k blocks of 32 so that
// four x3 stages (48 KB each) fit the ring; K-major tiles then have 64-byte rows and use the 64-byte swizzle.
constexpr int TC_EPI_WARPS = 8;
constexpr int TC_THREADS = 128 + 32 * TC_EPI_WARPS;
constexpr int TC_CONSUMER_WARP0 = 4;
constexpr uint32_t TC_A_BYTES = TC_BM * TC_BK * 2;   // 16 KB; rows 64..127 start at +8 KB in both majornesses

template <int BM>
struct TcTile {
  static constexpr int BK = BM == 256 ? 32 : TC_BK;
  static constexpr int MT = BM / 128;                         // m64 accumulators per consumer warpgroup
  static constexpr uint32_t A64_BYTES = 64 * BK * 2;          // 64 rows of A: the next 64 start here (both majornesses)
  static constexpr uint32_t A_BYTES = BM * BK * 2;
  static constexpr uint32_t KROW_BYTES = BK * 2;              // K-major row = swizzle span
  static constexpr uint32_t LAYOUT = BK == 64 ? 1u : 2u;      // K-major descriptor layout: 128- / 64-byte swizzle
  static constexpr uint32_t MN_BOX_BYTES = BK * 128;          // MN-major box: BK k rows of 64 mn
};

// Consumer main loop over k blocks [kb0, kb1) of one tile.  Every stage of the ring holds A_hi [A_lo] B_hi
// [B_lo] (x3 adds the lo tiles), each 1024-byte aligned in the swizzle TMA writes.  A stage is released (one
// arrive per consumer warp) once the wgmmas that read it have retired; the wgmmas of the next k block are already
// issued by then.  `stage` / `phase` carry the ring position across calls.
//   K-major SW128 / SW64 : rows of BK * 2 bytes, 8-row groups 8 rows apart (SBO); a 16-wide k step = +32 B.
//   MN-major SW128       : [BK k rows][64 mn] boxes; 8-row k groups 1024 B apart (SBO), 64-wide mn blocks one box
//                          apart (LBO); a 16-deep k step = +2048 B.
// Every accumulator sees the same k16 sequence, and per k16 lo*hi, hi*lo, hi*hi, whatever BM and BK are: a
// 256-row tile gives the bits of two 128-row tiles.
template <int BM, int BN, int TA, int TB>
__device__ __forceinline__ void tc_mainloop_t(float (&d)[TcTile<BM>::MT][BN / 2], bool x3, uint32_t ring,
                                              uint32_t stage_bytes, int stages, uint32_t bar_full, uint32_t bar_empty,
                                              int kb0, int kb1, int& stage, uint32_t& phase, int wg, int lane) {
  using T = TcTile<BM>;
  constexpr int MT = T::MT;
  constexpr uint32_t B_BYTES = BN * T::BK * 2;
  constexpr uint32_t a_lbo = TA ? T::MN_BOX_BYTES : 16u, b_lbo = TB ? T::MN_BOX_BYTES : 16u;
  constexpr uint32_t a_sbo = TA ? 1024u : 8 * T::KROW_BYTES, b_sbo = TB ? 1024u : 8 * T::KROW_BYTES;
  constexpr uint32_t a_lay = TA ? 1u : T::LAYOUT, b_lay = TB ? 1u : T::LAYOUT;
  int prev = -1;
  for (int kb = kb0; kb < kb1; ++kb) {
    mbar_wait(bar_full + 8 * stage, phase);
    __syncwarp();
    const uint32_t sa_hi = ring + stage * stage_bytes + (uint32_t)(wg * MT) * T::A64_BYTES;
    const uint32_t sa_lo = sa_hi + T::A_BYTES;
    const uint32_t sb_hi = ring + stage * stage_bytes + (x3 ? 2u : 1u) * T::A_BYTES;
    const uint32_t sb_lo = sb_hi + B_BYTES;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < T::BK / 16; ++k) {
      const uint32_t a_off = TA ? k * 2048u : k * 32u;
      const uint32_t b_off = TB ? k * 2048u : k * 32u;
      const uint64_t bh = make_smem_desc(sb_hi + b_off, b_lbo, b_sbo, b_lay);
      if (x3) {
        const uint64_t bl = make_smem_desc(sb_lo + b_off, b_lbo, b_sbo, b_lay);
#pragma unroll
        for (int j = 0; j < MT; ++j)
          wgmma_bf16<TA, TB>(d[j], make_smem_desc(sa_lo + j * T::A64_BYTES + a_off, a_lbo, a_sbo, a_lay), bh);
#pragma unroll
        for (int j = 0; j < MT; ++j)
          wgmma_bf16<TA, TB>(d[j], make_smem_desc(sa_hi + j * T::A64_BYTES + a_off, a_lbo, a_sbo, a_lay), bl);
      }
#pragma unroll
      for (int j = 0; j < MT; ++j)
        wgmma_bf16<TA, TB>(d[j], make_smem_desc(sa_hi + j * T::A64_BYTES + a_off, a_lbo, a_sbo, a_lay), bh);
    }
    wgmma_commit();
    wgmma_wait<1>();                              // the previous k block's wgmmas have retired
    if (prev >= 0 && lane == 0) mbar_arrive(bar_empty + 8 * prev);
    prev = stage;
    if (++stage == stages) { stage = 0; phase ^= 1; }
  }
  wgmma_wait<0>();
  if (prev >= 0 && lane == 0) mbar_arrive(bar_empty + 8 * prev);
}

template <int BM, int BN>
__device__ __forceinline__ void tc_mainloop(float (&d)[TcTile<BM>::MT][BN / 2], const TcArgs& g, uint32_t ring,
                                            uint32_t stage_bytes, int stages, uint32_t bar_full, uint32_t bar_empty,
                                            int kb0, int kb1, int& stage, uint32_t& phase, int wg, int lane) {
#pragma unroll
  for (int i = 0; i < TcTile<BM>::MT; ++i)
#pragma unroll
    for (int j = 0; j < BN / 2; ++j) d[i][j] = 0.f;
  const bool x3 = g.x3 != 0;
  if (!g.a_mn && !g.b_mn)
    tc_mainloop_t<BM, BN, 0, 0>(d, x3, ring, stage_bytes, stages, bar_full, bar_empty, kb0, kb1, stage, phase, wg, lane);
  else if (!g.a_mn)
    tc_mainloop_t<BM, BN, 0, 1>(d, x3, ring, stage_bytes, stages, bar_full, bar_empty, kb0, kb1, stage, phase, wg, lane);
  else if (!g.b_mn)
    tc_mainloop_t<BM, BN, 1, 0>(d, x3, ring, stage_bytes, stages, bar_full, bar_empty, kb0, kb1, stage, phase, wg, lane);
  else
    tc_mainloop_t<BM, BN, 1, 1>(d, x3, ring, stage_bytes, stages, bar_full, bar_empty, kb0, kb1, stage, phase, wg, lane);
}

// ------------------------------------------------------------------------------------------ epilogue
// The accumulator tile is staged in shared memory as fp32 [BM][BN + 4] (the 4-float pad makes the epilogue's
// row-per-lane 16-byte reads conflict-free), then every consumer warp reads ONE ROW per lane, 32 consecutive
// columns at a time.
__host__ __device__ constexpr int tc_acc_ld(int bn) { return bn + 4; }
__host__ __device__ constexpr int tc_acc_bytes(int bm, int bn) { return bm * tc_acc_ld(bn) * 4; }

// a consumer warp stores one m64 wgmma fragment of its warpgroup: rows row0 + lane / 4 (+ 8), columns
// 8 j + 2 (lane % 4), where row0 = the fragment's first tile row + 16 x (the warp's rank in its warpgroup)
template <int BN>
__device__ __forceinline__ void tc_stage_acc(const float (&d)[BN / 2], float* acc, int row0, int lane) {
  float* r0 = acc + (size_t)(row0 + (lane >> 2)) * tc_acc_ld(BN) + 2 * (lane & 3);
  float* r1 = r0 + 8 * tc_acc_ld(BN);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    *reinterpret_cast<float2*>(r0 + 8 * j) = make_float2(d[4 * j], d[4 * j + 1]);
    *reinterpret_cast<float2*>(r1 + 8 * j) = make_float2(d[4 * j + 2], d[4 * j + 3]);
  }
}

// Staged tile (BM rows x bn columns) -> global memory.
//
// Storing straight from the row-per-lane layout would make each warp-wide 16-byte store hit 32 different rows
// (32 half-written sectors per instruction).  Instead every 32 x 32 chunk is transposed through a per-warp
// shared-memory tile (padded rows: conflict-free 16-byte accesses) so that a warp store covers whole row
// segments: 8 rows x 64 B for the bf16 (hi, lo) operands, 4 rows x 128 B for fp32; the activation-gradient
// mask is read the same way.  Chunks that are ragged (N tail, the diverted bias-gradient column) or whose rows
// are not 16-byte aligned use element-wise but still row-contiguous accesses.
constexpr int TC_EPI_ROW_F32 = 20;                 // floats per staged fp32 half-row (16 + 4 pad)
constexpr int TC_EPI_ROW_BF16 = 40;                // bf16 per staged bf16 row (32 + 8 pad)
constexpr int TC_EPI_WARP_BYTES = 32 * TC_EPI_ROW_BF16 * 2;  // 2560 B per epilogue warp (fp32: two 16-column passes)
constexpr int TC_EPI_BYTES = TC_EPI_WARPS * TC_EPI_WARP_BYTES;
// the accumulator is staged in the operand ring, idle once the last wgmma has retired
__host__ __device__ constexpr size_t tc_ring_bytes(size_t ring, int bm, int bn) {
  return ring > (size_t)tc_acc_bytes(bm, bn) ? ring : (size_t)tc_acc_bytes(bm, bn);
}

// 32 x 32 bf16 chunk, one row per thread in `mine` -> global rows [mrow0, mrow0 + 32) x columns [nb, nb + 32)
__device__ __forceinline__ void tc_epi_store_bf16(const __nv_bfloat16 (&mine)[32], __nv_bfloat16* dst, long long ld,
                                                  long long mrow0, long long nb, long long M, long long N, bool vec,
                                                  int lane, __nv_bfloat16* sb) {
#pragma unroll
  for (int q = 0; q < 4; ++q)
    *reinterpret_cast<uint4*>(sb + lane * TC_EPI_ROW_BF16 + q * 8) = reinterpret_cast<const uint4*>(mine)[q];
  __syncwarp();
  if (vec) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {     // 8 rows x 64 B per warp store
      const int row = i * 8 + (lane >> 2), seg = lane & 3;
      if (mrow0 + row < M)
        *reinterpret_cast<uint4*>(dst + (mrow0 + row) * ld + nb + seg * 8) =
            *reinterpret_cast<const uint4*>(sb + row * TC_EPI_ROW_BF16 + seg * 8);
    }
  } else {
    const long long col = nb + lane;
    const int nrow = (int)min(32ll, M - mrow0);
    if (col < N)
      for (int row = 0; row < nrow; ++row) dst[(mrow0 + row) * ld + col] = sb[row * TC_EPI_ROW_BF16 + lane];
  }
  __syncwarp();
}

// This warp handles rows [32 quad, 32 quad + 32) of the tile and its 32-column chunks c0, c0 + cstep, ... (in a
// 128-row tile two warps per 32-row block split the chunks between them; in a 256-row tile each warp has a block).
__device__ __forceinline__ void tc_epilogue_tile(const TcArgs& g, int bn, int m0, int n0, int bz, const float* acc,
                                                 int quad, int lane, uint8_t* stage_warp, int c0, int cstep) {
  // Every field is copied into a register ONCE: `g` lives in kernel-parameter space and the mbarrier asm
  // statements clobber memory, so reading g.act or g.bias inside the element loops costs a constant-bank load +
  // a branch PER ELEMENT.
  const long long M = g.M, N = g.N;
  const int act = g.act, mask_act = g.mask_act;
  const __nv_bfloat16* const mask_hi = g.mask_hi;
  const __nv_bfloat16* const mask_lo = g.mask_lo;
  const long long ldmask = g.ldmask, ld_f32 = g.ld_f32, ld_out = g.ld_out, ld_outT = g.ld_outT;
  __nv_bfloat16* const out_hi = g.out_hi;
  __nv_bfloat16* const out_lo = g.out_lo;
  __nv_bfloat16* const outT_hi = g.outT_hi;
  __nv_bfloat16* const outT_lo = g.outT_lo;
  const float* const bias = g.bias;
  const long long col_index = g.col_index;
  float* const of32 = g.out_f32 ? g.out_f32 + (long long)bz * g.slab_stride : nullptr;
  float* const ocol = g.out_col ? g.out_col + (long long)bz * g.col_slab_stride : nullptr;

  const long long mrow0 = (long long)m0 + quad * 32;   // first row of this warp
  const long long m = mrow0 + lane;
  const bool m_ok = m < M;
  float* sf = reinterpret_cast<float*>(stage_warp);
  __nv_bfloat16* sb = reinterpret_cast<__nv_bfloat16*>(stage_warp);
  const bool f32_vec = of32 && (ld_f32 & 3) == 0 && (reinterpret_cast<uintptr_t>(of32) & 15) == 0;
  const bool bf_vec = out_hi && (ld_out & 7) == 0 && (reinterpret_cast<uintptr_t>(out_hi) & 15) == 0 &&
                      (!out_lo || (reinterpret_cast<uintptr_t>(out_lo) & 15) == 0);
  const bool mask_vec = mask_act != DLRM_ACT_NONE && (ldmask & 7) == 0 &&
                        (reinterpret_cast<uintptr_t>(mask_hi) & 15) == 0 &&
                        (!mask_lo || (reinterpret_cast<uintptr_t>(mask_lo) & 15) == 0);
  const bool bias_vec = bias && (reinterpret_cast<uintptr_t>(bias) & 15) == 0;
#pragma unroll 1
  for (int c = c0; c < bn / 32; c += cstep) {
    const long long nb = (long long)n0 + c * 32;
    if (nb >= N) break;
    uint32_t r[32];
    const float4* arow = reinterpret_cast<const float4*>(acc + (size_t)(quad * 32 + lane) * tc_acc_ld(bn) + c * 32);
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const float4 t = arow[q];
      r[4 * q] = __float_as_uint(t.x); r[4 * q + 1] = __float_as_uint(t.y);
      r[4 * q + 2] = __float_as_uint(t.z); r[4 * q + 3] = __float_as_uint(t.w);
    }
    float v[32];
    const bool full = nb + 32 <= N;
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = __uint_as_float(r[j]);
    if (bias) {       // nn.Linear bias: the same 32 values for every row -> 8 broadcast 16-byte loads
      if (full && bias_vec) {
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const float4 b4 = __ldg(reinterpret_cast<const float4*>(bias + nb) + q);
          v[4 * q] += b4.x; v[4 * q + 1] += b4.y; v[4 * q + 2] += b4.z; v[4 * q + 3] += b4.w;
        }
      } else {
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] += (nb + j < N) ? __ldg(bias + nb + j) : 0.f;
      }
    }
    if (act == DLRM_ACT_RELU) {
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
    } else if (act == DLRM_ACT_SIGMOID) {
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = 1.0f / (1.0f + expf(-v[j]));
    }
    // ---------------------------------------------------------------- activation-gradient mask
    if (mask_act != DLRM_ACT_NONE) {
      if (full && mask_vec) {
        const int passes = (mask_act == DLRM_ACT_SIGMOID && mask_lo) ? 2 : 1;
        for (int pass = 0; pass < passes; ++pass) {
          const __nv_bfloat16* src = pass ? mask_lo : mask_hi;
#pragma unroll
          for (int i = 0; i < 4; ++i) {       // 8 rows x 64 B per warp load
            const int row = i * 8 + (lane >> 2), seg = lane & 3;
            uint4 t = make_uint4(0, 0, 0, 0);
            if (mrow0 + row < M) t = *reinterpret_cast<const uint4*>(src + (mrow0 + row) * ldmask + nb + seg * 8);
            *reinterpret_cast<uint4*>(sb + row * TC_EPI_ROW_BF16 + seg * 8) = t;
          }
          __syncwarp();
          __align__(16) __nv_bfloat16 y[32];
#pragma unroll
          for (int q = 0; q < 4; ++q)
            reinterpret_cast<uint4*>(y)[q] = *reinterpret_cast<const uint4*>(sb + lane * TC_EPI_ROW_BF16 + q * 8);
          __syncwarp();
          if (mask_act == DLRM_ACT_RELU) {
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = __bfloat162float(y[j]) > 0.f ? v[j] : 0.f;
          } else if (passes == 1) {
#pragma unroll
            for (int j = 0; j < 32; ++j) { const float yy = __bfloat162float(y[j]); v[j] *= (1.0f - yy) * yy; }
          } else if (pass == 0) {
#pragma unroll
            for (int j = 0; j < 32; ++j) r[j] = __float_as_uint(__bfloat162float(y[j]));   // keep hi, add lo next pass
          } else {
#pragma unroll
            for (int j = 0; j < 32; ++j) {
              const float yy = __uint_as_float(r[j]) + __bfloat162float(y[j]);
              v[j] *= (1.0f - yy) * yy;
            }
          }
        }
      } else if (m_ok) {
        for (int j = 0; j < 32; ++j) {
          if (nb + j < N) {
            const long long o = m * ldmask + nb + j;
            float y = __bfloat162float(mask_hi[o]);
            if (mask_act == DLRM_ACT_RELU) {
              v[j] = y > 0.f ? v[j] : 0.f;
            } else {
              if (mask_lo) y += __bfloat162float(mask_lo[o]);
              v[j] *= (1.0f - y) * y;
            }
          }
        }
      }
    }
    // ---------------------------------------------------------------- fp32 output (+ diverted column)
    if (of32) {
      const bool vec = full && f32_vec && (!ocol || nb + 32 <= col_index);
      const int nrow = (int)min(32ll, M - mrow0);
#pragma unroll
      for (int h = 0; h < 2; ++h) {           // two 16-column passes through the 2560-byte staging tile
#pragma unroll
        for (int q = 0; q < 4; ++q)
          *reinterpret_cast<float4*>(sf + lane * TC_EPI_ROW_F32 + q * 4) =
              make_float4(v[16 * h + 4 * q], v[16 * h + 4 * q + 1], v[16 * h + 4 * q + 2], v[16 * h + 4 * q + 3]);
        __syncwarp();
        if (vec) {
#pragma unroll
          for (int i = 0; i < 4; ++i) {       // 8 rows x 64 B per warp store
            const int row = i * 8 + (lane >> 2), seg = lane & 3;
            if (row < nrow)
              *reinterpret_cast<float4*>(of32 + (mrow0 + row) * ld_f32 + nb + 16 * h + seg * 4) =
                  *reinterpret_cast<const float4*>(sf + row * TC_EPI_ROW_F32 + seg * 4);
          }
        } else {                              // 2 rows x 16 consecutive floats per store
          const long long col = nb + 16 * h + (lane & 15);
          const bool to_col = ocol && col == col_index;
          const bool to_out = col < N && (!ocol || col < col_index);
          for (int row = lane >> 4; row < nrow; row += 2) {
            const float x = sf[row * TC_EPI_ROW_F32 + (lane & 15)];
            if (to_col) ocol[mrow0 + row] = x;
            else if (to_out) of32[(mrow0 + row) * ld_f32 + col] = x;
          }
        }
        __syncwarp();
      }
    }
    // ---------------------------------------------------------------- (hi, lo) bf16 operand outputs
    if (out_hi || outT_hi) {
      __align__(16) __nv_bfloat16 hi[32], lo[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        hi[j] = __float2bfloat16_rn(v[j]);
        lo[j] = __float2bfloat16_rn(v[j] - __bfloat162float(hi[j]));
      }
      if (out_hi) {
        tc_epi_store_bf16(hi, out_hi, ld_out, mrow0, nb, M, N, full && bf_vec, lane, sb);
        if (out_lo) tc_epi_store_bf16(lo, out_lo, ld_out, mrow0, nb, M, N, full && bf_vec, lane, sb);
      }
      if (outT_hi && m_ok) {                  // transposed copy: consecutive lanes = consecutive rows = contiguous
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          if (full || nb + j < N) {
            const long long o = (nb + j) * ld_outT + m;
            outT_hi[o] = hi[j];
            if (outT_lo) outT_lo[o] = lo[j];
          }
        }
      }
    }
  }
}

struct TcPlan {
  CUtensorMap tmAh, tmAl, tmBh, tmBl;
  TcArgs args;
  int bm, bn, stages, splits;
  size_t smem;
  dim3 grid;
};

}  // namespace dlrm
