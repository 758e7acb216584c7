// wgmma / TMA GEMM for the MLP layers (forward, dgrad, wgrad) on sm_90a.
//
//   D[M,N] = sum_k A(m,k) * B(n,k)        bf16 operands, fp32 accumulation in registers.
//
// Precision modes
//   BF16   : one MMA per k-step (operands rounded to bf16).
//   BF16X3 : fp32-grade result from bf16 tensor cores.  Every fp32 operand x is stored as the pair
//            hi = bf16(x), lo = bf16(x - hi); the kernel issues hi*hi + hi*lo + lo*hi per k-step
//            (the dropped lo*lo and residual terms are <= 2^-16 relative per product), which keeps
//            the logits within 1e-5 of the reference's fp32 CPU forward (BASELINE.json north_star;
//            measured in tests/test_gpu_gemm_tc.py).  4 operand tiles per stage instead of 2.
//
// Structure (one 128 x BN output tile per CTA, optional split-K over gridDim.z):
//   warp 0      : TMA producer -- cp.async.bulk.tensor.2d into a 128B-swizzled smem ring, mbarrier
//                 complete_tx signalling.
//   warps 4..11 : two consumer warpgroups; warpgroup w issues wgmma.mma_async m64nBNk16 for rows
//                 [64 w, 64 w + 64) of the tile and releases each ring stage once its wgmmas retire.
//                 Then the accumulators go through shared memory to the epilogue on the same 8 warps:
//                 fused bias / activation / activation-gradient mask, fp32 and/or (hi,lo) bf16 stores
//                 in normal and transposed layout (the operand layouts of the next GEMMs).
// Operands may be K-major ([rows, K] with K contiguous) or MN-major ([K, rows] with rows
// contiguous, e.g. dY^T read straight from dY): the smem descriptors and the wgmma transpose
// immediates carry the majorness, so no transposed copy is needed for MN-major inputs.
#include <string.h>

#include "gemm_tc_common.cuh"

namespace dlrm {

// ------------------------------------------------------------------------------------------ kernel
// smem per stage: A_hi [A_lo] B_hi [B_lo]; every tile 1024-byte aligned.
template <int BN>
__global__ void __launch_bounds__(TC_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmAh, const __grid_constant__ CUtensorMap tmAl,
               const __grid_constant__ CUtensorMap tmBh, const __grid_constant__ CUtensorMap tmBl,
               const TcArgs g, int stages) {
#define TCB_BX blockIdx.x
#define TCB_BY blockIdx.y
#define TCB_BZ blockIdx.z
#define TCB_MAP_AH (&tmAh)
#define TCB_MAP_AL (&tmAl)
#define TCB_MAP_BH (&tmBh)
#define TCB_MAP_BL (&tmBl)
#include "gemm_tc_body.cuh"
#undef TCB_BX
#undef TCB_BY
#undef TCB_BZ
#undef TCB_MAP_AH
#undef TCB_MAP_AL
#undef TCB_MAP_BH
#undef TCB_MAP_BL
}

// ------------------------------------------------------------------------------------------ host
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// 2-D bf16 tensor [outer, inner] with `ld` elements between outer rows; box {box_inner, box_outer}
static int make_map(CUtensorMap* map, const void* ptr, long long inner, long long outer, long long ld,
                    int box_inner, int box_outer) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return set_error("gemm_tc: cuTensorMapEncodeTiled not available");
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) || (ld * 2) % 16)
    return set_error("gemm_tc: operand pointer/ld not 16-byte aligned (ld=%lld)", ld);
  cuuint64_t dims[2] = {(cuuint64_t)inner, (cuuint64_t)outer};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {(cuuint32_t)box_inner, (cuuint32_t)box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error("gemm_tc: cuTensorMapEncodeTiled failed (%d)", (int)r);
  return 0;
}


template <int BN>
static int launch_tc(const TcPlan& p, cudaStream_t st) {
  static bool configured = false;
  if (!configured) {
    DLRM_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_MAX_SMEM));
    configured = true;
  }
  (void)launch_chain(gemm_tc_kernel<BN>, p.grid, dim3(TC_THREADS), p.smem, st, p.tmAh, p.tmAl, p.tmBh, p.tmBl, p.args, p.stages);
  DLRM_CHECK_LAUNCH("gemm_tc_kernel");
  return 0;
}

}  // namespace dlrm

extern "C" int dlrm_b200_gemm_tc_plan_create(const dlrm_gemm_tc_desc_t* d, void** plan_out) {
  using namespace dlrm;
  if (!d || !plan_out) return set_error("gemm_tc_plan_create: NULL argument");
  if (d->M <= 0 || d->N <= 0 || d->K <= 0) return set_error("gemm_tc: empty problem M=%lld N=%lld K=%lld", (long long)d->M, (long long)d->N, (long long)d->K);
  if (!d->A_hi || !d->B_hi || (d->mode_x3 && (!d->A_lo || !d->B_lo)))
    return set_error("gemm_tc: NULL operand");
  TcPlan* p = new TcPlan();
  TcArgs& a = p->args;
  a.M = d->M; a.N = d->N; a.K = d->K;
  a.x3 = d->mode_x3 ? 1 : 0;
  a.a_mn = d->a_mn_major ? 1 : 0;
  a.b_mn = d->b_mn_major ? 1 : 0;
  a.act = d->act; a.mask_act = d->mask_act;
  a.mask_hi = static_cast<const __nv_bfloat16*>(d->mask_hi);
  a.mask_lo = static_cast<const __nv_bfloat16*>(d->mask_lo);
  a.ldmask = d->ldmask;
  a.out_f32 = d->out_f32; a.ld_f32 = d->ld_f32; a.slab_stride = d->slab_stride;
  a.out_hi = static_cast<__nv_bfloat16*>(d->out_hi); a.out_lo = static_cast<__nv_bfloat16*>(d->out_lo);
  a.ld_out = d->ld_out;
  a.outT_hi = static_cast<__nv_bfloat16*>(d->outT_hi); a.outT_lo = static_cast<__nv_bfloat16*>(d->outT_lo);
  a.ld_outT = d->ld_outT;
  a.out_col = d->out_col; a.col_index = d->col_index; a.col_slab_stride = d->col_slab_stride;
  a.bias = d->bias;
  if (a.mask_act != DLRM_ACT_NONE && !a.mask_hi) { delete p; return set_error("gemm_tc: mask_act without mask_hi"); }
  // the diverted column is stored by the fp32 store path, and every column right of it would be dropped
  if (a.out_col && !a.out_f32) { delete p; return set_error("gemm_tc: out_col needs out_f32"); }
  if (a.out_col && a.col_index != a.N - 1) {
    delete p;
    return set_error("gemm_tc: out_col diverts the last column: col_index=%lld, N=%lld", (long long)a.col_index, (long long)a.N);
  }
  if (a.out_hi && (a.ld_out % 8)) { delete p; return set_error("gemm_tc: ld_out must be a multiple of 8"); }
  // tile width: keep >= ~64 CTAs when N is small
  const long long mt = (d->M + TC_BM - 1) / TC_BM;
  int bn = 128;
  if (d->tile_n == 32 || d->tile_n == 64 || d->tile_n == 128) bn = d->tile_n;
  else {
    while (bn > 32 && mt * ((d->N + bn - 1) / bn) < 96) bn >>= 1;
    if (d->N <= 32) bn = 32; else if (d->N <= 64 && bn > 64) bn = 64;
  }
  if (a.b_mn && bn < 64) bn = 64;  // MN-major boxes are 64 wide
  // operand-ring budget (default 200 KB, the deepest ring).  The accumulator is staged in the ring once the last
  // wgmma has retired, so only the barriers and the epilogue's per-warp staging sit beside it.  A smaller budget
  // no longer lets two CTAs share an SM: 384 threads at ~160 registers take more than half the register file.
  int budget_kb = get_tunable(TUNE_GEMM_SMEM_KB);
  if (budget_kb <= 0 || budget_kb > 200) budget_kb = 200;
  if (budget_kb < 48) budget_kb = 48;
  const size_t ring_cap = TC_MAX_SMEM - (256 + TC_EPI_BYTES + 1024);
  const size_t ring_budget = (size_t)budget_kb * 1024 < ring_cap ? (size_t)budget_kb * 1024 : ring_cap;
  if (!(d->tile_n == 128) && bn == 128 &&
      ring_budget < 2 * (size_t)(a.x3 ? 2 : 1) * (TC_BM * TC_BK * 2 + 128 * TC_BK * 2))
    bn = 64;                       // two stages of a 128-wide tile would not fit the budget
  p->bn = bn;
  a.num_kb = (int)((d->K + TC_BK - 1) / TC_BK);
  int splits = d->split_k > 1 ? d->split_k : 1;
  if (splits > a.num_kb) splits = a.num_kb;
  a.kb_per_split = (a.num_kb + splits - 1) / splits;
  splits = (a.num_kb + a.kb_per_split - 1) / a.kb_per_split;  // no empty split
  p->splits = splits;
  if (splits > 1 && (a.out_hi || a.outT_hi || a.act != DLRM_ACT_NONE || a.mask_act != DLRM_ACT_NONE || a.bias)) {
    delete p; return set_error("gemm_tc: split-K only supports fp32 slab outputs");
  }
  const size_t stage_bytes = (size_t)(a.x3 ? 2 : 1) * (TC_BM * TC_BK * 2 + bn * TC_BK * 2);
  int stages = (int)(ring_budget / stage_bytes);
  if (stages > 8) stages = 8;
  if (stages < 2) stages = 2;
  if (stages > a.kb_per_split) stages = a.kb_per_split < 2 ? 2 : a.kb_per_split;
  p->stages = stages;
  // ring (also holds the staged accumulator) | barriers (<= 256 B) | per-warp staging | alignment
  p->smem = tc_ring_bytes(stages * stage_bytes, bn) + 256 + TC_EPI_BYTES + 1024;
  if (p->smem > (size_t)TC_MAX_SMEM) { delete p; return set_error("gemm_tc: %zu bytes of shared memory", p->smem); }
  p->grid = dim3((unsigned)((d->N + bn - 1) / bn), (unsigned)mt, (unsigned)splits);
  int rc = 0;
  // operand maps.  K-major: tensor [rows, K]; MN-major: tensor [K, rows].
  if (!a.a_mn) {
    rc |= make_map(&p->tmAh, d->A_hi, d->K, d->M, d->lda, TC_BK, TC_BM);
    rc |= make_map(&p->tmAl, a.x3 ? d->A_lo : d->A_hi, d->K, d->M, d->lda, TC_BK, TC_BM);
  } else {
    rc |= make_map(&p->tmAh, d->A_hi, d->M, d->K, d->lda, 64, TC_BK);
    rc |= make_map(&p->tmAl, a.x3 ? d->A_lo : d->A_hi, d->M, d->K, d->lda, 64, TC_BK);
  }
  if (!a.b_mn) {
    rc |= make_map(&p->tmBh, d->B_hi, d->K, d->N, d->ldb, TC_BK, bn);
    rc |= make_map(&p->tmBl, a.x3 ? d->B_lo : d->B_hi, d->K, d->N, d->ldb, TC_BK, bn);
  } else {
    rc |= make_map(&p->tmBh, d->B_hi, d->N, d->K, d->ldb, 64, TC_BK);
    rc |= make_map(&p->tmBl, a.x3 ? d->B_lo : d->B_hi, d->N, d->K, d->ldb, 64, TC_BK);
  }
  if (rc) { delete p; return -1; }
  *plan_out = p;
  return 0;
}

extern "C" int dlrm_b200_gemm_tc_plan_info(void* plan, int* tile_n, int* stages, int* splits, int* ctas) {
  using namespace dlrm;
  if (!plan) return set_error("gemm_tc_plan_info: NULL plan");
  TcPlan* p = static_cast<TcPlan*>(plan);
  if (tile_n) *tile_n = p->bn;
  if (stages) *stages = p->stages;
  if (splits) *splits = p->splits;
  if (ctas) *ctas = (int)(p->grid.x * p->grid.y * p->grid.z);
  return 0;
}

extern "C" int dlrm_b200_gemm_tc_run(void* plan, void* stream) {
  using namespace dlrm;
  if (!plan) return set_error("gemm_tc_run: NULL plan");
  TcPlan* p = static_cast<TcPlan*>(plan);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (p->bn == 128) return launch_tc<128>(*p, st);
  if (p->bn == 64) return launch_tc<64>(*p, st);
  return launch_tc<32>(*p, st);
}

extern "C" int dlrm_b200_gemm_tc_plan_destroy(void* plan) {
  delete static_cast<dlrm::TcPlan*>(plan);
  return 0;
}
