// Embedding backward + sparse optimizer for TINY tables (a few to a few hundred rows).
//
// The MLPerf-DLRM table list (torchrec_dlrm/README.MD:45) holds tables of 3, 4, 10, 14, 36, 63, 108 and
// 155 rows.  At a global batch of 65536 every one of their rows is hit hundreds to tens of thousands of times
// per step, so the list walk of emb_bwd.cu (one warp follows the occurrences of a row one link at a time)
// would serialise: 21845 dependent hops for a row of the 3-row table.  grad.coalesce() + the row update
// (optim/rwsadagrad.py:117-143) is done here as a dense, deterministic two-pass reduction instead:
//
//   accumulate : grid = (sample chunks, tables).  The CTA keeps a private [rows, dim] fp32 accumulator in
//                shared memory.  Warp w owns the rows r with r % 8 == w: every warp scans the chunk's index
//                stream (coalesced, 32 indices per load), compacts the positions whose row it owns with a
//                ballot and adds their dY rows (512-byte warp loads, up to 8 in flight) in sample order --
//                each dY row is read once, no atomics, a fixed summation order.  The accumulator is written
//                to partial[chunk][row][:].
//   apply      : one warp per row: sum the chunk partials in chunk order (= ascending position, the order
//                grad.coalesce() sums duplicates in), then the same row update as emb_update_kernel.
//                Rows nobody touched see g = 0 and are left bit-identical.
#include "common.cuh"

namespace dlrm {

constexpr int SMALL_CHUNK = 128;        // samples per accumulate CTA (512 would leave 16 chunks x 8 tables at MLPerf batch 8192: too few CTAs to fill the SMs)
constexpr int SMALL_MAX_TABLES = 32;

struct SmallTable {
  float* w;
  float* mom;
  const void* idx;
  const void* off;
  long long nnz;
  long long ld, mom_stride;
  long long dy_off;
  long long row_lo;
  int row_n;
  int part_row0;        // first row of this table in the partial buffer's row space
};

struct SmallParams {
  SmallTable t[SMALL_MAX_TABLES];
  const float* dY;
  long long dy_stride_sample;
  const float* peer_dY[DLRM_B200_MAX_PEERS];
  long long peer_batch;
  long long batch;
  int dim, include_last, optimizer;
  float lr, eps;
  float* partial;       // [chunks][total small rows][dim]
  int total_rows, chunks;
};

__device__ __forceinline__ const float* small_dy_row(const SmallParams& P, long long bag) {
  if (P.peer_batch > 0) {
    const int src = (int)(bag / P.peer_batch);
    return P.peer_dY[src] + (bag - src * P.peer_batch) * P.dy_stride_sample;
  }
  return P.dY + bag * P.dy_stride_sample;
}

// NV float4 per lane: dim = 128 * NV (columns >= dim masked)
template <int NV, typename idx_t>
__global__ void __launch_bounds__(256) emb_small_accum_kernel(const __grid_constant__ SmallParams P) {
  extern __shared__ __align__(16) float acc[];   // [row_n][dim]
  const SmallTable& tb = P.t[blockIdx.y];
  const int D = P.dim;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const idx_t* __restrict__ idx = static_cast<const idx_t*>(tb.idx);
  const idx_t* __restrict__ off = static_cast<const idx_t*>(tb.off);
  for (int e = threadIdx.x; e < tb.row_n * D; e += blockDim.x) acc[e] = 0.f;
  __syncthreads();
  const long long b0 = (long long)blockIdx.x * SMALL_CHUNK;
  const long long b1 = min(P.batch, b0 + SMALL_CHUNK);
  if (b0 < b1) {
    // positions of this chunk: [off[b0], end of bag b1-1)
    const long long p0 = (long long)off[b0];
    const long long p1 = (P.include_last || b1 < P.batch) ? (long long)off[b1] : tb.nnz;
    long long bag_lo = b0;     // bag of the first position of the current 32-wide window (monotone)
    for (long long w0 = p0; w0 < p1; w0 += 32) {
      const long long pos = w0 + lane;
      long long r = -1;
      long long bag = 0;
      if (pos < p1) {
        r = (long long)idx[pos] - tb.row_lo;
        // bag of pos: largest b in [bag_lo, b1) with off[b] <= pos (bags are short: linear probe from a
        // binary-search start is overkill for L = 1; plain binary search over the chunk)
        long long lo = bag_lo, hi = b1 - 1;
        while (lo < hi) {
          const long long mid = (lo + hi + 1) >> 1;
          if ((long long)off[mid] <= pos) lo = mid; else hi = mid - 1;
        }
        bag = lo;
      }
      const bool mine = r >= 0 && r < tb.row_n && (int)(r & 7) == warp;
      unsigned live = __ballot_sync(0xffffffffu, mine);
      bag_lo = __shfl_sync(0xffffffffu, bag, 0);
      while (live) {
        float4 val[8][NV];
        int row[8];
        bool on[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          on[u] = live != 0u;
          const int src = on[u] ? __ffs(live) - 1 : 0;
          live &= live - 1u;
          const long long bg = __shfl_sync(0xffffffffu, bag, src);
          row[u] = (int)__shfl_sync(0xffffffffu, r, src);
          if (on[u]) {
            const float* gp = small_dy_row(P, bg) + tb.dy_off + lane * 4;
#pragma unroll
            for (int v = 0; v < NV; ++v)
              if (lane * 4 + v * 128 < D) val[u][v] = *reinterpret_cast<const float4*>(gp + v * 128);
          }
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          if (on[u]) {
            float* a = acc + (size_t)row[u] * D + lane * 4;
#pragma unroll
            for (int v = 0; v < NV; ++v) {
              if (lane * 4 + v * 128 < D) {
                float4 t = *reinterpret_cast<float4*>(a + v * 128);
                t.x += val[u][v].x; t.y += val[u][v].y; t.z += val[u][v].z; t.w += val[u][v].w;
                *reinterpret_cast<float4*>(a + v * 128) = t;
              }
            }
          }
        }
      }
    }
  }
  __syncthreads();
  float* dst = P.partial + ((size_t)blockIdx.x * P.total_rows + tb.part_row0) * D;
  for (int e = threadIdx.x * 4; e < tb.row_n * D; e += blockDim.x * 4)
    *reinterpret_cast<float4*>(dst + e) = *reinterpret_cast<const float4*>(acc + e);
}

template <int NV>
__global__ void __launch_bounds__(256) emb_small_apply_kernel(const __grid_constant__ SmallParams P, int num_tables) {
  const int lane = threadIdx.x & 31;
  const int grow = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);   // row in the partial row space
  if (grow >= P.total_rows) return;
  int k = 0;
  while (k + 1 < num_tables && grow >= P.t[k + 1].part_row0) ++k;
  const SmallTable& tb = P.t[k];
  const int r = grow - tb.part_row0;
  const int D = P.dim;
  float4 g[NV];
#pragma unroll
  for (int v = 0; v < NV; ++v) g[v] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int c = 0; c < P.chunks; ++c) {      // fixed order: chunk 0 first (ascending sample = ascending position)
    const float* p = P.partial + ((size_t)c * P.total_rows + grow) * D + lane * 4;
#pragma unroll
    for (int v = 0; v < NV; ++v)
      if (lane * 4 + v * 128 < D) {
        const float4 t = *reinterpret_cast<const float4*>(p + v * 128);
        g[v].x += t.x; g[v].y += t.y; g[v].z += t.z; g[v].w += t.w;
      }
  }
  float* wrow = tb.w + (long long)r * tb.ld + lane * 4;
  const float nlr = -P.lr;
  if (P.optimizer == DLRM_OPT_RWSADAGRAD) {
    float sq = 0.f;
#pragma unroll
    for (int v = 0; v < NV; ++v)
      if (lane * 4 + v * 128 < D)
        sq = fmaf(g[v].x, g[v].x, fmaf(g[v].y, g[v].y, fmaf(g[v].z, g[v].z, fmaf(g[v].w, g[v].w, sq))));
    sq = warp_sum(sq);
    if (sq == 0.f) return;                  // untouched row (or an all-zero gradient): nothing changes
    const float m_new = tb.mom[(long long)r * tb.mom_stride] + sq * (1.0f / (float)D);
    const float stdv = sqrtf(m_new) + P.eps;
#pragma unroll
    for (int v = 0; v < NV; ++v)
      if (lane * 4 + v * 128 < D) {
        float4 w = *reinterpret_cast<float4*>(wrow + v * 128);
        w.x = fmaf(nlr, g[v].x / stdv, w.x); w.y = fmaf(nlr, g[v].y / stdv, w.y);
        w.z = fmaf(nlr, g[v].z / stdv, w.z); w.w = fmaf(nlr, g[v].w / stdv, w.w);
        *reinterpret_cast<float4*>(wrow + v * 128) = w;
      }
    if (lane == 0) tb.mom[(long long)r * tb.mom_stride] = m_new;
  } else {
#pragma unroll
    for (int v = 0; v < NV; ++v)
      if (lane * 4 + v * 128 < D) {
        float4 w = *reinterpret_cast<float4*>(wrow + v * 128);
        w.x = fmaf(nlr, g[v].x, w.x); w.y = fmaf(nlr, g[v].y, w.y);
        w.z = fmaf(nlr, g[v].z, w.z); w.w = fmaf(nlr, g[v].w, w.w);
        *reinterpret_cast<float4*>(wrow + v * 128) = w;
      }
  }
}

}  // namespace dlrm

extern "C" int64_t dlrm_b200_emb_bwd_small_scratch_bytes(int64_t total_small_rows, int dim, int64_t batch) {
  const int64_t chunks = (batch + dlrm::SMALL_CHUNK - 1) / dlrm::SMALL_CHUNK;
  return chunks * total_small_rows * dim * 4;
}

extern "C" int dlrm_b200_emb_bwd_small_update(const dlrm_emb_bwd_table_t* tables, int num_tables, int dim,
                                              int64_t batch, int idx_bytes, int include_last, const float* dY,
                                              const float* const* peer_dY, int world, int64_t batch_local,
                                              int64_t dy_stride_sample, int optimizer, float lr, float eps,
                                              float* scratch, int64_t scratch_bytes, void* stream) {
  using namespace dlrm;
  if (num_tables == 0 || batch == 0) return 0;
  if (num_tables < 0 || num_tables > SMALL_MAX_TABLES) return set_error("emb_bwd_small_update: num_tables=%d (max %d)", num_tables, SMALL_MAX_TABLES);
  if (idx_bytes != 4 && idx_bytes != 8) return set_error("emb_bwd_small_update: idx_bytes=%d", idx_bytes);
  if (optimizer != DLRM_OPT_SGD && optimizer != DLRM_OPT_RWSADAGRAD) return set_error("emb_bwd_small_update: optimizer=%d", optimizer);
  if (dim <= 0 || dim % 4 || dim > 512) return set_error("emb_bwd_small_update: dim=%d (multiple of 4, <= 512)", dim);
  if (!tables || !scratch || (!dY && !peer_dY)) return set_error("emb_bwd_small_update: NULL pointer");
  if (dy_stride_sample % 4) return set_error("emb_bwd_small_update: dY rows must be 16-byte aligned");
  SmallParams P{};
  int total_rows = 0, max_rows = 0;
  for (int k = 0; k < num_tables; ++k) {
    const dlrm_emb_bwd_table_t& s = tables[k];
    if (!s.weight || !s.offsets || (!s.indices && s.nnz > 0)) return set_error("emb_bwd_small_update: table %d NULL pointer", k);
    if (optimizer == DLRM_OPT_RWSADAGRAD && !s.momentum) return set_error("emb_bwd_small_update: table %d momentum NULL", k);
    const int64_t rn = s.row_n > 0 ? s.row_n : s.rows;
    if (rn <= 0 || rn > 4096) return set_error("emb_bwd_small_update: table %d has %lld rows (1..4096)", k, (long long)rn);
    if (!s.use_dy_off || s.dy_off % 4) return set_error("emb_bwd_small_update: table %d needs a 16-byte aligned dy_off", k);
    SmallTable& t = P.t[k];
    t.w = s.weight; t.mom = s.momentum; t.idx = s.indices; t.off = s.offsets; t.nnz = s.nnz;
    t.ld = s.ld > 0 ? s.ld : dim; t.mom_stride = s.mom_stride > 0 ? s.mom_stride : 1;
    t.dy_off = s.dy_off; t.row_lo = s.row_n > 0 ? s.row_lo : 0; t.row_n = (int)rn; t.part_row0 = total_rows;
    if (t.ld % 4 || (reinterpret_cast<uintptr_t>(t.w) & 15)) return set_error("emb_bwd_small_update: table %d rows not 16-byte aligned", k);
    total_rows += (int)rn;
    max_rows = (int)rn > max_rows ? (int)rn : max_rows;
  }
  const size_t smem = (size_t)max_rows * dim * 4;
  if (smem > 200 * 1024) return set_error("emb_bwd_small_update: %d rows x dim %d do not fit shared memory", max_rows, dim);
  const int chunks = (int)((batch + SMALL_CHUNK - 1) / SMALL_CHUNK);
  if ((int64_t)chunks * total_rows * dim * 4 > scratch_bytes)
    return set_error("emb_bwd_small_update: scratch %lld B < %lld B", (long long)scratch_bytes, (long long)chunks * total_rows * dim * 4);
  P.dY = dY; P.dy_stride_sample = dy_stride_sample; P.peer_batch = 0;
  if (peer_dY) {
    if (world < 1 || world > DLRM_B200_MAX_PEERS || batch_local <= 0 || batch_local * world != batch)
      return set_error("emb_bwd_small_update: world=%d batch_local=%lld batch=%lld", world, (long long)batch_local, (long long)batch);
    for (int d = 0; d < world; ++d) {
      if (!peer_dY[d]) return set_error("emb_bwd_small_update: peer %d pointer is NULL", d);
      P.peer_dY[d] = peer_dY[d];
    }
    P.peer_batch = batch_local;
  }
  P.batch = batch; P.dim = dim; P.include_last = include_last; P.optimizer = optimizer; P.lr = lr; P.eps = eps;
  P.partial = scratch; P.total_rows = total_rows; P.chunks = chunks;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int nv = (dim + 127) / 128;
#define SMALL_LAUNCH(NV, IDX)                                                                                         \
  do {                                                                                                                \
    if (smem > 48 * 1024)                                                                                             \
      DLRM_CUDA(cudaFuncSetAttribute(emb_small_accum_kernel<NV, IDX>, cudaFuncAttributeMaxDynamicSharedMemorySize,     \
                                     200 * 1024));                                                                    \
    emb_small_accum_kernel<NV, IDX><<<dim3((unsigned)chunks, (unsigned)num_tables), 256, smem, st>>>(P);              \
    DLRM_CHECK_LAUNCH("emb_small_accum_kernel");                                                                      \
    emb_small_apply_kernel<NV><<<(unsigned)((total_rows + 7) / 8), 256, 0, st>>>(P, num_tables);                      \
    DLRM_CHECK_LAUNCH("emb_small_apply_kernel");                                                                      \
    return 0;                                                                                                         \
  } while (0)
  if (idx_bytes == 8) {
    if (nv == 1) SMALL_LAUNCH(1, long long);
    if (nv == 2) SMALL_LAUNCH(2, long long);
    SMALL_LAUNCH(4, long long);
  }
  if (nv == 1) SMALL_LAUNCH(1, int);
  if (nv == 2) SMALL_LAUNCH(2, int);
  SMALL_LAUNCH(4, int);
#undef SMALL_LAUNCH
}
