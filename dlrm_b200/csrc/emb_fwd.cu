// Batched multi-table EmbeddingBag(sum) forward -- replaces the T separate
// nn.EmbeddingBag calls of DLRM_Net.apply_emb (dlrm_s_pytorch.py:407-462).
//
// One launch covers every table.  A "lane group" of G = dim/4 lanes (32 for dim 128) owns a
// bag: each lane keeps ONE float4 accumulator per 4G columns and adds the rows of the bag in
// index order, so the result is bit-identical to the reference CPU kernel (sequential fp32).
// A row of dim 128 is a single 512-byte, fully coalesced warp request (4 x 128B lines).
// Memory-level parallelism comes from (a) up to U rows in flight per group (indices are read
// with one coalesced load per G positions and broadcast with warp shuffles), (b) the indices
// of the next bag being prefetched while the rows of the current bag are in flight, and
// (c) 8..16 warps per CTA x many CTAs per SM.
#include "common.cuh"

namespace dlrm {

struct EmbFwdTable {
  const float* w;
  const void* idx;
  const void* off;
  const float* rw;
  long long nnz;
  int* head;            // training: per-row list heads of this table (see emb_bwd.cu); null = do not link
  long long hs;         // elements between the list heads of consecutive rows (1, or the row stride when the
                        // head lives inside the row's own DRAM page: [weights | accumulator | head | pad])
  long long pair_base;  // training: first slot of this table in link[]
  long long ld;         // row stride in floats
  long long out_off;    // pooled row of bag b goes to out_row(b) [+ b_local * out_stride] + out_off
  long long out_stride; // elements between consecutive samples of THIS table's output
  long long rows;       // rows of the whole table: an index outside [0, rows) is an error
  long long row_lo;     // this shard stores rows [row_lo, row_lo + row_n) at local index (row - row_lo)
  long long row_n;
};

struct EmbFwdParams {
  EmbFwdTable t[DLRM_B200_MAX_TABLES_PER_CALL];
  float* out;
  long long stride_sample;
  long long stride_table;
  long long batch;
  int dim;
  int include_last;
  int bags_per_group;
  int2* link;  // training: link[pos] = {previous head of the row, bag}
  // table-wise sharded runs: bag b belongs to rank b / peer_batch and its pooled row is stored straight
  // into that rank's buffer through peer-mapped memory (NVLink store).  peer_batch == 0: local output.
  float* peer_out[DLRM_B200_MAX_PEERS];
  long long peer_batch;
  unsigned* filter;   // training with a duplicate filter: count instead of linking
  int filter_log2;
  unsigned* err;      // device error word: bit 0 = an index was outside its table
};

// training: either thread the occurrence onto its row's list (returns the previous head) or, with a
// duplicate filter, just bump the row's hashed counter (no return value -> RED, nothing to wait for)
__device__ __forceinline__ int note_occurrence(const EmbFwdParams& P, const EmbFwdTable& tb, long long row,
                                               long long pos_local) {
  if (P.filter) {
    atomicAdd(P.filter + filter_slot(tb.head + row * tb.hs, P.filter_log2), 1u);
    return 0;
  }
  return atomicExch(tb.head + row * tb.hs, (int)(tb.pair_base + pos_local + 1));
}

// Where the pooled row of (table tb, global bag b) goes: buffer of the rank that owns the sample (peer-mapped
// on a sharded run), sample-local row, per-table offset/stride (whole tables land in feature slot 1+t of the
// interaction operand, row-split shards in their slab of the partial-sum area behind it).
__device__ __forceinline__ float* out_ptr(const EmbFwdParams& P, const EmbFwdTable& tb, long long b) {
  if (P.peer_batch > 0) {
    const int dst = (int)(b / P.peer_batch);
    return P.peer_out[dst] + (b - dst * P.peer_batch) * tb.out_stride + tb.out_off;
  }
  return P.out + b * tb.out_stride + tb.out_off;
}

__device__ __forceinline__ void flag_bad_index(const EmbFwdParams& P) {
  if (P.err) atomicOr(P.err, 1u);
}



template <typename idx_t>
__device__ __forceinline__ long long bag_end(const idx_t* off, long long b, long long batch,
                                             long long nnz, int include_last) {
  return (include_last || b + 1 < batch) ? (long long)off[b + 1] : nnz;
}

// G lanes per bag, NV float4 per lane (dim = 4*G*NV when exact; columns >= dim are masked).
// grid = (groups of S bags, table): a plain grid at 64 registers / 4 CTAs per SM rather than a persistent one-wave
// grid with more registers per thread -- the gather is latency-bound, so resident warps matter most.
template <int G, int NV, int U, typename idx_t, bool WEIGHTED, bool LINK>
__global__ void __launch_bounds__(256, (G == 32 && NV == 1) ? 4 : 1) emb_fwd_vec_kernel(
    const __grid_constant__ EmbFwdParams P, int num_tables) {
  const int D = P.dim;
  constexpr int GROUPS_PER_WARP = 32 / G;
  const int lane = threadIdx.x & 31;
  const int gl = lane % G;   // lane inside the group
  const int grp = lane / G;  // group inside the warp
  const unsigned gmask = (G == 32) ? 0xffffffffu : (((1u << G) - 1u) << (grp * G));
  const int S = P.bags_per_group;
  const int table = blockIdx.y;
  {
    const EmbFwdTable& tb = P.t[table];
    const idx_t* __restrict__ idx = static_cast<const idx_t*>(tb.idx);
    const idx_t* __restrict__ off = static_cast<const idx_t*>(tb.off);
    const float* __restrict__ W = tb.w;
    const long long b0 =
        (((long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * GROUPS_PER_WARP + grp) * S;
    if (b0 >= P.batch) return;
    const int nb = (int)min((long long)S, P.batch - b0);

    // bag boundaries of this run of bags: one coalesced load, then shuffles (S < G, host-enforced).
    // positions inside one call fit 31 bits (host-checked: nnz < 2^31); rows stay 64-bit
    int my_bound = 0;
    if (gl <= nb) {
      const long long b = b0 + gl;
      my_bound = (b < P.batch) ? (int)off[b] : 0;
      if (gl == nb) my_bound = (int)bag_end<idx_t>(off, b - 1, P.batch, tb.nnz, P.include_last);
    }
    int start = __shfl_sync(gmask, my_bound, 0, G);
    int end = __shfl_sync(gmask, my_bound, 1, G);
    // first index chunk of bag 0 (+ fused link: the atomic's result is only stored after the rows)
    // an index outside the table is reported through the error word and read as row 0 (never out of bounds)
    long long my_row = (start + gl < end) ? (long long)idx[start + gl] : 0;
    bool bad = (unsigned long long)my_row >= (unsigned long long)tb.rows;   // never linked, never updated
    if (bad) { flag_bad_index(P); my_row = 0; }
    int my_prev = 0;
    const bool link_tb = LINK && tb.head != nullptr;
    if (link_tb && start + gl < end && !bad) my_prev = note_occurrence(P, tb, my_row, start + gl);

    for (int s = 0; s < nb; ++s) {
      // prefetch boundaries + first index chunk of the next bag
      int nstart = 0, nend = 0, next_prev = 0;
      long long next_row = 0;
      if (s + 1 < nb) {
        nstart = end;
        nend = __shfl_sync(gmask, my_bound, s + 2, G);
        next_row = (nstart + gl < nend) ? (long long)idx[nstart + gl] : 0;
        bad = (unsigned long long)next_row >= (unsigned long long)tb.rows;
        if (bad) { flag_bad_index(P); next_row = 0; }
        if (link_tb && nstart + gl < nend && !bad)
          next_prev = note_occurrence(P, tb, next_row, nstart + gl);
      }
      float4 acc[NV];
#pragma unroll
      for (int v = 0; v < NV; ++v) acc[v] = make_float4(0.f, 0.f, 0.f, 0.f);

      for (int j0 = start; j0 < end; j0 += G) {
        if (j0 != start) {
          my_row = (j0 + gl < end) ? (long long)idx[j0 + gl] : 0;
          bad = (unsigned long long)my_row >= (unsigned long long)tb.rows;
          if (bad) { flag_bad_index(P); my_row = 0; }
          my_prev = (link_tb && j0 + gl < end && !bad) ? note_occurrence(P, tb, my_row, j0 + gl) : 0;
        }
        const int n = min(G, end - j0);
        for (int jj = 0; jj < n; jj += U) {
          float4 val[U][NV];
          float wgt[U];
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const long long r = __shfl_sync(gmask, my_row, jj + u, G);  // jj+u < G always (U | G)
            if (jj + u < n) {
              const float* rp = W + r * tb.ld + gl * 4;
#pragma unroll
              for (int v = 0; v < NV; ++v) {
                if (gl * 4 + v * G * 4 < D) val[u][v] = ldg_stream_f4(rp + v * G * 4);
              }
              if (WEIGHTED) wgt[u] = __ldg(tb.rw + r);
            }
          }
#pragma unroll
          for (int u = 0; u < U; ++u) {
            if (jj + u < n) {
#pragma unroll
              for (int v = 0; v < NV; ++v) {
                if (WEIGHTED) {
                  acc[v].x = fmaf(wgt[u], val[u][v].x, acc[v].x);
                  acc[v].y = fmaf(wgt[u], val[u][v].y, acc[v].y);
                  acc[v].z = fmaf(wgt[u], val[u][v].z, acc[v].z);
                  acc[v].w = fmaf(wgt[u], val[u][v].w, acc[v].w);
                } else {
                  acc[v].x += val[u][v].x;
                  acc[v].y += val[u][v].y;
                  acc[v].z += val[u][v].z;
                  acc[v].w += val[u][v].w;
                }
              }
            }
          }
        }
        if (link_tb && j0 + gl < end)
          P.link[tb.pair_base + j0 + gl] = make_int2(my_prev, (int)(b0 + s));
      }
      float* op = out_ptr(P, tb, b0 + s) + gl * 4;
#pragma unroll
      for (int v = 0; v < NV; ++v) {
        if (gl * 4 + v * G * 4 < D) *reinterpret_cast<float4*>(op + v * G * 4) = acc[v];
      }
      start = nstart;
      end = nend;
      my_row = next_row;
      my_prev = next_prev;
    }
  }
}

// Row-split shard: this rank stores rows [row_lo, row_lo + row_n) of the table and pools, for EVERY bag of the
// global batch, only the indices that fall into its range (a partial sum; the N partials of a bag are added on the
// rank that owns the sample).  The indices of a 32-wide chunk that are "mine" are compacted with a ballot so
// that up to U row loads stay in flight however sparse the hits are (L = 100 over 8 shards: ~4 of 32).
template <int G, int NV, int U, typename idx_t, bool WEIGHTED, bool LINK>
__global__ void __launch_bounds__(256) emb_fwd_shard_kernel(const __grid_constant__ EmbFwdParams P, int num_tables) {
  const int D = P.dim;
  constexpr int GROUPS_PER_WARP = 32 / G;
  const int lane = threadIdx.x & 31;
  const int gl = lane % G;
  const int grp = lane / G;
  const unsigned gbits = (G == 32) ? 0xffffffffu : ((1u << G) - 1u);
  const unsigned gmask = gbits << (grp * G);
  const EmbFwdTable& tb = P.t[blockIdx.y];
  const idx_t* __restrict__ idx = static_cast<const idx_t*>(tb.idx);
  const idx_t* __restrict__ off = static_cast<const idx_t*>(tb.off);
  const float* __restrict__ W = tb.w;
  const bool link_tb = LINK && tb.head != nullptr;
  const int S = P.bags_per_group;
  const long long b0 = (((long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * GROUPS_PER_WARP + grp) * S;
  for (int s = 0; s < S; ++s) {
    const long long b = b0 + s;
    if (b >= P.batch) return;
    const long long start = (long long)off[b];
    const long long end = bag_end<idx_t>(off, b, P.batch, tb.nnz, P.include_last);
    float4 acc[NV];
#pragma unroll
    for (int v = 0; v < NV; ++v) acc[v] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (long long j0 = start; j0 < end; j0 += G) {
      const bool valid = j0 + gl < end;
      const long long rg = valid ? (long long)idx[j0 + gl] : -1;
      const long long lr = rg - tb.row_lo;
      const bool mine = valid && (unsigned long long)lr < (unsigned long long)tb.row_n;
      if (valid && !mine && (unsigned long long)rg >= (unsigned long long)tb.rows) flag_bad_index(P);
      if (link_tb && mine)      // occurrences of other shards' rows are never looked at by the update
        P.link[tb.pair_base + j0 + gl] = make_int2(note_occurrence(P, tb, lr, j0 + gl), (int)b);
      unsigned live = (__ballot_sync(gmask, mine) >> (grp * G)) & gbits;
      while (live) {
        float4 val[U][NV];
        float wgt[U];
        bool on[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          on[u] = live != 0u;
          const int src = on[u] ? __ffs(live) - 1 : 0;
          live &= live - 1u;                      // clears the lowest set bit (0 stays 0)
          const long long r = __shfl_sync(gmask, lr, src, G);
          if (on[u]) {
            const float* rp = W + r * tb.ld + gl * 4;
#pragma unroll
            for (int v = 0; v < NV; ++v)
              if (gl * 4 + v * G * 4 < D) val[u][v] = ldg_stream_f4(rp + v * G * 4);
            if (WEIGHTED) wgt[u] = __ldg(tb.rw + r);
          }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          if (on[u]) {
#pragma unroll
            for (int v = 0; v < NV; ++v) {
              if (WEIGHTED) {
                acc[v].x = fmaf(wgt[u], val[u][v].x, acc[v].x);
                acc[v].y = fmaf(wgt[u], val[u][v].y, acc[v].y);
                acc[v].z = fmaf(wgt[u], val[u][v].z, acc[v].z);
                acc[v].w = fmaf(wgt[u], val[u][v].w, acc[v].w);
              } else {
                acc[v].x += val[u][v].x;
                acc[v].y += val[u][v].y;
                acc[v].z += val[u][v].z;
                acc[v].w += val[u][v].w;
              }
            }
          }
        }
      }
    }
    float* op = out_ptr(P, tb, b) + gl * 4;
#pragma unroll
    for (int v = 0; v < NV; ++v)
      if (gl * 4 + v * G * 4 < D) *reinterpret_cast<float4*>(op + v * G * 4) = acc[v];
  }
}

// Row-split table, REMOTE-READ forward (BASELINE.json north_star: "P2P reads of remote rows over NVSwitch"):
// the rank that owns a sample pools the whole bag itself, in index order (bit-identical to the reference CPU
// kernel, like the local gather), loading each row from the rank that stores it through peer-mapped memory --
// 512-byte NVLink reads, up to U in flight per lane group.  No partial sums, no reduction; NVLink carries
// L x 512 B per sample instead of (N-1) x 512 B of partial sums (better for short bags, worse for L = 100).
struct EmbRemoteTable {
  const float* shard_w[DLRM_B200_MAX_PEERS];   // base of shard s (rows [s*rps, (s+1)*rps))
  const void* idx;
  const void* off;
  long long nnz, ld, out_off, out_stride, rows, rps;
};
struct EmbRemoteParams {
  EmbRemoteTable t[4];
  float* out;
  long long batch;
  int dim, include_last, bags_per_group;
  unsigned* err;
};

template <int G, int NV, int U, typename idx_t>
__global__ void __launch_bounds__(256) emb_fwd_remote_kernel(const __grid_constant__ EmbRemoteParams P) {
  const int D = P.dim;
  constexpr int GROUPS_PER_WARP = 32 / G;
  const int lane = threadIdx.x & 31;
  const int gl = lane % G;
  const int grp = lane / G;
  const unsigned gmask = (G == 32) ? 0xffffffffu : (((1u << G) - 1u) << (grp * G));
  const EmbRemoteTable& tb = P.t[blockIdx.y];
  const idx_t* __restrict__ idx = static_cast<const idx_t*>(tb.idx);
  const idx_t* __restrict__ off = static_cast<const idx_t*>(tb.off);
  const int S = P.bags_per_group;
  const long long b0 = (((long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * GROUPS_PER_WARP + grp) * S;
  for (int s = 0; s < S; ++s) {
    const long long b = b0 + s;
    if (b >= P.batch) return;
    const long long start = (long long)off[b];
    const long long end = bag_end<idx_t>(off, b, P.batch, tb.nnz, P.include_last);
    float4 acc[NV];
#pragma unroll
    for (int v = 0; v < NV; ++v) acc[v] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (long long j0 = start; j0 < end; j0 += G) {
      long long my_row = (j0 + gl < end) ? (long long)idx[j0 + gl] : 0;
      if ((unsigned long long)my_row >= (unsigned long long)tb.rows) {
        if (P.err) atomicOr(P.err, 1u);
        my_row = 0;
      }
      const int n = (int)min((long long)G, end - j0);
      for (int jj = 0; jj < n; jj += U) {
        float4 val[U][NV];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const long long r = __shfl_sync(gmask, my_row, jj + u, G);
          if (jj + u < n) {
            const long long sh = r / tb.rps;
            const float* rp = tb.shard_w[sh] + (r - sh * tb.rps) * tb.ld + gl * 4;
#pragma unroll
            for (int v = 0; v < NV; ++v)
              if (gl * 4 + v * G * 4 < D) val[u][v] = ldg_stream_f4(rp + v * G * 4);
          }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          if (jj + u < n) {
#pragma unroll
            for (int v = 0; v < NV; ++v) {
              acc[v].x += val[u][v].x; acc[v].y += val[u][v].y; acc[v].z += val[u][v].z; acc[v].w += val[u][v].w;
            }
          }
        }
      }
    }
    float* op = P.out + b * tb.out_stride + tb.out_off + gl * 4;
#pragma unroll
    for (int v = 0; v < NV; ++v)
      if (gl * 4 + v * G * 4 < D) *reinterpret_cast<float4*>(op + v * G * 4) = acc[v];
  }
}

// any dim / any alignment: one thread per output element, sequential over the bag
template <typename idx_t, bool WEIGHTED, bool LINK>
__global__ void emb_fwd_scalar_kernel(const __grid_constant__ EmbFwdParams P) {
  const EmbFwdTable& tb = P.t[blockIdx.y];
  const idx_t* __restrict__ idx = static_cast<const idx_t*>(tb.idx);
  const idx_t* __restrict__ off = static_cast<const idx_t*>(tb.off);
  const int D = P.dim;
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= P.batch * D) return;
  const long long b = e / D;
  const int d = (int)(e % D);
  const long long start = off[b];
  const long long end = bag_end<idx_t>(off, b, P.batch, tb.nnz, P.include_last);
  float acc = 0.f;
  for (long long j = start; j < end; ++j) {
    const long long rg = idx[j];
    const long long r = rg - tb.row_lo;
    const bool mine = (unsigned long long)r < (unsigned long long)tb.row_n;
    if (!mine && (unsigned long long)rg >= (unsigned long long)tb.rows && d == 0) flag_bad_index(P);
    if (LINK && tb.head && d == 0) P.link[tb.pair_base + j] = make_int2(mine ? note_occurrence(P, tb, r, j) : 0, (int)b);
    if (!mine) continue;
    const float x = tb.w[r * tb.ld + d];
    acc = WEIGHTED ? fmaf(tb.rw[r], x, acc) : acc + x;
  }
  out_ptr(P, tb, b)[d] = acc;
}

template <int G, int NV, int U, typename idx_t, bool WEIGHTED, bool LINK>
static int launch_vec(const EmbFwdParams& P, int num_tables, bool shard, cudaStream_t st) {
  const int block = 256;
  const long long groups_per_block = (long long)(block / 32) * (32 / G);
  const long long groups = (P.batch + P.bags_per_group - 1) / P.bags_per_group;
  dim3 grid((unsigned)((groups + groups_per_block - 1) / groups_per_block), (unsigned)num_tables);
  if (shard) {
    emb_fwd_shard_kernel<G, NV, U, idx_t, WEIGHTED, LINK><<<grid, block, 0, st>>>(P, num_tables);
    DLRM_CHECK_LAUNCH("emb_fwd_shard_kernel");
    return 0;
  }
  emb_fwd_vec_kernel<G, NV, U, idx_t, WEIGHTED, LINK><<<grid, block, 0, st>>>(P, num_tables);
  DLRM_CHECK_LAUNCH("emb_fwd_vec_kernel");
  return 0;
}

template <typename idx_t, bool WEIGHTED, bool LINK>
static int dispatch(const EmbFwdParams& Pin, int num_tables, bool vec_ok, bool shard, cudaStream_t st) {
  EmbFwdParams P = Pin;
  const int D = P.dim;
  if (vec_ok) {
    const int u8 = get_tunable(TUNE_EMB_UNROLL) != 4;
    int S = get_tunable(TUNE_EMB_BAGS_PER_GROUP);
    if (S <= 0) S = 4;  // bags handled back to back by one lane group
#define VEC(G, NV)                                                                   \
  do {                                                                               \
    P.bags_per_group = S < (G) ? S : (G)-1;                                          \
    if ((G) >= 8 && u8) return launch_vec<G, NV, 8, idx_t, WEIGHTED, LINK>(P, num_tables, shard, st); \
    return launch_vec<G, NV, ((G) >= 4 ? 4 : (G)), idx_t, WEIGHTED, LINK>(P, num_tables, shard, st);  \
  } while (0)
    if (D == 16) VEC(4, 1);  // dim 4 / 8: scalar kernel (a group must hold S+1 bag bounds)
    if (D == 32) VEC(8, 1);
    if (D == 64) VEC(16, 1);
    if (D > 64 && D <= 128) VEC(32, 1);
    if (D > 128 && D <= 256) VEC(32, 2);
    if (D > 256 && D <= 512) VEC(32, 4);
#undef VEC
  }
  const int block = 256;
  const long long n = P.batch * D;
  dim3 grid((unsigned)((n + block - 1) / block), (unsigned)num_tables);
  emb_fwd_scalar_kernel<idx_t, WEIGHTED, LINK><<<grid, block, 0, st>>>(P);
  DLRM_CHECK_LAUNCH("emb_fwd_scalar_kernel");
  return 0;
}

}  // namespace dlrm

static int emb_fwd_impl(const dlrm_emb_fwd_table_t* tables, const dlrm_emb_bwd_table_t* train,
                        int32_t* link, int num_tables, int dim, int64_t batch, int idx_bytes,
                        int include_last, float* out, int64_t out_stride_sample,
                        int64_t out_stride_table, void* stream, float* const* peer_out = nullptr,
                        int world = 0, int64_t batch_local = 0, const dlrm_emb_dedup_t* dedup = nullptr) {
  using namespace dlrm;
  if (num_tables < 0 || num_tables > DLRM_B200_MAX_TABLES_PER_CALL)
    return set_error("emb_bag_fwd: num_tables=%d out of range [0,%d]", num_tables,
                     DLRM_B200_MAX_TABLES_PER_CALL);
  if (dim <= 0) return set_error("emb_bag_fwd: dim=%d", dim);
  if (idx_bytes != 4 && idx_bytes != 8) return set_error("emb_bag_fwd: idx_bytes=%d", idx_bytes);
  if (batch == 0 || num_tables == 0) return 0;
  if (batch < 0 || batch * (int64_t)dim > (int64_t)0x7fffffff * 256)
    return set_error("emb_bag_fwd: batch=%lld too large", (long long)batch);
  if (train && !link) return set_error("emb_bag_fwd_train: link is NULL");
  EmbFwdParams P;
  bool weighted = false, any_unweighted = false, any_shard = false;
  bool vec_ok = (dim % 4 == 0) && dim <= 512 && (peer_out || aligned16(out)) && out_stride_sample % 4 == 0 &&
                out_stride_table % 4 == 0;
  for (int k = 0; k < num_tables; ++k) {
    P.t[k].w = tables[k].weight;
    P.t[k].idx = tables[k].indices;
    P.t[k].off = tables[k].offsets;
    P.t[k].rw = tables[k].row_weights;
    P.t[k].nnz = tables[k].nnz;
    P.t[k].ld = tables[k].ld > 0 ? tables[k].ld : dim;
    if (P.t[k].ld < dim) return set_error("emb_bag_fwd: table %d: ld=%lld < dim", k, (long long)tables[k].ld);
    vec_ok = vec_ok && (P.t[k].ld % 4 == 0);
    P.t[k].head = train ? train[k].head : nullptr;   // train[k].head == NULL: this table is not linked
    P.t[k].hs = (train && train[k].head_stride > 0) ? train[k].head_stride : 1;
    P.t[k].pair_base = train ? train[k].pair_base : 0;
    // per-table output routing (0 = the call-level layout out[b, k, :])
    P.t[k].out_stride = tables[k].out_stride > 0 ? tables[k].out_stride : out_stride_sample;
    P.t[k].out_off = tables[k].out_stride > 0 ? tables[k].out_off : (int64_t)k * out_stride_table;
    vec_ok = vec_ok && (P.t[k].out_stride % 4 == 0) && (P.t[k].out_off % 4 == 0);
    // row range of a shard; rows <= 0: unchecked (legacy callers)
    P.t[k].rows = tables[k].rows > 0 ? tables[k].rows : 0x7fffffffffffffffLL;
    P.t[k].row_lo = tables[k].row_n > 0 ? tables[k].row_lo : 0;
    P.t[k].row_n = tables[k].row_n > 0 ? tables[k].row_n : P.t[k].rows;
    if (P.t[k].row_lo < 0 || (tables[k].rows > 0 && P.t[k].row_lo + P.t[k].row_n > tables[k].rows))
      return set_error("emb_bag_fwd: table %d: row range [%lld, +%lld) outside %lld rows", k,
                       (long long)P.t[k].row_lo, (long long)P.t[k].row_n, (long long)tables[k].rows);
    any_shard = any_shard || P.t[k].row_lo != 0 || P.t[k].row_n != P.t[k].rows;
    if (!tables[k].weight || !tables[k].offsets || (!tables[k].indices && tables[k].nnz > 0))
      return set_error("emb_bag_fwd: table %d has a NULL pointer", k);
    if (tables[k].nnz > 0x7ffffffeLL) return set_error("emb_bag_fwd: table %d: nnz >= 2^31 per call", k);
    if (train && train[k].pair_base + tables[k].nnz > 0x7ffffffeLL)
      return set_error("emb_bag_fwd_train: more than 2^31-2 index occurrences");
    if (tables[k].row_weights) weighted = true; else any_unweighted = true;
    vec_ok = vec_ok && aligned16(tables[k].weight);
  }
  if (weighted && any_unweighted)
    return set_error("emb_bag_fwd: row_weights must be given for all tables of a call or none");
  P.out = out;
  P.stride_sample = out_stride_sample;
  P.stride_table = out_stride_table;
  P.batch = batch;
  P.dim = dim;
  P.include_last = include_last;
  P.bags_per_group = 1;
  P.link = reinterpret_cast<int2*>(link);
  P.filter = nullptr;
  P.filter_log2 = 0;
  P.err = err_word_device();
  if (train && dedup && dedup->filter) {
    if (dedup->log2_size < 10 || dedup->log2_size > 30)
      return set_error("emb_bag_fwd_train: dedup log2_size=%d out of range [10,30]", dedup->log2_size);
    P.filter = dedup->filter;
    P.filter_log2 = dedup->log2_size;
  }
  P.peer_batch = 0;
  for (int d = 0; d < DLRM_B200_MAX_PEERS; ++d) P.peer_out[d] = nullptr;
  if (peer_out) {
    if (world < 1 || world > DLRM_B200_MAX_PEERS || batch_local <= 0 || batch_local * world != batch)
      return set_error("emb_bag_fwd_p2p: world=%d batch_local=%lld batch=%lld", world, (long long)batch_local,
                       (long long)batch);
    for (int d = 0; d < world; ++d) {
      if (!peer_out[d]) return set_error("emb_bag_fwd_p2p: peer %d pointer is NULL", d);
      vec_ok = vec_ok && aligned16(peer_out[d]);
      P.peer_out[d] = peer_out[d];
    }
    P.peer_batch = batch_local;
    P.out = peer_out[0];
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
#define DISPATCH(IDX)                                                                          \
  do {                                                                                         \
    if (train) return weighted ? dispatch<IDX, true, true>(P, num_tables, vec_ok, any_shard, st)          \
                               : dispatch<IDX, false, true>(P, num_tables, vec_ok, any_shard, st);        \
    return weighted ? dispatch<IDX, true, false>(P, num_tables, vec_ok, any_shard, st)                    \
                    : dispatch<IDX, false, false>(P, num_tables, vec_ok, any_shard, st);                  \
  } while (0)
  if (idx_bytes == 8) DISPATCH(long long);
  DISPATCH(int);
#undef DISPATCH
}

extern "C" int dlrm_b200_emb_bag_fwd(const dlrm_emb_fwd_table_t* tables, int num_tables, int dim,
                                     int64_t batch, int idx_bytes, int include_last, float* out,
                                     int64_t out_stride_sample, int64_t out_stride_table,
                                     void* stream) {
  return emb_fwd_impl(tables, nullptr, nullptr, num_tables, dim, batch, idx_bytes, include_last, out,
                      out_stride_sample, out_stride_table, stream);
}

extern "C" int dlrm_b200_emb_bag_fwd_train(const dlrm_emb_fwd_table_t* tables,
                                           const dlrm_emb_bwd_table_t* train, int num_tables, int dim,
                                           int64_t batch, int idx_bytes, int include_last, int32_t* next,
                                           float* out, int64_t out_stride_sample,
                                           int64_t out_stride_table, const dlrm_emb_dedup_t* dedup,
                                           void* stream) {
  if (!train) return dlrm::set_error("emb_bag_fwd_train: train descriptors are NULL");
  return emb_fwd_impl(tables, train, next, num_tables, dim, batch, idx_bytes, include_last, out,
                      out_stride_sample, out_stride_table, stream, nullptr, 0, 0, dedup);
}

extern "C" int dlrm_b200_emb_bag_fwd_p2p(const dlrm_emb_fwd_table_t* tables,
                                         const dlrm_emb_bwd_table_t* train, int num_tables, int dim,
                                         int64_t batch_global, int idx_bytes, int include_last, int32_t* next,
                                         float* const* peer_out, int world, int64_t batch_local,
                                         int64_t out_stride_sample, int64_t out_stride_table,
                                         const dlrm_emb_dedup_t* dedup, void* stream) {
  if (!peer_out) return dlrm::set_error("emb_bag_fwd_p2p: peer_out is NULL");
  return emb_fwd_impl(tables, train, next, num_tables, dim, batch_global, idx_bytes, include_last, nullptr,
                      out_stride_sample, out_stride_table, stream, peer_out, world, batch_local, dedup);
}

extern "C" int dlrm_b200_emb_bag_fwd_remote(const dlrm_emb_remote_table_t* tables, int num_tables, int dim,
                                            int64_t batch, int idx_bytes, int include_last, float* out,
                                            void* stream) {
  using namespace dlrm;
  if (num_tables == 0 || batch == 0) return 0;
  if (num_tables < 0 || num_tables > 4) return set_error("emb_bag_fwd_remote: num_tables=%d (max 4 per call)", num_tables);
  if (idx_bytes != 4 && idx_bytes != 8) return set_error("emb_bag_fwd_remote: idx_bytes=%d", idx_bytes);
  if (!tables || !out) return set_error("emb_bag_fwd_remote: NULL pointer");
  if (dim <= 0 || dim % 4 || dim > 512 || !aligned16(out)) return set_error("emb_bag_fwd_remote: dim=%d (multiple of 4, <= 512)", dim);
  EmbRemoteParams P{};
  for (int k = 0; k < num_tables; ++k) {
    const dlrm_emb_remote_table_t& s = tables[k];
    if (s.num_shards < 1 || s.num_shards > DLRM_B200_MAX_PEERS || s.rows_per_shard <= 0 || s.rows <= 0 ||
        s.rows_per_shard * s.num_shards < s.rows)
      return set_error("emb_bag_fwd_remote: table %d: %d shards of %lld rows for %lld rows", k, s.num_shards,
                       (long long)s.rows_per_shard, (long long)s.rows);
    if (!s.offsets || (!s.indices && s.nnz > 0)) return set_error("emb_bag_fwd_remote: table %d has a NULL pointer", k);
    EmbRemoteTable& t = P.t[k];
    for (int d = 0; d < DLRM_B200_MAX_PEERS; ++d) {
      t.shard_w[d] = d < s.num_shards ? s.shard_weight[d] : s.shard_weight[0];
      if (d < s.num_shards && (!s.shard_weight[d] || !aligned16(s.shard_weight[d])))
        return set_error("emb_bag_fwd_remote: table %d shard %d pointer NULL / unaligned", k, d);
    }
    t.idx = s.indices; t.off = s.offsets; t.nnz = s.nnz; t.ld = s.ld > 0 ? s.ld : dim;
    t.out_off = s.out_off; t.out_stride = s.out_stride; t.rows = s.rows; t.rps = s.rows_per_shard;
    if (t.ld % 4 || t.out_off % 4 || t.out_stride % 4) return set_error("emb_bag_fwd_remote: table %d: unaligned strides", k);
  }
  P.out = out; P.batch = batch; P.dim = dim; P.include_last = include_last; P.err = err_word_device();
  cudaStream_t st = static_cast<cudaStream_t>(stream);
#define REMOTE(G, NV, IDX)                                                                                 \
  do {                                                                                                     \
    P.bags_per_group = 2;                                                                                  \
    const long long gpb = (256 / 32) * (32 / (G));                                                         \
    const long long groups = (batch + 1) / 2;                                                              \
    dim3 grid((unsigned)((groups + gpb - 1) / gpb), (unsigned)num_tables);                                 \
    emb_fwd_remote_kernel<G, NV, ((G) >= 8 ? 8 : (G)), IDX><<<grid, 256, 0, st>>>(P);                       \
    DLRM_CHECK_LAUNCH("emb_fwd_remote_kernel");                                                            \
    return 0;                                                                                              \
  } while (0)
#define REMOTE_D(IDX)                      \
  do {                                     \
    if (dim <= 16) REMOTE(4, 1, IDX);      \
    if (dim <= 32) REMOTE(8, 1, IDX);      \
    if (dim <= 64) REMOTE(16, 1, IDX);     \
    if (dim <= 128) REMOTE(32, 1, IDX);    \
    if (dim <= 256) REMOTE(32, 2, IDX);    \
    REMOTE(32, 4, IDX);                    \
  } while (0)
  if (idx_bytes == 8) REMOTE_D(long long);
  REMOTE_D(int);
#undef REMOTE_D
#undef REMOTE
}
