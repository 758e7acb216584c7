// Embedding backward fused with the sparse optimizer step.
//
// Replaces: autograd _embedding_bag_backward -> sparse COO grad (dlrm_s_pytorch.py:1613) and
// optimizer.step() (:1620): optim/rwsadagrad.py:117-143 (coalesce, mean of squares, momentum,
// scaled sparse add) or torch.optim.SGD's sparse add.  No [nnz, D] gradient tensor is ever
// materialised: the gradient of a (table,row) occurrence IS the dY row of its bag.
//
// Coalescing (the update is non-linear, so occurrences of the same row must be summed first,
// optim/rwsadagrad.py:118-120) is done without a sort:
//   link   : every occurrence `pos` of a row threads itself onto a per-row list with one
//            atomicExch on head[row] (int32 per table row, zero between steps):
//                link[pos] = { previous head, bag of pos };  head[row] = pos + 1
//            and, when the previous head p + 1 is not 0, marks occurrence p as superseded:
//                mark[p] = 1     (one byte per position, zero between steps)
//            Every position is superseded by at most one successor, so a plain store does; only
//            duplicate occurrences write, and the array (1 byte x occurrences) stays in L2.
//            Depends on the indices only -> can overlap the forward pass (or ride in the gather).
//   update : a warp takes 32 consecutive positions and reads index, link entry and mark of each
//            (coalesced), clearing the marks it read.  Occurrence `pos` owns its row iff it is not
//            marked (the last arrival): ownership is decided without touching the table.  The owner
//            issues the loads of the weight row and of the row's accumulator together (with the
//            interleaved layout the accumulator and the list head sit right behind the row, in the
//            same DRAM page), walks the list when there is one, sorts the members by position when
//            there are <= 32 (deterministic sum in ascending position == grad.coalesce() order; a
//            longer list takes the order-independent fixed-point sum of list_sum_exact), adds their
//            dY rows, applies the optimizer in registers and stores the row, the accumulator and
//            head[row] = 0 together.  Two random DRAM accesses per updated row: row + words in,
//            row + words out.  Non-owners do nothing.  Rows without duplicates (the common case at
//            1e6-row tables) never touch link[] beyond their own entry.
//   fp16 tables (template row type wt = __half): the owner widens the row to fp32, applies the same fp32 step and
//            stores the row with stochastic rounding (st_row4, common.cuh); the accumulator and the head stay
//            fp32 / int32 words behind the row.  The float instantiations are the fp32 kernels.
//   element-wise Adagrad (DLRM_OPT_ADAGRAD, template flag EW): the same coalesce and ownership; the owner also loads
//            its row of per-element accumulators (momentum + r * mom_stride, a separate arena: 512 more bytes per row
//            at D = 128, one more random access in and one out) in the same batch as the weight row, applies
//            adagrad_ew (common.cuh: s += g*g with two roundings, IEEE sqrt, + eps, IEEE division, one fmaf) per
//            element and stores both rows.  The EW = false instantiations are the SGD / RWSAdagrad kernels unchanged.
#include "common.cuh"

namespace dlrm {

// A per-row occurrence list is acyclic by construction (every gather+link is followed by the update that resets
// the heads it used).  If a caller breaks that contract (indices rewritten between link and update, a skipped
// update), stale heads can close a cycle and the walk would spin for ever: past 2^17 members the walk checks the
// clock and traps after 20 s instead of hanging the GPU.
__device__ __forceinline__ void list_walk_guard(unsigned& chunks, unsigned long long& t0) {
  if (++chunks >= 4096u && (chunks & 4095u) == 0u) {
    unsigned long long now;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
    if (t0 == 0) t0 = now;
    else if (now - t0 > 20000000000ULL) {
      if ((threadIdx.x & 31) == 0) printf("dlrm_b200: emb update: a row's occurrence list does not end (stale list heads?)\n");
      __trap();
    }
  }
}

// Sum of the dY rows of a row's occurrence list longer than 32 (the owner `self_bag` first, then the list from
// `nxt`).  The list is built by atomicExch, so its order changes from run to run; summing it in list order would
// make the update -- and every later step -- differ between runs.  Instead every value is converted to 64-bit fixed
// point with a per-column scale taken from the column's largest magnitude (a max, independent of order), the
// integers are added exactly and the sum is rounded to fp32 once: the result depends only on the set of members.
// The conversion truncates at 2^-62 x n of the column's largest |value|, far below one fp32 ulp of the sum.
// Called by a whole warp.  The walk gathers 32 members per chunk into the lanes (one dependent link load each);
// the bags of the first LS_KEEP chunks stay in registers, so the second pass over them only reloads dY rows.
// load(bag, t) fills t[0..N) with this lane's columns of the dY row of `bag` (0 for columns outside the row).
constexpr int LS_KEEP = 4;

struct ListWalk {
  const int2* link;
  int cur, self_bag;
  bool first;
  unsigned chunks;
  unsigned long long t0;
  // next <= 32 members into the lanes (member i of the chunk -> lane i's `bag`); returns their number
  __device__ __forceinline__ int chunk(int lane, int& bag) {
    int cnt = 0;
    while (cnt < 32 && (first || cur != 0)) {
      int b;
      if (first) { b = self_bag; first = false; }
      else { const int2 e = link[cur - 1]; b = e.y; cur = e.x; }
      if (lane == cnt) bag = b;
      ++cnt;
    }
    list_walk_guard(chunks, t0);
    return cnt;
  }
  __device__ __forceinline__ bool done() const { return !first && cur == 0; }
};

template <int N, class Load>
__device__ __forceinline__ void list_sum_exact(const int2* link, int nxt, int self_bag, const Load& load, float (&out)[N]) {
  const int lane = threadIdx.x & 31;
  float mx[N];
#pragma unroll
  for (int j = 0; j < N; ++j) mx[j] = 0.f;
  int keep[LS_KEEP];
  int cnt_keep[LS_KEEP];
  ListWalk w{link, nxt, self_bag, true, 0u, 0ull};
  ListWalk resume = w;
  int n = 0;
  // members of a chunk are visited LB at a time: their dY rows are all loaded before the first is used
  constexpr int LB = N <= 4 ? 4 : 1;
  auto visit = [&](int bag, int cnt, auto&& use) {
    for (int q0 = 0; q0 < cnt; q0 += LB) {
      float t[LB][N];
#pragma unroll
      for (int u = 0; u < LB; ++u) {
        const int b = __shfl_sync(0xffffffffu, bag, (q0 + u) & 31);
        if (q0 + u < cnt) load(b, t[u]);
      }
#pragma unroll
      for (int u = 0; u < LB; ++u)
        if (q0 + u < cnt) use(t[u]);
    }
  };
  for (int c = 0; !w.done(); ++c) {                    // pass 1: column maxima
    int bag = 0;
    const int cnt = w.chunk(lane, bag);
    if (c < LS_KEEP) { keep[c] = bag; cnt_keep[c] = cnt; resume = w; }
    visit(bag, cnt, [&](const float (&t)[N]) {
#pragma unroll
      for (int j = 0; j < N; ++j) mx[j] = fmaxf(mx[j], fabsf(t[j]));
    });
    n += cnt;
  }
  const int L = 32 - __clz(n);                          // n < 2^L
  double sc[N];
  long long s[N];
  float f[N];                                          // plain sum: only to carry an inf / nan through
#pragma unroll
  for (int j = 0; j < N; ++j) {
    int E;
    frexpf(mx[j], &E);                                  // |value| < 2^E  ->  |sum| x 2^k < 2^62
    sc[j] = ldexp(1.0, 62 - L - E);
    s[j] = 0;
    f[j] = 0.f;
  }
  auto add_chunk = [&](int bag, int cnt) {
    visit(bag, cnt, [&](const float (&t)[N]) {
#pragma unroll
      for (int j = 0; j < N; ++j) { s[j] += (long long)((double)t[j] * sc[j]); f[j] += t[j]; }
    });
  };
#pragma unroll
  for (int c = 0; c < LS_KEEP; ++c)                    // pass 2: the kept chunks, then the rest of the list
    if (c * 32 < n) add_chunk(keep[c], cnt_keep[c]);
  while (!resume.done()) {
    int bag = 0;
    const int cnt = resume.chunk(lane, bag);
    add_chunk(bag, cnt);
  }
#pragma unroll
  for (int j = 0; j < N; ++j) out[j] = isfinite(f[j]) ? (float)((double)s[j] / sc[j]) : f[j];
}

struct EmbBwdTable {
  void* w;               // rows of the row type (float or __half)
  float* mom;
  int* head;
  const void* idx;
  const void* off;
  long long nnz;
  long long pair_base;
  long long ld;          // row stride of w in elements of the row type
  long long mom_stride;  // elements between consecutive rows' accumulators
  long long hs;          // elements between consecutive rows' list heads
  long long dy_off;      // the dY row of (bag, this table) is dy_row(bag) + dy_off
  long long rows;        // rows of the whole table
  long long row_lo;      // this shard stores rows [row_lo, row_lo + row_n) at local index (row - row_lo);
  long long row_n;       //   occurrences of other rows belong to another shard and are ignored
  unsigned char* mark;   // superseded marks, indexed like link[]
};

struct EmbBwdParams {
  EmbBwdTable t[DLRM_B200_MAX_TABLES_PER_CALL];
  int2* link;        // [total nnz] {next, bag}
  const float* dY;
  long long dy_stride_sample;
  long long dy_stride_table;
  long long batch;
  int dim;
  int include_last;
  int optimizer;
  float lr;
  float eps;
  // table-wise sharded runs: the dY row of global bag b is read from rank b / peer_batch through
  // peer-mapped memory (NVLink load).  peer_batch == 0: local dY.
  const float* peer_dY[DLRM_B200_MAX_PEERS];
  long long peer_batch;
  // duplicate filter (optional): occurrences with flags[pos] == 0 are the only occurrence of their row
  const unsigned char* flags;
  int debug;   // TIMING EXPERIMENTS ONLY (tunable upd_debug): 1 = no weight store, 2 = no weight load, 4 = no
               // accumulator / list-head stores, 8 = no gradient load.  Results are wrong when non-zero.
  // fp16 tables: stochastic-rounding key of table k for this step (kept out of EmbBwdTable, so that the fp32
  // kernels see the parameter layout they always had)
  unsigned long long round_key[DLRM_B200_MAX_TABLES_PER_CALL];
  // learning rate in device memory (CUDA-graph steps whose rate changes between replays); NULL: lr above
  const float* lr_dev;
  // learned weighted pooling (the RW instantiations only): v of table k and its Adagrad sum (NULL for SGD), kept out
  // of EmbBwdTable for the same reason as round_key
  float* row_w[DLRM_B200_MAX_TABLES_PER_CALL];
  float* row_w_sum[DLRM_B200_MAX_TABLES_PER_CALL];
};

__device__ __forceinline__ float step_lr(const EmbBwdParams& P) { return P.lr_dev ? *P.lr_dev : P.lr; }

// Learned weighted pooling: the step of the row weight v (old value v, gradient dv = <S, W_old>) and of its Adagrad
// sum s (RWSAdagrad / Adagrad: the dense branch, as dense_update_kernel; SGD: s unused).  Returns v'.
__device__ __forceinline__ float row_weight_step(const EmbBwdParams& P, float v, float dv, float& s) {
  const float lr = step_lr(P);
  if (P.optimizer == DLRM_OPT_SGD) return fmaf(-lr, dv, v);
  s = fmaf(dv, dv, s);
  return fmaf(-lr, dv / (sqrtf(s) + P.eps), v);
}

__device__ __forceinline__ const float* dy_row(const EmbBwdParams& P, long long bag) {
  if (P.peer_batch > 0) {
    const int src = (int)(bag / P.peer_batch);
    return P.peer_dY[src] + (bag - src * P.peer_batch) * P.dy_stride_sample;
  }
  return P.dY + bag * P.dy_stride_sample;
}

template <typename idx_t>
__device__ __forceinline__ long long bag_end2(const idx_t* off, long long b, long long batch,
                                              long long nnz, int include_last) {
  return (include_last || b + 1 < batch) ? (long long)off[b + 1] : nnz;
}

// ---------------------------------------------------------------------------------------------
// link: one thread per occurrence; its bag is found by binary search in the offsets (L2 hits).
// ---------------------------------------------------------------------------------------------
template <typename idx_t>
__global__ void __launch_bounds__(256) emb_link_kernel(const __grid_constant__ EmbBwdParams P) {
  const EmbBwdTable& tb = P.t[blockIdx.y];
  const idx_t* __restrict__ idx = static_cast<const idx_t*>(tb.idx);
  const idx_t* __restrict__ off = static_cast<const idx_t*>(tb.off);
  // packed format: offsets are global positions into one shared index array, so a table's
  // occurrences are [off[0], off[batch]); reference format: [0, nnz)
  const long long jbeg = (long long)off[0];
  const long long nnz = P.include_last ? (long long)off[P.batch] : tb.nnz;
  for (long long j = jbeg + (long long)blockIdx.x * blockDim.x + threadIdx.x; j < nnz;
       j += (long long)gridDim.x * blockDim.x) {
    // largest b with off[b] <= j  (empty bags share an offset: pick the last of the run)
    long long lo = 0, hi = P.batch - 1;
    while (lo < hi) {
      const long long mid = (lo + hi + 1) >> 1;
      if ((long long)off[mid] <= j) lo = mid; else hi = mid - 1;
    }
    const long long r = (long long)idx[j] - tb.row_lo;
    const long long pos = tb.pair_base + j;
    const bool mine = tb.head != nullptr && (unsigned long long)r < (unsigned long long)tb.row_n;
    const int prev = mine ? atomicExch(tb.head + r * tb.hs, (int)(pos + 1)) : 0;
    P.link[pos] = make_int2(prev, (int)lo);
    if (prev) tb.mark[prev - 1] = 1;          // that occurrence is no longer the last one of its row
  }
}

// ---------------------------------------------------------------------------------------------
// update.  W = elements per lane per step (4 = float4 path, 1 = scalar path), NV steps.
// lane columns: c(v) = lane*W + v*32*W.
// ---------------------------------------------------------------------------------------------
template <int W>
struct Pack {
  float x[W];
};

template <int W, typename wt = float>
__device__ __forceinline__ Pack<W> ld_pack(const wt* p) {
  Pack<W> r;
  if constexpr (is_f16<wt>::value) {
    static_assert(W == 4, "fp16 rows take the 4-wide path");
    const float4 v = ld_row4(p);
    r.x[0] = v.x; r.x[1 % W] = v.y; r.x[2 % W] = v.z; r.x[3 % W] = v.w;
  } else if (W == 4) {
    const float4 v = *reinterpret_cast<const float4*>(p);
    r.x[0] = v.x; r.x[1 % W] = v.y; r.x[2 % W] = v.z; r.x[3 % W] = v.w;
  } else {
    r.x[0] = *p;
  }
  return r;
}
template <int W, typename wt = float>
__device__ __forceinline__ void st_pack(wt* p, const Pack<W>& r, unsigned long long bits = 0) {
  if constexpr (is_f16<wt>::value) {
    st_row4(p, make_float4(r.x[0], r.x[1 % W], r.x[2 % W], r.x[3 % W]), bits);
  } else if (W == 4) {
    *reinterpret_cast<float4*>(p) = make_float4(r.x[0], r.x[1 % W], r.x[2 % W], r.x[3 % W]);
  } else {
    *p = r.x[0];
  }
}

// first global position of every table of the call (+ the end of the last) in shared memory; tend[k] = end of
// table k's own positions.  The tables of a call need not be adjacent in the position space (tiny tables are
// updated by another kernel and leave gaps): a position p belongs to table k = table_of(p) only if p < tend[k].
template <typename idx_t>
__device__ __forceinline__ void load_bounds(long long* bound, long long* tend, const EmbBwdParams& P, int num_tables,
                                            long long total_hint) {
  if ((int)threadIdx.x < num_tables) {
    const int k = threadIdx.x;
    const idx_t* off = static_cast<const idx_t*>(P.t[k].off);
    const long long b = P.include_last ? (long long)off[0] : P.t[k].pair_base;
    const long long e = P.include_last ? (long long)off[P.batch] : P.t[k].pair_base + P.t[k].nnz;
    bound[k] = b;
    tend[k] = e;
    if (k == num_tables - 1) bound[num_tables] = e;
  }
  (void)total_hint;
  __syncthreads();
}
// table of a position: largest k with bound[k] <= pos (empty tables share a bound)
__device__ __forceinline__ int table_of(const long long* bound, int num_tables, long long pos) {
  int lo = 0, hi = num_tables - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (bound[mid] <= pos) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// ---------------------------------------------------------------------------------------------
// duplicate filter, step 2: flag the occurrences whose hashed counter is > 1 and collect them
// ---------------------------------------------------------------------------------------------
template <typename idx_t>
__global__ void __launch_bounds__(256) emb_classify_kernel(const __grid_constant__ EmbBwdParams P, int num_tables,
                                                           long long total_hint, const unsigned* filter,
                                                           int log2_size, unsigned char* flags, int* suspects,
                                                           int* n_suspects) {
  __shared__ long long bound[DLRM_B200_MAX_TABLES_PER_CALL + 1], tend[DLRM_B200_MAX_TABLES_PER_CALL + 1];
  load_bounds<idx_t>(bound, tend, P, num_tables, total_hint);
  const int lane = threadIdx.x & 31;
  const long long first = bound[0], total = bound[num_tables];
  const long long warp0 = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long wstride = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long base = first + warp0 * 32; base < total; base += wstride * 32) {
    const long long pos = base + lane;
    bool susp = false;
    const int kk = table_of(bound, num_tables, pos < total ? pos : first);
    if (pos < total && pos < tend[kk]) {
      const EmbBwdTable& tb = P.t[kk];
      // local row, as the gather counted it; rows of another shard and tables without lists are never linked
      const long long r = (long long)static_cast<const idx_t*>(tb.idx)[pos - tb.pair_base] - tb.row_lo;
      if (tb.head != nullptr && (unsigned long long)r < (unsigned long long)tb.row_n)
        susp = filter[filter_slot(tb.head + r * tb.hs, log2_size)] > 1u;
      flags[pos] = susp ? 1 : 0;
    }
    const unsigned m = __ballot_sync(0xffffffffu, susp);
    if (m) {
      int slot0 = 0;
      if (lane == 0) slot0 = atomicAdd(n_suspects, __popc(m));
      slot0 = __shfl_sync(0xffffffffu, slot0, 0);
      if (susp) suspects[slot0 + __popc(m & ((1u << lane) - 1u))] = (int)pos;
    }
  }
}

// step 3: thread ONLY the suspects onto the per-row lists (link[pos].x; .y = bag was written by the gather)
template <typename idx_t>
__global__ void __launch_bounds__(256) emb_link_suspects_kernel(const __grid_constant__ EmbBwdParams P,
                                                                int num_tables, long long total_hint,
                                                                const int* suspects, const int* n_suspects) {
  __shared__ long long bound[DLRM_B200_MAX_TABLES_PER_CALL + 1], tend[DLRM_B200_MAX_TABLES_PER_CALL + 1];
  load_bounds<idx_t>(bound, tend, P, num_tables, total_hint);
  const int n = *n_suspects;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const long long pos = suspects[i];
    const EmbBwdTable& tb = P.t[table_of(bound, num_tables, pos)];
    const long long r = (long long)static_cast<const idx_t*>(tb.idx)[pos - tb.pair_base] - tb.row_lo;   // in range: classify
    const int prev = atomicExch(tb.head + r * tb.hs, (int)(pos + 1));
    P.link[pos].x = prev;
    if (prev) tb.mark[prev - 1] = 1;
  }
}

// Occurrence-centric: a warp takes 32 consecutive index positions (all tables share one global
// position space: reference format = per-table arrays + pair_base, packed format = one array),
// reads index / link / head with coalesced + gathered loads, and processes the rows it owns with
// up to PF weight rows AND their dY rows in flight.  The bag of an occurrence comes from link[],
// so the offsets are not needed (packed format reads only the per-table bounds).
// Out of line: the long-list sum must not take registers from the update kernel's hot path.
template <int NV, int W>
__device__ __noinline__ void dup_sum_long(const EmbBwdParams& P, int nxt, int self_bag, long long dyk_off,
                                          const bool (&col_ok)[NV], Pack<W> (&g)[NV]) {
  const int lane = threadIdx.x & 31;
  auto load = [&](int bag, float (&t)[NV * W]) {
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      Pack<W> p;
#pragma unroll
      for (int e = 0; e < W; ++e) p.x[e] = 0.f;
      if (col_ok[v]) p = ld_pack<W>(dy_row(P, bag) + dyk_off + lane * W + v * 32 * W);
#pragma unroll
      for (int e = 0; e < W; ++e) t[v * W + e] = p.x[e];
    }
  };
  float acc[NV * W];
  list_sum_exact<NV * W>(P.link, nxt, self_bag, load, acc);
#pragma unroll
  for (int v = 0; v < NV; ++v)
#pragma unroll
    for (int e = 0; e < W; ++e) g[v].x[e] = acc[v * W + e];
}

// EW: the element-wise Adagrad instantiation (DLRM_OPT_ADAGRAD): every lane also moves its columns of the row's
// accumulator row, loaded with the weight row and stored with it.  EW = false is the SGD / RWSAdagrad kernel.
// RW: learned weighted pooling: the owner also loads v[r] (and its sum) with the row, takes dv = <S, W_old> over the
// warp, scales S by v[r] and steps v[r].  RW = false is the unweighted kernel unchanged.
template <typename wt, int W, int NV, typename idx_t, bool EW = false, bool RW = false>
__global__ void __launch_bounds__(256, NV == 1 ? (EW ? 2 : 3) : 1) emb_update_kernel(const __grid_constant__ EmbBwdParams P,
                                                                          int num_tables, long long total_hint) {
  __shared__ long long bound[DLRM_B200_MAX_TABLES_PER_CALL + 1], tend[DLRM_B200_MAX_TABLES_PER_CALL + 1];
  load_bounds<idx_t>(bound, tend, P, num_tables, total_hint);
  const int D = P.dim;
  const int lane = threadIdx.x & 31;
  const long long first = bound[0], total = bound[num_tables];
  const long long warp0 = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long wstride = (long long)gridDim.x * (blockDim.x >> 5);
  bool col_ok[NV];
#pragma unroll
  for (int v = 0; v < NV; ++v) col_ok[v] = lane * W + v * 32 * W < D;
  const float inv_d = 1.0f / (float)D;
  // EW carries the accumulators too: 2 rows in flight at 2 CTAs per SM keep it free of spills (4 at 3 spill)
  constexpr int PF = NV == 1 ? (EW ? 2 : 4) : 1;

  for (long long base = first + warp0 * 32; base < total; base += wstride * 32) {
    const long long pos = base + lane;
    const int k = table_of(bound, num_tables, pos < total ? pos : first);
    const bool valid = pos < total && pos < tend[k];
    long long my_r = 0;
    int2 my_link = make_int2(0, 0);
    bool my_susp = true;
    bool owner = false;
    if (valid) {
      const EmbBwdTable& tb = P.t[k];
      my_r = (long long)static_cast<const idx_t*>(tb.idx)[pos - tb.pair_base] - tb.row_lo;
      // rows of another shard, and tables updated by the small-table path (head == null), are not ours
      if (tb.head != nullptr && (unsigned long long)my_r < (unsigned long long)tb.row_n) {
        my_link = P.link[pos];
        const unsigned char superseded = tb.mark[pos];
        if (superseded) tb.mark[pos] = 0;
        owner = !superseded;
        // an unflagged occurrence is the only one of its row (never linked, never marked): head[] is never touched
        if (P.flags) my_susp = P.flags[pos] != 0;
        if (!my_susp) my_link.x = 0;
      }
    }
    const unsigned owners = __ballot_sync(0xffffffffu, owner);
    const unsigned susp_mask = __ballot_sync(0xffffffffu, my_susp);
    for (int u0 = 0; u0 < 32; u0 += PF) {
      if (((owners >> u0) & ((1u << PF) - 1u)) == 0u) continue;
      Pack<W> wpf[PF][NV], gpf[PF][NV];
      Pack<W> spf[EW ? PF : 1][EW ? NV : 1];     // EW: the accumulators of the lane's columns
      float mpf[PF];
      float vpf[RW ? PF : 1], vspf[RW ? PF : 1];  // RW: v[r] and its sum (every lane loads the same word)
#pragma unroll
      for (int u = 0; u < PF; ++u) {
        const int src = u0 + u;
        const long long r = __shfl_sync(0xffffffffu, my_r, src);
        const int ku = __shfl_sync(0xffffffffu, k, src);
        const int bag = __shfl_sync(0xffffffffu, my_link.y, src);
        if ((owners >> src) & 1u) {
          const EmbBwdTable& tb = P.t[ku];
          const wt* wrow = static_cast<const wt*>(tb.w) + r * tb.ld;
          const float* grow = dy_row(P, bag) + tb.dy_off;
#pragma unroll
          for (int v = 0; v < NV; ++v)
            if (col_ok[v]) {
              wpf[u][v] = ld_pack<W>(wrow + lane * W + v * 32 * W);
              gpf[u][v] = ld_pack<W>(grow + lane * W + v * 32 * W);
            }
          if constexpr (EW) {
            const float* srow = tb.mom + r * tb.mom_stride;
#pragma unroll
            for (int v = 0; v < NV; ++v)
              if (col_ok[v]) spf[u][v] = ld_pack<W>(srow + lane * W + v * 32 * W);
            mpf[u] = 0.f;
          } else {
            mpf[u] = (P.optimizer == DLRM_OPT_RWSADAGRAD) ? tb.mom[r * tb.mom_stride] : 0.f;
          }
          if constexpr (RW) {
            vpf[u] = P.row_w[ku][r];
            vspf[u] = P.optimizer != DLRM_OPT_SGD ? P.row_w_sum[ku][r] : 0.f;
          }
        }
      }
#pragma unroll
      for (int u = 0; u < PF; ++u) {
        const int src = u0 + u;
        const long long r = __shfl_sync(0xffffffffu, my_r, src);
        const int ku = __shfl_sync(0xffffffffu, k, src);
        int nxt = __shfl_sync(0xffffffffu, my_link.x, src);
        const int self_bag = __shfl_sync(0xffffffffu, my_link.y, src);
        if (!((owners >> src) & 1u)) continue;
        const EmbBwdTable& tb = P.t[ku];
        wt* wrow = static_cast<wt*>(tb.w) + r * tb.ld;
        const long long dyk_off = tb.dy_off;
        // fp16: random bits of column group q = lane + 32 v (columns 4q..4q+3) of this global row
        const unsigned long long rkey = is_f16<wt>::value ? sr_row_key(P.round_key[ku], r + tb.row_lo) : 0ull;
        Pack<W> w[NV], g[NV];
#pragma unroll
        for (int v = 0; v < NV; ++v) { w[v] = wpf[u][v]; g[v] = gpf[u][v]; }
        const float m_old = mpf[u];
        if (nxt != 0) {
          // duplicates: up to 32 members (self first) are summed in ascending position (== grad.coalesce());
          // a longer list takes the order-independent sum
#pragma unroll
          for (int v = 0; v < NV; ++v)
#pragma unroll
            for (int e = 0; e < W; ++e) g[v].x[e] = 0.f;
          const int nxt0 = nxt;
          int cnt = 1;
          int mpos = (lane == 0) ? (int)(base + src) : 0x7fffffff;
          int mbag = self_bag;
          while (nxt != 0 && cnt < 32) {
            const int2 e = P.link[nxt - 1];
            if (lane == cnt) { mpos = nxt - 1; mbag = e.y; }
            ++cnt;
            nxt = e.x;
          }
          if (nxt == 0) {
            int rank = 0;  // positions are unique -> ranks are a permutation
            for (int i = 0; i < cnt; ++i) rank += (__shfl_sync(0xffffffffu, mpos, i) < mpos) ? 1 : 0;
            for (int q = 0; q < cnt; ++q) {
              const unsigned who = __ballot_sync(0xffffffffu, lane < cnt && rank == q);
              const int bag = __shfl_sync(0xffffffffu, mbag, __ffs(who) - 1);
#pragma unroll
              for (int v = 0; v < NV; ++v) {
                if (col_ok[v]) {
                  const Pack<W> t = ld_pack<W>(dy_row(P, bag) + dyk_off + lane * W + v * 32 * W);
#pragma unroll
                  for (int e = 0; e < W; ++e) g[v].x[e] += t.x[e];
                }
              }
            }
          } else {
            dup_sum_long<NV, W>(P, nxt0, self_bag, dyk_off, col_ok, g);
          }
        }
        if constexpr (RW) {
          float dv = 0.f;
#pragma unroll
          for (int v = 0; v < NV; ++v)
            if (col_ok[v])
#pragma unroll
              for (int e = 0; e < W; ++e) dv = fmaf(g[v].x[e], w[v].x[e], dv);
          dv = warp_sum(dv);
          const float vr = vpf[u];
#pragma unroll
          for (int v = 0; v < NV; ++v)
#pragma unroll
            for (int e = 0; e < W; ++e) g[v].x[e] *= vr;
          float s = vspf[u];
          const float v_new = row_weight_step(P, vr, dv, s);
          if (lane == 0) {
            P.row_w[ku][r] = v_new;
            if (P.optimizer != DLRM_OPT_SGD) P.row_w_sum[ku][r] = s;
          }
        }
        if constexpr (EW) {
          (void)m_old;
          const float nlr = -step_lr(P);
          float* srow = tb.mom + r * tb.mom_stride;
#pragma unroll
          for (int v = 0; v < NV; ++v)
            if (col_ok[v]) {
              Pack<W> s = spf[u][v];
#pragma unroll
              for (int e = 0; e < W; ++e) w[v].x[e] = adagrad_ew(g[v].x[e], s.x[e], w[v].x[e], nlr, P.eps);
              st_pack<W>(wrow + lane * W + v * 32 * W, w[v], is_f16<wt>::value ? sr_bits(rkey, lane + 32 * v) : 0ull);
              st_pack<W>(srow + lane * W + v * 32 * W, s);
            }
        } else if (P.optimizer == DLRM_OPT_RWSADAGRAD) {
          float sq = 0.f;
#pragma unroll
          for (int v = 0; v < NV; ++v)
            if (col_ok[v])
#pragma unroll
              for (int e = 0; e < W; ++e) sq = fmaf(g[v].x[e], g[v].x[e], sq);
          sq = warp_sum(sq);
          const float m_new = m_old + sq * inv_d;
          const float stdv = sqrtf(m_new) + P.eps;
          const float nlr = -step_lr(P);
#pragma unroll
          for (int v = 0; v < NV; ++v)
            if (col_ok[v]) {
#pragma unroll
              for (int e = 0; e < W; ++e) w[v].x[e] = fmaf(nlr, g[v].x[e] / stdv, w[v].x[e]);
              st_pack<W>(wrow + lane * W + v * 32 * W, w[v], is_f16<wt>::value ? sr_bits(rkey, lane + 32 * v) : 0ull);
            }
          if (lane == 0) tb.mom[r * tb.mom_stride] = m_new;
        } else {
          const float nlr = -step_lr(P);
#pragma unroll
          for (int v = 0; v < NV; ++v)
            if (col_ok[v]) {
#pragma unroll
              for (int e = 0; e < W; ++e) w[v].x[e] = fmaf(nlr, g[v].x[e], w[v].x[e]);
              st_pack<W>(wrow + lane * W + v * 32 * W, w[v], is_f16<wt>::value ? sr_bits(rkey, lane + 32 * v) : 0ull);
            }
        }
        if (lane == 0 && ((susp_mask >> src) & 1u)) tb.head[r * tb.hs] = 0;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Lean variant for dim <= 128 (one float4 per lane), the shape of every BASELINE config.
//
// In the kernel above the table descriptor is re-read from parameter space for every row, rows / tables / bags
// travel through 64-bit shuffles twice and the optimizer divides per element: at MLPerf sizes (1.75 M occurrences
// per step and GPU) that makes the update instruction-bound instead of bound by random DRAM accesses.  Here
//   * the per-table fields live in shared memory, a 32-position window takes its table from lane 0 unless
//     the window straddles a table boundary;
//   * every lane resolves ITS occurrence once (ownership from the coalesced mark, no table access) into
//     pointers to the weight row, gradient row, accumulator and list head; owners are compacted with
//     ballot/ffs and processed PF at a time: 2 pointer broadcasts + 2 row loads each, the owning lane loads
//     the accumulator, all issued before the first use;
//   * the row update is w += (-lr / (sqrt(m) + eps)) * g -- one reciprocal per row instead of a division per
//     element (differs from g / std by <= 1 ulp per element; the tests' tolerance is 2e-5 relative);
//   * the owning lane itself stores the accumulator and clears the list head with the row's store (no
//     pointer broadcast);
//   * rows with duplicates (rare at large tables) take an out-of-line path.
// ---------------------------------------------------------------------------------------------
struct UpdTableS {
  void* w;
  float* mom;
  int* head;
  unsigned char* mark;
  const void* idx;
  long long pair_base, ld, mom_stride, hs, dy_off, row_lo, row_n;
};

__device__ __noinline__ float4 upd_sum_long(const EmbBwdParams& P, int nxt, int self_bag, long long dy_off,
                                            bool col_ok) {
  const int lane = threadIdx.x & 31;
  auto load = [&](int bag, float (&t)[4]) {
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (col_ok) v = *reinterpret_cast<const float4*>(dy_row(P, bag) + dy_off + lane * 4);
    t[0] = v.x; t[1] = v.y; t[2] = v.z; t[3] = v.w;
  };
  float s[4];
  list_sum_exact<4>(P.link, nxt, self_bag, load, s);
  return make_float4(s[0], s[1], s[2], s[3]);
}

__device__ __noinline__ float4 upd_sum_duplicates(const EmbBwdParams& P, int nxt, int self_pos, int self_bag,
                                                  long long dy_off, int lane, bool col_ok) {
  // up to 32 members of the row's list (self first) are summed in ascending position (== grad.coalesce());
  // a longer list takes the order-independent sum
  float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
  const int nxt0 = nxt;
  int cnt = 1;
  int mpos = (lane == 0) ? self_pos : 0x7fffffff;
  int mbag = self_bag;
  while (nxt != 0 && cnt < 32) {
    const int2 e = P.link[nxt - 1];
    if (lane == cnt) { mpos = nxt - 1; mbag = e.y; }
    ++cnt;
    nxt = e.x;
  }
  if (nxt != 0) return upd_sum_long(P, nxt0, self_bag, dy_off, col_ok);
  int rank = 0;
  for (int i = 0; i < cnt; ++i) rank += (__shfl_sync(0xffffffffu, mpos, i) < mpos) ? 1 : 0;
  // the dY rows of DUP_BATCH members are loaded before any of them is added (one round trip per batch instead of
  // one per member); the adds keep the ascending-position order
  constexpr int DUP_BATCH = 4;
  for (int q0 = 0; q0 < cnt; q0 += DUP_BATCH) {
    float4 t[DUP_BATCH];
#pragma unroll
    for (int u = 0; u < DUP_BATCH; ++u) {
      const unsigned who = __ballot_sync(0xffffffffu, lane < cnt && rank == q0 + u);
      const int bag = __shfl_sync(0xffffffffu, mbag, who ? __ffs(who) - 1 : 0);
      t[u] = (who && col_ok) ? *reinterpret_cast<const float4*>(dy_row(P, bag) + dy_off + lane * 4)
                             : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int u = 0; u < DUP_BATCH; ++u)
      if (q0 + u < cnt && col_ok) { g.x += t[u].x; g.y += t[u].y; g.z += t[u].z; g.w += t[u].w; }
  }
  return g;
}

// PF: row PAIRS in flight per warp.  EW: element-wise Adagrad (DLRM_OPT_ADAGRAD): every lane also loads its 8
// accumulators (two float4 behind the row's accumulator pointer) in the same batch as the rows and stores them with
// the row.  EW = false is the SGD / RWSAdagrad kernel.  RW: learned weighted pooling (see emb_update_kernel): the
// owning lanes load v[r] and its sum with the row's accumulator and store them with it.
template <typename wt, typename idx_t, int PF, int MINB, bool EW = false, bool RW = false>
__global__ void __launch_bounds__(256, MINB) emb_update_lean_kernel(const __grid_constant__ EmbBwdParams P, int num_tables,
                                                                    long long total_hint) {
  __shared__ long long bound[DLRM_B200_MAX_TABLES_PER_CALL + 1], tend[DLRM_B200_MAX_TABLES_PER_CALL + 1];
  __shared__ UpdTableS ts[DLRM_B200_MAX_TABLES_PER_CALL];
  for (int k = threadIdx.x; k < num_tables; k += blockDim.x) {
    UpdTableS t;
    t.w = P.t[k].w; t.mom = P.t[k].mom; t.head = P.t[k].head; t.mark = P.t[k].mark; t.idx = P.t[k].idx;
    t.pair_base = P.t[k].pair_base; t.ld = P.t[k].ld; t.mom_stride = P.t[k].mom_stride; t.hs = P.t[k].hs;
    t.dy_off = P.t[k].dy_off; t.row_lo = P.t[k].row_lo; t.row_n = P.t[k].row_n;
    ts[k] = t;
  }
  load_bounds<idx_t>(bound, tend, P, num_tables, total_hint);     // ends with __syncthreads()
  const int D = P.dim;
  const int lane = threadIdx.x & 31;
  // Rows WITHOUT duplicates (almost all of them at large tables) are processed TWO per warp step: lanes 0-15
  // take one row, lanes 16-31 another, 8 columns (two float4; one 16-byte load of an fp16 row) per lane.  Every shuffle / FMA / branch of the
  // step then serves two rows, and twice as many rows are in flight per warp.
  const int half = lane >> 4, l16 = lane & 15;
  const bool c0_ok = l16 * 8 < D, c1_ok = l16 * 8 + 4 < D;
  const bool col_ok = lane * 4 < D;                          // full-warp layout of the duplicate path
  const long long first = bound[0], total = bound[num_tables];
  const long long warp0 = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long wstep = (long long)gridDim.x * (blockDim.x >> 5) * 32;
  const float inv_d = 1.0f / (float)D;
  const float nlr = -step_lr(P);
  const bool adagrad = !EW && P.optimizer == DLRM_OPT_RWSADAGRAD;    // row-wise
  const int dbg = P.debug;

  for (long long base = first + warp0 * 32; base < total; base += wstep) {
    // index, list entry and mark of the 32 positions of the window: coalesced, and all that ownership needs
    const long long pos = base + lane;
    // table of this window: lane 0's, unless the window crosses into the next table
    int k = table_of(bound, num_tables, base);
    if (base + 31 >= bound[k + 1]) k = table_of(bound, num_tables, pos < total ? pos : base);
    const UpdTableS& tb = ts[k];
    int r = 0;
    int2 lk = make_int2(0, 0);
    bool owner = false;
    if (pos < total && pos < tend[k] && tb.head != nullptr) {   // positions between two tables of the call are not ours
      const long long rr = (long long)static_cast<const idx_t*>(tb.idx)[pos - tb.pair_base] - tb.row_lo;
      lk = P.link[pos];
      const unsigned char superseded = tb.mark[pos];
      if (superseded) tb.mark[pos] = 0;
      // the last occurrence to arrive (never superseded) owns the row; rows of another shard are not ours
      owner = (unsigned long long)rr < (unsigned long long)tb.row_n && !superseded;
      r = (int)rr;
    }
    const int nxt = owner ? lk.x : 0, bag = lk.y;
    wt* wptr = owner ? static_cast<wt*>(tb.w) + (long long)r * tb.ld : nullptr;
    // fp16: the key of the owned GLOBAL row for the stochastic rounding of its columns
    const unsigned long long rkey =
        (is_f16<wt>::value && owner) ? sr_row_key(P.round_key[k], (long long)r + tb.row_lo) : 0ull;
    const float* gptr = owner ? dy_row(P, bag) + tb.dy_off : nullptr;
    float* mptr = (owner && (adagrad || EW)) ? tb.mom + (long long)r * tb.mom_stride : nullptr;
    int* hptr = owner ? tb.head + (long long)r * tb.hs : nullptr;
    float* vptr = (RW && owner) ? P.row_w[k] + r : nullptr;
    float* vsptr = (RW && owner && P.optimizer != DLRM_OPT_SGD) ? P.row_w_sum[k] + r : nullptr;
    unsigned simple = __ballot_sync(0xffffffffu, owner && nxt == 0);
    unsigned dups = __ballot_sync(0xffffffffu, owner && nxt != 0);

    // ---------------------------------------------------------------- rows without duplicates, two per step
    while (simple) {
      float4 wv[PF][2], gv[PF][2];
      float4 sv[EW ? PF : 1][2];                   // EW: the lane's 8 accumulators
      float mv[PF];
      float vv[RW ? PF : 1], vs[RW ? PF : 1];     // RW: the owning lanes' v[r] and sum
      int sa[PF], sb[PF];
#pragma unroll
      for (int u = 0; u < PF; ++u) {
        sa[u] = simple ? __ffs(simple) - 1 : -1;
        simple &= simple - 1u;
        sb[u] = simple ? __ffs(simple) - 1 : -1;
        simple &= simple - 1u;
        const int s_ = half ? sb[u] : sa[u];
        const int sc = s_ < 0 ? 0 : s_;
        const wt* wp = reinterpret_cast<const wt*>(__shfl_sync(0xffffffffu, (unsigned long long)wptr, sc)) + l16 * 8;
        const float* gp = reinterpret_cast<const float*>(__shfl_sync(0xffffffffu, (unsigned long long)gptr, sc)) + l16 * 8;
        const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
        const bool ldw = !(dbg & 2), ldg = !(dbg & 8);
        if constexpr (is_f16<wt>::value) {      // 8 halves = one 16-byte load (c1_ok == c0_ok: dim % 8 == 0)
          if (s_ >= 0 && c0_ok && ldw) {
            const uint4 h = *reinterpret_cast<const uint4*>(wp);
            wv[u][0] = h4_to_f4(make_uint2(h.x, h.y));
            wv[u][1] = h4_to_f4(make_uint2(h.z, h.w));
          } else {
            wv[u][0] = z; wv[u][1] = z;
          }
        } else {
          wv[u][0] = (s_ >= 0 && c0_ok && ldw) ? *reinterpret_cast<const float4*>(wp) : z;
          wv[u][1] = (s_ >= 0 && c1_ok && ldw) ? *reinterpret_cast<const float4*>(wp + 4) : z;
        }
        gv[u][0] = (s_ >= 0 && c0_ok && ldg) ? *reinterpret_cast<const float4*>(gp) : z;
        gv[u][1] = (s_ >= 0 && c1_ok && ldg) ? *reinterpret_cast<const float4*>(gp + 4) : z;
        // the owning lanes load their accumulators in the same batch as the rows
        mv[u] = (adagrad && (lane == sa[u] || lane == sb[u])) ? *mptr : 0.f;
        if constexpr (RW) {
          vv[u] = (lane == sa[u] || lane == sb[u]) ? *vptr : 0.f;
          vs[u] = ((lane == sa[u] || lane == sb[u]) && vsptr) ? *vsptr : 0.f;
        }
        if constexpr (EW) {
          const float* sp = reinterpret_cast<const float*>(__shfl_sync(0xffffffffu, (unsigned long long)mptr, sc)) + l16 * 8;
          sv[u][0] = (s_ >= 0 && c0_ok) ? *reinterpret_cast<const float4*>(sp) : z;
          sv[u][1] = (s_ >= 0 && c1_ok) ? *reinterpret_cast<const float4*>(sp + 4) : z;
        }
      }
#pragma unroll
      for (int u = 0; u < PF; ++u) {
        if (sa[u] < 0) break;
        const int s_ = half ? sb[u] : sa[u];
        const int sc = s_ < 0 ? 0 : s_;
        float4 g0 = gv[u][0], g1 = gv[u][1];
        if constexpr (RW) {       // dv = <S, W_old> within the half; S *= v[r]; the owning lanes store v' and s'
          const float4 w0 = wv[u][0], w1 = wv[u][1];
          float dv = fmaf(g0.x, w0.x, fmaf(g0.y, w0.y, fmaf(g0.z, w0.z, g0.w * w0.w)));
          dv = fmaf(g1.x, w1.x, fmaf(g1.y, w1.y, fmaf(g1.z, w1.z, fmaf(g1.w, w1.w, dv))));
#pragma unroll
          for (int o = 8; o > 0; o >>= 1) dv += __shfl_xor_sync(0xffffffffu, dv, o);
          const float vr = __shfl_sync(0xffffffffu, vv[u], sc);
          float s = __shfl_sync(0xffffffffu, vs[u], sc);
          const float v_new = row_weight_step(P, vr, dv, s);
          g0.x *= vr; g0.y *= vr; g0.z *= vr; g0.w *= vr;
          g1.x *= vr; g1.y *= vr; g1.z *= vr; g1.w *= vr;
          const float vA = __shfl_sync(0xffffffffu, v_new, 0), vB = __shfl_sync(0xffffffffu, v_new, 16);
          const float sA = __shfl_sync(0xffffffffu, s, 0), sB = __shfl_sync(0xffffffffu, s, 16);
          if (lane == sa[u]) { *vptr = vA; if (vsptr) *vsptr = sA; }
          if (lane == sb[u]) { *vptr = vB; if (vsptr) *vsptr = sB; }
        }
        float scale = nlr;
        if (adagrad) {
          float sq = fmaf(g0.x, g0.x, fmaf(g0.y, g0.y, fmaf(g0.z, g0.z, g0.w * g0.w)));
          sq = fmaf(g1.x, g1.x, fmaf(g1.y, g1.y, fmaf(g1.z, g1.z, fmaf(g1.w, g1.w, sq))));
#pragma unroll
          for (int o = 8; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);     // within the half
          const float m_new = __shfl_sync(0xffffffffu, mv[u], sc) + sq * inv_d;
          scale = nlr / (sqrtf(m_new) + P.eps);
          const float mA = __shfl_sync(0xffffffffu, m_new, 0), mB = __shfl_sync(0xffffffffu, m_new, 16);
          if (lane == sa[u] && !(dbg & 4)) *mptr = mA;               // the owning lanes store their accumulators
          if (lane == sb[u] && !(dbg & 4)) *mptr = mB;
        }
        wt* wp = reinterpret_cast<wt*>(__shfl_sync(0xffffffffu, (unsigned long long)wptr, sc)) + l16 * 8;
        float* spw = nullptr;
        float4 s0, s1;
        if constexpr (EW) {                  // element-wise step: the accumulators move with the row
          spw = reinterpret_cast<float*>(__shfl_sync(0xffffffffu, (unsigned long long)mptr, sc)) + l16 * 8;
          s0 = sv[u][0]; s1 = sv[u][1];
        }
        if constexpr (is_f16<wt>::value) {
          const unsigned long long rk = __shfl_sync(0xffffffffu, rkey, sc);
          if (s_ >= 0) {
            float4 w0 = wv[u][0], w1 = wv[u][1];
            if constexpr (EW) {
              w0 = adagrad_ew4(g0, s0, w0, nlr, P.eps);
              w1 = adagrad_ew4(g1, s1, w1, nlr, P.eps);
              if (c0_ok && !(dbg & 4)) {
                *reinterpret_cast<float4*>(spw) = s0;
                *reinterpret_cast<float4*>(spw + 4) = s1;
              }
            } else {
              w0.x = fmaf(scale, g0.x, w0.x); w0.y = fmaf(scale, g0.y, w0.y); w0.z = fmaf(scale, g0.z, w0.z); w0.w = fmaf(scale, g0.w, w0.w);
              w1.x = fmaf(scale, g1.x, w1.x); w1.y = fmaf(scale, g1.y, w1.y); w1.z = fmaf(scale, g1.z, w1.z); w1.w = fmaf(scale, g1.w, w1.w);
            }
            if (c0_ok && !(dbg & 1)) {
              uint2 a, b;
              st_row4(reinterpret_cast<__half*>(&a), w0, sr_bits(rk, l16 * 2));
              st_row4(reinterpret_cast<__half*>(&b), w1, sr_bits(rk, l16 * 2 + 1));
              *reinterpret_cast<uint4*>(wp) = make_uint4(a.x, a.y, b.x, b.y);
            }
          }
        } else if (s_ >= 0) {
          float4 w0 = wv[u][0], w1 = wv[u][1];
          if constexpr (EW) {
            w0 = adagrad_ew4(g0, s0, w0, nlr, P.eps);
            w1 = adagrad_ew4(g1, s1, w1, nlr, P.eps);
            if (c0_ok && !(dbg & 4)) *reinterpret_cast<float4*>(spw) = s0;
            if (c1_ok && !(dbg & 4)) *reinterpret_cast<float4*>(spw + 4) = s1;
          } else {
            w0.x = fmaf(scale, g0.x, w0.x); w0.y = fmaf(scale, g0.y, w0.y); w0.z = fmaf(scale, g0.z, w0.z); w0.w = fmaf(scale, g0.w, w0.w);
            w1.x = fmaf(scale, g1.x, w1.x); w1.y = fmaf(scale, g1.y, w1.y); w1.z = fmaf(scale, g1.z, w1.z); w1.w = fmaf(scale, g1.w, w1.w);
          }
          if (c0_ok && !(dbg & 1)) *reinterpret_cast<float4*>(wp) = w0;
          if (c1_ok && !(dbg & 1)) *reinterpret_cast<float4*>(wp + 4) = w1;
        }
        if ((lane == sa[u] || lane == sb[u]) && !(dbg & 4)) *hptr = 0;
      }
    }

    // ---------------------------------------------------------------- rows with duplicates, one per step
    while (dups) {
      const int s_ = __ffs(dups) - 1;
      dups &= dups - 1u;
      const int nx = __shfl_sync(0xffffffffu, nxt, s_);
      const int sbg = __shfl_sync(0xffffffffu, bag, s_);
      const long long dyo = __shfl_sync(0xffffffffu, tb.dy_off, s_);       // the OWNER's table (windows may straddle)
      wt* wp = reinterpret_cast<wt*>(__shfl_sync(0xffffffffu, (unsigned long long)wptr, s_));
      float4 w = col_ok ? ld_row4(wp + lane * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
      const float m_old = (adagrad && lane == s_) ? *mptr : 0.f;
      const float v_old = (RW && lane == s_) ? *vptr : 0.f;
      const float vs_old = (RW && lane == s_ && vsptr) ? *vsptr : 0.f;
      float* spd = nullptr;
      float4 sd = make_float4(0.f, 0.f, 0.f, 0.f);
      if constexpr (EW) {
        spd = reinterpret_cast<float*>(__shfl_sync(0xffffffffu, (unsigned long long)mptr, s_)) + lane * 4;
        if (col_ok) sd = *reinterpret_cast<const float4*>(spd);
      }
      float4 g = upd_sum_duplicates(P, nx, (int)(base + s_), sbg, dyo, lane, col_ok);
      if constexpr (RW) {
        const float dv = warp_sum(col_ok ? fmaf(g.x, w.x, fmaf(g.y, w.y, fmaf(g.z, w.z, g.w * w.w))) : 0.f);
        const float vr = __shfl_sync(0xffffffffu, v_old, s_);
        float s = __shfl_sync(0xffffffffu, vs_old, s_);
        const float v_new = row_weight_step(P, vr, dv, s);
        g.x *= vr; g.y *= vr; g.z *= vr; g.w *= vr;
        if (lane == s_) { *vptr = v_new; if (vsptr) *vsptr = s; }
      }
      if constexpr (EW) {
        w = adagrad_ew4(g, sd, w, nlr, P.eps);
        if (col_ok) *reinterpret_cast<float4*>(spd) = sd;
      } else {
        float scale = nlr;
        if (adagrad) {
          float sq = fmaf(g.x, g.x, fmaf(g.y, g.y, fmaf(g.z, g.z, g.w * g.w)));
          sq = warp_sum(sq);
          const float m_new = __shfl_sync(0xffffffffu, m_old, s_) + sq * inv_d;
          scale = nlr / (sqrtf(m_new) + P.eps);
          if (lane == s_) *mptr = m_new;
        }
        w.x = fmaf(scale, g.x, w.x); w.y = fmaf(scale, g.y, w.y);
        w.z = fmaf(scale, g.z, w.z); w.w = fmaf(scale, g.w, w.w);
      }
      if constexpr (is_f16<wt>::value) {
        const unsigned long long rk = __shfl_sync(0xffffffffu, rkey, s_);
        if (col_ok) st_row4(wp + lane * 4, w, sr_bits(rk, lane));
      } else {
        if (col_ok) *reinterpret_cast<float4*>(wp + lane * 4) = w;
      }
      if (lane == s_) *hptr = 0;
    }
  }
}

static int fill_params(EmbBwdParams& P, const dlrm_emb_bwd_table_t* tables, int num_tables,
                       const char* who) {
  if (num_tables < 0 || num_tables > DLRM_B200_MAX_TABLES_PER_CALL)
    return set_error("%s: num_tables=%d out of range [0,%d]", who, num_tables,
                     DLRM_B200_MAX_TABLES_PER_CALL);
  for (int k = 0; k < num_tables; ++k) {
    if (!tables[k].offsets || (!tables[k].indices && tables[k].nnz > 0))
      return set_error("%s: table %d has a NULL pointer", who, k);
    if (tables[k].pair_base + tables[k].nnz > 0x7ffffffeLL)
      return set_error("%s: more than 2^31-2 index occurrences in one call", who);
    P.t[k].w = tables[k].weight;
    P.t[k].mom = tables[k].momentum;
    P.t[k].head = tables[k].head;
    P.t[k].mark = tables[k].mark;
    if (tables[k].head && !tables[k].mark) return set_error("%s: table %d: head without a mark array", who, k);
    P.t[k].idx = tables[k].indices;
    P.t[k].off = tables[k].offsets;
    P.t[k].nnz = tables[k].nnz;
    P.t[k].pair_base = tables[k].pair_base;
    P.t[k].ld = tables[k].ld;   // 0 -> dim, resolved by the update entry point
    P.t[k].mom_stride = tables[k].mom_stride > 0 ? tables[k].mom_stride : 1;
    P.t[k].hs = tables[k].head_stride > 0 ? tables[k].head_stride : 1;
    P.t[k].dy_off = 0;          // resolved by the update entry point
    P.t[k].rows = tables[k].rows > 0 ? tables[k].rows : 0x7fffffffffffffffLL;
    P.t[k].row_lo = tables[k].row_n > 0 ? tables[k].row_lo : 0;
    P.t[k].row_n = tables[k].row_n > 0 ? tables[k].row_n : P.t[k].rows;
    P.round_key[k] = tables[k].round_key;
    if (tables[k].weight_dtype != tables[0].weight_dtype)
      return set_error("%s: table %d: weight_dtype differs from table 0's (one row type per call)", who, k);
  }
  if (num_tables > 0 && tables[0].weight_dtype != DLRM_DTYPE_F32 && tables[0].weight_dtype != DLRM_DTYPE_F16)
    return set_error("%s: weight_dtype=%d", who, tables[0].weight_dtype);
  return 0;
}

}  // namespace dlrm

extern "C" int dlrm_b200_emb_bwd_link(const dlrm_emb_bwd_table_t* tables, int num_tables,
                                      int64_t batch, int idx_bytes, int include_last,
                                      int32_t* next, void* stream) {
  using namespace dlrm;
  EmbBwdParams P{};
  if (int rc = fill_params(P, tables, num_tables, "emb_bwd_link")) return rc;
  if (idx_bytes != 4 && idx_bytes != 8) return set_error("emb_bwd_link: idx_bytes=%d", idx_bytes);
  if (num_tables == 0 || batch == 0) return 0;
  if (!next) return set_error("emb_bwd_link: next is NULL");
  P.link = reinterpret_cast<int2*>(next);
  P.batch = batch;
  P.include_last = include_last;
  long long max_nnz = 0;
  for (int k = 0; k < num_tables; ++k) max_nnz = tables[k].nnz > max_nnz ? tables[k].nnz : max_nnz;
  if (max_nnz == 0) return 0;
  const int block = 256;
  long long gx = (max_nnz + block - 1) / block;
  if (gx > 65535) gx = 65535;  // grid-stride loop covers the rest
  dim3 grid((unsigned)gx, (unsigned)num_tables);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (idx_bytes == 8) emb_link_kernel<long long><<<grid, block, 0, st>>>(P);
  else emb_link_kernel<int><<<grid, block, 0, st>>>(P);
  DLRM_CHECK_LAUNCH("emb_link_kernel");
  return 0;
}

// Lean-kernel shape of the element-wise Adagrad instantiation: row pairs in flight per warp, CTAs per SM.
constexpr int EW_PF = 2, EW_MINB = 2;
// and of the learned-weight instantiation: v and its sum per row pair spill at 3 CTAs per SM (80 registers)
constexpr int RW_PF = 2, RW_MINB = 2;

static int emb_update_impl(const dlrm_emb_bwd_table_t* tables, int num_tables, int dim, int64_t batch,
                           int idx_bytes, int include_last, const int32_t* next, const float* dY,
                           int64_t dy_stride_sample, int64_t dy_stride_table, int optimizer, float lr,
                           float eps, void* stream, const float* const* peer_dY, int world,
                           int64_t batch_local, const dlrm_emb_dedup_t* dedup, const float* lr_dev = nullptr) {
  using namespace dlrm;
  EmbBwdParams P{};
  if (int rc = fill_params(P, tables, num_tables, "emb_bwd_update")) return rc;
  if (idx_bytes != 4 && idx_bytes != 8) return set_error("emb_bwd_update: idx_bytes=%d", idx_bytes);
  if (optimizer != DLRM_OPT_SGD && optimizer != DLRM_OPT_RWSADAGRAD && optimizer != DLRM_OPT_ADAGRAD)
    return set_error("emb_bwd_update: optimizer=%d", optimizer);
  const bool ew = optimizer == DLRM_OPT_ADAGRAD;
  if (dim <= 0 || dim > 1024) return set_error("emb_bwd_update: dim=%d unsupported (1..1024)", dim);
  const bool f16 = num_tables > 0 && tables[0].weight_dtype == DLRM_DTYPE_F16;
  if (f16 && dim % 8) return set_error("emb_bwd_update: fp16 tables need dim %% 8 == 0 (dim=%d)", dim);
  bool lean_rows = true;
  if (num_tables == 0 || batch == 0) return 0;
  if (!next || (!dY && !peer_dY)) return set_error("emb_bwd_update: NULL next/dY");
  bool vec = (dim % 4 == 0) && (peer_dY || aligned16(dY)) && dy_stride_sample % 4 == 0 && dy_stride_table % 4 == 0;
  P.flags = (dedup && dedup->flags) ? dedup->flags : nullptr;
  bool rw = false;
  for (int k = 0; k < num_tables; ++k) rw = rw || tables[k].row_weights != nullptr;
  if (rw) {
    if (peer_dY) return set_error("emb_bwd_update_p2p: row_weights (learned weighted pooling) is not supported");
    if (P.flags) return set_error("emb_bwd_update: the duplicate filter does not support row_weights");
    for (int k = 0; k < num_tables; ++k) {
      if (!tables[k].row_weights)
        return set_error("emb_bwd_update: table %d: row_weights must be set for every table of a call or for none", k);
      if (optimizer != DLRM_OPT_SGD && !tables[k].row_weight_sum)
        return set_error("emb_bwd_update: table %d: row_weight_sum NULL (needed by optimizer=%d)", k, optimizer);
      P.row_w[k] = tables[k].row_weights;
      P.row_w_sum[k] = tables[k].row_weight_sum;
    }
  }
  P.peer_batch = 0;
  for (int d = 0; d < DLRM_B200_MAX_PEERS; ++d) P.peer_dY[d] = nullptr;
  if (peer_dY) {
    if (world < 1 || world > DLRM_B200_MAX_PEERS || batch_local <= 0 || batch_local * world != batch)
      return set_error("emb_bwd_update_p2p: world=%d batch_local=%lld batch=%lld", world, (long long)batch_local,
                       (long long)batch);
    for (int d = 0; d < world; ++d) {
      if (!peer_dY[d]) return set_error("emb_bwd_update_p2p: peer %d pointer is NULL", d);
      vec = vec && aligned16(peer_dY[d]);
      P.peer_dY[d] = peer_dY[d];
    }
    P.peer_batch = batch_local;
    dY = peer_dY[0];
  }
  for (int k = 0; k < num_tables; ++k) {
    P.t[k].dy_off = tables[k].use_dy_off ? tables[k].dy_off : (int64_t)k * dy_stride_table;
    vec = vec && (P.t[k].dy_off % 4 == 0);
    if (!tables[k].weight) return set_error("emb_bwd_update: table %d weight NULL", k);
    if ((optimizer == DLRM_OPT_RWSADAGRAD || ew) && !tables[k].momentum)
      return set_error("emb_bwd_update: table %d momentum NULL", k);
    if (ew) {     // one accumulator per element: rows of at least dim floats, the vector kernels need 16-byte ones
      P.t[k].mom_stride = tables[k].mom_stride > 0 ? tables[k].mom_stride : dim;
      if (P.t[k].mom_stride < dim) return set_error("emb_bwd_update: table %d: Adagrad mom_stride < dim", k);
      vec = vec && aligned16(tables[k].momentum) && P.t[k].mom_stride % 4 == 0;
    }
    vec = vec && aligned16(tables[k].weight);
    if (P.t[k].ld <= 0) P.t[k].ld = dim;
    if (P.t[k].ld < dim) return set_error("emb_bwd_update: table %d: ld < dim", k);
    vec = vec && (P.t[k].ld % 4 == 0);
    // the lean kernel moves 8 columns per lane in one 16-byte access: fp16 rows must start on 16-byte boundaries
    // (ld % 8 halves); fp16 rows that are only 8-byte aligned take the general kernel (8-byte accesses)
    lean_rows = lean_rows && (!f16 || P.t[k].ld % 8 == 0);
  }
  P.link = reinterpret_cast<int2*>(const_cast<int32_t*>(next));
  P.dY = dY;
  P.dy_stride_sample = dy_stride_sample;
  P.dy_stride_table = dy_stride_table;
  P.batch = batch;
  P.dim = dim;
  P.include_last = include_last;
  P.optimizer = optimizer;
  P.lr = lr;
  P.lr_dev = lr_dev;
  P.eps = eps;
  P.debug = get_tunable(TUNE_UPD_DEBUG);
  const int block = 256;
  long long total = 0;
  for (int k = 0; k < num_tables; ++k) total += tables[k].nnz;   // reference format: exact; packed: capacity
  if (include_last) {
    total = 0;
    for (int k = 0; k < num_tables; ++k) total = tables[k].nnz > total ? tables[k].nnz : total;
  }
  if (total == 0) return 0;
  int dev = 0, sms = 0;
  DLRM_CUDA(cudaGetDevice(&dev));
  DLRM_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  long long gridx = (total / 32 + block / 32) / (block / 32);
  if (gridx > (long long)sms * 3) gridx = (long long)sms * 3;
  if (gridx < 1) gridx = 1;
  const long long total_hint = include_last ? 0 : (tables[num_tables - 1].pair_base + tables[num_tables - 1].nnz);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
#define UPD_R(WT, Wd, NV, EW, RW)                                                                                 \
  do {                                                                                                               \
    if (idx_bytes == 8)                                                                                              \
      emb_update_kernel<WT, Wd, NV, long long, EW, RW><<<(unsigned)gridx, block, 0, st>>>(P, num_tables, total_hint); \
    else                                                                                                             \
      emb_update_kernel<WT, Wd, NV, int, EW, RW><<<(unsigned)gridx, block, 0, st>>>(P, num_tables, total_hint);      \
    DLRM_CHECK_LAUNCH("emb_update_kernel");                                                                          \
    return 0;                                                                                                        \
  } while (0)
#define UPD_E(WT, Wd, NV, EW)              \
  do {                                     \
    if (rw) UPD_R(WT, Wd, NV, EW, true);   \
    UPD_R(WT, Wd, NV, EW, false);          \
  } while (0)
#define UPD_T(WT, Wd, NV)   \
  do {                      \
    if (ew) UPD_E(WT, Wd, NV, true); \
    UPD_E(WT, Wd, NV, false);        \
  } while (0)
#define UPD(Wd, NV) UPD_T(float, Wd, NV)
#define LEAN(WT, IDX)                                                                                              \
  do {                                                                                                             \
    if (ew && rw) emb_update_lean_kernel<WT, IDX, EW_PF, EW_MINB, true, true><<<(unsigned)gl, block, 0, st>>>(P, num_tables, total_hint); \
    else if (ew) emb_update_lean_kernel<WT, IDX, EW_PF, EW_MINB, true><<<(unsigned)gl, block, 0, st>>>(P, num_tables, total_hint); \
    else if (rw) emb_update_lean_kernel<WT, IDX, RW_PF, RW_MINB, false, true><<<(unsigned)gl, block, 0, st>>>(P, num_tables, total_hint); \
    else emb_update_lean_kernel<WT, IDX, 2, 3><<<(unsigned)gl, block, 0, st>>>(P, num_tables, total_hint);        \
  } while (0)
  if (f16 && !vec)
    return set_error("emb_bwd_update: fp16 tables need a 16-byte aligned weight pointer, ld %% 4 == 0 (8-byte rows) "
                     "and 16-byte aligned gradient rows%s", ew ? " and accumulators (momentum, mom_stride % 4 == 0)" : "");
  if (vec && lean_rows && dim <= 128 && !P.flags && get_tunable(TUNE_UPD_LEAN) != 2) {
    long long gl = (total / 32 + block / 32) / (block / 32);
    if (gl > (long long)sms * 3) gl = (long long)sms * 3;
    if (gl < 1) gl = 1;
    // 3 CTAs of 256 threads per SM (<= 85 registers), 2 row pairs in flight per warp: on H100 (cfg3) 3 pairs /
    // 3 CTAs and 4 pairs / 2 CTAs per SM were measured no faster and 8 % slower.  The kernel is bound by the RATE of random accesses
    // (row + accumulator read, row + accumulator + head write), not by the latency of any one of them.
    // Element-wise Adagrad carries 16 more floats per row pair (the accumulators): EW_PF / EW_MINB above.
    if (f16) {
      if (idx_bytes == 8) LEAN(__half, long long);
      else LEAN(__half, int);
    } else if (idx_bytes == 8) {
      LEAN(float, long long);
    } else {
      LEAN(float, int);
    }
    DLRM_CHECK_LAUNCH("emb_update_lean_kernel");
    return 0;
  }
  if (f16) {
    if (dim <= 128) UPD_T(__half, 4, 1);
    if (dim <= 256) UPD_T(__half, 4, 2);
    if (dim <= 512) UPD_T(__half, 4, 4);
    UPD_T(__half, 4, 8);
  }
  if (vec) {
    if (dim <= 128) UPD(4, 1);
    if (dim <= 256) UPD(4, 2);
    if (dim <= 512) UPD(4, 4);
    UPD(4, 8);
  }
  if (dim <= 32) UPD(1, 1);
  if (dim <= 64) UPD(1, 2);
  if (dim <= 128) UPD(1, 4);
  if (dim <= 256) UPD(1, 8);
  if (dim <= 512) UPD(1, 16);
  UPD(1, 32);
#undef LEAN
#undef UPD
#undef UPD_T
#undef UPD_E
#undef UPD_R
}

extern "C" int dlrm_b200_emb_bwd_update(const dlrm_emb_bwd_table_t* tables, int num_tables, int dim,
                                        int64_t batch, int idx_bytes, int include_last,
                                        const int32_t* next, const float* dY,
                                        int64_t dy_stride_sample, int64_t dy_stride_table,
                                        int optimizer, float lr, float eps, const dlrm_emb_dedup_t* dedup,
                                        void* stream) {
  return emb_update_impl(tables, num_tables, dim, batch, idx_bytes, include_last, next, dY, dy_stride_sample,
                         dy_stride_table, optimizer, lr, eps, stream, nullptr, 0, 0, dedup);
}

extern "C" int dlrm_b200_emb_bwd_update_lr_dev(const dlrm_emb_bwd_table_t* tables, int num_tables, int dim,
                                               int64_t batch, int idx_bytes, int include_last,
                                               const int32_t* next, const float* dY,
                                               int64_t dy_stride_sample, int64_t dy_stride_table,
                                               int optimizer, float lr, const float* lr_dev, float eps,
                                               const dlrm_emb_dedup_t* dedup, void* stream) {
  return emb_update_impl(tables, num_tables, dim, batch, idx_bytes, include_last, next, dY, dy_stride_sample,
                         dy_stride_table, optimizer, lr, eps, stream, nullptr, 0, 0, dedup, lr_dev);
}

extern "C" int dlrm_b200_emb_bwd_classify(const dlrm_emb_bwd_table_t* tables, int num_tables, int64_t batch,
                                          int idx_bytes, int include_last, int32_t* next,
                                          const dlrm_emb_dedup_t* dedup, void* stream) {
  using namespace dlrm;
  EmbBwdParams P{};
  if (int rc = fill_params(P, tables, num_tables, "emb_bwd_classify")) return rc;
  if (idx_bytes != 4 && idx_bytes != 8) return set_error("emb_bwd_classify: idx_bytes=%d", idx_bytes);
  if (!dedup || !dedup->filter || !dedup->flags || !dedup->suspects || !next)
    return set_error("emb_bwd_classify: NULL dedup buffers");
  if (num_tables == 0 || batch == 0) return 0;
  P.link = reinterpret_cast<int2*>(next);
  P.batch = batch;
  P.include_last = include_last;
  long long total = 0;
  for (int k = 0; k < num_tables; ++k) total += tables[k].nnz;
  if (include_last) {
    total = 0;
    for (int k = 0; k < num_tables; ++k) total = tables[k].nnz > total ? tables[k].nnz : total;
  }
  if (total == 0) return 0;
  const long long total_hint = include_last ? 0 : (tables[num_tables - 1].pair_base + tables[num_tables - 1].nnz);
  int dev = 0, sms = 0;
  DLRM_CUDA(cudaGetDevice(&dev));
  DLRM_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  long long gridx = (total / 32 + 7) / 8;
  if (gridx > (long long)sms * 8) gridx = (long long)sms * 8;
  if (gridx < 1) gridx = 1;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int* n_susp = reinterpret_cast<int*>(dedup->filter + ((size_t)1 << dedup->log2_size));
  if (idx_bytes == 8) {
    emb_classify_kernel<long long><<<(unsigned)gridx, 256, 0, st>>>(P, num_tables, total_hint, dedup->filter,
                                                                    dedup->log2_size, dedup->flags, dedup->suspects, n_susp);
    DLRM_CHECK_LAUNCH("emb_classify_kernel");
    emb_link_suspects_kernel<long long><<<sms, 256, 0, st>>>(P, num_tables, total_hint, dedup->suspects, n_susp);
  } else {
    emb_classify_kernel<int><<<(unsigned)gridx, 256, 0, st>>>(P, num_tables, total_hint, dedup->filter,
                                                              dedup->log2_size, dedup->flags, dedup->suspects, n_susp);
    DLRM_CHECK_LAUNCH("emb_classify_kernel");
    emb_link_suspects_kernel<int><<<sms, 256, 0, st>>>(P, num_tables, total_hint, dedup->suspects, n_susp);
  }
  DLRM_CHECK_LAUNCH("emb_link_suspects_kernel");
  return 0;
}

extern "C" int dlrm_b200_emb_bwd_update_p2p(const dlrm_emb_bwd_table_t* tables, int num_tables, int dim,
                                            int64_t batch_global, int idx_bytes, int include_last,
                                            const int32_t* next, const float* const* peer_dY, int world,
                                            int64_t batch_local, int64_t dy_stride_sample,
                                            int64_t dy_stride_table, int optimizer, float lr, float eps,
                                            const dlrm_emb_dedup_t* dedup, void* stream) {
  if (!peer_dY) return dlrm::set_error("emb_bwd_update_p2p: peer_dY is NULL");
  return emb_update_impl(tables, num_tables, dim, batch_global, idx_bytes, include_last, next, nullptr,
                         dy_stride_sample, dy_stride_table, optimizer, lr, eps, stream, peer_dY, world,
                         batch_local, dedup);
}
