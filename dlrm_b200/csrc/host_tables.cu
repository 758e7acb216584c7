// Embedding tables in pinned host memory ("host tables"): the rows a batch touches are staged through an HBM
// arena, so the gather and the fused update run unchanged on device addresses.  An optional row cache keeps the
// recently used rows in the same arena between steps.
//
// Arena: N cache slots (N = cache_rows, 0 without a cache) followed by one staging slot per position of the batch;
// the gather and the update see it as one table of N + capacity rows.  map[row] (int32 per host row) is
//   0            the row is in host memory only;
//   1 .. N       slot + 1 of the cache slot that holds the row (kept across steps);
//   N + 1 ..     slot + 1 = N + p + 1 of this step's staging slot (p: the position that claimed the row).
//
//   stage_in   before the gather, one pass over the batch's occurrences of the host tables.  For occurrence p of
//              host table t (p = its global position: packed batches share one index array; reference-format
//              batches number the tables' positions back to back, pos_base = pair_base):
//                row outside [0, rows)  -> device error bit 0 (as the gather), slot index -1, no host access;
//                else atomicCAS(map[row], 0, N + p + 1):
//                  0 before: a miss.  p claims the row: slot N + p (positions are distinct and < capacity, so no
//                     sort is needed), appends the slot to the list through the one counter, and copies the row --
//                     weights and its in-row accumulator / separate accumulator / element-wise Adagrad row -- from
//                     host memory with zero-copy reads through the UVA pointer; the staged list head is zero.  With
//                     a cache, a training pass also threads p onto the per-set list of the row's set;
//                  1 .. N: a hit, slot = map - 1.  A training pass stamps the slot's last use with the step; the
//                     occurrence that stamps first counts the hit;
//                  else: another occurrence's staging slot;
//                every occurrence writes its slot into slot_idx[p], parallel to the batch's index array.
//   write_back after the update, on the same stream.  With a cache, insert first: one warp per set with misses picks
//              the set's 32 smallest misses by (table, row), orders the ways not used in this step by (last use,
//              way) -- an empty way has last use 0 -- and gives the i-th miss the i-th way.  A victim's row and
//              words go to host memory and its map entry is cleared; the miss moves HBM-to-HBM into the slot and its
//              map entry becomes the cache slot.  Then every listed slot whose map entry still names it goes back to
//              its host row (list head written as zero) and its entry is reset.  release: the reset alone (forward
//              only).  flush: every resident row goes home and the cache is emptied.
//
// Invariants between steps: the map holds no staging entry (stage_in claims, write_back / release clears exactly the
// entries it claimed and the inserts turned into cache entries); a cache entry's slot holds the row's current values
// with a zero list head, its tag names the row and its last use is the step that last used it; the host copy of a
// cached row is stale until it is evicted or flushed; set lists are empty.  The counter, the set count and the step
// change in-stream (a memset, or the begin kernel of a training pass with a cache), so a captured step replays
// correctly.  Host rows no occurrence touched are never read or written, except victims and flushed rows.  The
// kernels that do arithmetic see the same values in the same order at different addresses, so a step is
// bit-identical to the device step.
//
// The hot path is latency-bound random reads and writes of ~528-byte rows over the host link: a warp copies the
// rows its lanes claimed as one flat list of 16-byte vectors, 8 vectors per lane in flight, and a grid of several
// warps per SM keeps thousands of rows outstanding (the gather keeps 8 rows in flight per lane group the same way).
// A set's misses are walked by one warp, so a cache with far fewer sets than a step has misses serializes there.
#include "common.cuh"

namespace dlrm {

constexpr int HT_THREADS = 256;
constexpr int HT_UNROLL = 8;
constexpr int HT_WARPS = HT_THREADS / 32;

struct HostTableDev {
  float* w;         // host rows [rows][ld] (UVA)
  float* mom;       // host separate row-wise accumulators [rows] or null
  float* acc;       // host element-wise accumulators [rows][dim] or null
  const void* idx;
  const void* off;
  long long nnz, rows, pos_base;
  int* map;         // [rows] slot + 1, 0 = host only
};

struct HostStageParams {
  HostTableDev t[DLRM_B200_MAX_TABLES_PER_CALL];
  float* sw;        // arena [ncache + cap][ld]
  float* smom;      // arena [ncache + cap] or null
  int* shead;       // arena [ncache + cap] or null (separate list heads)
  float* sacc;      // arena [ncache + cap][dim] or null
  void* slot_idx;   // [cap] in the index dtype
  int* list;        // [cap] staged slots in claim order
  long long* key;   // [cap] row * 64 + table of the row position p staged
  int* count;
  long long cap, ld, batch;
  int dim, include_last, head_col;
  unsigned* err;
  // row cache (ncache == 0: none)
  long long ncache;
  long long* tag;   // [ncache] row * 64 + table, -1 = empty
  int* used;        // [ncache] last training step, 0 = empty
  int* step;
  int* set_head;    // [ncache / 32] position + 1
  int* set_next;    // [cap]
  int* sets;
  int* nsets;
  unsigned long long* stats;   // hits, inserts, evictions, staged
  int train;        // a cache and a training pass: stamp hits, thread misses
};

// set of a row key (row * 64 + table) in a cache of nsets sets
__device__ __forceinline__ int set_of(long long key, long long nsets) {
  return (int)(splitmix64((unsigned long long)key) % (unsigned long long)nsets);
}

// Copies n rows (row i: src + rs[i] * sstride -> dst + rd[i] * dstride, `words` floats each) as one flat list of
// float4 (VEC) or float work items over the warp, HT_UNROLL items per lane in flight.  zero_col >= 0: that word of
// every row is stored as zero (the list head).  src and dst may be the same arena when no row is both read and
// written.
template <bool VEC>
__device__ __forceinline__ void copy_rows(const float* src, long long sstride, float* dst, long long dstride,
                                          const long long* rs, const long long* rd, int n, int words, int zero_col,
                                          int lane) {
  constexpr int W = VEC ? 4 : 1;
  const int per_row = words / W;
  const int total = n * per_row;
  for (int base = 0; base < total; base += 32 * HT_UNROLL) {
    float4 v[HT_UNROLL];
#pragma unroll
    for (int u = 0; u < HT_UNROLL; ++u) {
      const int i = base + u * 32 + lane;
      if (i < total) {
        const int r = i / per_row, c = i - r * per_row;
        const float* p = src + rs[r] * sstride + c * W;
        if (VEC) v[u] = *reinterpret_cast<const float4*>(p);
        else v[u].x = *p;
      }
    }
#pragma unroll
    for (int u = 0; u < HT_UNROLL; ++u) {
      const int i = base + u * 32 + lane;
      if (i < total) {
        const int r = i / per_row, c = i - r * per_row;
        float* p = dst + rd[r] * dstride + c * W;
        if (VEC) {
          float4 x = v[u];
          if (zero_col >= 0 && zero_col / 4 == c) {
            const int q = zero_col & 3;
            if (q == 0) x.x = 0.f; else if (q == 1) x.y = 0.f; else if (q == 2) x.z = 0.f; else x.w = 0.f;
          }
          *reinterpret_cast<float4*>(p) = x;
        } else {
          *p = (c == zero_col) ? 0.f : v[u].x;
        }
      }
    }
  }
}

// n arena slots -> their host rows (slot[i] -> row[i] of call table tab[i]): weights with the list head as zero, the
// separate accumulator and the element-wise Adagrad row.  Rows of one warp may belong to different tables: copied
// run by run of equal table.
template <bool VEC>
__device__ __forceinline__ void rows_home(const HostStageParams& P, const long long* slot, const long long* row,
                                          const int* tab, int n, int lane) {
  if (P.smom)
    for (int i = lane; i < n; i += 32) P.t[tab[i]].mom[row[i]] = P.smom[slot[i]];
  for (int r0 = 0; r0 < n;) {
    const int t = tab[r0];
    int r1 = r0 + 1;
    while (r1 < n && tab[r1] == t) ++r1;
    copy_rows<VEC>(P.sw, P.ld, P.t[t].w, P.ld, slot + r0, row + r0, r1 - r0, (int)P.ld, P.head_col, lane);
    if (P.sacc)
      copy_rows<VEC>(P.sacc, P.dim, P.t[t].acc, P.dim, slot + r0, row + r0, r1 - r0, P.dim, -1, lane);
    r0 = r1;
  }
}

template <typename idx_t, bool VEC>
__global__ void __launch_bounds__(HT_THREADS) host_stage_in_kernel(const __grid_constant__ HostStageParams P) {
  __shared__ long long s_src[HT_WARPS][32];
  __shared__ long long s_dst[HT_WARPS][32];
  const HostTableDev& tb = P.t[blockIdx.y];
  const idx_t* idx = static_cast<const idx_t*>(tb.idx);
  const idx_t* off = static_cast<const idx_t*>(tb.off);
  idx_t* sidx = static_cast<idx_t*>(P.slot_idx);
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const long long N = P.ncache;
  const int step = P.train ? *P.step : 0;
  // the positions the gather reads: [off[0], end of the last bag)
  const long long start = P.batch > 0 ? (long long)off[0] : 0;
  const long long end = P.batch <= 0 ? 0 : (P.include_last ? (long long)off[P.batch] : tb.nnz);
  const long long warps = (long long)gridDim.x * HT_WARPS;
  for (long long c0 = start + ((long long)blockIdx.x * HT_WARPS + wib) * 32; c0 < end; c0 += warps * 32) {
    const long long p = c0 + lane;
    bool win = false, hit = false;
    long long row = 0, slot = -1;
    if (p < end) {
      row = (long long)idx[p];
      const long long g = tb.pos_base + p;
      if ((unsigned long long)row >= (unsigned long long)tb.rows || g >= P.cap) {
        if (P.err) atomicOr(P.err, 1u);
      } else {
        const int old = atomicCAS(tb.map + row, 0, (int)(N + g + 1));
        win = old == 0;
        slot = win ? N + g : (long long)(old - 1);
        // the first occurrence to stamp a resident row in this step counts its hit
        hit = P.train && !win && slot < N && atomicExch(P.used + slot, step) != step;
      }
      if (tb.pos_base + p < P.cap) sidx[tb.pos_base + p] = (idx_t)slot;
    }
    if (P.train) {
      const unsigned hits = __ballot_sync(0xffffffffu, hit);
      if (lane == 0 && hits) atomicAdd(P.stats, (unsigned long long)__popc(hits));
    }
    const unsigned wins = __ballot_sync(0xffffffffu, win);
    if (wins == 0u) continue;
    if (win) {
      const int rank = __popc(wins & ((1u << lane) - 1u));
      const long long g = slot - N;
      const long long key = row * 64 + blockIdx.y;
      s_src[wib][rank] = row;
      s_dst[wib][rank] = slot;
      P.list[atomicAdd(P.count, 1)] = (int)slot;
      P.key[g] = key;
      if (P.smom) P.smom[slot] = tb.mom[row];
      if (P.shead) P.shead[slot] = 0;
      if (P.train) {
        const int set = set_of(key, N / 32);
        const int prev = atomicExch(P.set_head + set, (int)(g + 1));
        P.set_next[g] = prev;
        if (prev == 0) P.sets[atomicAdd(P.nsets, 1)] = set;
      }
    }
    __syncwarp();
    const int n = __popc(wins);
    copy_rows<VEC>(tb.w, P.ld, P.sw, P.ld, s_src[wib], s_dst[wib], n, (int)P.ld, P.head_col, lane);
    if (P.sacc) copy_rows<VEC>(tb.acc, P.dim, P.sacc, P.dim, s_src[wib], s_dst[wib], n, P.dim, -1, lane);
    __syncwarp();
  }
}

// A training pass with a cache: reset the counters and advance the step, in-stream.
__global__ void host_cache_begin_kernel(int* count, int* nsets, int* step) {
  *count = 0;
  *nsets = 0;
  *step += 1;
}

// (table, row) order of a key row * 64 + table
__device__ __forceinline__ long long table_row(long long key) { return ((key & 63) << 32) | (key >> 6); }

// After the update of a training pass: one warp per set with misses inserts the set's misses into its ways (see the
// comment at the top).  Runs before host_write_back_kernel, which returns the misses left over.
template <bool VEC>
__global__ void __launch_bounds__(HT_THREADS, 2) host_cache_insert_kernel(const __grid_constant__ HostStageParams P) {
  __shared__ long long s_ord[HT_WARPS][32];
  __shared__ int s_pos[HT_WARPS][32];
  __shared__ long long s_slot[HT_WARPS][32];
  __shared__ long long s_row[HT_WARPS][32];
  __shared__ int s_tab[HT_WARPS][32];
  constexpr long long NONE = 0x7fffffffffffffffll;
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const long long N = P.ncache;
  const int nsets = *P.nsets, step = *P.step;
  const int warps = gridDim.x * HT_WARPS;
  for (int si = blockIdx.x * HT_WARPS + wib; si < nsets; si += warps) {
    const int set = P.sets[si];
    // 1. the (up to) 32 smallest misses of the set by (table, row), ascending over the lanes: the list is walked 32
    //    nodes at a time (every lane follows it, lane j keeps node j) and merged by rank into the best 32 so far.
    long long best = NONE;
    int bpos = -1;
    int node = P.set_head[set];
    while (node != 0) {
      int cpos = -1;
      for (int j = 0; j < 32 && node != 0; ++j) {
        if (lane == j) cpos = node - 1;
        node = P.set_next[node - 1];
      }
      const long long c = cpos >= 0 ? table_row(P.key[cpos]) : NONE;
      int rb = lane, rc = 0;
#pragma unroll 8
      for (int j = 0; j < 32; ++j) {
        const long long bj = __shfl_sync(0xffffffffu, best, j), cj = __shfl_sync(0xffffffffu, c, j);
        rb += cj < best;
        rc += (bj < c) + (cj < c);
      }
      s_ord[wib][lane] = NONE;
      s_pos[wib][lane] = -1;
      __syncwarp();
      // distinct ranks for every real key; only NONE entries may share one (and write the same values)
      if (rb < 32) { s_ord[wib][rb] = best; s_pos[wib][rb] = bpos; }
      if (rc < 32) { s_ord[wib][rc] = c; s_pos[wib][rc] = cpos; }
      __syncwarp();
      best = s_ord[wib][lane];
      bpos = s_pos[wib][lane];
      __syncwarp();
    }
    const int nmiss = __popc(__ballot_sync(0xffffffffu, bpos >= 0));
    // 2. the ways not used in this step, ordered by (last use, way); the i-th takes the i-th miss
    const long long way = (long long)set * 32 + lane;
    const long long tag = P.tag[way];
    const int used = P.used[way];
    const bool free_way = used != step;
    int r = 0;
    for (int j = 0; j < 32; ++j) {
      const int uj = __shfl_sync(0xffffffffu, used, j);
      r += uj != step && (uj < used || (uj == used && j < lane));
    }
    const int nins = min(nmiss, __popc(__ballot_sync(0xffffffffu, free_way)));
    const bool take = free_way && r < nins;
    const bool evict = take && tag >= 0;
    // 3. victims go home, then leave the map
    const unsigned ev = __ballot_sync(0xffffffffu, evict);
    if (evict) {
      const int e = __popc(ev & ((1u << lane) - 1u));
      s_slot[wib][e] = way;
      s_row[wib][e] = tag >> 6;
      s_tab[wib][e] = (int)(tag & 63);
    }
    __syncwarp();
    rows_home<VEC>(P, s_slot[wib], s_row[wib], s_tab[wib], __popc(ev), lane);
    __syncwarp();     // the victims' slots are read before the misses overwrite them
    if (evict) P.t[tag & 63].map[tag >> 6] = 0;
    // 4. the misses move into their ways: s_slot = staged slot, s_row = way
    const unsigned in = __ballot_sync(0xffffffffu, take);
    long long key = -1;
    int pos = -1;
    if (take) {
      const int e = __popc(in & ((1u << lane) - 1u));
      pos = s_pos[wib][r];
      key = P.key[pos];
      s_slot[wib][e] = N + pos;
      s_row[wib][e] = way;
    }
    __syncwarp();
    const int n = __popc(in);
    for (int i = lane; i < n; i += 32) {
      if (P.smom) P.smom[s_row[wib][i]] = P.smom[s_slot[wib][i]];
      if (P.shead) P.shead[s_row[wib][i]] = 0;
    }
    copy_rows<VEC>(P.sw, P.ld, P.sw, P.ld, s_slot[wib], s_row[wib], n, (int)P.ld, P.head_col, lane);
    if (P.sacc) copy_rows<VEC>(P.sacc, P.dim, P.sacc, P.dim, s_slot[wib], s_row[wib], n, P.dim, -1, lane);
    if (take) {
      P.t[key & 63].map[key >> 6] = (int)(way + 1);
      P.tag[way] = key;
      P.used[way] = step;
    }
    if (lane == 0) {
      P.set_head[set] = 0;
      if (n) atomicAdd(P.stats + 1, (unsigned long long)n);
      if (ev) atomicAdd(P.stats + 2, (unsigned long long)__popc(ev));
    }
    __syncwarp();
  }
}

// write == true: staged rows back to host + map reset; false: map reset only.  With a cache, a listed slot whose
// row's map entry no longer names it was inserted into the cache and is skipped.
template <bool VEC>
__global__ void __launch_bounds__(HT_THREADS, 2) host_write_back_kernel(const __grid_constant__ HostStageParams P,
                                                                     bool write) {
  __shared__ long long s_slot[HT_WARPS][32];
  __shared__ long long s_row[HT_WARPS][32];
  __shared__ int s_tab[HT_WARPS][32];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const long long n_all = *P.count;
  const long long warps = (long long)gridDim.x * HT_WARPS;
  for (long long c0 = ((long long)blockIdx.x * HT_WARPS + wib) * 32; c0 < n_all; c0 += warps * 32) {
    const long long i = c0 + lane;
    bool go = i < n_all;
    long long slot = 0, row = 0;
    int t = 0;
    if (go) {
      slot = P.list[i];
      const long long k = P.key[slot - P.ncache];
      t = (int)(k & 63);
      row = k >> 6;
      if (P.ncache) go = P.t[t].map[row] == (int)(slot + 1);
    }
    const unsigned gos = __ballot_sync(0xffffffffu, go);
    if (go) {
      const int e = __popc(gos & ((1u << lane) - 1u));
      s_slot[wib][e] = slot;
      s_row[wib][e] = row;
      s_tab[wib][e] = t;
    }
    __syncwarp();
    if (write) rows_home<VEC>(P, s_slot[wib], s_row[wib], s_tab[wib], __popc(gos), lane);
    if (write && P.ncache && lane == 0 && gos) atomicAdd(P.stats + 3, (unsigned long long)__popc(gos));
    // every host access of this warp is issued before the entries are released for the next step's claims
    __syncwarp();
    if (go) P.t[t].map[row] = 0;
    __syncwarp();
  }
}

// Every resident row home, then the cache emptied.
template <bool VEC>
__global__ void __launch_bounds__(HT_THREADS) host_cache_flush_kernel(const __grid_constant__ HostStageParams P) {
  __shared__ long long s_slot[HT_WARPS][32];
  __shared__ long long s_row[HT_WARPS][32];
  __shared__ int s_tab[HT_WARPS][32];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const long long warps = (long long)gridDim.x * HT_WARPS;
  for (long long c0 = ((long long)blockIdx.x * HT_WARPS + wib) * 32; c0 < P.ncache; c0 += warps * 32) {
    const long long slot = c0 + lane;       // ncache is a multiple of 32
    const long long tag = P.tag[slot];
    const bool go = tag >= 0;
    const unsigned gos = __ballot_sync(0xffffffffu, go);
    if (go) {
      const int e = __popc(gos & ((1u << lane) - 1u));
      s_slot[wib][e] = slot;
      s_row[wib][e] = tag >> 6;
      s_tab[wib][e] = (int)(tag & 63);
    }
    __syncwarp();
    rows_home<VEC>(P, s_slot[wib], s_row[wib], s_tab[wib], __popc(gos), lane);
    __syncwarp();
    if (go) {
      P.t[tag & 63].map[tag >> 6] = 0;
      P.tag[slot] = -1;
      P.used[slot] = 0;
    }
    __syncwarp();
  }
}

static int fill_params(HostStageParams& P, const char* who, const dlrm_host_table_t* tables, int num_tables,
                       const dlrm_host_stage_t* st, int dim, int64_t batch, int include_last, bool* vec) {
  if (num_tables < 1 || num_tables > DLRM_B200_MAX_TABLES_PER_CALL)
    return set_error("%s: num_tables=%d (1..%d)", who, num_tables, DLRM_B200_MAX_TABLES_PER_CALL);
  if (!tables || !st) return set_error("%s: NULL descriptor", who);
  if (dim <= 0) return set_error("%s: dim=%d", who, dim);
  const long long ld = st->ld > 0 ? st->ld : dim;
  if (ld < dim) return set_error("%s: ld=%lld < dim=%d", who, (long long)ld, dim);
  if (st->head_col >= ld || (st->head_col >= 0 && st->head_col < dim))
    return set_error("%s: head_col=%lld must lie in the row's words past dim (or be -1)", who, (long long)st->head_col);
  if (st->capacity <= 0 || st->capacity > 0x7ffffffeLL)
    return set_error("%s: capacity=%lld (1..2^31-2)", who, (long long)st->capacity);
  if (!st->weight || !st->slot_idx || !st->list || !st->key || !st->count)
    return set_error("%s: NULL staging pointer", who);
  const long long N = st->cache_rows;
  if (N < 0 || N % 32) return set_error("%s: cache_rows=%lld (a multiple of 32, 0 = no cache)", who, (long long)N);
  if (N > 0x7ffffffeLL - st->capacity)
    return set_error("%s: cache_rows + capacity = %lld does not fit the int32 slot map (<= 2^31-2)", who,
                     (long long)(N + st->capacity));
  if (N && (!st->cache_tag || !st->cache_used || !st->step || !st->set_head || !st->set_next || !st->sets ||
            !st->num_sets || !st->stats))
    return set_error("%s: NULL cache pointer", who);
  P = HostStageParams{};
  P.sw = st->weight; P.smom = st->momentum; P.shead = st->head; P.sacc = st->acc_ew;
  P.slot_idx = st->slot_idx; P.list = st->list; P.key = reinterpret_cast<long long*>(st->key); P.count = st->count;
  P.cap = st->capacity; P.ld = ld; P.batch = batch; P.dim = dim; P.include_last = include_last;
  P.head_col = (int)st->head_col;
  P.err = err_word_device();
  P.ncache = N;
  P.tag = reinterpret_cast<long long*>(st->cache_tag); P.used = st->cache_used; P.step = st->step;
  P.set_head = st->set_head; P.set_next = st->set_next; P.sets = st->sets; P.nsets = st->num_sets;
  P.stats = reinterpret_cast<unsigned long long*>(st->stats);
  P.train = N > 0 && !st->forward_only;
  bool v = ld % 4 == 0 && dim % 4 == 0 && aligned16(st->weight) && (!st->acc_ew || aligned16(st->acc_ew));
  for (int k = 0; k < num_tables; ++k) {
    const dlrm_host_table_t& s = tables[k];
    if (!s.weight || !s.map || !s.offsets || (!s.indices && s.nnz > 0))
      return set_error("%s: table %d has a NULL pointer", who, k);
    if (s.rows <= 0 || s.rows > 0x7ffffffeLL) return set_error("%s: table %d: rows=%lld", who, k, (long long)s.rows);
    if ((st->momentum != nullptr) != (s.momentum != nullptr))
      return set_error("%s: table %d: a separate accumulator must be given for the staging and every table", who, k);
    if ((st->acc_ew != nullptr) != (s.acc_ew != nullptr))
      return set_error("%s: table %d: element-wise accumulators must be given for the staging and every table", who, k);
    if (s.pos_base < 0 || s.nnz < 0) return set_error("%s: table %d: negative pos_base / nnz", who, k);
    P.t[k].w = s.weight; P.t[k].mom = s.momentum; P.t[k].acc = s.acc_ew; P.t[k].idx = s.indices;
    P.t[k].off = s.offsets; P.t[k].nnz = s.nnz; P.t[k].rows = s.rows; P.t[k].pos_base = s.pos_base;
    P.t[k].map = s.map;
    v = v && aligned16(s.weight) && (!s.acc_ew || aligned16(s.acc_ew));
  }
  *vec = v;
  return 0;
}

static unsigned grid_for(long long work) {
  const long long b = (work + HT_THREADS - 1) / HT_THREADS;
  return (unsigned)max(1ll, min(b, 2048ll));
}

}  // namespace dlrm

extern "C" int dlrm_b200_host_stage_in(const dlrm_host_table_t* tables, int num_tables, const dlrm_host_stage_t* st,
                                       int dim, int64_t batch, int idx_bytes, int include_last, void* stream) {
  using namespace dlrm;
  HostStageParams P;
  bool vec = false;
  if (int rc = fill_params(P, "host_stage_in", tables, num_tables, st, dim, batch, include_last, &vec)) return rc;
  if (idx_bytes != 4 && idx_bytes != 8) return set_error("host_stage_in: idx_bytes=%d (4 or 8)", idx_bytes);
  if (!P.err) return set_error("host_stage_in: no device error word");
  long long bound = 0;   // positions of one table: at most its nnz (reference format) or the capacity (packed)
  for (int k = 0; k < num_tables; ++k) bound = max(bound, include_last ? P.cap : (long long)tables[k].nnz);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (P.train) {
    host_cache_begin_kernel<<<1, 1, 0, s>>>(P.count, P.nsets, P.step);
    DLRM_CHECK_LAUNCH("host_cache_begin_kernel");
  } else {
    DLRM_CUDA(cudaMemsetAsync(P.count, 0, sizeof(int), s));
  }
  const dim3 grid(grid_for(bound), num_tables);
  if (idx_bytes == 8) {
    if (vec) host_stage_in_kernel<long long, true><<<grid, HT_THREADS, 0, s>>>(P);
    else host_stage_in_kernel<long long, false><<<grid, HT_THREADS, 0, s>>>(P);
  } else {
    if (vec) host_stage_in_kernel<int, true><<<grid, HT_THREADS, 0, s>>>(P);
    else host_stage_in_kernel<int, false><<<grid, HT_THREADS, 0, s>>>(P);
  }
  DLRM_CHECK_LAUNCH("host_stage_in_kernel");
  return 0;
}

static int host_finish(const char* who, const dlrm_host_table_t* tables, int num_tables, const dlrm_host_stage_t* st,
                       int dim, bool write, void* stream) {
  using namespace dlrm;
  HostStageParams P;
  bool vec = false;
  if (int rc = fill_params(P, who, tables, num_tables, st, dim, 0, 0, &vec)) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (write && P.train) {
    const unsigned g = grid_for(min(P.ncache / 32, P.cap) * 32);
    if (vec) host_cache_insert_kernel<true><<<g, HT_THREADS, 0, s>>>(P);
    else host_cache_insert_kernel<false><<<g, HT_THREADS, 0, s>>>(P);
    DLRM_CHECK_LAUNCH("host_cache_insert_kernel");
  }
  if (vec) host_write_back_kernel<true><<<grid_for(P.cap), HT_THREADS, 0, s>>>(P, write);
  else host_write_back_kernel<false><<<grid_for(P.cap), HT_THREADS, 0, s>>>(P, write);
  DLRM_CHECK_LAUNCH("host_write_back_kernel");
  return 0;
}

extern "C" int dlrm_b200_host_write_back(const dlrm_host_table_t* tables, int num_tables, const dlrm_host_stage_t* st,
                                         int dim, void* stream) {
  return host_finish("host_write_back", tables, num_tables, st, dim, true, stream);
}

extern "C" int dlrm_b200_host_release(const dlrm_host_table_t* tables, int num_tables, const dlrm_host_stage_t* st,
                                      int dim, void* stream) {
  return host_finish("host_release", tables, num_tables, st, dim, false, stream);
}

extern "C" int dlrm_b200_host_cache_flush(const dlrm_host_table_t* tables, int num_tables,
                                          const dlrm_host_stage_t* st, int dim, void* stream) {
  using namespace dlrm;
  HostStageParams P;
  bool vec = false;
  if (int rc = fill_params(P, "host_cache_flush", tables, num_tables, st, dim, 0, 0, &vec)) return rc;
  if (P.ncache == 0) return set_error("host_cache_flush: no cache (cache_rows = 0)");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (vec) host_cache_flush_kernel<true><<<grid_for(P.ncache), HT_THREADS, 0, s>>>(P);
  else host_cache_flush_kernel<false><<<grid_for(P.ncache), HT_THREADS, 0, s>>>(P);
  DLRM_CHECK_LAUNCH("host_cache_flush_kernel");
  return 0;
}

extern "C" int dlrm_b200_host_register(void* ptr, int64_t bytes) {
  using namespace dlrm;
  if (!ptr || bytes <= 0) return set_error("host_register: NULL pointer or %lld bytes", (long long)bytes);
  DLRM_CUDA(cudaHostRegister(ptr, (size_t)bytes, cudaHostRegisterMapped | cudaHostRegisterPortable));
  void* dev = nullptr;
  cudaError_t e = cudaHostGetDevicePointer(&dev, ptr, 0);
  if (e != cudaSuccess || dev != ptr) {
    cudaHostUnregister(ptr);
    return set_error("host_register: the device address of %p is %p (%s): host tables need unified addressing",
                     ptr, dev, cudaGetErrorString(e));
  }
  return 0;
}

extern "C" int dlrm_b200_host_unregister(void* ptr) {
  using namespace dlrm;
  if (!ptr) return set_error("host_unregister: NULL pointer");
  DLRM_CUDA(cudaHostUnregister(ptr));
  return 0;
}
