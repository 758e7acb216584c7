// Embedding tables in pinned host memory ("host tables"): the rows a batch touches are staged through an HBM
// arena, so the gather and the fused update run unchanged on device addresses.
//
//   stage_in   before the gather, one pass over the batch's occurrences of the host tables.  For occurrence p of
//              host table t (p = its global position: packed batches share one index array; reference-format
//              batches number the tables' positions back to back, pos_base = pair_base):
//                row outside [0, rows)  -> device error bit 0 (as the gather), slot index -1, no host access;
//                else atomicCAS(map[row], 0, p + 1): the first occurrence to claim the row makes p the row's SLOT
//                     (slot ids are positions, so they are distinct and < capacity without a sort), appends
//                     (slot) to the list through the one counter, and copies the row -- weights and its in-row
//                     accumulator / separate accumulator / element-wise Adagrad row -- from host memory into
//                     staging slot p with zero-copy reads through the UVA pointer; the staged list head is zero;
//                every occurrence writes its slot into slot_idx[p], parallel to the batch's index array.
//   write_back after the update, on the same stream: every listed slot's row and words go back to their host row
//              (list head written as zero) and its map entry is reset.  release: the map reset alone (forward only).
//
// Invariants: the map is all zero between steps (stage_in claims, write_back / release clears exactly the entries
// it claimed); the counter is reset in-stream by a memset inside dlrm_b200_host_stage_in, so a captured step
// replays correctly; host rows no occurrence touched are never read or written.  The kernels that do arithmetic
// see the same values in the same order at different addresses, so a step is bit-identical to the device step.
//
// The hot path is latency-bound random reads and writes of ~528-byte rows over the host link: a warp copies the
// rows its lanes claimed as one flat list of 16-byte vectors, 8 vectors per lane in flight, and a grid of several
// warps per SM keeps thousands of rows outstanding (the gather keeps 8 rows in flight per lane group the same way).
#include "common.cuh"

namespace dlrm {

constexpr int HT_THREADS = 256;
constexpr int HT_UNROLL = 8;

struct HostTableDev {
  float* w;         // host rows [rows][ld] (UVA)
  float* mom;       // host separate row-wise accumulators [rows] or null
  float* acc;       // host element-wise accumulators [rows][dim] or null
  const void* idx;
  const void* off;
  long long nnz, rows, pos_base;
  int* map;         // [rows] slot + 1, 0 = not staged
};

struct HostStageParams {
  HostTableDev t[DLRM_B200_MAX_TABLES_PER_CALL];
  float* sw;        // staging [cap][ld]
  float* smom;      // staging [cap] or null
  int* shead;       // staging [cap] or null (separate list heads)
  float* sacc;      // staging [cap][dim] or null
  void* slot_idx;   // [cap] in the index dtype
  int* list;        // [cap] staged slots in claim order
  long long* key;   // [cap] row * 64 + table of a staged slot
  int* count;
  long long cap, ld, batch;
  int dim, include_last, head_col;
  unsigned* err;
};

// Copies n rows (row i: src + rs[i] * sstride -> dst + rd[i] * dstride, `words` floats each) as one flat list of
// float4 (VEC) or float work items over the warp, HT_UNROLL items per lane in flight.  zero_col >= 0: that word of
// every row is stored as zero (the list head).
template <bool VEC>
__device__ __forceinline__ void copy_rows(const float* __restrict__ src, long long sstride, float* __restrict__ dst,
                                          long long dstride, const long long* rs, const long long* rd, int n,
                                          int words, int zero_col, int lane) {
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

template <typename idx_t, bool VEC>
__global__ void __launch_bounds__(HT_THREADS) host_stage_in_kernel(const __grid_constant__ HostStageParams P) {
  __shared__ long long s_src[HT_THREADS / 32][32];
  __shared__ long long s_dst[HT_THREADS / 32][32];
  const HostTableDev& tb = P.t[blockIdx.y];
  const idx_t* idx = static_cast<const idx_t*>(tb.idx);
  const idx_t* off = static_cast<const idx_t*>(tb.off);
  idx_t* sidx = static_cast<idx_t*>(P.slot_idx);
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  // the positions the gather reads: [off[0], end of the last bag)
  const long long start = P.batch > 0 ? (long long)off[0] : 0;
  const long long end = P.batch <= 0 ? 0 : (P.include_last ? (long long)off[P.batch] : tb.nnz);
  const long long warps = (long long)gridDim.x * (HT_THREADS / 32);
  for (long long c0 = start + ((long long)blockIdx.x * (HT_THREADS / 32) + wib) * 32; c0 < end; c0 += warps * 32) {
    const long long p = c0 + lane;
    bool win = false;
    long long row = 0, slot = -1;
    if (p < end) {
      row = (long long)idx[p];
      const long long g = tb.pos_base + p;
      if ((unsigned long long)row >= (unsigned long long)tb.rows || g >= P.cap) {
        if (P.err) atomicOr(P.err, 1u);
      } else {
        const int old = atomicCAS(tb.map + row, 0, (int)(g + 1));
        win = old == 0;
        slot = win ? g : (long long)(old - 1);
      }
      if (tb.pos_base + p < P.cap) sidx[tb.pos_base + p] = (idx_t)slot;
    }
    const unsigned wins = __ballot_sync(0xffffffffu, win);
    if (wins == 0u) continue;
    if (win) {
      const int rank = __popc(wins & ((1u << lane) - 1u));
      s_src[wib][rank] = row;
      s_dst[wib][rank] = slot;
      P.list[atomicAdd(P.count, 1)] = (int)slot;
      P.key[slot] = row * 64 + blockIdx.y;
      if (P.smom) P.smom[slot] = tb.mom[row];
      if (P.shead) P.shead[slot] = 0;
    }
    __syncwarp();
    const int n = __popc(wins);
    copy_rows<VEC>(tb.w, P.ld, P.sw, P.ld, s_src[wib], s_dst[wib], n, (int)P.ld, P.head_col, lane);
    if (P.sacc) copy_rows<VEC>(tb.acc, P.dim, P.sacc, P.dim, s_src[wib], s_dst[wib], n, P.dim, -1, lane);
    __syncwarp();
  }
}

// write == true: staged rows back to host + map reset; false: map reset only.
template <bool VEC>
__global__ void __launch_bounds__(HT_THREADS) host_write_back_kernel(const __grid_constant__ HostStageParams P,
                                                                     bool write) {
  __shared__ long long s_slot[HT_THREADS / 32][32];
  __shared__ long long s_row[HT_THREADS / 32][32];
  __shared__ int s_tab[HT_THREADS / 32][32];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const long long n_all = *P.count;
  const long long warps = (long long)gridDim.x * (HT_THREADS / 32);
  for (long long c0 = ((long long)blockIdx.x * (HT_THREADS / 32) + wib) * 32; c0 < n_all; c0 += warps * 32) {
    const long long i = c0 + lane;
    const bool have = i < n_all;
    if (have) {
      const long long slot = P.list[i];
      const long long k = P.key[slot];
      const int t = (int)(k & 63);
      const long long row = k >> 6;
      s_slot[wib][lane] = slot;
      s_row[wib][lane] = row;
      s_tab[wib][lane] = t;
      if (write && P.smom) P.t[t].mom[row] = P.smom[slot];
    }
    __syncwarp();
    const int n = (int)min(32ll, n_all - c0);
    if (write) {
      // rows of one warp may belong to different tables: copy run by run of equal table
      for (int r0 = 0; r0 < n;) {
        const int t = s_tab[wib][r0];
        int r1 = r0 + 1;
        while (r1 < n && s_tab[wib][r1] == t) ++r1;
        copy_rows<VEC>(P.sw, P.ld, P.t[t].w, P.ld, s_slot[wib] + r0, s_row[wib] + r0, r1 - r0, (int)P.ld,
                       P.head_col, lane);
        if (P.sacc)
          copy_rows<VEC>(P.sacc, P.dim, P.t[t].acc, P.dim, s_slot[wib] + r0, s_row[wib] + r0, r1 - r0, P.dim, -1,
                         lane);
        r0 = r1;
      }
    }
    // every host access of this warp is issued before the entries are released for the next step's claims
    __syncwarp();
    if (have) P.t[s_tab[wib][lane]].map[s_row[wib][lane]] = 0;
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
  P = HostStageParams{};
  P.sw = st->weight; P.smom = st->momentum; P.shead = st->head; P.sacc = st->acc_ew;
  P.slot_idx = st->slot_idx; P.list = st->list; P.key = reinterpret_cast<long long*>(st->key); P.count = st->count;
  P.cap = st->capacity; P.ld = ld; P.batch = batch; P.dim = dim; P.include_last = include_last;
  P.head_col = (int)st->head_col;
  P.err = err_word_device();
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
  DLRM_CUDA(cudaMemsetAsync(P.count, 0, sizeof(int), s));
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
