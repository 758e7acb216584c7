// Decode of MLPerf binary records (data_loader_terabyte.py:74-93 _transform_features, :229-240 __getitem__)
// into the packed device batch of dlrm_b200/data.py, so that only the raw int32 records cross the bus.
#include "common.cuh"

namespace dlrm {

// One thread per record word, then one per offset: record word w of sample b goes to
//   w == 0            target[b]
//   1 <= w <= nd      X[b, w-1] = log((float)x + 1)
//   w > nd            indices[(w-1-nd) * n + b]  (table-major)
// and offsets[k, b] = k*n + b for b in 0..n.
__global__ void __launch_bounds__(256) decode_records_kernel(const int32_t* __restrict__ rec, long long n, int nd,
                                                             int ns, long long max_ind_range,
                                                             float* __restrict__ X, float* __restrict__ target,
                                                             long long* __restrict__ offsets,
                                                             long long* __restrict__ indices) {
  const long long words = (long long)(1 + nd + ns);
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < n * words) {
    const long long b = e / words;
    const int w = (int)(e - b * words);
    const int32_t v = rec[e];
    if (w == 0) {
      target[b] = (float)v;
    } else if (w <= nd) {
      // fp32 conversion first, then the add in fp32: torch.log(x.to(torch.float) + 1)
      X[b * nd + (w - 1)] = logf(__fadd_rn(__int2float_rn(v), 1.0f));
    } else {
      long long id = v;
      if (max_ind_range > 0) {  // floor modulo (Python / torch `%`): never negative
        id %= max_ind_range;
        if (id < 0) id += max_ind_range;
      }
      indices[(long long)(w - 1 - nd) * n + b] = id;
    }
    return;
  }
  const long long o = e - n * words;
  if (o < (long long)ns * (n + 1)) {
    const long long k = o / (n + 1);
    offsets[o] = o - k;  // k*(n+1) + b  ->  k*n + b
  }
}

// Batch assembly from a split resident in device memory (dlrm_data_pytorch.py:293-296 __getitem__ + :324-337
// collate_wrapper_criteo_offset): sample b of the batch is row ids[b] of X_int [N, nd], X_cat [N, ns], y [N].
// One block per tile of GATHER_TILE samples.  The ids of a shuffled split point at random rows, so each row is
// read as a run of consecutive words (coalesced) into a shared-memory tile, which is then written out the way
// decode_records_kernel writes it: X and target row-major, ids table-major (coalesced along the batch).
constexpr int GATHER_TILE = 64;
constexpr int GATHER_THREADS = 256;

__device__ __forceinline__ long long fold_id(long long id, long long max_ind_range) {
  if (max_ind_range > 0) {  // floor modulo (Python / torch `%`): never negative
    id %= max_ind_range;
    if (id < 0) id += max_ind_range;
  }
  return id;
}

__global__ void __launch_bounds__(GATHER_THREADS) gather_records_kernel(
    const int32_t* __restrict__ X_int, const int32_t* __restrict__ X_cat, const int32_t* __restrict__ y,
    const long long* __restrict__ ids, long long n, int nd, int ns, long long max_ind_range,
    float* __restrict__ X, float* __restrict__ target, long long* __restrict__ offsets,
    long long* __restrict__ indices) {
  extern __shared__ int32_t tile[];  // [GATHER_TILE][pitch]: nd dense words, ns ids, the label
  const int words = nd + ns + 1;
  const int pitch = words | 1;       // odd pitch: the column reads of the write phase are conflict-free
  const long long b0 = (long long)blockIdx.x * GATHER_TILE;
  const int m = (int)min((long long)GATHER_TILE, n - b0);
  for (int t = threadIdx.x; t < m * words; t += GATHER_THREADS) {
    const int s = t / words, w = t - s * words;
    const long long r = ids[b0 + s];
    tile[s * pitch + w] = w < nd ? X_int[r * nd + w] : w < nd + ns ? X_cat[r * ns + (w - nd)] : y[r];
  }
  __syncthreads();
  for (int t = threadIdx.x; t < m * nd; t += GATHER_THREADS) {
    const int s = t / nd, d = t - s * nd;
    // fp32 conversion first, then the add in fp32: torch.log(torch.tensor(x, dtype=torch.float) + 1)
    X[(b0 + s) * nd + d] = logf(__fadd_rn(__int2float_rn(tile[s * pitch + d]), 1.0f));
  }
  for (int t = threadIdx.x; t < ns * GATHER_TILE; t += GATHER_THREADS) {
    const int k = t / GATHER_TILE, s = t - k * GATHER_TILE;
    if (s < m) indices[(long long)k * n + b0 + s] = fold_id(tile[s * pitch + nd + k], max_ind_range);
  }
  if (threadIdx.x < m) target[b0 + threadIdx.x] = (float)tile[threadIdx.x * pitch + nd + ns];
  for (long long o = (long long)blockIdx.x * GATHER_THREADS + threadIdx.x; o < (long long)ns * (n + 1);
       o += (long long)gridDim.x * GATHER_THREADS)
    offsets[o] = o - o / (n + 1);  // k*(n+1) + b  ->  k*n + b
}


// Per-day Criteo chunks (the reference's `*_{d}_reordered.npz`, dlrm_data_pytorch.py:270-289) into a device ring of
// int32 rows: one thread per element of the chunk, members in order X_int [n, nd], X_cat [n, ns], y [n], each in
// the dtype its file stores.  Row r goes to ring row (dst + r) mod capacity.  A value that is not an exact integer
// in int32 range, a negative id or a label outside {0, 1} is not written; the smallest `r * 4 + member` of such
// values is kept in *bad (atomicMin), so the host learns the first bad row and which member holds it.
enum : int { INGEST_F64 = 0, INGEST_I64 = 1, INGEST_I32 = 2 };

__device__ __forceinline__ bool ingest_load(const void* p, int dtype, long long i, int32_t* out) {
  if (dtype == INGEST_I32) {
    *out = static_cast<const int32_t*>(p)[i];
    return true;
  }
  if (dtype == INGEST_I64) {
    const long long v = static_cast<const long long*>(p)[i];
    *out = (int32_t)v;
    return v >= INT32_MIN && v <= INT32_MAX;
  }
  const double v = static_cast<const double*>(p)[i];
  // NaN fails both comparisons; inside the range the cast is exact iff v has no fraction
  if (!(v >= -2147483648.0 && v <= 2147483647.0)) return false;
  *out = (int32_t)v;
  return (double)*out == v;
}

__global__ void __launch_bounds__(256) ingest_records_kernel(
    const void* __restrict__ x_int, int int_dtype, const void* __restrict__ x_cat, int cat_dtype,
    const void* __restrict__ y, int y_dtype, long long n, int nd, int ns, int32_t* __restrict__ ring_int,
    int32_t* __restrict__ ring_cat, int32_t* __restrict__ ring_y, long long capacity, long long dst,
    unsigned long long* __restrict__ bad) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long n_int = n * nd, n_cat = n * ns;
  int member, w;
  long long r, i;
  const void* src;
  int dtype;
  if (e < n_int) {
    member = 0, src = x_int, dtype = int_dtype, i = e, r = e / nd, w = (int)(e - r * nd);
  } else if (e < n_int + n_cat) {
    member = 1, src = x_cat, dtype = cat_dtype, i = e - n_int, r = i / ns, w = (int)(i - r * ns);
  } else if (e < n_int + n_cat + n) {
    member = 2, src = y, dtype = y_dtype, i = e - n_int - n_cat, r = i, w = 0;
  } else {
    return;
  }
  int32_t v;
  bool ok = ingest_load(src, dtype, i, &v);
  if (member == 1) ok = ok && v >= 0;
  if (member == 2) ok = ok && (v == 0 || v == 1);
  if (!ok) {
    atomicMin(bad, (unsigned long long)(r * 4 + member));
    return;
  }
  long long row = dst + r;
  if (row >= capacity) row -= capacity;
  if (member == 0)
    ring_int[row * nd + w] = v;
  else if (member == 1)
    ring_cat[row * ns + w] = v;
  else
    ring_y[row] = v;
}

}  // namespace dlrm

extern "C" int dlrm_b200_gather_records(const int32_t* X_int, const int32_t* X_cat, const int32_t* y,
                                        const int64_t* ids, int64_t n, int num_dense, int num_sparse,
                                        int64_t max_ind_range, float* X, float* target, int64_t* offsets,
                                        int64_t* indices, void* stream) {
  using namespace dlrm;
  if (n <= 0) return set_error("gather_records: n=%lld samples (must be > 0)", (long long)n);
  if (num_dense <= 0 || num_sparse <= 0 || num_dense + num_sparse + 1 > 128)
    return set_error("gather_records: num_dense=%d, num_sparse=%d (both > 0, at most 127 words per sample)",
                     num_dense, num_sparse);
  if (!X_int || !X_cat || !y || !ids || !X || !target || !offsets || !indices)
    return set_error("gather_records: NULL pointer");
  const long long blocks = (n + GATHER_TILE - 1) / GATHER_TILE;
  if (blocks >= (1ll << 31)) return set_error("gather_records: %lld samples is too many for one call", (long long)n);
  const size_t smem = sizeof(int32_t) * GATHER_TILE * ((num_dense + num_sparse + 1) | 1);
  gather_records_kernel<<<(unsigned)blocks, GATHER_THREADS, smem, static_cast<cudaStream_t>(stream)>>>(
      X_int, X_cat, y, reinterpret_cast<const long long*>(ids), (long long)n, num_dense, num_sparse,
      (long long)max_ind_range, X, target, reinterpret_cast<long long*>(offsets),
      reinterpret_cast<long long*>(indices));
  DLRM_CHECK_LAUNCH("gather_records_kernel");
  return 0;
}

extern "C" int dlrm_b200_decode_records(const int32_t* records, int64_t n, int num_dense, int num_sparse,
                                        int64_t max_ind_range, float* X, float* target, int64_t* offsets,
                                        int64_t* indices, void* stream) {
  using namespace dlrm;
  if (n <= 0) return set_error("decode_records: n=%lld records (must be > 0)", (long long)n);
  if (num_dense <= 0 || num_sparse <= 0)
    return set_error("decode_records: num_dense=%d, num_sparse=%d (both must be > 0)", num_dense, num_sparse);
  if (!records || !X || !target || !offsets || !indices) return set_error("decode_records: NULL pointer");
  const long long total = n * (1ll + num_dense + num_sparse) + (long long)num_sparse * (n + 1);
  const long long blocks = (total + 255) / 256;
  if (blocks >= (1ll << 31)) return set_error("decode_records: %lld records is too many for one call", (long long)n);
  decode_records_kernel<<<(unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      records, (long long)n, num_dense, num_sparse, (long long)max_ind_range, X, target,
      reinterpret_cast<long long*>(offsets), reinterpret_cast<long long*>(indices));
  DLRM_CHECK_LAUNCH("decode_records_kernel");
  return 0;
}

extern "C" int dlrm_b200_ingest_records(const void* x_int, int x_int_dtype, const void* x_cat, int x_cat_dtype,
                                        const void* y, int y_dtype, int64_t n, int num_dense, int num_sparse,
                                        int32_t* ring_int, int32_t* ring_cat, int32_t* ring_y, int64_t capacity,
                                        int64_t dst, uint64_t* bad, void* stream) {
  using namespace dlrm;
  if (n <= 0 || n > capacity)
    return set_error("ingest_records: n=%lld rows for a ring of %lld (must be in 1..capacity)", (long long)n,
                     (long long)capacity);
  if (dst < 0 || dst >= capacity)
    return set_error("ingest_records: dst=%lld outside the ring [0, %lld)", (long long)dst, (long long)capacity);
  if (num_dense <= 0 || num_sparse <= 0)
    return set_error("ingest_records: num_dense=%d, num_sparse=%d (both must be > 0)", num_dense, num_sparse);
  for (int d : {x_int_dtype, x_cat_dtype, y_dtype})
    if (d != INGEST_F64 && d != INGEST_I64 && d != INGEST_I32)
      return set_error("ingest_records: dtype code %d (0 float64, 1 int64, 2 int32)", d);
  if (!x_int || !x_cat || !y || !ring_int || !ring_cat || !ring_y || !bad)
    return set_error("ingest_records: NULL pointer");
  const long long total = n * (1ll + num_dense + num_sparse);
  const long long blocks = (total + 255) / 256;
  if (blocks >= (1ll << 31)) return set_error("ingest_records: %lld rows is too many for one call", (long long)n);
  ingest_records_kernel<<<(unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x_int, x_int_dtype, x_cat, x_cat_dtype, y, y_dtype, (long long)n, num_dense, num_sparse, ring_int, ring_cat,
      ring_y, (long long)capacity, (long long)dst, reinterpret_cast<unsigned long long*>(bad));
  DLRM_CHECK_LAUNCH("ingest_records_kernel");
  return 0;
}
