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

}  // namespace dlrm

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
