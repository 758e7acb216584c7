// Glue kernels of the sharded (table-wise + row-split) embedding placement (dlrm_b200/placement.py):
//
//   reduce_partials : T[b, 1+t, :] = sum over the shards p of a row-split table t of partial[p][b][:]
//                     (fixed shard order -> deterministic).  Replaces, for those tables, the pooled vector
//                     the reference's single EmbeddingBag call returns (dlrm_s_pytorch.py:452-457).
//   block_copy      : up to 64 contiguous blocks copied in one launch (16-byte vector accesses); with
//                     peer-mapped destinations this is the index exchange of a sharded step: every rank
//                     uploads the indices of ITS samples and pushes each table's block to the rank(s)
//                     storing that table (the reference broadcasts the whole batch to every rank,
//                     dlrm_s_pytorch.py:528-544).
//   gen_multihot    : device-side synthetic batches of the MLPerf multi-hot distribution
//                     (torchrec_dlrm/multi_hot.py:80-127), bit-identical to dlrm_b200/mlperf.py.
#include "common.cuh"

namespace dlrm {

struct ReduceSlots {
  int feature[16];     // destination feature of slot s
  int first[17];       // slabs [first[s], first[s+1]) of the partial area belong to slot s
  int n;
};

__global__ void __launch_bounds__(256) reduce_partials_kernel(const float* __restrict__ part, float* __restrict__ T,
                                                              long long ldt, long long B, int D,
                                                              const __grid_constant__ ReduceSlots S) {
  pdl_launch_dependents();
  pdl_wait();
  const int s = blockIdx.y;
  const int d4 = D >> 2;
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= B * d4) return;
  const long long b = e / d4;
  const int c = (int)(e - b * d4) * 4;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int p = S.first[s]; p < S.first[s + 1]; ++p) {
    const float4 v = *reinterpret_cast<const float4*>(part + ((long long)p * B + b) * D + c);
    acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
  }
  *reinterpret_cast<float4*>(T + b * ldt + (long long)S.feature[s] * D + c) = acc;
}

struct CopyList {
  const uint4* src[64];
  uint4* dst[64];
  long long n16[64];
  int n;
};

__global__ void __launch_bounds__(256) block_copy_kernel(const __grid_constant__ CopyList L) {
  const int k = blockIdx.y;
  const uint4* __restrict__ s = L.src[k];
  uint4* __restrict__ d = L.dst[k];
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < L.n16[k]; i += (long long)gridDim.x * blockDim.x)
    d[i] = s[i];
}

// ---- counter-based generator (mirror of dlrm_b200/mlperf.py: keep the two in sync, tests compare them bit for bit;
// splitmix64 is in common.cuh)
constexpr unsigned long long K_TABLE = 0x9E3779B97F4A7C15ull, K_ROW = 0xC2B2AE3D27D4EB4Full,
                             K_SLOT = 0x165667B19E3779F9ull, K_STEP = 0xD6E8FEB86659FD93ull;

struct GenTable {
  void* out;            // [batch, L] indices
  long long rows;
  int L, table;
};
struct GenParams {
  GenTable t[64];
  int n, idx_bytes;
  unsigned long long seed, step, sample0;
  long long batch;
  float* X;             // [batch, m_den] or null
  float* target;        // [batch] or null
  int m_den;
};

__global__ void __launch_bounds__(256) gen_multihot_kernel(const __grid_constant__ GenParams P) {
  if ((int)blockIdx.y == P.n) {       // dense features + targets
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int cols = P.m_den + 1;
    if (!P.X || e >= P.batch * cols) return;
    const long long b = e / cols;
    const int c = (int)(e - b * cols);
    const unsigned long long base = (P.seed * K_STEP) ^ ((P.step + 1) * K_TABLE) ^ 0x5DEECE66Dull;
    const unsigned long long h = splitmix64(splitmix64(base ^ ((P.sample0 + b) * K_ROW) ^ ((unsigned long long)c * K_SLOT)));
    const float u = (float)(h >> 40) * (1.0f / 16777216.0f);
    if (c < P.m_den) P.X[b * P.m_den + c] = u;
    else if (P.target) P.target[b] = rintf(u);
    return;
  }
  const GenTable& tb = P.t[blockIdx.y];
  const long long n = P.batch * tb.L;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const long long b = e / tb.L;
    const int j = (int)(e - b * tb.L);
    const unsigned long long base = (P.seed * K_STEP) ^ ((P.step + 1) * K_TABLE) ^ ((unsigned long long)(tb.table + 1) * K_SLOT);
    const unsigned long long id = __umul64hi(splitmix64(splitmix64(base ^ ((P.sample0 + b) * K_ROW))), (unsigned long long)tb.rows);
    unsigned long long v = id;
    if (j > 0) {
      const unsigned long long base2 = ((unsigned long long)(tb.table + 1) * K_TABLE) ^ 0xA5A5A5A5A5A5A5A5ull;
      v = __umul64hi(splitmix64(base2 ^ (id * K_ROW) ^ ((unsigned long long)j * K_SLOT)), (unsigned long long)tb.rows);
    }
    if (P.idx_bytes == 8) static_cast<long long*>(tb.out)[e] = (long long)v;
    else static_cast<int*>(tb.out)[e] = (int)v;
  }
}

}  // namespace dlrm

extern "C" int dlrm_b200_emb_reduce_partials(const float* partial, float* T, int64_t ldt, int64_t batch, int dim,
                                             const int* slot_feature, const int* slot_first, int num_slots,
                                             void* stream) {
  using namespace dlrm;
  if (num_slots == 0 || batch == 0) return 0;
  if (num_slots < 0 || num_slots > 16) return set_error("emb_reduce_partials: num_slots=%d (max 16)", num_slots);
  if (!partial || !T || !slot_feature || !slot_first) return set_error("emb_reduce_partials: NULL pointer");
  if (dim % 4 || ldt % 4 || !aligned16(partial) || !aligned16(T)) return set_error("emb_reduce_partials: needs 16-byte aligned rows");
  ReduceSlots S{};
  for (int s = 0; s < num_slots; ++s) { S.feature[s] = slot_feature[s]; S.first[s] = slot_first[s]; }
  S.first[num_slots] = slot_first[num_slots];
  S.n = num_slots;
  const long long n = batch * (dim / 4);
  (void)launch_chain(reduce_partials_kernel, dim3((unsigned)((n + 255) / 256), (unsigned)num_slots), dim3(256), 0,
                     static_cast<cudaStream_t>(stream), partial, T, (long long)ldt, (long long)batch, dim, S);
  DLRM_CHECK_LAUNCH("reduce_partials_kernel");
  return 0;
}

extern "C" int dlrm_b200_block_copy(const void* const* src, void* const* dst, const int64_t* nbytes, int n, void* stream) {
  using namespace dlrm;
  if (n == 0) return 0;
  if (n < 0 || n > 64) return set_error("block_copy: n=%d (max 64 per call)", n);
  if (!src || !dst || !nbytes) return set_error("block_copy: NULL argument");
  CopyList L{};
  long long mx = 0;
  for (int k = 0; k < n; ++k) {
    if (!src[k] || !dst[k]) return set_error("block_copy: block %d has a NULL pointer", k);
    if (nbytes[k] % 16 || !aligned16(src[k]) || !aligned16(dst[k]))
      return set_error("block_copy: block %d is not 16-byte aligned / sized", k);
    L.src[k] = static_cast<const uint4*>(src[k]);
    L.dst[k] = static_cast<uint4*>(dst[k]);
    L.n16[k] = nbytes[k] / 16;
    mx = L.n16[k] > mx ? L.n16[k] : mx;
  }
  L.n = n;
  if (mx == 0) return 0;
  long long gx = (mx + 255) / 256;
  if (gx > 296) gx = 296;          // 2 CTAs per SM per block; the grid-stride loop covers the rest
  block_copy_kernel<<<dim3((unsigned)gx, (unsigned)n), 256, 0, static_cast<cudaStream_t>(stream)>>>(L);
  DLRM_CHECK_LAUNCH("block_copy_kernel");
  return 0;
}

extern "C" int dlrm_b200_gen_multihot(void* const* out, const int64_t* rows, const int* hot, const int* table_ids,
                                      int num_tables, int idx_bytes, uint64_t seed, uint64_t step, int64_t sample0,
                                      int64_t batch, float* X, float* target, int m_den, void* stream) {
  using namespace dlrm;
  if (batch == 0) return 0;
  if (num_tables < 0 || num_tables > 64) return set_error("gen_multihot: num_tables=%d (max 64)", num_tables);
  if (idx_bytes != 4 && idx_bytes != 8) return set_error("gen_multihot: idx_bytes=%d", idx_bytes);
  GenParams P{};
  long long mx = X ? batch * (m_den + 1) : 0;
  for (int k = 0; k < num_tables; ++k) {
    if (!out[k] || rows[k] <= 0 || rows[k] >= (1ll << 32) || hot[k] <= 0)
      return set_error("gen_multihot: table %d: out=%p rows=%lld L=%d", k, out[k], (long long)rows[k], hot[k]);
    if (idx_bytes == 4 && rows[k] > 0x7fffffffLL) return set_error("gen_multihot: table %d needs 64-bit indices", k);
    P.t[k].out = out[k]; P.t[k].rows = rows[k]; P.t[k].L = hot[k]; P.t[k].table = table_ids[k];
    mx = batch * hot[k] > mx ? batch * hot[k] : mx;
  }
  P.n = num_tables; P.idx_bytes = idx_bytes; P.seed = seed; P.step = step; P.sample0 = (unsigned long long)sample0;
  P.batch = batch; P.X = X; P.target = target; P.m_den = m_den;
  long long gx = (mx + 255) / 256;
  if (gx > 1184) gx = 1184;
  if (X && gx * 256 < batch * (m_den + 1)) gx = (batch * (m_den + 1) + 255) / 256;
  gen_multihot_kernel<<<dim3((unsigned)gx, (unsigned)(num_tables + 1)), 256, 0, static_cast<cudaStream_t>(stream)>>>(P);
  DLRM_CHECK_LAUNCH("gen_multihot_kernel");
  return 0;
}
