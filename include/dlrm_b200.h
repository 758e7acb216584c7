/*
 * dlrm_b200.h -- C ABI of libdlrm_b200.so: the H100 (sm_90a) kernels behind the
 * DLRM_Net forward/backward hot path of facebookresearch/dlrm.
 *
 * The reference has NO native interface for this path: every op below replaces an
 * ATen call made from dlrm_s_pytorch.py (cited per entry point).  A maintainer of
 * the reference binds these with ctypes (see INTEGRATION.md); dlrm_b200/_lib.py is
 * exactly that binding.
 *
 * Conventions
 *   - extern "C", plain pointers and sizes; no torch types.
 *   - every pointer is a DEVICE pointer on the current CUDA device unless marked
 *     [host]; the caller (PyTorch) owns all memory, the library allocates nothing
 *     and keeps no pointer beyond the call (except inside explicit handles).
 *   - `stream` is a cudaStream_t passed as void* (0 = legacy default stream).
 *     All work is enqueued asynchronously on it; no hidden synchronisation, so
 *     every entry point is legal inside CUDA-graph stream capture.
 *   - return 0 on success, <0 on error; dlrm_b200_last_error() gives the text
 *     (thread-local).  Unsupported shapes are errors, never silent fallbacks.
 *   - float = IEEE fp32.  Index/offset tensors are int64 (idx_bytes=8) or int32
 *     (idx_bytes=4), both arrays of one call having the same width, exactly as
 *     nn.EmbeddingBag accepts them; they are consumed bit-for-bit, never copied.
 *   - Embedding tables are fp32 or IEEE fp16 (weight_dtype, DLRM_DTYPE_*; all tables of one call
 *     share it).  fp16 rows are widened to fp32 for every sum and every optimizer step; the row-wise
 *     accumulator, the list head and all arithmetic stay fp32 / int32.  The `weight` fields keep their
 *     float* type and then point at halves; `ld` always counts elements of the row type.  fp16 needs
 *     dim % 8 == 0.  A zero-initialised descriptor means fp32.
 */
#ifndef DLRM_B200_H_
#define DLRM_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DLRM_B200_ABI_VERSION 1
#define DLRM_B200_MAX_TABLES_PER_CALL 64 /* larger T: split into several calls */
#define DLRM_B200_MAX_PEERS 8            /* GPUs of one NVSwitch box */

/* activations of create_mlp (dlrm_s_pytorch.py:237-241) */
enum { DLRM_ACT_NONE = 0, DLRM_ACT_RELU = 1, DLRM_ACT_SIGMOID = 2 };
/* loss functions (dlrm_s_pytorch.py:385-393) */
enum { DLRM_LOSS_MSE = 0, DLRM_LOSS_BCE = 1, DLRM_LOSS_WBCE = 2 };
/* sparse optimizers: torch.optim.SGD (dlrm_s_pytorch.py:1343) / optim/rwsadagrad.py / torch.optim.Adagrad (:1345) */
enum { DLRM_OPT_SGD = 0, DLRM_OPT_RWSADAGRAD = 1, DLRM_OPT_ADAGRAD = 2 };
/* GEMM back ends */
enum { DLRM_GEMM_SIMT_FP32 = 0, DLRM_GEMM_TC_BF16X3 = 1, DLRM_GEMM_TC_BF16 = 2 };
/* storage type of embedding table rows (weight_dtype of the table descriptors).  The row-wise quantized types are
 * fbgemm's packed rows (torch.ops.quantized.embedding_bag_{byte,4bit}_prepack), forward-only, `ld` in bytes:
 *   DLRM_DTYPE_Q8: [dim uint8 | fp32 scale | fp32 bias], dim % 4 == 0, 4-byte aligned rows;
 *   DLRM_DTYPE_Q4: [dim/2 bytes, column 2j in the low nibble of byte j | fp16 scale | fp16 bias], dim % 8 == 0. */
enum { DLRM_DTYPE_F32 = 0, DLRM_DTYPE_F16 = 1, DLRM_DTYPE_Q8 = 2, DLRM_DTYPE_Q4 = 3 };

int dlrm_b200_abi_version(void);
const char* dlrm_b200_last_error(void);
/* Reads and clears the device error word of the current device (synchronises `stream`): bit 0 = an embedding
 * index outside its table since the last check.  The only hidden state of the library: 256 bytes of device
 * memory per GPU, allocated on first use. */
int dlrm_b200_check_device_errors(void* stream);
/* sm count / compute capability of `device`; error unless cc == 9.0 (the library is built for sm_90a) */
int dlrm_b200_device_info(int device, int* sm_count, int* cc_major, int* cc_minor);
/* Experiment knobs of the kernels (ids: csrc/common.cuh `enum Tunable`; dlrm_b200/_lib.py TUNE; env DLRM_TUNE).
 * Process-wide, read at launch time; 0 restores the default of every knob.  Not part of the reference's surface. */
int dlrm_b200_set_tunable(int id, int value);

/* ------------------------------------------------------------------------------------------
 * apply_emb  (dlrm_s_pytorch.py:407-462: one nn.EmbeddingBag(mode="sum") call per table)
 * ONE launch for all tables:  out[b, k, :] = sum_{j in bag(k,b)} rw_k[idx_k[j]] * W_k[idx_k[j], :]
 * accumulated sequentially in index order (bit-identical to the reference CPU kernel when
 * row_weights == NULL).  Bag b of table k is idx[off[b] .. off[b+1]) and the last bag runs to
 * nnz (EmbeddingBag without include_last_offset) unless include_last != 0, in which case
 * offsets has batch+1 entries and `nnz` is ignored (graph-replay friendly).  Empty bag -> 0.
 * ------------------------------------------------------------------------------------------ */
typedef struct {
  const float* weight;      /* [rows, dim] row-major (fp32, or fp16 per weight_dtype), 16-byte aligned when dim % 4 == 0 */
  const void* indices;      /* [nnz]   int64 / int32 */
  const void* offsets;      /* [batch] (or [batch+1] when include_last) same type */
  const float* row_weights; /* NULL, or [rows]: v_W_l[k] (weighted pooling, :425-428) */
  int64_t nnz;
  int64_t rows;             /* rows of the WHOLE table: an index outside [0, rows) sets the device error word
                             * (dlrm_b200_check_device_errors) and is read as row 0 / skipped; 0 = unchecked */
  int64_t ld;               /* row stride of `weight` in elements of the row type; 0 = dim (dense rows) */
  /* Sharded placement (dlrm_b200/placement.py).  All zero = the call-level layout out[b, k, :].
   * out_stride > 0: the pooled row of bag b goes to out (or the owner's peer buffer) + b_local*out_stride + out_off
   *   -- a whole table lands in feature slot 1+t of the interaction operand, a row-split shard in its slab of
   *   the partial-sum area (dlrm_b200_emb_reduce_partials adds the slabs).
   * row_n > 0: `weight` holds rows [row_lo, row_lo + row_n) of the table; indices outside the range belong
   *   to another shard and are skipped (a partial sum over this shard's rows). */
  int64_t out_off, out_stride;
  int64_t row_lo, row_n;
  int32_t weight_dtype;     /* DLRM_DTYPE_F32 (0) or DLRM_DTYPE_F16: fp16 rows are widened to fp32 and summed as above,
                             * so the pooled output equals the fp32 gather over the widened table bit for bit.
                             * DLRM_DTYPE_Q8 / Q4 (dlrm_b200_emb_bag_fwd only; whole tables, no row range): every
                             * occurrence j of row r adds, column by column and in index order,
                             *   acc = fmaf(s, q, acc + b),  s = scale_r * w_j,  b = bias_r * w_j  (both rounded to fp32)
                             * with w_j = row_weights[r] (1 without them) and the fp16 scale / bias of Q4 widened first:
                             * bit-identical to torch.ops.quantized.embedding_bag_{byte,4bit}_rowwise_offsets on the
                             * CPU.  ld = 0 means the packed width (dim + 8 or dim/2 + 4 bytes). */
} dlrm_emb_fwd_table_t;

int dlrm_b200_emb_bag_fwd(const dlrm_emb_fwd_table_t* tables /*[host]*/, int num_tables, int dim,
                          int64_t batch, int idx_bytes, int include_last,
                          float* out, int64_t out_stride_sample, int64_t out_stride_table,
                          void* stream);

/* Row-wise quantization of `rows` float rows (src_dtype DLRM_DTYPE_F32 or F16, row stride ld_src in elements, so
 * the engine's interleaved rows work as they are) into packed rows of dst_dtype DLRM_DTYPE_Q8 / Q4 (row stride
 * ld_dst bytes, 0 = the packed width).  Byte-identical to torch.ops.quantized.embedding_bag_{byte,4bit}_prepack of
 * the same (widened) values for finite rows; a caller quantizes a table in chunks by offsetting both pointers.
 *   Q8: bias = min, scale = (max - min) / 255, q = rint((x - min) * (255 / ((max - min) + 1e-8))).
 *   Q4: bias = fp16(min), scale = fp16((max - bias) / 15) (1 when the range or that is 0, or 1 / scale is inf),
 *       q = clamp(rint((x - bias) * (1 / scale)), 0, 15). */
int dlrm_b200_emb_quantize_rows(const void* src, int src_dtype, int64_t ld_src, int64_t rows, int dim, void* dst,
                                int dst_dtype, int64_t ld_dst, void* stream);

/* ------------------------------------------------------------------------------------------
 * Embedding backward fused with the sparse optimizer
 * (autograd _embedding_bag_backward, dlrm_s_pytorch.py:1613 + optimizer.step() :1620:
 *  optim/rwsadagrad.py:117-143 or torch.optim.SGD sparse add).
 *
 * Step 1, dlrm_b200_emb_bwd_link: depends on the indices only (can run on a side stream
 * during the forward pass).  Threads every (table,row) occurrence of the batch onto a
 * per-row list: prev = atomicExch(&head[row], pos+1); next[pos] = prev; and, when prev != 0,
 * mark[prev-1] = 1 (that occurrence is no longer the last one of its row).  `head` is an int32
 * array over all rows of the table, `mark` a byte per occurrence position; both are zero on
 * entry and zero again after step 2.
 * Step 2, dlrm_b200_emb_bwd_update: the last occurrence of a row (the unmarked one) owns it,
 * known from the coalesced mark[] without touching the table; it
 * sums dY over the row's occurrences: up to 32 in ascending position (== grad.coalesce()), more
 * with an order-independent fixed-point sum (the same result on every run), then
 *   RWSAdagrad: momentum[row] += mean_d(g^2); W[row] -= lr * g / (sqrt(momentum[row]) + eps)
 *   SGD:        W[row] -= lr * g
 *   Adagrad (element-wise, torch.optim.Adagrad on a sparse gradient): for every column j of the row,
 *               s = momentum[row * mom_stride + j]
 *               s = __fadd_rn(s, __fmul_rn(g[j], g[j]))       (two roundings, no FMA: grad.pow(2), then the add)
 *               d = sqrtf(s) + eps                             (IEEE sqrt, then one rounding)
 *               W[row][j] = fmaf(-lr, g[j] / d, W[row][j])     (IEEE division; one fused step)
 *             `momentum` then points at a [rows][mom_stride] fp32 array (one accumulator per element; mom_stride 0
 *             means dim, otherwise it must be >= dim); NULL momentum or 0 < mom_stride < dim is an error without a
 *             launch.  The vector kernels need a 16-byte aligned momentum and mom_stride % 4 == 0; other
 *             accumulators take the scalar kernel (fp16 tables and the tiny-table path have none: an error).
 *             Rows that do not occur are not touched, neither their weights nor their accumulators.
 * `lr` is the already-decayed clr of optim/rwsadagrad.py:115 (torch.optim.Adagrad: lr / (1 + (step - 1) lr_decay)).
 * fp16 tables (weight_dtype = DLRM_DTYPE_F16): the row is widened to fp32, the step above runs in fp32 with the
 * operations of the fp32 kernel, and the result x is stored with STOCHASTIC ROUNDING: x itself when it is an
 * fp16 value, else lo (the fp16 neighbour toward zero) or hi (the one away from zero), hi iff
 *   r < floor(2^16 * (|x| - |lo|) / (|hi| - |lo|)),
 * |x| > 65504 -> +-inf, NaN stays NaN.  r = 16 bits of h = splitmix64(round_key ^ R * 0xC2B2AE3D27D4EB4F ^
 * (c / 4) * 0x165667B19E3779F9) for global row R = row_lo + local row and column c: bits [16 (c % 4), +16) of h.
 * Rows that are not updated are not rewritten.
 * Learned weighted pooling (row_weights != NULL, v = v_W_l[k] of dlrm_s_pytorch.py:425-428): the forward pooled
 * v[row] * W[row] per occurrence, so with S = the coalesced sum of dY above (v scales every occurrence alike)
 *               g      = v[row] * S                              (fp32 product per element; the step above takes g)
 *               dv     = <S, W_old[row]>                         (the row BEFORE its step; fp16: the widened row)
 *   SGD:        v[row] = fmaf(-lr, dv, v[row])
 *   RWSAdagrad, Adagrad (the dense branch of optim/rwsadagrad.py:145-148 and torch.optim.Adagrad on the [rows]
 *   parameter v; both keep a [rows] 'sum'):
 *               s = fmaf(dv, dv, row_weight_sum[row]);  v[row] = fmaf(-lr, dv / (sqrtf(s) + eps), v[row])
 * with the same lr as the rows.  Only the owner of a row writes v[row] and row_weight_sum[row]: the entries of rows
 * that do not occur stay bit-identical (their gradient is 0 in the reference).  row_weights == NULL runs the
 * unweighted kernels unchanged.  The duplicate filter and dlrm_b200_emb_bwd_update_p2p refuse row_weights.
 * dY[b, k, :] is read at dY + b*dy_stride_sample + k*dy_stride_table.
 * ------------------------------------------------------------------------------------------ */
typedef struct {
  float* weight;        /* [rows, dim] updated in place */
  float* momentum;      /* [rows] (RWSAdagrad), [rows][mom_stride] (Adagrad) or NULL (SGD) */
  int32_t* head;        /* [rows] zero-initialised scratch, self-cleaning */
  const void* indices;  /* as in forward */
  const void* offsets;
  int64_t nnz;
  int64_t rows;
  int64_t pair_base;    /* first slot of this table in next[] / (sum of nnz of earlier tables) */
  int64_t ld;           /* row stride of `weight` in elements of the row type; 0 = dim.  fp16: the weight pointer
                         * 16-byte aligned and ld % 4 == 0 (rows on 8-byte boundaries); ld % 8 == 0 (16-byte rows, the
                         * engine's layout) lets dim <= 128 take the faster kernel with one 16-byte access per lane */
  int64_t mom_stride;   /* elements between consecutive rows' accumulators in `momentum`; 0 = 1 (Adagrad: 0 = dim).
                         * ld = dim + 4 with momentum = weight + dim and mom_stride = ld keeps the
                         * row-wise Adagrad accumulator in the SAME DRAM burst as its row: the update then
                         * costs one activation per row instead of two. */
  /* Sharded placement.  use_dy_off != 0: the gradient row of (bag b, this table) is at dY(b) + dy_off instead
   * of dY(b) + k*dy_stride_table.  row_n > 0: `weight`/`momentum`/`head` hold rows [row_lo, row_lo + row_n)
   * of the table; occurrences of other rows are another shard's.  head == NULL: this table is not linked and
   * not updated by dlrm_b200_emb_bwd_update (tiny tables: dlrm_b200_emb_bwd_small_update). */
  int64_t use_dy_off, dy_off;
  int64_t row_lo, row_n;
  /* elements between consecutive rows' list heads; 0 = 1.  head = (int32*)weight + dim + 1 with head_stride = ld
   * (and momentum = weight + dim, mom_stride = ld, ld = dim + 4) keeps BOTH per-row words inside the row's own
   * DRAM page.  The update is bound by the RATE of random DRAM accesses (the gather's 512-byte rows and the
   * update's 4-byte words cost about the same), and with the marks below the owner of a row reads the two words
   * in the same batch as the row and writes them with the row: two random accesses per updated row (row +
   * words in, row + words out) instead of four. */
  int64_t head_stride;
  /* [positions] superseded marks, indexed like next[] (pair_base + j): mark[p] = 1 once a later occurrence of
   * the same row was linked.  Zero-initialised scratch, all zero between steps (the update clears what the
   * link set).  Required whenever head != NULL. */
  uint8_t* mark;
  /* DLRM_DTYPE_F32 (0) or DLRM_DTYPE_F16 (weight points at halves; ld in halves; momentum / head keep their own
   * fp32 / int32 strides -- the interleaved fp16 row is [dim halves | fp32 accumulator | int32 head | pad]). */
  int32_t weight_dtype;
  /* fp16 only: stochastic-rounding key of this table for this step (see above), the hash prefix
   * splitmix64(seed * 0xD6E8FEB86659FD93 ^ (step + 1) * 0x9E3779B97F4A7C15 ^ (global table + 1) * 0x165667B19E3779F9) */
  uint64_t round_key;
  /* learned weighted pooling (see above): [rows] fp32 v of this table (local rows of a shard), read and updated in
   * place, or NULL (unweighted, or fixed weights of one); row_weight_sum: [rows] fp32 Adagrad 'sum' of v for
   * RWSAdagrad / Adagrad, NULL for SGD.  Ignored by the training gather. */
  float* row_weights;
  float* row_weight_sum;
} dlrm_emb_bwd_table_t;

/* Optional duplicate filter (dlrm_emb_dedup_t): at 1e6-row tables almost every row of a batch is
 * touched once, and the gather's atomicExch on head[] is a random 4-byte access per occurrence.
 * With a filter the training gather only bumps a counter in an L2-sized hashed array
 * (fire-and-forget RED), dlrm_b200_emb_bwd_classify() -- right after the gather, while the
 * counters are L2-hot -- marks the occurrences whose counter is > 1 as suspects (hash collisions
 * only add false suspects) and threads ONLY those onto the per-row lists; the update then treats
 * unflagged occurrences as sole owners of their row and leaves their head[] and link[].x alone.
 *   filter   : uint32 [2^log2_size + 1], zeroed by the caller before every training gather
 *              (the last element is the suspect counter)
 *   flags    : uint8  [nnz capacity]   suspects : int32 [nnz capacity]
 * dedup == NULL everywhere: every occurrence is linked (the original scheme). */
typedef struct {
  uint32_t* filter;
  int32_t log2_size;
  uint8_t* flags;
  int32_t* suspects;
} dlrm_emb_dedup_t;

/* Training forward: the gather of dlrm_b200_emb_bag_fwd AND step 1 (link) in the same launch --
 * the index of every occurrence is already in a register, so linking costs one atomicExch. */
int dlrm_b200_emb_bag_fwd_train(const dlrm_emb_fwd_table_t* tables /*[host]*/,
                                const dlrm_emb_bwd_table_t* train /*[host]*/, int num_tables, int dim,
                                int64_t batch, int idx_bytes, int include_last, int32_t* next,
                                float* out, int64_t out_stride_sample, int64_t out_stride_table,
                                const dlrm_emb_dedup_t* dedup /*[host] or NULL*/, void* stream);

/* After a filtered training gather: flag suspects and link them (two small launches). */
int dlrm_b200_emb_bwd_classify(const dlrm_emb_bwd_table_t* tables /*[host]*/, int num_tables,
                               int64_t batch, int idx_bytes, int include_last, int32_t* next,
                               const dlrm_emb_dedup_t* dedup /*[host]*/, void* stream);

int dlrm_b200_emb_bwd_link(const dlrm_emb_bwd_table_t* tables /*[host]*/, int num_tables,
                           int64_t batch, int idx_bytes, int include_last,
                           int32_t* next /*[total nnz]*/, void* stream);

int dlrm_b200_emb_bwd_update(const dlrm_emb_bwd_table_t* tables /*[host]*/, int num_tables, int dim,
                             int64_t batch, int idx_bytes, int include_last,
                             const int32_t* next, const float* dY, int64_t dy_stride_sample,
                             int64_t dy_stride_table, int optimizer, float lr, float eps,
                             const dlrm_emb_dedup_t* dedup /*[host] or NULL*/, void* stream);
/* _lr_dev variants (here and for dlrm_b200_emb_bwd_small_update, dlrm_b200_dense_update and
 * dlrm_b200_dense_update_pack): the kernels read the learning rate from the device float *lr_dev when it is not
 * NULL, so that a captured CUDA graph can change it between replays; lr_dev == NULL runs exactly the by-value
 * entry point with `lr`.  The same value gives bit-identical results either way. */
int dlrm_b200_emb_bwd_update_lr_dev(const dlrm_emb_bwd_table_t* tables /*[host]*/, int num_tables, int dim,
                                    int64_t batch, int idx_bytes, int include_last,
                                    const int32_t* next, const float* dY, int64_t dy_stride_sample,
                                    int64_t dy_stride_table, int optimizer, float lr,
                                    const float* lr_dev /*[device] or NULL*/, float eps,
                                    const dlrm_emb_dedup_t* dedup /*[host] or NULL*/, void* stream);

/* ------------------------------------------------------------------------------------------
 * Table-wise sharded runs (replaces extend_distributed.alltoall, extend_distributed.py:389-486, and
 * the butterfly shuffle of parallel_forward, dlrm_s_pytorch.py:693-699): the exchange is fused into
 * the kernels through peer-mapped memory (cudaIpc / NVLink), no staging buffer, no collective.
 *   fwd : this rank pools ITS tables for the GLOBAL batch; bag b is stored into rank (b / batch_local)'s
 *         buffer: peer_out[d] + (b % batch_local) * out_stride_sample + k * out_stride_table.
 *   bwd : the dY row of global bag b is loaded from peer_dY[b / batch_local] with the same strides.
 * The caller synchronises the ranks (a barrier after fwd, before bwd).  train may be NULL (inference).
 * ------------------------------------------------------------------------------------------ */
int dlrm_b200_emb_bag_fwd_p2p(const dlrm_emb_fwd_table_t* tables /*[host]*/,
                              const dlrm_emb_bwd_table_t* train /*[host] or NULL*/, int num_tables, int dim,
                              int64_t batch_global, int idx_bytes, int include_last, int32_t* next,
                              float* const* peer_out /*[host][world]*/, int world, int64_t batch_local,
                              int64_t out_stride_sample, int64_t out_stride_table,
                              const dlrm_emb_dedup_t* dedup /*[host] or NULL*/, void* stream);
int dlrm_b200_emb_bwd_update_p2p(const dlrm_emb_bwd_table_t* tables /*[host]*/, int num_tables, int dim,
                                 int64_t batch_global, int idx_bytes, int include_last, const int32_t* next,
                                 const float* const* peer_dY /*[host][world]*/, int world,
                                 int64_t batch_local, int64_t dy_stride_sample, int64_t dy_stride_table,
                                 int optimizer, float lr, float eps,
                                 const dlrm_emb_dedup_t* dedup /*[host] or NULL*/, void* stream);

/* NCCL-free cross-GPU steps over the same peer mappings (graph-capturable):
 *   barrier        : peer_sig[r] = int32[world] on rank r (zero-initialised once); epoch = device int32.
 *   allreduce_mean : peer_grad[r] = dense-gradient arena of rank r (n floats); every rank ends with
 *                    the mean over ranks (DDP semantics), summed in rank order.  The caller places a
 *                    barrier before and after. */
/* kernels running on `device` may dereference memory of `peer_device` (cudaDeviceEnablePeerAccess);
 * needed once per peer before passing IPC-mapped peer pointers to the entry points above. */
int dlrm_b200_enable_peer_access(int device, int peer_device);
/* Export the cudaMalloc allocation that holds device pointer `ptr` of this process: a 64-byte
 * cudaIpcMemHandle_t and ptr's byte offset inside the allocation (send both to the peer process). */
int dlrm_b200_ipc_export(const void* ptr, void* handle64_out /*[host, 64 bytes]*/, int64_t* offset_out /*[host]*/);
/* Open such a handle in another process with `device` current, so that kernels launched on `device`
 * can dereference the mapping (base_out + offset = the peer's ptr).  One open per allocation. */
int dlrm_b200_ipc_open(const void* handle64 /*[host]*/, int device, void** base_out /*[host]*/);
int dlrm_b200_ipc_close(void* base);
int dlrm_b200_p2p_barrier(void* const* peer_sig /*[host][world]*/, int rank, int world, int32_t* epoch,
                          void* stream);
int dlrm_b200_p2p_allreduce_mean(void* const* peer_grad /*[host][world]*/, int rank, int world, int64_t n,
                                 void* stream);

/* ------------------------------------------------------------------------------------------
 * apply_mlp layer (dlrm_s_pytorch.py:399-405: nn.Linear -> addmm, + ReLU / Sigmoid modules)
 *   fwd  : Y[M,N]  = act(X[M,K] W[N,K]^T + bias[N])
 *   dgrad: dX[M,K] = (dY[M,N] W[N,K]) * act'(Xact[M,K])   (Xact = output of the previous
 *          layer, NULL / DLRM_ACT_NONE when the input is not an activation)
 *   wgrad: dW[N,K] = dY[M,N]^T X[M,K];  dbias[N] = sum_m dY[m,n]
 * ld* are row strides in elements.  backend = DLRM_GEMM_*.
 * ------------------------------------------------------------------------------------------ */
int dlrm_b200_linear_fwd(const float* X, int64_t ldx, const float* W, int64_t ldw, const float* bias,
                         float* Y, int64_t ldy, int64_t M, int64_t N, int64_t K, int act,
                         int backend, void* stream);
int dlrm_b200_linear_dgrad(const float* dY, int64_t lddy, const float* W, int64_t ldw,
                           const float* Xact, int64_t ldxa, int act_prev,
                           float* dX, int64_t lddx, int64_t M, int64_t N, int64_t K,
                           int backend, void* stream);
int dlrm_b200_linear_wgrad(const float* dY, int64_t lddy, const float* X, int64_t ldx,
                           float* dW, int64_t lddw, float* dbias, int64_t M, int64_t N, int64_t K,
                           int backend, void* stream);

/* ------------------------------------------------------------------------------------------
 * interact_features (dlrm_s_pytorch.py:483-515), op == "dot":
 *   T[b] = [x[b]; ly_0[b]; ...] (F x D, read in place at T + b*ldt, feature stride D)
 *   R[b, 0:D] = x[b];  R[b, D + tri(i,j)] = <T[b,i], T[b,j]>  for j < i (+ diagonal if itself),
 *   row-major strict lower triangle (1,0),(2,0),(2,1),...  (cat/bmm/index/cat fused: K3-K6).
 * bwd: dT[b] = (dZ + dZ^T) T[b] (+ dR[b,0:D] on feature 0), with dZ scattered from dR[b, D:];
 *   feature 0 of dT is multiplied by act'(x), act = mask_feature0 (DLRM_ACT_*: the bottom MLP's
 *   last activation; DLRM_ACT_NONE = no mask).
 * op == "cat" is a pure layout (R == T flattened): no kernel, handled by strides on the host.
 * ------------------------------------------------------------------------------------------ */
int dlrm_b200_interact_fwd(const float* T, int64_t ldt, float* R, int64_t ldr, int64_t batch,
                           int num_features, int dim, int itself, void* stream);
/* _ex variants: additionally emit the (hi, lo) bf16 operand pair consumed by the wgmma GEMMs
 * (R for the first top-MLP layer; feature 0 of dT for the bottom MLP's backward).  R may be NULL
 * when only the bf16 pair is wanted. */
int dlrm_b200_interact_fwd_ex(const float* T, int64_t ldt, float* R, int64_t ldr, void* R_hi, void* R_lo,
                              int64_t ld_rb, int64_t batch, int num_features, int dim, int itself,
                              void* stream);
int dlrm_b200_interact_bwd_ex(const float* T, int64_t ldt, const float* dR, int64_t lddr, float* dT,
                              int64_t lddt, int64_t batch, int num_features, int dim, int itself,
                              int mask_feature0, void* g0_hi, void* g0_lo, int64_t ld_g0, void* stream);
/* Sharded variant: feature i's gradient rows are stored at feat_dst[q] + sample * feat_ld[q] (floats) for
 * every destination q in [feat_first[i], feat_first[i+1]) instead of dT (at most 128 destinations in all).
 * On a sharded run the destinations of feature 1 + t point into the receive buffers of the rank(s) storing
 * table t (peer-mapped over NVLink; a row-split table has one on every rank), which replaces the backward
 * all-to-all of dlrm_s_pytorch.py:545-560 / extend_distributed.py:alltoall backward; feature 0 stays local.
 * emb_grad_scale multiplies the rows of features >= 1: 1 = the reference's distributed semantics (every rank's
 * loss is the mean over ITS batch slice and the embedding gradients of the ranks are SUMMED, i.e. world x the
 * single-process gradient); 1/world = the gradient of the global mean loss (equals a single-process run). */
int dlrm_b200_interact_bwd_p2p(const float* T, int64_t ldt, const float* dR, int64_t lddr,
                               void* const* feat_dst /*[host][ndst]*/, const int64_t* feat_ld /*[host][ndst]*/,
                               const int* feat_first /*[host][F+1]*/, float emb_grad_scale, int64_t batch,
                               int num_features, int dim,
                               int itself, int mask_feature0, void* g0_hi, void* g0_lo, int64_t ld_g0,
                               void* stream);
int dlrm_b200_interact_bwd(const float* T, int64_t ldt, const float* dR, int64_t lddr,
                           float* dT, int64_t lddt, int64_t batch, int num_features, int dim,
                           int itself, int mask_feature0, void* stream);

/* ------------------------------------------------------------------------------------------
 * loss_fn_wrap (dlrm_s_pytorch.py:148-156; MSELoss/BCELoss(mean), wbce) + clamp (:607-610)
 * + backward through the loss, the clamp and the last activation:
 *   z = clamp(p, thr, 1-thr) iff 0 < thr < 1;  loss = mean(l(z,t) [* ws[t]])
 *   gz[i] = dloss/dz[i] * [thr <= p <= 1-thr] * act'(p[i])     (act = last layer's activation)
 * n = batch * outputs (contiguous).  loss_out: 1 float; gz may be NULL (inference).
 * `scratch` >= 1024 floats.  Deterministic (fixed reduction tree).
 * ------------------------------------------------------------------------------------------ */
int dlrm_b200_loss_fwd_bwd(const float* p, const float* target, const float* loss_ws /*[2] or NULL*/,
                           int64_t n, int loss_kind, float loss_threshold, int last_act,
                           float* loss_out, float* gz, float* scratch, void* stream);

/* gz = gy * [thr <= y <= 1-thr] * act'(y): entry of the backward pass when the loss is computed
 * OUTSIDE the library (autograd of DLRM_Net.forward: `E.backward()` hands us dE/d(clamped p)).
 * clamp_threshold outside (0,1) disables the clamp mask. */
int dlrm_b200_act_bwd(const float* gy, const float* y, float* gz, int64_t n, int act,
                      float clamp_threshold, void* stream);

/* ------------------------------------------------------------------------------------------
 * Dense parameters of optimizer.step(): flat arenas (all bot/top W and b, contiguous).
 *   SGD:        p -= lr * g
 *   RWSAdagrad dense branch (optim/rwsadagrad.py:145-148): s += g*g; p -= lr * g / (sqrt(s)+eps)
 *   Adagrad: the same algorithm, so DLRM_OPT_ADAGRAD runs exactly what DLRM_OPT_RWSADAGRAD runs here and in
 *   dlrm_b200_dense_update_pack.
 * ------------------------------------------------------------------------------------------ */
/* ------------------------------------------------------------------------------------------
 * Fused head for a top MLP whose last layer has one output: Linear(K->1) + act + clamp + loss
 * + d(loss) + wgrad/bias-grad/dgrad of that layer in ONE launch (see csrc/head.cu).
 * target == NULL: inference (p only).  dW == NULL: loss (+ gz) only.  gprev (fp32) and/or
 * gprev_hi/lo (bf16 pair) receive gz * w * act_prev'(h).  scratch: dlrm_b200_head_scratch_bytes()
 * bytes, zero-initialised once.
 * ------------------------------------------------------------------------------------------ */
int64_t dlrm_b200_head_scratch_bytes(int64_t batch, int64_t K);
int dlrm_b200_head_fused(const float* h, int64_t ldh, const float* w, const float* bias,
                         const float* target, const float* loss_ws, int64_t batch, int64_t K,
                         int act_last, int act_prev, int loss_kind, float loss_threshold,
                         float* p, float* loss_out, float* gz, float* dW, float* db,
                         float* gprev, int64_t ld_gprev, void* gprev_hi, void* gprev_lo,
                         int64_t ld_gprev_bf16, void* scratch, void* stream);

int dlrm_b200_dense_update(float* param, const float* grad, float* state /*NULL for SGD*/,
                           int64_t n, int optimizer, float lr, float eps, void* stream);
int dlrm_b200_dense_update_lr_dev(float* param, const float* grad, float* state /*NULL for SGD*/,
                                  int64_t n, int optimizer, float lr, const float* lr_dev /*[device] or NULL*/,
                                  float eps, void* stream);


/* ------------------------------------------------------------------------------------------
 * wgmma GEMM back end of apply_mlp and its autograd (aten::addmm, dlrm_s_pytorch.py:399-405):
 *   D[M,N] = sum_k A(m,k) * B(n,k),  bf16 operands staged by TMA, fp32 accumulation in registers.
 * Operands are (hi, lo) bf16 pairs of fp32 values (hi = bf16(x), lo = bf16(x - hi)); mode_x3
 * computes hi*hi + hi*lo + lo*hi (fp32-grade), otherwise hi*hi only.  An operand is K-major
 * ([rows, K], ld = row stride) or MN-major ([K, rows]); ld in elements, multiple of 8.
 * Bias: forward layers add `bias` (fp32) in the epilogue; the weight-gradient GEMMs get the bias gradient
 * for free from a constant-1 column of the activations ([dW | db] = gz^T [X | 1]).
 * Epilogue (all optional): act(); multiply by act'(y), y = mask_hi + mask_lo [M, ldmask];
 * fp32 store (split-K: one slab per split, reduced by dense_update_pack); the last column diverted to
 * out_col (bias gradient: needs out_f32, col_index = N - 1); (hi, lo) bf16 stores in normal [M, ld_out] and
 * transposed [N, ld_outT] layout.  A plan holds the TMA descriptors: create once per buffer set, run every step.
 * split_k is an upper bound: no split is left without a k block, so a plan may write fewer slabs than asked
 * (K = 700, split_k = 8: 11 k blocks, 2 per split, 6 slabs).  plan_info reports the slabs a run writes; slabs
 * past that count are never touched, and the caller reduces exactly that many (dlrm_dense_layer_t.num_slabs).
 * Only operand elements inside [rows, K] are read and only output elements inside [M, N] are written: the
 * padding up to the leading dimensions may hold anything and is left as it is.
 * ------------------------------------------------------------------------------------------ */
typedef struct {
  const void* A_hi; const void* A_lo; int64_t lda; int a_mn_major;
  const void* B_hi; const void* B_lo; int64_t ldb; int b_mn_major;
  int64_t M, N, K;
  int mode_x3;
  int split_k;      /* >= 1: at most this many slabs; plan_info gives the number written */
  int tile_n;       /* 0 = auto, or 32 / 64 / 128 */
  int act;          /* DLRM_ACT_* applied to the accumulator */
  int mask_act;     /* DLRM_ACT_*: multiply by act'(y) */
  const void* mask_hi; const void* mask_lo; int64_t ldmask;
  float* out_f32; int64_t ld_f32; int64_t slab_stride;
  void* out_hi; void* out_lo; int64_t ld_out;
  void* outT_hi; void* outT_lo; int64_t ld_outT;
  float* out_col; int64_t col_index; int64_t col_slab_stride;
  const float* bias;  /* optional fp32 [N] added to the accumulator before act (nn.Linear bias in fp32) */
  int tile_m;       /* rows per CTA tile: 0 = auto, 128 or 256.  256 needs a 128-wide tile and no split-K (refused
                       otherwise); auto picks it for such plans when M >= 256, the grid keeps >= 120 CTAs and every
                       K-major operand's ld is a multiple of 64 (128-byte rows).  Both heights give bit-identical
                       results. */
} dlrm_gemm_tc_desc_t;

int dlrm_b200_gemm_tc_plan_create(const dlrm_gemm_tc_desc_t* desc /*[host]*/, void** plan);
/* tile_m (appended): the plan's rows per CTA tile, 128 or 256.  Any output pointer may be NULL. */
int dlrm_b200_gemm_tc_plan_info(void* plan, int* tile_n, int* stages, int* splits, int* ctas, int* tile_m);
int dlrm_b200_gemm_tc_run(void* plan, void* stream);
int dlrm_b200_gemm_tc_plan_destroy(void* plan);

/* fp32 [M,N] (row stride ldx) -> (hi, lo) bf16 [M, ld_out]; lo may be NULL */
int dlrm_b200_split_bf16(const float* X, int64_t ldx, int64_t M, int64_t N, void* hi, void* lo,
                         int64_t ld_out, void* stream);

/* Dense optimizer step fused with the split-K slab reduction of dW/db and the refresh of the
 * [N, K+1] = [W | bias] (hi, lo) operand copies.  optimizer = DLRM_OPT_*, -1 (pack only) or
 * -2 (only fold the slabs into slab 0, for a cross-rank all-reduce before the update). */
typedef struct {
  float* W; float* b; float* sW; float* sb;
  const float* dW; const float* db;
  void* pack_hi; void* pack_lo;
  int64_t slab_stride; int64_t N; int64_t K; int64_t ld_pack; int64_t num_slabs;
} dlrm_dense_layer_t;
int dlrm_b200_dense_update_pack(const dlrm_dense_layer_t* layers /*[host]*/, int num_layers, int optimizer,
                                float lr, float eps, void* stream);
int dlrm_b200_dense_update_pack_lr_dev(const dlrm_dense_layer_t* layers /*[host]*/, int num_layers, int optimizer,
                                       float lr, const float* lr_dev /*[device] or NULL*/, float eps, void* stream);

/* ------------------------------------------------------------------------------------------
 * Sharded placement (dlrm_b200/placement.py): the pieces around the gather / update kernels.
 * ------------------------------------------------------------------------------------------ */
/* Row-split table, remote-read forward: the rank that owns the samples pools each bag itself, in index order,
 * reading every row from the rank that stores it (shard_weight[s] = base of rows [s*rows_per_shard, ...), a
 * peer-mapped pointer for s != own rank): 512-byte NVLink loads inside the gather kernel instead of partial sums
 * + reduction.  out[b*out_stride + out_off .. +dim) for the `batch` bags described by offsets / indices. */
typedef struct {
  const float* shard_weight[DLRM_B200_MAX_PEERS];
  int32_t num_shards;
  int64_t rows_per_shard;
  int64_t rows;
  int64_t ld;
  const void* indices; const void* offsets; int64_t nnz;
  int64_t out_off, out_stride;
  int32_t weight_dtype;     /* DLRM_DTYPE_F32 (0) or DLRM_DTYPE_F16; ld in elements of the row type */
} dlrm_emb_remote_table_t;
int dlrm_b200_emb_bag_fwd_remote(const dlrm_emb_remote_table_t* tables /*[host]*/, int num_tables, int dim,
                                 int64_t batch, int idx_bytes, int include_last, float* out, void* stream);

/* Tiny tables (a few to a few hundred rows, hit thousands of times per step at MLPerf batch sizes): dense
 * two-pass coalesce + row update instead of the per-row list walk (csrc/emb_small.cu).  Same semantics as
 * dlrm_b200_emb_bwd_update (grad.coalesce() + optim/rwsadagrad.py:117-143 / sparse SGD), deterministic.
 * Every table needs use_dy_off; `scratch` holds the per-chunk partial sums
 * (dlrm_b200_emb_bwd_small_scratch_bytes(total rows of the call, dim, batch) bytes).
 * dY (or every peer_dY[d], d < world) must be 16-byte aligned and dy_stride_sample / dy_off multiples of 4:
 * otherwise an error without a launch (the rows are read with 16-byte loads; there is no scalar kernel). */
int64_t dlrm_b200_emb_bwd_small_scratch_bytes(int64_t total_small_rows, int dim, int64_t batch);
int dlrm_b200_emb_bwd_small_update(const dlrm_emb_bwd_table_t* tables /*[host]*/, int num_tables, int dim,
                                   int64_t batch, int idx_bytes, int include_last, const float* dY,
                                   const float* const* peer_dY /*[host][world] or NULL*/, int world,
                                   int64_t batch_local, int64_t dy_stride_sample, int optimizer, float lr,
                                   float eps, float* scratch, int64_t scratch_bytes, void* stream);
int dlrm_b200_emb_bwd_small_update_lr_dev(const dlrm_emb_bwd_table_t* tables /*[host]*/, int num_tables, int dim,
                                          int64_t batch, int idx_bytes, int include_last, const float* dY,
                                          const float* const* peer_dY /*[host][world] or NULL*/, int world,
                                          int64_t batch_local, int64_t dy_stride_sample, int optimizer, float lr,
                                          const float* lr_dev /*[device] or NULL*/, float eps, float* scratch,
                                          int64_t scratch_bytes, void* stream);
/* Row-split tables: T[b, slot_feature[s], :] = sum of the slabs [slot_first[s], slot_first[s+1]) of
 * partial ([slab][batch][dim]), in slab order. */
int dlrm_b200_emb_reduce_partials(const float* partial, float* T, int64_t ldt, int64_t batch, int dim,
                                  const int* slot_feature /*[host]*/, const int* slot_first /*[host][n+1]*/,
                                  int num_slots, void* stream);
/* n <= 64 contiguous blocks (16-byte aligned pointers and sizes) copied in ONE launch; destinations may be
 * peer-mapped (the index exchange of a sharded step). */
int dlrm_b200_block_copy(const void* const* src /*[host]*/, void* const* dst /*[host]*/,
                         const int64_t* nbytes /*[host]*/, int n, void* stream);
/* Device-side synthetic batch of the MLPerf multi-hot distribution (torchrec_dlrm/multi_hot.py:80-127):
 * out[k] = [batch, hot[k]] indices (idx_bytes wide) of table table_ids[k] for global samples
 * [sample0, sample0 + batch) of `step`; optional dense features X [batch, m_den] and rounded targets [batch].
 * Bit-identical to dlrm_b200/mlperf.py (host). */
int dlrm_b200_gen_multihot(void* const* out /*[host]*/, const int64_t* rows /*[host]*/, const int* hot /*[host]*/,
                           const int* table_ids /*[host]*/, int num_tables, int idx_bytes, uint64_t seed,
                           uint64_t step, int64_t sample0, int64_t batch, float* X, float* target, int m_den,
                           void* stream);

/* ------------------------------------------------------------------------------------------
 * MLPerf binary records -> one packed batch (data_loader_terabyte.py:74-93 _transform_features,
 * :229-240 CriteoBinDataset.__getitem__).  records = n int32 records [label | num_dense | num_sparse ids]:
 *   X[b, d]            = logf((float)x + 1.0f)   (fp32 conversion, then an fp32 add; IEEE logf)
 *   target[b]          = (float)label
 *   indices[k*n + b]   = id mod max_ind_range (floor modulo, never negative) if max_ind_range > 0, else id
 *   offsets[k*(n+1)+b] = k*n + b for b in 0..n   (the include_last layout of dlrm_b200/data.py)
 * A negative id with max_ind_range <= 0 is passed through; the gather's range check reports it.
 * n <= 0, non-positive num_dense / num_sparse or a NULL pointer is an error without a launch.
 * ------------------------------------------------------------------------------------------ */
int dlrm_b200_decode_records(const int32_t* records, int64_t n, int num_dense, int num_sparse,
                             int64_t max_ind_range, float* X, float* target, int64_t* offsets,
                             int64_t* indices, void* stream);

/* ------------------------------------------------------------------------------------------
 * One packed batch from a processed Criteo split resident in device memory (dlrm_data_pytorch.py:293-296
 * CriteoDataset.__getitem__, :324-337 collate_wrapper_criteo_offset).  X_int [N, num_dense], X_cat
 * [N, num_sparse] and y [N] are int32 row-major; sample b of the batch is row ids[b] (int64 [n], device).
 * The outputs are exactly those of dlrm_b200_decode_records for the records [y | X_int | X_cat] of rows
 * ids[0..n).  The ids are not checked: the caller guarantees 0 <= ids[b] < N.
 * n <= 0, non-positive num_dense / num_sparse, more than 127 words per sample or a NULL pointer is an
 * error without a launch.
 * ------------------------------------------------------------------------------------------ */
int dlrm_b200_gather_records(const int32_t* X_int, const int32_t* X_cat, const int32_t* y, const int64_t* ids,
                             int64_t n, int num_dense, int num_sparse, int64_t max_ind_range, float* X,
                             float* target, int64_t* offsets, int64_t* indices, void* stream);

/* ------------------------------------------------------------------------------------------
 * One chunk of a per-day Criteo file (the reference's `*_{d}_reordered.npz`, read with --memory-map) into a
 * device ring of int32 rows.  x_int [n, num_dense], x_cat [n, num_sparse] and y [n] are row-major device arrays
 * in the dtype the file stores: 0 float64, 1 int64, 2 int32.  Chunk row r goes to ring row
 * (dst + r) mod capacity of ring_int [capacity, num_dense], ring_cat [capacity, num_sparse], ring_y [capacity];
 * no other ring row is written.
 * Every value is checked: an exact integer inside int32 range, and in addition an id >= 0 and a label in {0, 1}.
 * A value that fails is not written, and *bad (device) becomes min(*bad, r * 4 + member), member 0 X_int,
 * 1 X_cat, 2 y: the caller sets *bad to UINT64_MAX first and reads it once the chunk's work has completed.
 * Rows whose values all pass are converted exactly, so dlrm_b200_gather_records over ring rows gives the
 * reference's collate of the same samples.
 * n outside 1..capacity, dst outside [0, capacity), non-positive num_dense / num_sparse, an unknown dtype code
 * or a NULL pointer is an error without a launch.
 * ------------------------------------------------------------------------------------------ */
int dlrm_b200_ingest_records(const void* x_int, int x_int_dtype, const void* x_cat, int x_cat_dtype, const void* y,
                             int y_dtype, int64_t n, int num_dense, int num_sparse, int32_t* ring_int,
                             int32_t* ring_cat, int32_t* ring_y, int64_t capacity, int64_t dst, uint64_t* bad,
                             void* stream);

/* ------------------------------------------------------------------------------------------
 * Host tables (csrc/host_tables.cu): fp32 tables whose rows live in pinned, mapped host memory.  The rows a batch
 * touches are staged into an HBM arena before the gather and written back after the update, so the gather and
 * update entry points above run unchanged on the staging arena (rows = capacity) with `slot_idx` as their indices.
 *   stage_in   : for every occurrence p (global position: pos_base + local position; a packed batch's offsets are
 *                already global, pos_base 0) of a host table, over the positions the gather reads
 *                ([offsets[0], end of the last bag)): an index outside [0, rows) sets the device error word and
 *                writes slot -1 (the gather then reports and skips it as well); otherwise the first occurrence of
 *                its row claims map[row] (0 -> p + 1), becomes the row's slot p, and copies the row (ld floats,
 *                the word head_col written as zero), its separate accumulator and its element-wise Adagrad row
 *                into slot p of the staging arrays.  slot_idx[p] = the slot, in the batch's index dtype.  The
 *                counter is reset by a memset on `stream` first; it ends as the number of distinct rows, and
 *                list[0 .. count) holds their slots.
 *   write_back : every listed slot back to its host row (head_col written as zero), and map[row] = 0.
 *   release    : map[row] = 0 for every listed slot only (a forward without an update).
 * The map of a table is int32 [rows], all zero between steps; untouched host rows are never read or written.
 * Host pointers must be device-accessible at the same address (unified addressing; dlrm_b200_host_register).
 * The tables of one call share the row layout: ld floats per row (dim when 0), separate accumulators either for
 * every table and the staging or for none, and the same for element-wise accumulators ([rows][dim]).
 * ------------------------------------------------------------------------------------------ */
typedef struct {
  float* weight;        /* [host] rows [rows][ld] */
  float* momentum;      /* [host] separate row-wise accumulators [rows], or NULL */
  float* acc_ew;        /* [host] element-wise Adagrad accumulators [rows][dim], or NULL */
  const void* indices;  /* as in dlrm_emb_fwd_table_t */
  const void* offsets;
  int64_t nnz;
  int64_t rows;
  int64_t pos_base;     /* first global position of this table (reference format: pair_base) */
  int32_t* map;         /* [rows] device, zero between steps */
} dlrm_host_table_t;

typedef struct {
  float* weight;        /* [capacity][ld] */
  float* momentum;      /* [capacity] or NULL */
  int32_t* head;        /* [capacity] separate list heads, set to zero for every staged slot, or NULL */
  float* acc_ew;        /* [capacity][dim] or NULL */
  void* slot_idx;       /* [capacity] slot of every position, the batch's index dtype */
  int32_t* list;        /* [capacity] staged slots */
  int64_t* key;         /* [capacity] row * 64 + table of a staged slot */
  int32_t* count;       /* one int32: staged rows */
  int64_t capacity;     /* positions (and slots); every global position must be below it */
  int64_t ld;           /* floats per row; 0 = dim */
  int64_t head_col;     /* word of the row holding the list head (interleaved rows), or -1 */
  /* Row cache (all zero: no cache, and every call behaves as described above).  With cache_rows = N > 0 the
   * staging arrays weight / momentum / head / acc_ew hold N + capacity rows: slots [0, N) are the cache, kept
   * across calls, and position p stages into slot N + p.  map[row] = slot + 1 then means a cache slot for 1..N
   * and this step's staging slot above N; only the latter are cleared by write_back / release.  key[] stays
   * [capacity], indexed by position.  The set of a row is splitmix64(row * 64 + table) mod (N / 32), 32 ways.
   *   stage_in, training (forward_only = 0): a one-thread kernel, in place of the counter memset, advances *step
   *                and resets count and num_sets; a resident row is a hit (its slot goes to slot_idx, its last use becomes *step); a missing row is
   *                staged as above and threaded onto its set's list.
   *   stage_in, forward_only = 1: hits are read from their slots, misses staged; no cache state changes.
   *   write_back : per set with misses, the misses in ascending (table, row) order take the ways not used in this
   *                step, empty ways first, then the oldest last use, ties to the lower way; a victim's row goes
   *                to host memory and leaves the map; the miss moves into the slot.  Misses left over go home.
   * stats: cumulative hits, inserts, evictions, staged (uncached) rows, each per distinct row of a training step. */
  int64_t cache_rows;   /* N: a multiple of 32, N + capacity <= 2^31 - 2; 0 = no cache */
  int64_t* cache_tag;   /* [N] row * 64 + table of a resident slot, -1 = empty */
  int32_t* cache_used;  /* [N] training step of the slot's last use, 0 = empty */
  int32_t* step;        /* one int32: the current training step, 0 before the first */
  int32_t* set_head;    /* [N / 32] position + 1 of a set's first miss, zero between steps */
  int32_t* set_next;    /* [capacity] */
  int32_t* sets;        /* [N / 32] the sets with a miss in this step */
  int32_t* num_sets;    /* one int32 */
  int64_t* stats;       /* [4] hits, inserts, evictions, staged */
  int64_t forward_only; /* 1: a pass without an update (see stage_in) */
} dlrm_host_stage_t;

int dlrm_b200_host_stage_in(const dlrm_host_table_t* tables /*[host]*/, int num_tables,
                            const dlrm_host_stage_t* stage /*[host]*/, int dim, int64_t batch, int idx_bytes,
                            int include_last, void* stream);
int dlrm_b200_host_write_back(const dlrm_host_table_t* tables /*[host]*/, int num_tables,
                              const dlrm_host_stage_t* stage /*[host]*/, int dim, void* stream);
int dlrm_b200_host_release(const dlrm_host_table_t* tables /*[host]*/, int num_tables,
                           const dlrm_host_stage_t* stage /*[host]*/, int dim, void* stream);
/* Row cache: every resident row and its accumulators back to host memory (list head as zero), then its map entry,
 * tag and last use cleared.  Counters and the step are kept.  Needs cache_rows > 0; no batch fields are read. */
int dlrm_b200_host_cache_flush(const dlrm_host_table_t* tables /*[host]*/, int num_tables,
                               const dlrm_host_stage_t* stage /*[host]*/, int dim, void* stream);
/* Page-lock [ptr, ptr + bytes) of ordinary host memory as mapped memory (cudaHostRegister) and check that the
 * device address equals ptr; error (and nothing stays registered) otherwise.  Synchronous. */
int dlrm_b200_host_register(void* ptr, int64_t bytes);
int dlrm_b200_host_unregister(void* ptr);

#ifdef __cplusplus
}
#endif
#endif /* DLRM_B200_H_ */
