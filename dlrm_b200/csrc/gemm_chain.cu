// Persistent tile-dataflow wgmma kernel: a whole MLP chain (forward layers, or the dgrad chain with
// all weight-gradient GEMMs beside it) in ONE launch.
//
// Why: at batch 2048 every layer of the DLRM MLPs is a 32-144-tile GEMM whose math takes a few us; as one
// launch per layer each pays launch + prologue (barrier init, descriptor fetch) + pipeline fill + drain.
// Here the tiles of ALL layers of a chain are one topologically ordered task list:
//
//   * grid = one CTA per SM (or fewer); warp 0 claims the next task from a device-side queue
//     (atomicAdd, claimed one task ahead so the round trip is hidden), publishes it to the consumer
//     warps through a 4-deep shared-memory ring guarded by mbarriers and streams its operands;
//   * a task whose A operand is produced inside this launch (layer l+1 reads layer l's activations;
//     a weight-gradient GEMM reads the dgrad chain's gz) spins on per-(producer, 128-row block)
//     completion counters (ld.acquire.gpu), then issues a async-proxy fence before its TMA loads.  Tasks
//     are claimed in topological order and a claimed task depends only on lower-numbered tasks, which are
//     owned by resident CTAs: no deadlock whatever the number of resident CTAs;
//   * the two consumer warpgroups run the wgmmas of tile i, stage the accumulator in shared memory and run
//     its epilogue (activation / activation-gradient mask, fp32 and (hi,lo) bf16 stores) while the producer
//     already streams the operands of tile i+1; after their stores they bump the completion counter
//     (fence + named barrier + release reduction);
//   * the last CTA to leave zeroes queue + counters, so a CUDA-graph replay needs no memset node.
//
// The CTA program per tile (TMA boxes, smem descriptors, main loop, epilogue) is the one of
// gemm_tc_body.cuh, so the results are bit-identical to the per-layer launches.
#include <string.h>

#include "gemm_tc_common.cuh"

namespace dlrm {

constexpr int CH_MAX_PROBLEMS = 16;
constexpr int CH_RING = 4;

struct ChProblem {
  CUtensorMap m[4];   // A_hi, A_lo, B_hi, B_lo
  TcArgs a;
  int bn;
  int gx, gy, gz;     // n tiles, m tiles, k splits
  int task_begin;
  int dep;            // producing problem or -1
  int dep_on_k;       // 0: A rows = this task's m tile; 1: A rows = this task's k range
  int dep_target;     // tiles per 128-row block of the producer
  int ctr_base;       // this problem's counters: ctr[2 + ctr_base + m_tile]
  int signal;         // some later problem depends on this one
};

// Task order.  A group of consecutive single-split problems with the same number of m tiles (the layers of a
// forward MLP, the dgrad chain) is enumerated M-TILE MAJOR: (m, problem, n tile).  Layer l+1 of m tile 0 is then
// claimed right after layer l of m tile 0 and can start as soon as those few tiles are done, while other CTAs
// work on the next m tiles: the layers pipeline across the batch instead of running as one wave per layer.
// Any other problem is a group of its own, enumerated (k split, m, n).
struct ChGroup {
  int task_begin, p0, np, per_m;
};

struct ChParams {
  ChProblem p[CH_MAX_PROBLEMS];
  ChGroup grp[CH_MAX_PROBLEMS];
  int ngroups;
  int n, total, stages;
  int max_bn;         // widest tile: size of the accumulator staging
  uint32_t stage_bytes;
  int* ctr;           // [0] task queue, [1] exit count, [2...] completion counters
  int n_ctr;
  // optional per-task timeline (globaltimer ns), 8 words per task: claim, deps ready, last TMA issued,
  // consumers start, wgmmas retired, accumulator staged, epilogue + signal done, SM id
  unsigned long long* trace;
};

__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.b32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_gpu_add(int* p, int v) {
  asm volatile("red.release.gpu.global.add.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

struct ChTask {
  int pi, bx, by, bz;
};
__device__ __forceinline__ ChTask ch_decode(const ChParams& P, int t) {
  ChTask k;
  int gi = 0;
  while (gi + 1 < P.ngroups && t >= P.grp[gi + 1].task_begin) ++gi;
  const ChGroup& G = P.grp[gi];
  const int local = t - G.task_begin;
  if (G.np == 1) {
    const ChProblem& Q = P.p[G.p0];
    k.pi = G.p0;
    k.bx = local % Q.gx;
    k.by = (local / Q.gx) % Q.gy;
    k.bz = local / (Q.gx * Q.gy);
  } else {
    k.by = local / G.per_m;
    int r = local - k.by * G.per_m;
    k.pi = G.p0;
    while (r >= P.p[k.pi].gx) { r -= P.p[k.pi].gx; ++k.pi; }
    k.bx = r;
    k.bz = 0;
  }
  return k;
}

constexpr int CH_EPI_WARPS = TC_EPI_WARPS;
constexpr int CH_THREADS = TC_THREADS;
constexpr int CH_HEAD = 512;        // barriers + task ring

template <int BN>
__device__ __forceinline__ void ch_mma_stage(const TcArgs& g, uint32_t ring, uint32_t stage_bytes, int stages,
                                             uint32_t bar_full, uint32_t bar_empty, int kb0, int kb1, int& stage,
                                             uint32_t& phase, float* acc, int cw, int lane) {
  float d[BN / 2];
  tc_mainloop<BN>(d, g, ring, stage_bytes, stages, bar_full, bar_empty, kb0, kb1, stage, phase, cw >> 2, lane);
  // the previous task's epilogue has read the staged accumulator before it is overwritten
  asm volatile("bar.sync 2, %0;" ::"n"(32 * CH_EPI_WARPS) : "memory");
  tc_stage_acc<BN>(d, acc, cw, lane);
}

__global__ void __launch_bounds__(CH_THREADS, 1) gemm_chain_kernel(const __grid_constant__ ChParams P) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int stages = P.stages;
  const uint32_t stage_bytes = P.stage_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)stages * stage_bytes);
  // bars: full[stages] | empty[stages] | task_full[4] | task_empty[4]
  int* ring = reinterpret_cast<int*>(bars + 2 * stages + 2 * CH_RING);
  float* acc = reinterpret_cast<float*>(smem + (size_t)stages * stage_bytes + CH_HEAD);
  uint8_t* epi_stage = smem + (size_t)stages * stage_bytes + CH_HEAD + tc_acc_bytes(P.max_bn);

  pdl_launch_dependents();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t smem_base = smem_u32(smem);
  const uint32_t bar_full = smem_u32(bars);
  const uint32_t bar_empty = bar_full + 8 * stages;
  const uint32_t bar_task_full = bar_empty + 8 * stages;
  const uint32_t bar_task_empty = bar_task_full + 8 * CH_RING;

  if (threadIdx.x == 0) {
    for (int s = 0; s < stages; ++s) {
      mbar_init(bar_full + 8 * s, 1);
      mbar_init(bar_empty + 8 * s, CH_EPI_WARPS);        // one arrive per consumer warp
    }
    for (int s = 0; s < CH_RING; ++s) {
      mbar_init(bar_task_full + 8 * s, 1);
      mbar_init(bar_task_empty + 8 * s, CH_EPI_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();   // barriers are set up; global memory is first touched below

  if (warp == 0) {
    // ------------------------------------------------------------------ task claim + TMA producer
    if (lane == 0) {
      int stage = 0, slot = 0;
      uint32_t phase = 0, tph = 0;
      int t = atomicAdd(P.ctr, 1);
      while (true) {
        mbar_wait(bar_task_empty + 8 * slot, tph ^ 1);
        ring[slot] = t;
        mbar_arrive(bar_task_full + 8 * slot);
        if (++slot == CH_RING) { slot = 0; tph ^= 1; }
        if (t >= P.total) break;
        if (P.trace) P.trace[(size_t)t * 8 + 0] = globaltimer_ns();
        const int tnext = atomicAdd(P.ctr, 1);    // claimed one task ahead: the round trip hides behind this task
        const ChTask k = ch_decode(P, t);
        const ChProblem& Q = P.p[k.pi];
        const TcArgs& g = Q.a;
        const uint32_t A_BYTES = TC_A_BYTES;
        const uint32_t B_BYTES = (uint32_t)Q.bn * TC_BK * 2;
        const uint32_t tx = (g.x3 ? 2u : 1u) * (A_BYTES + B_BYTES);
        const int m0 = k.by * TC_BM, n0 = k.bx * Q.bn;
        const int kb0 = k.bz * g.kb_per_split;
        const int kb1 = min(g.num_kb, kb0 + g.kb_per_split);
        if (Q.dep >= 0) {
          long long r0, r1;
          if (Q.dep_on_k) { r0 = (long long)kb0 * TC_BK; r1 = min((long long)kb1 * TC_BK, g.K); }
          else { r0 = m0; r1 = min((long long)m0 + TC_BM, g.M); }
          const int* cbase = P.ctr + 2 + P.p[Q.dep].ctr_base;
          for (int c = (int)(r0 / TC_BM); c < (int)((r1 + TC_BM - 1) / TC_BM); ++c) {
            unsigned long long t0 = 0;
            while (ld_acquire_gpu(cbase + c) < Q.dep_target) {
              __nanosleep(40);
              const unsigned long long now = globaltimer_ns();
              if (t0 == 0) t0 = now;
              else if (now - t0 > 2000000000ull) __trap();   // a protocol bug must trap, not hang the GPU
            }
          }
          asm volatile("fence.proxy.async;" ::: "memory");   // producer's generic-proxy stores -> our TMA reads
        }
        if (P.trace) P.trace[(size_t)t * 8 + 1] = globaltimer_ns();
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(bar_empty + 8 * stage, phase ^ 1);
          const uint32_t full = bar_full + 8 * stage;
          mbar_expect_tx(full, tx);
          uint32_t dst = smem_base + stage * stage_bytes;
          const int k0 = kb * TC_BK;
          for (int part = 0; part < (g.x3 ? 2 : 1); ++part) {
            const CUtensorMap* map = &Q.m[part];
            if (!g.a_mn) {
              tma_load_2d(dst, map, full, k0, m0);
            } else {
              tma_load_2d(dst, map, full, m0, k0);
              tma_load_2d(dst + A_BYTES / 2, map, full, m0 + 64, k0);
            }
            dst += A_BYTES;
          }
          for (int part = 0; part < (g.x3 ? 2 : 1); ++part) {
            const CUtensorMap* map = &Q.m[2 + part];
            if (!g.b_mn) {
              tma_load_2d(dst, map, full, k0, n0);
            } else {
              for (int h = 0; h < Q.bn / 64; ++h) tma_load_2d(dst + h * 8192, map, full, n0 + 64 * h, k0);
            }
            dst += B_BYTES;
          }
          if (++stage == stages) { stage = 0; phase ^= 1; }
        }
        if (P.trace) P.trace[(size_t)t * 8 + 2] = globaltimer_ns();
        t = tnext;
      }
    }
  } else if (warp >= TC_CONSUMER_WARP0) {
    // ------------------------------------------------------------------ wgmma consumers + epilogue (warps 4..11)
    const int cw = warp - TC_CONSUMER_WARP0;
    const bool rec = P.trace && cw == 0 && lane == 0;
    int stage = 0, slot = 0;
    uint32_t phase = 0, tph = 0;
    while (true) {
      mbar_wait(bar_task_full + 8 * slot, tph);
      const int t = __shfl_sync(0xffffffffu, ring[slot], 0);   // warp-uniform: the wgmma paths below branch on it
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_task_empty + 8 * slot);
      if (++slot == CH_RING) { slot = 0; tph ^= 1; }
      if (t >= P.total) break;
      const ChTask k = ch_decode(P, t);
      const ChProblem& Q = P.p[k.pi];
      const int kb0 = k.bz * Q.a.kb_per_split;
      const int kb1 = min(Q.a.num_kb, kb0 + Q.a.kb_per_split);
      if (rec) P.trace[(size_t)t * 8 + 3] = globaltimer_ns();
      if (Q.bn == 128)
        ch_mma_stage<128>(Q.a, smem_base, stage_bytes, stages, bar_full, bar_empty, kb0, kb1, stage, phase, acc, cw, lane);
      else if (Q.bn == 64)
        ch_mma_stage<64>(Q.a, smem_base, stage_bytes, stages, bar_full, bar_empty, kb0, kb1, stage, phase, acc, cw, lane);
      else
        ch_mma_stage<32>(Q.a, smem_base, stage_bytes, stages, bar_full, bar_empty, kb0, kb1, stage, phase, acc, cw, lane);
      if (rec) P.trace[(size_t)t * 8 + 4] = globaltimer_ns();
      asm volatile("bar.sync 1, %0;" ::"n"(32 * CH_EPI_WARPS) : "memory");
      if (rec) P.trace[(size_t)t * 8 + 5] = globaltimer_ns();
      tc_epilogue_tile(Q.a, Q.bn, k.by * TC_BM, k.bx * Q.bn, k.bz, acc, cw & 3, lane,
                       epi_stage + (size_t)cw * TC_EPI_WARP_BYTES, cw >> 2, CH_EPI_WARPS / 4);
      if (Q.signal) {
        // grid-sync idiom: every epilogue thread has issued its stores (barrier), then ONE thread makes them
        // visible GPU-wide (cumulative fence) and publishes the tile with a release reduction
        asm volatile("bar.sync 1, %0;" ::"n"(32 * CH_EPI_WARPS) : "memory");
        if (cw == 0 && lane == 0) {
          __threadfence();
          asm volatile("fence.proxy.async;" ::: "memory");
          red_release_gpu_add(P.ctr + 2 + Q.ctr_base + k.by, 1);
        }
      }
      if (rec) {
        unsigned smid;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
        P.trace[(size_t)t * 8 + 6] = globaltimer_ns();
        P.trace[(size_t)t * 8 + 7] = smid;
      }
    }
  }
  __syncthreads();
  // the last CTA to leave resets queue + counters for the next launch / graph replay
  if (threadIdx.x == 0) {
    __threadfence();
    const int left = atomicAdd(P.ctr + 1, 1);
    if (left == (int)gridDim.x - 1) {
      __threadfence();
      for (int i = 0; i < P.n_ctr; ++i) P.ctr[i] = 0;
      __threadfence();
    }
  }
}

struct Chain {
  ChParams P;
  unsigned grid;
  size_t smem;
};

}  // namespace dlrm

extern "C" int dlrm_b200_gemm_chain_create(void* const* plans, const int* dep, const int* dep_on_k, int n,
                                           int32_t* counters, int64_t counters_len, void** chain_out) {
  using namespace dlrm;
  if (!plans || !dep || !dep_on_k || !counters || !chain_out) return set_error("gemm_chain_create: NULL argument");
  if (n < 1 || n > CH_MAX_PROBLEMS) return set_error("gemm_chain_create: n=%d (1..%d)", n, CH_MAX_PROBLEMS);
  Chain* c = new Chain();
  memset(&c->P, 0, sizeof(c->P));
  ChParams& P = c->P;
  long long total = 0, nctr = 0;
  uint32_t stage_bytes = 0;
  int max_bn = 32;
  for (int i = 0; i < n; ++i) {
    const TcPlan* p = static_cast<const TcPlan*>(plans[i]);
    if (!p) { delete c; return set_error("gemm_chain_create: plan %d is NULL", i); }
    if (p->bn != 32 && p->bn != 64 && p->bn != 128) { delete c; return set_error("gemm_chain_create: plan %d tile_n=%d", i, p->bn); }
    ChProblem& Q = P.p[i];
    Q.m[0] = p->tmAh; Q.m[1] = p->tmAl; Q.m[2] = p->tmBh; Q.m[3] = p->tmBl;
    Q.a = p->args;
    Q.bn = p->bn;
    Q.gx = (int)p->grid.x; Q.gy = (int)p->grid.y; Q.gz = (int)p->grid.z;
    Q.task_begin = (int)total;
    total += (long long)Q.gx * Q.gy * Q.gz;
    Q.ctr_base = (int)nctr;
    nctr += Q.gy;
    Q.dep = dep[i];
    Q.dep_on_k = dep_on_k[i] ? 1 : 0;
    Q.signal = 0;
    if (Q.dep >= i) { delete c; return set_error("gemm_chain_create: plan %d depends on plan %d (must be earlier)", i, Q.dep); }
    if (Q.dep >= 0) {
      ChProblem& Dp = P.p[Q.dep];
      if (Dp.gz != 1) { delete c; return set_error("gemm_chain_create: plan %d is split-K and cannot be a producer", Q.dep); }
      Dp.signal = 1;
      Q.dep_target = Dp.gx;
      // the rows this problem reads must be rows the producer writes
      const long long rows = Q.dep_on_k ? Q.a.K : Q.a.M;
      if (rows > Dp.a.M) { delete c; return set_error("gemm_chain_create: plan %d reads %lld rows, producer %d has %lld", i, rows, Q.dep, (long long)Dp.a.M); }
    }
    const uint32_t sb = (uint32_t)((Q.a.x3 ? 2 : 1) * (TC_BM * TC_BK * 2 + Q.bn * TC_BK * 2));
    stage_bytes = sb > stage_bytes ? sb : stage_bytes;
    max_bn = Q.bn > max_bn ? Q.bn : max_bn;
  }
  // groups (see ChGroup): maximal runs of single-split problems with equal m tiles, m-tile major
  {
    int gi = 0, i = 0;
    long long t0 = 0;
    const bool mmajor = get_tunable(TUNE_CHAIN_ORDER) == 2;   // measured slower (blocking claims): opt-in
    while (i < n) {
      int j = i + 1;
      // only row-linked problems (a task depends on ITS m tile of the producer) may be interleaved by m tile:
      // a problem that reduces over the batch (dep_on_k) needs ALL m tiles of its producer first
      if (mmajor && P.p[i].gz == 1 && !P.p[i].dep_on_k)
        while (j < n && P.p[j].gz == 1 && !P.p[j].dep_on_k && P.p[j].gy == P.p[i].gy) ++j;
      ChGroup& G = P.grp[gi++];
      G.task_begin = (int)t0; G.p0 = i; G.np = j - i; G.per_m = 0;
      for (int q = i; q < j; ++q) {
        G.per_m += P.p[q].gx;
        t0 += (long long)P.p[q].gx * P.p[q].gy * P.p[q].gz;
      }
      i = j;
    }
    P.ngroups = gi;
  }
  if (total <= 0 || total >= (1ll << 30)) { delete c; return set_error("gemm_chain_create: %lld tasks", total); }
  if (counters_len < 2 + nctr) { delete c; return set_error("gemm_chain_create: counters_len=%lld < %lld", (long long)counters_len, 2 + nctr); }
  P.n = n;
  P.total = (int)total;
  P.stage_bytes = stage_bytes;
  P.max_bn = max_bn;
  int budget_kb = get_tunable(TUNE_GEMM_SMEM_KB);
  if (budget_kb <= 0 || budget_kb > 200) budget_kb = 200;
  size_t ring_bytes = (size_t)budget_kb * 1024;
  if (ring_bytes > TC_MAX_SMEM - tc_extra_smem(max_bn, CH_HEAD)) ring_bytes = TC_MAX_SMEM - tc_extra_smem(max_bn, CH_HEAD);
  int stages = (int)(ring_bytes / stage_bytes);
  if (stages > 8) stages = 8;
  if (stages < 2) stages = 2;
  P.stages = stages;
  P.ctr = counters;
  P.n_ctr = (int)(2 + nctr);
  c->smem = (size_t)stages * stage_bytes + tc_extra_smem(max_bn, CH_HEAD);   // ring | barriers, task ring | accumulator | staging
  if (c->smem > (size_t)TC_MAX_SMEM) { delete c; return set_error("gemm_chain_create: %zu bytes of shared memory", c->smem); }
  int dev = 0, sms = 0;
  DLRM_CUDA(cudaGetDevice(&dev));
  DLRM_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  c->grid = (unsigned)(total < sms ? total : sms);
  *chain_out = c;
  return 0;
}

extern "C" int dlrm_b200_gemm_chain_info(void* chain, int* tasks, int* ctas, int* stages, int* smem_bytes) {
  using namespace dlrm;
  if (!chain) return set_error("gemm_chain_info: NULL chain");
  Chain* c = static_cast<Chain*>(chain);
  if (tasks) *tasks = c->P.total;
  if (ctas) *ctas = (int)c->grid;
  if (stages) *stages = c->P.stages;
  if (smem_bytes) *smem_bytes = (int)c->smem;
  return 0;
}

extern "C" int dlrm_b200_gemm_chain_set_trace(void* chain, uint64_t* trace) {
  using namespace dlrm;
  if (!chain) return set_error("gemm_chain_set_trace: NULL chain");
  static_cast<Chain*>(chain)->P.trace = reinterpret_cast<unsigned long long*>(trace);
  return 0;
}

extern "C" int dlrm_b200_gemm_chain_run(void* chain, void* stream) {
  using namespace dlrm;
  if (!chain) return set_error("gemm_chain_run: NULL chain");
  Chain* c = static_cast<Chain*>(chain);
  static bool configured = false;
  if (!configured) {
    DLRM_CUDA(cudaFuncSetAttribute(gemm_chain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_MAX_SMEM));
    configured = true;
  }
  (void)launch_chain(gemm_chain_kernel, dim3(c->grid), dim3(CH_THREADS), c->smem, static_cast<cudaStream_t>(stream), c->P);
  DLRM_CHECK_LAUNCH("gemm_chain_kernel");
  return 0;
}

extern "C" int dlrm_b200_gemm_chain_destroy(void* chain) {
  delete static_cast<dlrm::Chain*>(chain);
  return 0;
}
