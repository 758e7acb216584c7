// Body of the wgmma GEMM CTA (see gemm_tc.cu for the design).  Textually included by the kernels
// that share it; the including kernel provides, as macros or locals:
//   TCB_BX / TCB_BY / TCB_BZ        tile coordinates (n tile, m tile, k split)
//   TCB_MAP_AH / _AL / _BH / _BL    const CUtensorMap* of the four operand maps (kernel-parameter space)
//   g       const TcArgs&           problem description
//   stages  int                     depth of the operand ring
//   BN      template int            tile width
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr uint32_t A_BYTES = TC_A_BYTES;
  constexpr uint32_t B_BYTES = BN * TC_BK * 2;
  const uint32_t stage_bytes = (g.x3 ? 2u : 1u) * (A_BYTES + B_BYTES);
  const size_t ring_bytes = tc_ring_bytes((size_t)stages * stage_bytes, BN);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + ring_bytes);
  // bars[0..stages) full, [stages..2*stages) empty
  float* acc = reinterpret_cast<float*>(smem);   // the ring, once every TMA load has landed and every wgmma retired
  uint8_t* epi = smem + ring_bytes + 256;

  pdl_launch_dependents();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = TCB_BY * TC_BM, n0 = TCB_BX * BN;
  const int kb0 = TCB_BZ * g.kb_per_split;
  const int kb1 = min(g.num_kb, kb0 + g.kb_per_split);
  const uint32_t smem_base = smem_u32(smem);
  const uint32_t bar_base = smem_u32(bars);

  if (threadIdx.x == 0) {
    for (int s = 0; s < stages; ++s) {
      mbar_init(bar_base + 8 * s, 1);
      mbar_init(bar_base + 8 * (stages + s), TC_EPI_WARPS);   // one arrive per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();   // barriers are set up; global memory is first touched below

  if (warp == 0) {
    // ------------------------------------------------------------------ TMA producer
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(bar_base + 8 * (stages + stage), phase ^ 1);
        const uint32_t full = bar_base + 8 * stage;
        mbar_expect_tx(full, stage_bytes);
        uint32_t dst = smem_base + stage * stage_bytes;
        const int k0 = kb * TC_BK;
        // A tile(s)
        for (int part = 0; part < (g.x3 ? 2 : 1); ++part) {
          const CUtensorMap* map = part ? TCB_MAP_AL : TCB_MAP_AH;
          if (!g.a_mn) {
            tma_load_2d(dst, map, full, k0, m0);                       // box {64 k, 128 m}
          } else {
            tma_load_2d(dst, map, full, m0, k0);                       // box {64 m, 64 k} x 2
            tma_load_2d(dst + A_BYTES / 2, map, full, m0 + 64, k0);
          }
          dst += A_BYTES;
        }
        for (int part = 0; part < (g.x3 ? 2 : 1); ++part) {
          const CUtensorMap* map = part ? TCB_MAP_BL : TCB_MAP_BH;
          if (!g.b_mn) {
            tma_load_2d(dst, map, full, k0, n0);                       // box {64 k, BN n}
          } else {
#pragma unroll
            for (int h = 0; h < BN / 64; ++h) tma_load_2d(dst + h * 8192, map, full, n0 + 64 * h, k0);
          }
          dst += B_BYTES;
        }
        if (++stage == stages) { stage = 0; phase ^= 1; }
      }
    }
  } else if (warp >= TC_CONSUMER_WARP0) {
    // ------------------------------------------------------------------ wgmma consumers + epilogue
    const int cw = warp - TC_CONSUMER_WARP0;
    float d[BN / 2];
    int stage = 0;
    uint32_t phase = 0;
    tc_mainloop<BN>(d, g, smem_base, stage_bytes, stages, bar_base, bar_base + 8 * stages, kb0, kb1, stage, phase,
                    cw >> 2, lane);
    // both warpgroups' wgmmas have retired (every operand the producer loaded was waited for): the ring is free
    asm volatile("bar.sync 2, %0;" ::"n"(32 * TC_EPI_WARPS) : "memory");
    tc_stage_acc<BN>(d, acc, cw, lane);
    asm volatile("bar.sync 1, %0;" ::"n"(32 * TC_EPI_WARPS) : "memory");
    tc_epilogue_tile(g, BN, m0, n0, TCB_BZ, acc, cw & 3, lane, epi + (size_t)cw * TC_EPI_WARP_BYTES, cw >> 2,
                     TC_EPI_WARPS / 4);
  }
