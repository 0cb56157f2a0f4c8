// lm_head GEMM for sm_90a as one persistent launch of one CTA per SM (ea_model.py:190 + utils.py:362).
//
// CTA c owns the whole 128-row vocabulary tiles c, c+G, c+2G, ... (G = SM count), so no tile is split over the reduction
// dimension and nothing is reduced across CTAs:
//   * the WEIGHT producer (one lane) streams the CTA's weight tiles into a shared-memory ring with TMA; it needs nothing from
//     the previous kernel, so under PDL it starts while that kernel drains;
//   * the ACTIVATION producer (another lane) waits for the previous kernel and TMA-loads the X tile of every k-block behind
//     the already-resident W tiles;
//   * an MMA warpgroup accumulates each tile with wgmma in registers and hands it to the epilogue warps through a
//     shared-memory staging tile, while the next tile's MMAs run;
//   * the epilogue warps finish the tile in one of two ways:
//       FIN_ARGMAX        per-row (max, first index) of the tile's 128 logits (rounded to the model dtype first), written to
//                         a [tiles][64] table; after a grid-wide arrival counter the first rows CTAs merge the table per row
//                         (and, vocabulary-parallel, exchange the pairs with the peers): the 15.4 MB logits round trip and
//                         the arg-max launch disappear (verify pass);
//       FIN_STORE_DIRECT  T(acc [+ bias]) stored as logits (sampling path).
// The counters reset themselves when the last CTA leaves, so the launch can be replayed from a CUDA graph.
#include <algorithm>

#include "gemm_common.cuh"

namespace eb {

constexpr int kChainThreads = 320;   // warps 0-3 MMA, warps 4-7 epilogue, warp 8 W producer, warp 9 X producer
constexpr int kChainMaxStages = 12;
constexpr int kChainCtrlBytes = 8192;  // mbarriers + arg-max pairs; the staging tile follows
constexpr int kSyncPartials = 0;     // CTAs that have written all their per-tile arg-max pairs
constexpr int kSyncExit = 1;         // CTAs that have left (the last one resets both counters)

// ------------------------------------------------------------------------------------------------------------
// small device helpers
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_gpu_add(int* p, int v) {
  asm volatile("red.release.gpu.global.add.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// Bounded spin: a mis-programmed launch traps (CUDA error on the host) instead of hanging the GPU.  No printf in this kernel:
// ptxas serialises every wgmma of a kernel in which a call may run while MMAs are in flight (see mbar_wait_mma).
__device__ __forceinline__ void spin_until_ge(const int* p, int target) {
  uint32_t n = 0;
  while (ld_acquire_gpu(p) < target) {
    __nanosleep(32);
    if (++n > (1u << 23)) __trap();
  }
}
__device__ __forceinline__ void chain_epi_bar() { asm volatile("bar.sync 1, 128;" ::: "memory"); }
// ---- system scope (other GPUs over NVLink peer memory) ----
__device__ __forceinline__ int ld_acquire_sys(const int* p) {
  int v;
  asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(int* p, int v) { asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ unsigned long long chain_gtimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// wait for a peer GPU: the peers run the same launch sequence but are not lock-stepped (host launch skew in eager mode), so the
// bound is wall-clock (20 s), not an iteration count
__device__ __forceinline__ void spin_until_ge_sys(const int* p, int target) {
  unsigned long long t0 = 0;
  uint32_t n = 0;
  while (ld_acquire_sys(p) - target < 0) {
    __nanosleep(64);
    if ((++n & 4095u) == 0) {
      const unsigned long long now = chain_gtimer();
      if (!t0) t0 = now;
      if (now - t0 > 20000000000ull) __trap();
    }
  }
}
__device__ __forceinline__ bool better(float v, int i, float bv, int bi) { return v > bv || (v == bv && i < bi); }

// merge the per-tile (max, first index) pairs of row m (torch.argmax: first maximal index; ea_model.py:190 + utils.py:362)
__device__ __forceinline__ void finish_argmax(const ChainPhase& ph, const ChainTP& tp, int epoch, int ntiles, int m, int etid, float* sval,
                                              int* sidx) {
  float bv = -INFINITY;
  int bi = 0x7fffffff;
  for (int t = etid; t < ntiles; t += 128) {
    const float v = __ldcg(ph.tile_val + static_cast<long>(t) * 64 + m);
    const int i = __ldcg(ph.tile_idx + static_cast<long>(t) * 64 + m);
    if (better(v, i, bv, bi)) {
      bv = v;
      bi = i;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (better(ov, oi, bv, bi)) {
      bv = ov;
      bi = oi;
    }
  }
  if ((etid & 31) == 0) {
    sval[etid >> 5] = bv;
    sidx[etid >> 5] = bi;
  }
  chain_epi_bar();
  if (etid == 0) {
    for (int w = 1; w < 4; ++w)
      if (better(sval[w], sidx[w], bv, bi)) {
        bv = sval[w];
        bi = sidx[w];
      }
    if (tp.size > 1) {
      // vocabulary-parallel lm_head: exchange the (value, global index) pairs of the shards; lowest index wins ties, like one GPU
      bi += ph.idx_offset;
      for (int r = 0; r < tp.size; ++r) {
        float* slot = reinterpret_cast<float*>(tp.win[r] + tp.am_off) + (static_cast<long>(tp.rank) * 64 + m) * 2;
        slot[0] = bv;
        reinterpret_cast<int*>(slot)[1] = bi;
        __threadfence_system();
        st_release_sys(reinterpret_cast<int*>(tp.win[r] + tp.am_off + static_cast<long>(kMaxTp) * 64 * 8) + tp.rank * 64 + m, epoch);
      }
      const int* flags = reinterpret_cast<const int*>(tp.win[tp.rank] + tp.am_off + static_cast<long>(kMaxTp) * 64 * 8);
      const float* mine = reinterpret_cast<const float*>(tp.win[tp.rank] + tp.am_off);
      bv = -INFINITY;
      bi = 0x7fffffff;
      for (int src = 0; src < tp.size; ++src) {
        spin_until_ge_sys(flags + src * 64 + m, epoch);
        const float v = __ldcg(mine + (static_cast<long>(src) * 64 + m) * 2);
        const int i = __ldcg(reinterpret_cast<const int*>(mine + (static_cast<long>(src) * 64 + m) * 2) + 1);
        if (better(v, i, bv, bi)) {
          bv = v;
          bi = i;
        }
      }
    }
    ph.out_idx[m] = bi;
  }
  chain_epi_bar();
}

// ------------------------------------------------------------------------------------------------------------
// the kernel
// ------------------------------------------------------------------------------------------------------------
template <typename T, int MPAD>
__global__ void __launch_bounds__(kChainThreads, 1)
gemm_chain_kernel(const __grid_constant__ ChainMaps maps, const __grid_constant__ ChainArgs args, const int stages) {
  constexpr int kXBytes = x_tile_bytes(MPAD);
  constexpr int kStageBytes = kWTileBytes + kXBytes;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* ctrl = smem + stages * kStageBytes;
  uint64_t* fullW = reinterpret_cast<uint64_t*>(ctrl);
  uint64_t* fullX = fullW + kChainMaxStages;
  uint64_t* empty = fullX + kChainMaxStages;
  uint64_t* acc_full = empty + kChainMaxStages;   // the staging tile holds a tile's accumulators (128 arrivals)
  uint64_t* acc_empty = acc_full + 1;             // the epilogue has drained it
  float* accbuf = reinterpret_cast<float*>(ctrl + kChainCtrlBytes);  // [MPAD][128] staged fp32 accumulators
  float* sval = reinterpret_cast<float*>(ctrl + 1024);              // [4][64]
  int* sidx = reinterpret_cast<int*>(ctrl + 1024 + 4 * 64 * 4);     // [4][64]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int cta = blockIdx.x, G = gridDim.x;
  const ChainPhase& ph = args.ph;
  const int nkb = (ph.K + kBlockK - 1) / kBlockK;
  const int ntiles = (ph.N + kBlockN - 1) / kBlockN;
  pdl_launch_dependents();

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&maps.w);
    tma_prefetch_desc(&maps.x);
    for (int i = 0; i < stages; ++i) {
      mbar_init(&fullW[i], 1);
      mbar_init(&fullX[i], 1);
      mbar_init(&empty[i], 1);
    }
    mbar_init(acc_full, 128);
    mbar_init(acc_empty, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ===== weight producer: weights depend on no earlier kernel, so no PDL wait =====
    if (lane == 0) {
      int s = 0;
      uint32_t par = 0;
      for (int t = cta; t < ntiles; t += G) {
        for (int kb = 0; kb < nkb; ++kb) {
          mbar_wait_mma(&empty[s], par ^ 1);
          mbar_arrive_expect_tx(&fullW[s], kWTileBytes);
          tma_load_2d(smem + s * kStageBytes, &maps.w, &fullW[s], kb * kBlockK, t * kBlockN, kEvictFirst);
          if (++s == stages) {
            s = 0;
            par ^= 1;
          }
        }
      }
    }
  } else if (warp == 9) {
    // ===== activation producer: the X operand is the previous kernel's output =====
    if (lane == 0) {
      pdl_wait();
      int s = 0;
      uint32_t par = 0;
      for (int t = cta; t < ntiles; t += G) {
        for (int kb = 0; kb < nkb; ++kb) {
          mbar_wait_mma(&empty[s], par ^ 1);
          mbar_arrive_expect_tx(&fullX[s], kXBytes);
          tma_load_2d(smem + s * kStageBytes + kWTileBytes, &maps.x, &fullX[s], kb * kBlockK, 0, kEvictLast);
          if (++s == stages) {
            s = 0;
            par ^= 1;
          }
        }
      }
    }
  } else if (warp < 4) {
    // ===== MMA warpgroup: both 64-row halves of each tile, fp32 accumulators in registers =====
    const bool lead = threadIdx.x == 0;
    int s = 0;
    uint32_t par = 0, seg = 0;
    for (int t = cta; t < ntiles; t += G) {
      float acc[2][MPAD / 2];
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < MPAD / 2; ++i) acc[h][i] = 0.f;
      int prev = -1;
      for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait_mma(&fullW[s], par);
        mbar_wait_mma(&fullX[s], par);
        const uint32_t st = smem_u32(smem + s * kStageBytes);
        const uint64_t b_desc = make_kmajor_sw128_desc(st + kWTileBytes);
        wgmma_fence();
#pragma unroll
        for (int h = 0; h < 2; ++h) wgmma_kblock<T, MPAD>(acc[h], make_kmajor_sw128_desc(st + h * (kWTileBytes / 2)), b_desc);
        wgmma_commit();
        wgmma_wait<1>();  // the previous k-block's MMAs have retired: its slot can be refilled
        if (prev >= 0 && lead) mbar_arrive(&empty[prev]);
        prev = s;
        if (++s == stages) {
          s = 0;
          par ^= 1;
        }
      }
      wgmma_wait<0>();
      if (prev >= 0 && lead) mbar_arrive(&empty[prev]);
#pragma unroll
      for (int h = 0; h < 2; ++h) wgmma_fence_acc(acc[h]);
      mbar_wait_mma(acc_empty, (seg & 1) ^ 1);  // the epilogue has drained the staging tile (first use passes)
#pragma unroll
      for (int h = 0; h < 2; ++h) wgmma_store_acc<MPAD>(acc[h], accbuf, kBlockN, h * 64);
      mbar_arrive(acc_full);
      ++seg;
    }
  } else if (warp >= 4) {
    // ===== epilogue warps (thread <-> weight row quad * 32 + lane) =====
    const int quad = warp & 3;
    const int etid = threadIdx.x - 128;
    const int row = quad * 32 + lane;  // weight row inside the tile
    pdl_wait();
    const int m_valid = args.m_idx >= 0 ? min(args.m_rows, ld_dep(args.st + args.m_idx)) : args.m_rows;
    if (args.timing && cta == 0 && etid == 0) *reinterpret_cast<volatile unsigned long long*>(args.timing + 2) = chain_gtimer();
    const int tp_epoch0 = args.tp.size > 1 ? ld_dep(args.tp.epoch) : 0;
    uint32_t seg = 0;
    for (int t = cta; t < ntiles; t += G) {
      mbar_wait_mma(acc_full, seg & 1);
      if (ph.fin == FIN_STORE_DIRECT) {
        GemmParams gp;
        gp.N = ph.N;
        gp.out = ph.out;
        gp.ld_out = ph.ld_out;
        gp.bias = ph.bias;
        float acc[16], acc2[16];
#pragma unroll 1
        for (int c = 0; c < MPAD / 16; ++c) {
          if (c * 16 >= m_valid) break;
          float r[16];
          acc_ld16(accbuf, kBlockN, row, c * 16, r);
#pragma unroll
          for (int j = 0; j < 16; ++j) acc[j] = acc2[j] = r[j];
          final_chunk<T, EPI_STORE>(gp, acc, acc2, c * 16, m_valid, row, t, nullptr);
        }
      } else {  // FIN_ARGMAX: per-row (max, first index) of this tile's 128 vocabulary rows
        const int n = t * kBlockN + row;
#pragma unroll 1
        for (int c = 0; c < MPAD / 16; ++c) {
          if (c * 16 >= m_valid) break;
          float r[16];
          acc_ld16(accbuf, kBlockN, row, c * 16, r);
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            float v = (n < ph.N) ? rnd<T>(r[j]) : -INFINITY;  // the logits tensor is model dtype (ea_model.py:190)
            int idx = n;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
              const float ov = __shfl_xor_sync(0xffffffffu, v, o);
              const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
              if (better(ov, oi, v, idx)) {
                v = ov;
                idx = oi;
              }
            }
            if (lane == 0) {
              sval[quad * 64 + c * 16 + j] = v;
              sidx[quad * 64 + c * 16 + j] = idx;
            }
          }
        }
        chain_epi_bar();
        if (etid < m_valid) {
          float bv = sval[etid];
          int bi = sidx[etid];
#pragma unroll
          for (int w = 1; w < 4; ++w)
            if (better(sval[w * 64 + etid], sidx[w * 64 + etid], bv, bi)) {
              bv = sval[w * 64 + etid];
              bi = sidx[w * 64 + etid];
            }
          __stcg(ph.tile_val + static_cast<long>(t) * 64 + etid, bv);
          __stcg(ph.tile_idx + static_cast<long>(t) * 64 + etid, bi);
        }
      }
      chain_epi_bar();  // every epilogue thread is done with the staging tile (and with sval/sidx)
      if (etid == 0) mbar_arrive(acc_empty);
      ++seg;
    }
    if (ph.fin == FIN_ARGMAX) {
      // ---- all tile results of this CTA are written; once every CTA's are, the first m_valid CTAs merge one row each ----
      __threadfence();
      chain_epi_bar();
      if (etid == 0) red_release_gpu_add(args.sync + kSyncPartials, 1);
      if (cta < m_valid) {
        if (etid == 0) spin_until_ge(args.sync + kSyncPartials, G);
        chain_epi_bar();
        __threadfence();
        for (int m = cta; m < m_valid; m += G) finish_argmax(ph, args.tp, tp_epoch0 + 1, ntiles, m, etid, sval, sidx);
      }
    }
  }

  __syncthreads();
  if (threadIdx.x == 0) {
    pdl_wait();  // (returns at once: the epilogue warps already waited) keeps every global access of this thread behind the wait
    // the last CTA to leave resets the counters for the next launch on this stream (nobody polls after its own exit ticket)
    const int old = atomicAdd(args.sync + kSyncExit, 1);
    if (old == G - 1) {
      args.sync[kSyncPartials] = 0;
      args.sync[kSyncExit] = 0;
      if (args.tp.size > 1) *args.tp.epoch += 1;
      if (args.timing) {
        volatile unsigned long long* tm = args.timing;
        const unsigned long long t0 = tm[2], t1 = chain_gtimer();
        if (t0 != 0 && t1 > t0) {
          tm[0] += t1 - t0;
          tm[1] += 1;
        }
        tm[2] = 0;
      }
      __threadfence();
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------------------
static int chain_grid_for(int dev) {
  static int sms[64] = {};
  if (dev < 0 || dev >= 64) return 0;
  if (!sms[dev]) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0;
    sms[dev] = n;
  }
  return sms[dev];
}
static int current_device() {
  int dev = 0;
  return cudaGetDevice(&dev) == cudaSuccess ? dev : -1;
}
bool chain_phase_ok(int N, int K) { return chain_grid_for(current_device()) > 0 && N >= 1 && K >= 8 && K % 8 == 0; }

template <typename T, int MPAD> static int launch_chain_t(const ChainMaps& maps, const ChainArgs& a, cudaStream_t s) {
  auto kern = gemm_chain_kernel<T, MPAD>;
  const int dev = current_device();
  const int G = chain_grid_for(dev);
  if (G <= 0) return static_cast<int>(cudaErrorInvalidDevice);
  constexpr int kStageBytes = kWTileBytes + x_tile_bytes(MPAD);
  constexpr int kAccBytes = MPAD * kBlockN * 4;
  const int max_smem = 227 * 1024;
  const int stages = std::min(kChainMaxStages, (max_smem - 1024 - kChainCtrlBytes - kAccBytes) / kStageBytes);
  const size_t smem = static_cast<size_t>(stages) * kStageBytes + kChainCtrlBytes + kAccBytes + 1024;
  static bool configured[64] = {};  // per device (and per instantiation: this is a template)
  if (!configured[dev]) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem);
    if (e != cudaSuccess) return static_cast<int>(e);
    configured[dev] = true;
  }
  return static_cast<int>(launch_k(kern, dim3(G), dim3(kChainThreads), smem, s, 1, maps, a, stages));
}

int launch_gemm_chain(int dtype, int mpad, const ChainMaps& maps, const ChainArgs& args, cudaStream_t s) {
  const ChainPhase& ph = args.ph;
  if (args.m_rows < 1 || args.m_rows > mpad || !args.sync || !chain_phase_ok(ph.N, ph.K) ||
      (ph.fin != FIN_ARGMAX && ph.fin != FIN_STORE_DIRECT))
    return static_cast<int>(cudaErrorInvalidValue);
  if (dtype == DT_BF16) {
    if (mpad == 16) return launch_chain_t<__nv_bfloat16, 16>(maps, args, s);
    if (mpad == 64) return launch_chain_t<__nv_bfloat16, 64>(maps, args, s);
  } else if (dtype == DT_FP16) {
    if (mpad == 16) return launch_chain_t<__half, 16>(maps, args, s);
    if (mpad == 64) return launch_chain_t<__half, 64>(maps, args, s);
  }
  return static_cast<int>(cudaErrorInvalidValue);
}

}  // namespace eb
