// Persistent stream-K variant of the skinny weight-streaming GEMM (same math, tiles, epilogues and rounding points as
// gemm.cu; see there for the swap-AB / TMA / wgmma layout).
//
// Why: the HBM roofline is only reachable when ALL SMs stream, evenly, for the whole kernel.  Tile-granular grids
// (48 / 32 / 112 tiles for the Llama-3-8B projections, times a power-of-two split) leave SMs idle or double-loaded.
// Here the iteration space  units = n_tiles x k_blocks  is cut into one contiguous, equal share per CTA (one CTA per
// SM).  A CTA walks its share k-fastest; every change of tile closes a SEGMENT:
//   * a segment that covers a whole tile runs the fused epilogue directly;
//   * a segment that starts inside a tile (k > 0) is a CONTRIBUTION: its fp32 partial goes to a per-CTA slot of an
//     L2-resident workspace, then the tile's arrival counter is bumped (release);
//   * the segment that starts a tile (k == 0) but does not finish it makes this CTA the tile's FINISHER: it waits
//     for the contributions (they come from the next CTAs, which process them FIRST, so the wait is short and can
//     never deadlock: contributors never wait), adds them in CTA order (deterministic) and runs the epilogue.
// Roles: warps 0..3 are the MMA warpgroup (wgmma, both 64-row halves of the tile, fp32 accumulators in registers), warps
// 4..7 the epilogue, warp 8 the TMA producer.  The TMA producer streams across segment boundaries without draining; at
// the end of a segment the MMA warpgroup hands its accumulators to the epilogue through a shared-memory staging tile and
// goes on with the next segment, so the MMAs of the next segment overlap the epilogue of the previous one.  Weight tiles are prefetched
// before the programmatic-dependent-launch wait (they do not depend on the previous kernel), activations after it.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "gemm_common.cuh"

namespace eb {

constexpr int kSkEpiScratch = 16 * kBlockN * 2 + 64;  // RoPE exchange strip + flag word

struct StreamK {
  int tiles, num_kb;
  long units;
  float* ws;    // [grid][2][acc][MPAD][128] fp32 partial slots: [c][0] contribution of CTA c, [c][1] its own finisher partial
  int* flags;   // [tiles] arrival counters (self-resetting)
};

__device__ __forceinline__ long sk_begin(long units, int cta, int grid) { return (units * cta) / grid; }
// CTA that owns unit u under the partition above
__device__ __forceinline__ int sk_owner(long units, long u, int grid) {
  return static_cast<int>(((u + 1) * grid + units - 1) / units) - 1;
}
__device__ __forceinline__ int ld_acquire(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

template <typename T, int MPAD, int EPI>
__global__ void __launch_bounds__(kGemmThreads, 1)
skinny_gemm_streamk(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmW2,
                    const __grid_constant__ CUtensorMap tmX, const GemmParams p, const int stages, const StreamK sk) {
  constexpr bool kDual = (EPI == EPI_SWIGLU);
  constexpr int kAcc = kDual ? 2 : 1;
  constexpr int kStageBytes = stage_bytes(MPAD, EPI);

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  float* accbuf = reinterpret_cast<float*>(smem + stages * kStageBytes);  // [acc][MPAD][128] staged accumulators
  uint8_t* scratch = smem + stages * kStageBytes + acc_tile_bytes(MPAD, EPI);  // epilogue exchange strip (never aliased with the ring)
  uint8_t* ctrl = scratch + kSkEpiScratch;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>((reinterpret_cast<uintptr_t>(ctrl) + 7) & ~static_cast<uintptr_t>(7));
  uint64_t* empty_bar = full_bar + kMaxStages;
  uint64_t* acc_full = empty_bar + kMaxStages;   // the staging tile holds a segment's accumulators (128 arrivals)
  uint64_t* acc_empty = acc_full + 1;            // the epilogue has drained it

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int cta = blockIdx.x, grid = gridDim.x;
  const long u0 = sk_begin(sk.units, cta, grid), u1 = sk_begin(sk.units, cta + 1, grid);
  pdl_launch_dependents();

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmW);
    tma_prefetch_desc(&tmX);
    if (kDual) tma_prefetch_desc(&tmW2);
    for (int i = 0; i < stages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 1);
    }
    mbar_init(acc_full, 128);
    mbar_init(acc_empty, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == kTmaWarp) {
    // ===== TMA producer: one contiguous stream of units, oblivious to segment boundaries =====
    if (lane == 0) {
      const long n_units = u1 - u0;
      const int pre = static_cast<int>(n_units < stages ? n_units : stages);
      for (int j = 0; j < pre; ++j) {  // weights first: they do not depend on the previous kernel
        const long u = u0 + j;
        const int tile = static_cast<int>(u / sk.num_kb), kb = static_cast<int>(u % sk.num_kb);
        uint8_t* st = smem + j * kStageBytes;
        mbar_arrive_expect_tx(&full_bar[j], kStageBytes);
        tma_load_2d(st, &tmW, &full_bar[j], kb * kBlockK, tile * kBlockN, kEvictFirst);
        if (kDual) tma_load_2d(st + kWTileBytes, &tmW2, &full_bar[j], kb * kBlockK, tile * kBlockN, kEvictFirst);
      }
      pdl_wait();
      for (int j = 0; j < pre; ++j) {
        const int kb = static_cast<int>((u0 + j) % sk.num_kb);
        tma_load_2d(smem + j * kStageBytes + kWTileBytes * kAcc, &tmX, &full_bar[j], kb * kBlockK, 0, kEvictLast);
      }
      int s = (pre == stages) ? 0 : pre;
      uint32_t ph = (pre == stages) ? 1 : 0;
      for (long u = u0 + pre; u < u1; ++u) {
        const int tile = static_cast<int>(u / sk.num_kb), kb = static_cast<int>(u % sk.num_kb);
        mbar_wait_mma(&empty_bar[s], ph ^ 1);
        uint8_t* st = smem + s * kStageBytes;
        mbar_arrive_expect_tx(&full_bar[s], kStageBytes);
        tma_load_2d(st, &tmW, &full_bar[s], kb * kBlockK, tile * kBlockN, kEvictFirst);
        if (kDual) tma_load_2d(st + kWTileBytes, &tmW2, &full_bar[s], kb * kBlockK, tile * kBlockN, kEvictFirst);
        tma_load_2d(st + kWTileBytes * kAcc, &tmX, &full_bar[s], kb * kBlockK, 0, kEvictLast);
        if (++s == stages) {
          s = 0;
          ph ^= 1;
        }
      }
    }
  } else if (warp < 4) {
    // ===== MMA warpgroup: one segment at a time, accumulators (both 64-row halves) in registers =====
    int s = 0;
    uint32_t ph = 0;
    int seg = 0;
    long u = u0;
    while (u < u1) {
      const int kb_lo = static_cast<int>(u % sk.num_kb);
      const long rem = u1 - u;
      const int kb_hi = static_cast<int>((sk.num_kb - kb_lo) < rem ? sk.num_kb : kb_lo + rem);
      float acc[2][MPAD / 2], acc2[2][kDual ? MPAD / 2 : 1];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int i = 0; i < MPAD / 2; ++i) acc[h][i] = 0.f;
#pragma unroll
        for (int i = 0; i < (kDual ? MPAD / 2 : 1); ++i) acc2[h][i] = 0.f;
      }
      int prev = -1;
      for (int kb = kb_lo; kb < kb_hi; ++kb) {
        mbar_wait_mma(&full_bar[s], ph);
        const uint32_t st = smem_u32(smem + s * kStageBytes);
        const uint64_t b_desc = make_kmajor_sw128_desc(st + kWTileBytes * kAcc);
        wgmma_fence();
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          wgmma_kblock<T, MPAD>(acc[h], make_kmajor_sw128_desc(st + h * (kWTileBytes / 2)), b_desc);
          if constexpr (kDual) wgmma_kblock<T, MPAD>(acc2[h], make_kmajor_sw128_desc(st + kWTileBytes + h * (kWTileBytes / 2)), b_desc);
        }
        wgmma_commit();
        wgmma_wait<1>();  // the previous k-block's MMAs have retired: its slot can be refilled
        if (prev >= 0 && threadIdx.x == 0) mbar_arrive(&empty_bar[prev]);
        prev = s;
        if (++s == stages) {
          s = 0;
          ph ^= 1;
        }
      }
      wgmma_wait<0>();
      if (prev >= 0 && threadIdx.x == 0) mbar_arrive(&empty_bar[prev]);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        wgmma_fence_acc(acc[h]);
        wgmma_fence_acc(acc2[h]);
      }
      mbar_wait_mma(acc_empty, (seg & 1) ^ 1);  // the epilogue has drained the staging tile (first use passes)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        wgmma_store_acc<MPAD>(acc[h], accbuf, kBlockN, h * 64);
        if constexpr (kDual) wgmma_store_acc<MPAD>(acc2[h], accbuf + MPAD * kBlockN, kBlockN, h * 64);
      }
      mbar_arrive(acc_full);
      u += kb_hi - kb_lo;
      ++seg;
    }
  } else {
    // ===== epilogue warps (thread <-> weight row quad * 32 + lane) =====
    const int quad = warp & 3;
    const int row = quad * 32 + lane;
    pdl_wait();
    const int m_valid = valid_rows(p);
    int* flag_word = reinterpret_cast<int*>(scratch + 16 * kBlockN * 2);
    int seg = 0;
    long u = u0;
    while (u < u1) {
      const int tile = static_cast<int>(u / sk.num_kb);
      const int kb_lo = static_cast<int>(u % sk.num_kb);
      const long rem = u1 - u;
      const int kb_hi = static_cast<int>((sk.num_kb - kb_lo) < rem ? sk.num_kb : kb_lo + rem);
      const bool whole = (kb_lo == 0 && kb_hi == sk.num_kb);
      mbar_wait_mma(acc_full, seg & 1);
      auto load_chunk = [&](int c, float(&acc)[16], float(&acc2)[16]) {
        acc_ld16(accbuf, kBlockN, row, c * 16, acc);
        if constexpr (kDual) acc_ld16(accbuf + MPAD * kBlockN, kBlockN, row, c * 16, acc2);
      };
      auto release_acc = [&]() {
        epi_bar();
        if (row == 0) mbar_arrive(acc_empty);
      };
      float acc[16], acc2[16];
      if (whole) {
#pragma unroll 1
        for (int c = 0; c < MPAD / 16; ++c) {
          if (c * 16 >= m_valid) break;
          load_chunk(c, acc, acc2);
          final_chunk<T, EPI>(p, acc, acc2, c * 16, m_valid, row, tile, scratch);
        }
        release_acc();
      } else {
        // park this segment's fp32 partial in one of the CTA's two workspace slots (a CTA can be contributor of its
        // first tile and finisher of its last one; the two partials must not share storage)
        constexpr long kSlot = static_cast<long>(kAcc) * MPAD * kBlockN;
        float* slot = sk.ws + (static_cast<long>(cta) * 2 + (kb_lo > 0 ? 0 : 1)) * kSlot;
#pragma unroll 1
        for (int c = 0; c < MPAD / 16; ++c) {
          if (c * 16 >= m_valid) break;
          load_chunk(c, acc, acc2);
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            __stcg(slot + (c * 16 + j) * kBlockN + row, acc[j]);
            if constexpr (kDual) __stcg(slot + (MPAD + c * 16 + j) * kBlockN + row, acc2[j]);
          }
        }
        release_acc();
        if (kb_lo > 0) {
          // contribution: publish and move on (never waits)
          __threadfence();
          epi_bar();
          if (row == 0) atomicAdd(sk.flags + tile, 1);
        } else {
          // finisher: wait for the CTAs that hold the rest of this tile's k range, add in CTA order, run the epilogue
          const int last = sk_owner(sk.units, static_cast<long>(tile) * sk.num_kb + sk.num_kb - 1, grid);
          const int expected = last - cta;
          if (row == 0) {
            uint32_t spins = 0;
            while (ld_acquire(sk.flags + tile) < expected) {
              if (++spins > (1u << 26)) __trap();  // no printf in a wgmma kernel (see mbar_wait_mma)
            }
            sk.flags[tile] = 0;  // self-reset for the next launch
          }
          epi_bar();
          __threadfence();
#pragma unroll 1
          for (int c = 0; c < MPAD / 16; ++c) {
            if (c * 16 >= m_valid) break;
#pragma unroll
            for (int j = 0; j < 16; ++j) acc[j] = acc2[j] = 0.f;
            for (int peer = cta; peer <= last; ++peer) {
              const float* ps = sk.ws + (static_cast<long>(peer) * 2 + (peer == cta ? 1 : 0)) * kSlot;
#pragma unroll
              for (int j = 0; j < 16; ++j) {
                if (c * 16 + j < m_valid) {
                  acc[j] += __ldcg(ps + (c * 16 + j) * kBlockN + row);
                  if constexpr (kDual) acc2[j] += __ldcg(ps + (MPAD + c * 16 + j) * kBlockN + row);
                }
              }
            }
            final_chunk<T, EPI>(p, acc, acc2, c * 16, m_valid, row, tile, scratch);
          }
        }
      }
      u += kb_hi - kb_lo;
      ++seg;
    }
    (void)flag_word;
  }
}

// ------------------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------------------
static int sk_grid_cap() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("EB200_SK_CTAS");  // tuning knob (default: one CTA per SM)
    v = e ? atoi(e) : 0;
    if (v < 1) v = 0;
  }
  return v ? v : device_sm_count();
}
static int sk_smem_kb() {
  static int v = 0;
  if (!v) {
    const char* e = getenv("EB200_SK_SMEM_KB");
    v = e ? atoi(e) : 200;
    if (v < 48) v = 48;
    if (v > 216) v = 216;
  }
  return v;
}

size_t streamk_ws_bytes() { return static_cast<size_t>(device_sm_count()) * 2 * 2 * 64 * kBlockN * 4 + 1024; }

template <typename T, int MPAD, int EPI>
static int launch_sk_one(const CUtensorMap* tmW, const CUtensorMap* tmW2, const CUtensorMap* tmX, const GemmParams& p,
                         float* ws, int* flags, cudaStream_t s) {
  auto kern = skinny_gemm_streamk<T, MPAD, EPI>;
  StreamK sk;
  sk.tiles = (p.N + kBlockN - 1) / kBlockN;
  sk.num_kb = (p.K + kBlockK - 1) / kBlockK;
  sk.units = static_cast<long>(sk.tiles) * sk.num_kb;
  sk.ws = ws;
  sk.flags = flags;
  long g = sk.units / 2;  // at least two k-blocks of work per CTA
  if (g < 1) g = 1;
  if (g > sk_grid_cap()) g = sk_grid_cap();
  if (g > device_sm_count()) g = device_sm_count();  // workspace slots per CTA; finisher waits need every CTA resident
  constexpr int kFixed = acc_tile_bytes(MPAD, EPI) + kSkEpiScratch + 512 + 1024;
  int stages = (sk_smem_kb() * 1024 - kFixed) / stage_bytes(MPAD, EPI);
  if (stages > kMaxStages) stages = kMaxStages;
  if (stages < 2) stages = 2;
  const int smem = stages * stage_bytes(MPAD, EPI) + kFixed;
  if (smem > 220 * 1024) return static_cast<int>(cudaErrorInvalidValue);
  static bool configured_dev[64] = {};  // per device (the attribute is per device) and per instantiation
  const int cur_dev = current_device_index();
  if (cur_dev < 0) return static_cast<int>(cudaErrorInvalidDevice);
  if (!configured_dev[cur_dev]) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
    if (e != cudaSuccess) return static_cast<int>(e);
    configured_dev[cur_dev] = true;
  }
  return static_cast<int>(launch_k(kern, dim3(static_cast<unsigned>(g)), dim3(kGemmThreads), static_cast<size_t>(smem), s, 1, *tmW,
                                   tmW2 ? *tmW2 : *tmW, *tmX, p, stages, sk));
}

template <typename T, int MPAD>
static int launch_sk_epi(int epi, const CUtensorMap* a, const CUtensorMap* b, const CUtensorMap* c, const GemmParams& p, float* ws,
                         int* flags, cudaStream_t s) {
  switch (epi) {
    case EPI_STORE: return launch_sk_one<T, MPAD, EPI_STORE>(a, b, c, p, ws, flags, s);
    case EPI_RESIDUAL: return launch_sk_one<T, MPAD, EPI_RESIDUAL>(a, b, c, p, ws, flags, s);
    case EPI_SWIGLU: return launch_sk_one<T, MPAD, EPI_SWIGLU>(a, b, c, p, ws, flags, s);
    case EPI_QKV_ROPE: return launch_sk_one<T, MPAD, EPI_QKV_ROPE>(a, b, c, p, ws, flags, s);
    case EPI_PARTIAL_F32: return launch_sk_one<T, MPAD, EPI_PARTIAL_F32>(a, b, c, p, ws, flags, s);
    case EPI_SWIGLU_IL: return launch_sk_one<T, MPAD, EPI_SWIGLU_IL>(a, b, c, p, ws, flags, s);
  }
  return static_cast<int>(cudaErrorInvalidValue);
}

int launch_gemm_streamk(int dtype, int mpad, int epi, const CUtensorMap* tmW, const CUtensorMap* tmW2, const CUtensorMap* tmX,
                        const GemmParams& p_in, float* ws, int* flags, cudaStream_t s) {
  GemmParams p = p_in;
  if (p.m_rows > mpad || !ws || !flags) return static_cast<int>(cudaErrorInvalidValue);
  if (epi == EPI_SWIGLU || epi == EPI_SWIGLU_IL) {
    p.silu_lut = silu_lut(dtype, s);
    if (!p.silu_lut) return static_cast<int>(cudaErrorNotReady);
  }
  if (dtype == DT_BF16) {
    if (mpad == 16) return launch_sk_epi<__nv_bfloat16, 16>(epi, tmW, tmW2, tmX, p, ws, flags, s);
    if (mpad == 64) return launch_sk_epi<__nv_bfloat16, 64>(epi, tmW, tmW2, tmX, p, ws, flags, s);
  } else if (dtype == DT_FP16) {
    if (mpad == 16) return launch_sk_epi<__half, 16>(epi, tmW, tmW2, tmX, p, ws, flags, s);
    if (mpad == 64) return launch_sk_epi<__half, 64>(epi, tmW, tmW2, tmX, p, ws, flags, s);
  }
  return static_cast<int>(cudaErrorInvalidValue);
}

}  // namespace eb
