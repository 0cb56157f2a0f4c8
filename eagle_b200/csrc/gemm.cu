// Skinny-M weight-streaming GEMM for sm_90a:  Y[m, n] = sum_k X[m, k] * W[n, k],  m <= MPAD in {16, 64, 256}.
//
// This is the dominant kernel of the draft -> verify -> accept cycle: at batch 1 every projection of the target
// verify pass (60 tree rows) and of the draft head (10 rows) is HBM-bound on its weight matrix, so the job of the
// kernel is to stream W once at HBM speed and keep the tensor pipe off the critical path.
//
//   * swap-AB: the 128 weight rows of a tile are the wgmma M dimension, the (padded) activation rows are wgmma N,
//     so a tile is two wgmma.m64nMPADk16 (one per MMA warpgroup) per 32 bytes of K.
//   * W and X tiles (64 K-elements = 128 B rows, SWIZZLE_128B) are staged by TMA into a multi-stage shared-memory
//     ring (mbarrier full/empty pairs); weights carry an L2 evict-first hint, activations evict-last.
//   * one producer lane (warp 8) issues TMA, two MMA warpgroups (warps 0..7) issue wgmma and hold the fp32 accumulators in
//     registers; at the end they park them in shared memory and warpgroup 0 runs the epilogue (thread <-> weight row).
//   * split-K fills the SMs for the small-N projections.  The CTAs that share an n-tile form a thread-block
//     CLUSTER (1 x splitk x 1): each parks its fp32 partial tile in its own shared memory, and after a cluster
//     barrier every CTA reduces a slice of the activation rows over all peers through distributed shared memory
//     (mapa + ld.shared::cluster) in fixed rank order -- deterministic, no global-memory workspace, no serial tail.
//   * two CTAs are co-resident per SM (<= ~100 KB of stages each) so one CTA's prologue/epilogue overlaps the
//     other's main loop.
//   * epilogues reproduce the reference's rounding points: plain store (+bias), residual add, SwiGLU (two
//     accumulators: gate and up tiles share the X tile), and fused RoPE + Q store / K,V cache append.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "gemm_common.cuh"

namespace eb {

// Stage memory per CTA.  Grids that fit one CTA per SM get a deep ring (one resident CTA, ~200 KB in flight);
// larger grids run two CTAs per SM with ~100 KB each so one CTA's prologue/epilogue hides under the other's loop.
static int env_kb(const char* name, int dflt) {
  const char* e = getenv(name);
  int kb = e ? atoi(e) : dflt;
  if (kb < 48) kb = 48;
  if (kb > 200) kb = 200;
  return kb;
}
static int smem_budget(int total_ctas) {
  static int small_kb = 0, big_kb = 0;
  if (!small_kb) {
    small_kb = env_kb("EB200_GEMM_SMEM_KB", 100);      // when the grid exceeds the SM count (two per SM)
    big_kb = env_kb("EB200_GEMM_SMEM_BIG_KB", 200);    // when it fits one CTA per SM
  }
  return (total_ctas <= device_sm_count() ? big_kb : small_kb) * 1024;
}
static int stage_count_for(int mpad, int epi, int total_ctas) {
  // 256 activation rows (prefill): a stage is 48 KB and the cluster reduction parks 128 KB of partials, so always one CTA per SM
  const int budget = mpad >= 256 ? 200 * 1024 : smem_budget(total_ctas);
  int s = (budget - kCtrlBytes - 1024) / stage_bytes(mpad, epi);
  if (s > kMaxStages) s = kMaxStages;
  if (s < 2) s = 2;
  return s;
}
int gemm_stage_count(int mpad, int epi) { return stage_count_for(mpad, epi, 1 << 30); }

// ------------------------------------------------------------------------------------------------------------
// wgmma + TMA kernel
// ------------------------------------------------------------------------------------------------------------
// Warps 0..7 are two MMA warpgroups: warpgroup g multiplies weight rows [64g, 64g + 64) of the tile with the X tile
// (wgmma m64 x MPAD x k16, fp32 accumulators in registers); warp 8 is the TMA producer.  After the main loop both
// warpgroups park their accumulators in the (then idle) stage memory as an fp32 [acc][MPAD][128] tile, and warpgroup 0
// runs the epilogue from there (thread <-> weight row).
// XMC: the two CTAs of neighbouring n-tiles (cluster dimension x = 2) stream the SAME activation k-range; each loads one half of
// every X tile (32 rows) and TMA-multicasts it into both CTAs' rings, so the L2 -> shared-memory ingress of an SM carries half
// the X bytes.
template <typename T, int MPAD, int EPI, bool XMC>
__global__ void __launch_bounds__(kGemmThreads, (MPAD >= 256 ? 1 : 2))
skinny_gemm_wgmma(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmW2,
                  const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmXh, const GemmParams p, const int stages) {
  constexpr bool kDual = (EPI == EPI_SWIGLU);
  static_assert(!XMC || (MPAD == 64 && !kDual), "X multicast: 64-row tiles, single accumulator");
  constexpr int kStageBytes = stage_bytes(MPAD, EPI);
  constexpr int kPartBytes = acc_tile_bytes(MPAD, EPI);

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* ctrl = smem + stages * kStageBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(ctrl);
  uint64_t* empty_bar = full_bar + kMaxStages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int n_tile = blockIdx.x;
  const int split = blockIdx.y;
  const int num_kb = (p.K + kBlockK - 1) / kBlockK;
  const int kb_begin = static_cast<int>((static_cast<long>(num_kb) * split) / p.splitk);
  const int kb_end = static_cast<int>((static_cast<long>(num_kb) * (split + 1)) / p.splitk);
  pdl_launch_dependents();  // let the next kernel start its own (independent) prologue and weight prefetch
  // cluster = (XMC ? 2 : 1) x splitk x 1; rank = x + 2 * y when XMC
  const uint32_t crank = (XMC || p.splitk > 1) ? cluster_ctarank() : 0u;
  const uint32_t xpar = XMC ? (crank & 1u) : 0u;
  const uint16_t pair_mask = XMC ? static_cast<uint16_t>(3u << (crank & ~1u)) : static_cast<uint16_t>(0);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmW);
    tma_prefetch_desc(XMC ? &tmXh : &tmX);
    if (kDual) tma_prefetch_desc(&tmW2);
    for (int i = 0; i < stages; ++i) {
      mbar_init(&full_bar[i], 1);
      // one arrival per MMA warpgroup; XMC: also the neighbour's (its half of the X tile lives here too)
      mbar_init(&empty_bar[i], XMC ? 4 : 2);
    }
    fence_barrier_init();
  }
  if (XMC) cluster_sync_all();  // the neighbour's barriers exist before anything is multicast into this CTA
  else __syncthreads();

  if (warp == kTmaWarp) {
    // ===== TMA producer =====
    if (lane == 0) {
      // The weight tiles do not depend on any earlier kernel: fill the whole ring with W before the programmatic
      // dependency wait, so this kernel's pipeline fill overlaps the tail of its predecessor.  Activation tiles
      // (written by the predecessor) follow after the wait; both land on the same full barrier (tx bytes add up).
      const int nkb = kb_end - kb_begin;
      const int pre = nkb < stages ? nkb : stages;
      for (int j = 0; j < pre; ++j) {
        uint8_t* st = smem + j * kStageBytes;
        mbar_arrive_expect_tx(&full_bar[j], kStageBytes);
        tma_load_2d(st, &tmW, &full_bar[j], (kb_begin + j) * kBlockK, n_tile * kBlockN, kEvictFirst);
        if (kDual) tma_load_2d(st + kWTileBytes, &tmW2, &full_bar[j], (kb_begin + j) * kBlockK, n_tile * kBlockN, kEvictFirst);
      }
      pdl_wait();
      auto load_x = [&](int stage, int kb) {
        uint8_t* xdst = smem + stage * kStageBytes + kWTileBytes * (kDual ? 2 : 1);
        if constexpr (XMC) {
          tma_load_2d_multicast(xdst + xpar * (32 * kBlockK * 2), &tmXh, &full_bar[stage], kb * kBlockK, static_cast<int>(xpar) * 32, pair_mask,
                                kEvictLast);
        } else {
          tma_load_2d(xdst, &tmX, &full_bar[stage], kb * kBlockK, 0, kEvictLast);
        }
      };
      for (int j = 0; j < pre; ++j) load_x(j, kb_begin + j);
      int s = (pre == stages) ? 0 : pre;
      uint32_t ph = (pre == stages) ? 1 : 0;
      for (int kb = kb_begin + pre; kb < kb_end; ++kb) {
        mbar_wait_mma(&empty_bar[s], ph ^ 1);
        uint8_t* st = smem + s * kStageBytes;
        mbar_arrive_expect_tx(&full_bar[s], kStageBytes);
        tma_load_2d(st, &tmW, &full_bar[s], kb * kBlockK, n_tile * kBlockN, kEvictFirst);
        if (kDual) tma_load_2d(st + kWTileBytes, &tmW2, &full_bar[s], kb * kBlockK, n_tile * kBlockN, kEvictFirst);
        load_x(s, kb);
        if (++s == stages) {
          s = 0;
          ph ^= 1;
        }
      }
    }
  } else {
    // ===== MMA warpgroups =====
    const int wg = warp >> 2;
    float acc[MPAD / 2], acc2[kDual ? MPAD / 2 : 1];
#pragma unroll
    for (int i = 0; i < MPAD / 2; ++i) acc[i] = 0.f;
#pragma unroll
    for (int i = 0; i < (kDual ? MPAD / 2 : 1); ++i) acc2[i] = 0.f;
    auto release = [&](int st) {
      if ((threadIdx.x & 127) == 0) {
        mbar_arrive(&empty_bar[st]);
        if constexpr (XMC) mbar_arrive_cluster(&empty_bar[st], crank ^ 1u);  // the neighbour's half of this slot is consumed too
      }
    };
    int s = 0, prev = -1;
    uint32_t ph = 0;
    for (int kb = kb_begin; kb < kb_end; ++kb) {
      mbar_wait_mma(&full_bar[s], ph);
      const uint32_t st = smem_u32(smem + s * kStageBytes);
      const uint32_t a_addr = st + wg * (kWTileBytes / 2);  // 64 weight rows = 8 KB = eight whole swizzle atoms
      const uint64_t b_desc = make_kmajor_sw128_desc(st + kWTileBytes * (kDual ? 2 : 1));
      wgmma_fence();
      wgmma_kblock<T, MPAD>(acc, make_kmajor_sw128_desc(a_addr), b_desc);
      if constexpr (kDual) wgmma_kblock<T, MPAD>(acc2, make_kmajor_sw128_desc(a_addr + kWTileBytes), b_desc);
      wgmma_commit();
      wgmma_wait<1>();  // the previous k-block's MMAs have retired: its slot can be refilled
      if (prev >= 0) release(prev);
      prev = s;
      if (++s == stages) {
        s = 0;
        ph ^= 1;
      }
    }
    wgmma_wait<0>();
    wgmma_fence_acc(acc);
    wgmma_fence_acc(acc2);
    // every MMA of both warpgroups has retired and every TMA load has landed: the stage memory becomes the fp32
    // accumulator tile part[acc][m][128], then scratch for the epilogue
    asm volatile("bar.sync 2, 256;" ::: "memory");
    float* part = reinterpret_cast<float*>(smem);
    wgmma_store_acc<MPAD>(acc, part, kBlockN, wg * 64);
    if constexpr (kDual) wgmma_store_acc<MPAD>(acc2, part + MPAD * kBlockN, kBlockN, wg * 64);
    asm volatile("bar.sync 2, 256;" ::: "memory");
    if (wg == 0) {
      pdl_wait();  // residual / device state / KV cache are produced by earlier kernels
      if (p.splitk == 1) {
        const int row = threadIdx.x;
        const int m_valid = valid_rows(p);
        float a[16], a2[16];
#pragma unroll 1
        for (int c = 0; c < MPAD / 16; ++c) {
          if (c * 16 >= m_valid) break;
          acc_ld16(part, kBlockN, row, c * 16, a);
          if constexpr (kDual) acc_ld16(part + MPAD * kBlockN, kBlockN, row, c * 16, a2);
          final_chunk<T, EPI>(p, a, a2, c * 16, m_valid, row, n_tile, smem + kPartBytes);
        }
      }
    }
  }

  if (p.splitk > 1) {
    // ===== cluster split-K reduction over distributed shared memory =====
    cluster_sync_all();  // every peer's partial tile is visible cluster-wide
    if (warp < 4) {
      const int row = threadIdx.x;
      const int m_valid = valid_rows(p);
      const int S = p.splitk;
      const int rank = static_cast<int>(XMC ? (crank >> 1) : crank);  // this CTA's index among the split-K peers of its n-tile
      const int per = (MPAD + S - 1) / S;  // activation rows reduced by each CTA
      const int m_lo = rank * per, m_hi = min(MPAD, m_lo + per);
      const uint32_t part_local = smem_u32(smem);
      float acc[16], acc2[16];
#pragma unroll 1
      for (int m0 = m_lo; m0 < m_hi; m0 += 16) {
        if (m0 >= m_valid) break;
        const int nrows = min(16, m_hi - m0);
#pragma unroll
        for (int j = 0; j < 16; ++j) acc[j] = acc2[j] = 0.f;
        for (int s = 0; s < S; ++s) {  // fixed rank order: deterministic sums
          const uint32_t peer = dsmem_map(part_local, XMC ? (xpar + 2u * static_cast<uint32_t>(s)) : static_cast<uint32_t>(s));
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            if (j < nrows && m0 + j < m_valid) {
              acc[j] += dsmem_ld_f32(peer + static_cast<uint32_t>(((m0 + j) * kBlockN + row) * 4));
              if constexpr (kDual) acc2[j] += dsmem_ld_f32(peer + static_cast<uint32_t>(((MPAD + m0 + j) * kBlockN + row) * 4));
            }
          }
        }
        final_chunk<T, EPI>(p, acc, acc2, m0, m_valid, row, n_tile, smem + kPartBytes, nrows);
      }
    }
    cluster_sync_all();  // no CTA may exit (and free its shared memory) while a peer still reads it
  } else if (XMC) {
    cluster_sync_all();  // the neighbour may still multicast into / arrive on this CTA's shared memory
  }
}

// ------------------------------------------------------------------------------------------------------------
// SIMT bring-up kernel: identical epilogue, naive main loop (debug aid; never on the product path)
// ------------------------------------------------------------------------------------------------------------
template <typename T, int MPAD, int EPI>
__global__ void __launch_bounds__(128) skinny_gemm_simt(const T* __restrict__ W, const T* __restrict__ W2,
                                                        const T* __restrict__ X, long ldx, const GemmParams p) {
  constexpr bool kDual = (EPI == EPI_SWIGLU);
  __shared__ __align__(16) uint8_t scratch[16 * kBlockN * 2 + 16];
  pdl_launch_dependents();
  pdl_wait();
  const int row = threadIdx.x;
  const int n_tile = blockIdx.x;
  const int split = blockIdx.y;
  const int n = n_tile * kBlockN + row;
  const int m_valid = valid_rows(p);
  const int num_kb = (p.K + kBlockK - 1) / kBlockK;
  const int k0 = static_cast<int>((static_cast<long>(num_kb) * split) / p.splitk) * kBlockK;
  const int k1 = min(p.K, static_cast<int>((static_cast<long>(num_kb) * (split + 1)) / p.splitk) * kBlockK);
  auto compute_chunk = [&](int c, float(&acc)[16], float(&acc2)[16]) {
#pragma unroll
    for (int j = 0; j < 16; ++j) acc[j] = acc2[j] = 0.f;
    if (n < p.N) {
      for (int k = k0; k < k1; ++k) {
        const float w = DT<T>::to_f(W[static_cast<long>(n) * p.K + k]);
        float w2 = 0.f;
        if constexpr (kDual) w2 = DT<T>::to_f(W2[static_cast<long>(n) * p.K + k]);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const float x = DT<T>::to_f(X[static_cast<long>(c * 16 + j) * ldx + k]);
          acc[j] = fmaf(w, x, acc[j]);
          if constexpr (kDual) acc2[j] = fmaf(w2, x, acc2[j]);
        }
      }
    }
  };
  float acc[16], acc2[16];
  if (p.splitk == 1) {
    for (int c = 0; c < MPAD / 16; ++c) {
      compute_chunk(c, acc, acc2);
      final_chunk<T, EPI>(p, acc, acc2, c * 16, m_valid, row, n_tile, scratch);
    }
  } else {
    for (int c = 0; c < MPAD / 16; ++c) {
      compute_chunk(c, acc, acc2);
      partial_store<MPAD, EPI>(p, acc, acc2, c * 16, m_valid, n, split);
    }
    if (splitk_arrive(p, n_tile, row, scratch)) {
      for (int c = 0; c < MPAD / 16; ++c) {
        partial_reduce<MPAD, EPI>(p, acc, acc2, c * 16, m_valid, n);
        final_chunk<T, EPI>(p, acc, acc2, c * 16, m_valid, row, n_tile, scratch);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// SiLU table: the activation is a function of a 16-bit value, so T(g / (1 + exp(-g))) is tabulated once per device
// with the exact expression the epilogue used to evaluate per element (LlamaMLP act_fn on a model-dtype tensor,
// modeling_llama_kv.py:501-535 / cnets.py:347-367)
// ------------------------------------------------------------------------------------------------------------
__device__ unsigned short g_silu_lut[2][65536];
template <typename T> __global__ void silu_lut_kernel(unsigned short* lut) {
  const unsigned i = blockIdx.x * 256u + threadIdx.x;
  const unsigned short b = static_cast<unsigned short>(i);
  const T g = *reinterpret_cast<const T*>(&b);
  const float gf = DT<T>::to_f(g);
  const T r = DT<T>::from_f(gf / (1.0f + expf(-gf)));
  lut[i] = *reinterpret_cast<const unsigned short*>(&r);
}
const void* silu_lut(int dtype, cudaStream_t s) {
  static const void* ready[64][2] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64 || dtype < 0 || dtype > 1) return nullptr;
  if (!ready[dev][dtype]) {
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(s, &cap) != cudaSuccess || cap != cudaStreamCaptureStatusNone) return nullptr;  // first use must be eager
    unsigned short* base = nullptr;
    if (cudaGetSymbolAddress(reinterpret_cast<void**>(&base), g_silu_lut) != cudaSuccess) return nullptr;
    unsigned short* lut = base + static_cast<size_t>(dtype) * 65536;
    if (dtype == DT_BF16) silu_lut_kernel<__nv_bfloat16><<<256, 256, 0, s>>>(lut);
    else silu_lut_kernel<__half><<<256, 256, 0, s>>>(lut);
    if (cudaGetLastError() != cudaSuccess || cudaStreamSynchronize(s) != cudaSuccess) return nullptr;
    ready[dev][dtype] = lut;
  }
  return ready[dev][dtype];
}

// ------------------------------------------------------------------------------------------------------------
// host launchers
// ------------------------------------------------------------------------------------------------------------
static bool xmc_enabled() {
  static int v = -1;
  if (v < 0) {
    // Opt-in: correct (all GEMM parity tests pass with it), but it doubles the cluster size of the split-K projections, which
    // constrains their scheduling, and has no measured gain on the H100.
    const char* e = getenv("EB200_GEMM_XMC");
    v = (e && atoi(e) == 1) ? 1 : 0;
  }
  return v == 1;
}
template <typename T, int MPAD, int EPI, bool XMC>
static int launch_one_x(const CUtensorMap* tmW, const CUtensorMap* tmW2, const CUtensorMap* tmX, const CUtensorMap* tmXh, const GemmParams& p,
                        cudaStream_t s);
template <typename T, int MPAD, int EPI>
static int launch_one(const CUtensorMap* tmW, const CUtensorMap* tmW2, const CUtensorMap* tmX, const GemmParams& p, cudaStream_t s,
                      const CUtensorMap* tmXh = nullptr) {
  if constexpr (MPAD == 64 && EPI != EPI_SWIGLU) {
    const int tiles = (p.N + kBlockN - 1) / kBlockN;
    if (tmXh && xmc_enabled() && tiles % 2 == 0 && 2 * p.splitk <= 8) return launch_one_x<T, MPAD, EPI, true>(tmW, tmW2, tmX, tmXh, p, s);
  }
  return launch_one_x<T, MPAD, EPI, false>(tmW, tmW2, tmX, tmX, p, s);
}
template <typename T, int MPAD, int EPI, bool XMC>
static int launch_one_x(const CUtensorMap* tmW, const CUtensorMap* tmW2, const CUtensorMap* tmX, const CUtensorMap* tmXh, const GemmParams& p,
                        cudaStream_t s) {
  auto kern = skinny_gemm_wgmma<T, MPAD, EPI, XMC>;
  dim3 grid((p.N + kBlockN - 1) / kBlockN, p.splitk);
  const int stages = stage_count_for(MPAD, EPI, static_cast<int>(grid.x * grid.y));
  const int smem = stages * stage_bytes(MPAD, EPI) + kCtrlBytes + 1024;
  if (p.splitk > 8) return static_cast<int>(cudaErrorInvalidValue);  // portable cluster size
  // the accumulators are parked as (1|2) x MPAD x 128 fp32 partials (+ a 4 KB exchange strip) in the stage memory
  if (stages * stage_bytes(MPAD, EPI) < acc_tile_bytes(MPAD, EPI) + 4096)
    return static_cast<int>(cudaErrorInvalidValue);
  static bool configured_dev[64] = {};  // per device (the attribute is per device) and per instantiation
  const int cur_dev = current_device_index();
  if (cur_dev < 0) return static_cast<int>(cudaErrorInvalidDevice);
  if (!configured_dev[cur_dev]) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024 + kCtrlBytes + 1024);
    if (e != cudaSuccess) return static_cast<int>(e);
    configured_dev[cur_dev] = true;
  }
  return static_cast<int>(launch_kc(kern, grid, dim3(kGemmThreads), static_cast<size_t>(smem), s, dim3(XMC ? 2 : 1, p.splitk, 1), *tmW,
                                    tmW2 ? *tmW2 : *tmW, *tmX, *tmXh, p, stages));
}

template <typename T, int MPAD>
static int launch_epi(int epi, const CUtensorMap* a, const CUtensorMap* b, const CUtensorMap* c, const GemmParams& p,
                      cudaStream_t s, const CUtensorMap* ch = nullptr) {
  switch (epi) {
    case EPI_STORE: return launch_one<T, MPAD, EPI_STORE>(a, b, c, p, s, ch);
    case EPI_RESIDUAL: return launch_one<T, MPAD, EPI_RESIDUAL>(a, b, c, p, s, ch);
    case EPI_SWIGLU: return launch_one<T, MPAD, EPI_SWIGLU>(a, b, c, p, s, ch);
    case EPI_QKV_ROPE: return launch_one<T, MPAD, EPI_QKV_ROPE>(a, b, c, p, s, ch);
    case EPI_PARTIAL_F32: return launch_one<T, MPAD, EPI_PARTIAL_F32>(a, b, c, p, s, ch);
    case EPI_SWIGLU_IL: return launch_one<T, MPAD, EPI_SWIGLU_IL>(a, b, c, p, s, ch);
  }
  return static_cast<int>(cudaErrorInvalidValue);
}

// 256 activation rows per launch (prompt prefill: wgmma N = 256, the weights are streamed once per 256 prompt tokens instead of
// once per 64): only the epilogues the target's decoder layer needs
template <typename T>
static int launch_epi256(int epi, const CUtensorMap* a, const CUtensorMap* c, const GemmParams& p, cudaStream_t s) {
  switch (epi) {
    case EPI_RESIDUAL: return launch_one<T, 256, EPI_RESIDUAL>(a, nullptr, c, p, s);
    case EPI_QKV_ROPE: return launch_one<T, 256, EPI_QKV_ROPE>(a, nullptr, c, p, s);
    case EPI_SWIGLU_IL: return launch_one<T, 256, EPI_SWIGLU_IL>(a, nullptr, c, p, s);
  }
  return static_cast<int>(cudaErrorInvalidValue);
}

int launch_gemm(int dtype, int mpad, int epi, const CUtensorMap* tmW, const CUtensorMap* tmW2, const CUtensorMap* tmX,
                const GemmParams& p_in, cudaStream_t s, const CUtensorMap* tmXh) {
  GemmParams p = p_in;
  if (p.splitk < 1 || p.m_rows > mpad) return static_cast<int>(cudaErrorInvalidValue);
  if (epi == EPI_SWIGLU || epi == EPI_SWIGLU_IL) {
    p.silu_lut = silu_lut(dtype, s);
    if (!p.silu_lut) return static_cast<int>(cudaErrorNotReady);
  }
  if (dtype == DT_BF16) {
    if (mpad == 16) return launch_epi<__nv_bfloat16, 16>(epi, tmW, tmW2, tmX, p, s);
    if (mpad == 64) return launch_epi<__nv_bfloat16, 64>(epi, tmW, tmW2, tmX, p, s, tmXh);
    if (mpad == 256) return launch_epi256<__nv_bfloat16>(epi, tmW, tmX, p, s);
  } else if (dtype == DT_FP16) {
    if (mpad == 16) return launch_epi<__half, 16>(epi, tmW, tmW2, tmX, p, s);
    if (mpad == 64) return launch_epi<__half, 64>(epi, tmW, tmW2, tmX, p, s, tmXh);
    if (mpad == 256) return launch_epi256<__half>(epi, tmW, tmX, p, s);
  }
  return static_cast<int>(cudaErrorInvalidValue);
}

template <typename T, int MPAD>
static int launch_simt_epi(int epi, const void* W, const void* W2, const void* X, long ldx, const GemmParams& p,
                           cudaStream_t s) {
  dim3 grid((p.N + kBlockN - 1) / kBlockN, p.splitk);
  const T* w = reinterpret_cast<const T*>(W);
  const T* w2 = reinterpret_cast<const T*>(W2);
  const T* x = reinterpret_cast<const T*>(X);
  switch (epi) {
    case EPI_STORE: skinny_gemm_simt<T, MPAD, EPI_STORE><<<grid, 128, 0, s>>>(w, w2, x, ldx, p); break;
    case EPI_RESIDUAL: skinny_gemm_simt<T, MPAD, EPI_RESIDUAL><<<grid, 128, 0, s>>>(w, w2, x, ldx, p); break;
    case EPI_SWIGLU: skinny_gemm_simt<T, MPAD, EPI_SWIGLU><<<grid, 128, 0, s>>>(w, w2, x, ldx, p); break;
    case EPI_QKV_ROPE: skinny_gemm_simt<T, MPAD, EPI_QKV_ROPE><<<grid, 128, 0, s>>>(w, w2, x, ldx, p); break;
    case EPI_PARTIAL_F32: skinny_gemm_simt<T, MPAD, EPI_PARTIAL_F32><<<grid, 128, 0, s>>>(w, w2, x, ldx, p); break;
    case EPI_SWIGLU_IL: skinny_gemm_simt<T, MPAD, EPI_SWIGLU_IL><<<grid, 128, 0, s>>>(w, w2, x, ldx, p); break;
    default: return static_cast<int>(cudaErrorInvalidValue);
  }
  return static_cast<int>(cudaGetLastError());
}

int launch_gemm_simt(int dtype, int mpad, int epi, const void* W, const void* W2, const void* X, long ldx,
                     const GemmParams& p_in, cudaStream_t s) {
  GemmParams p = p_in;
  if (p.splitk < 1 || p.m_rows > mpad) return static_cast<int>(cudaErrorInvalidValue);
  if (epi == EPI_SWIGLU || epi == EPI_SWIGLU_IL) {
    p.silu_lut = silu_lut(dtype, s);
    if (!p.silu_lut) return static_cast<int>(cudaErrorNotReady);
  }
  if (dtype == DT_BF16) {
    if (mpad == 16) return launch_simt_epi<__nv_bfloat16, 16>(epi, W, W2, X, ldx, p, s);
    if (mpad == 64) return launch_simt_epi<__nv_bfloat16, 64>(epi, W, W2, X, ldx, p, s);
  } else if (dtype == DT_FP16) {
    if (mpad == 16) return launch_simt_epi<__half, 16>(epi, W, W2, X, ldx, p, s);
    if (mpad == 64) return launch_simt_epi<__half, 64>(epi, W, W2, X, ldx, p, s);
  }
  return static_cast<int>(cudaErrorInvalidValue);
}

}  // namespace eb
