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

#include <algorithm>

#include "gemm_common.cuh"

namespace eb {

// Stage memory per CTA: ~100 KB, so two CTAs fit on an SM.  For grids larger than the SM count one CTA's prologue/epilogue hides
// under the other's loop.  Grids that fit one CTA per SM (EB200_GEMM_SMEM_BIG_KB) take the same budget: the next kernel's CTAs then
// become resident next to them and fill their own rings while these drain.  With a 200 KB ring they waited for these to exit, and
// the cycle was 5 % slower on the H100 (DESIGN.md §5).
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
    big_kb = env_kb("EB200_GEMM_SMEM_BIG_KB", 100);    // when it fits one CTA per SM
  }
  return (total_ctas <= device_sm_count() ? big_kb : small_kb) * 1024;
}
static int stage_count_for(int mpad, int epi, int total_ctas, int wq = WQ_NONE) {
  // 256 activation rows (prefill): a stage is 48 KB and the cluster reduction parks 128 KB of partials, so always one CTA per SM
  const int budget = mpad >= 256 ? 200 * 1024 : smem_budget(total_ctas);
  int s = wq == WQ_INT8   ? (budget - kCtrlBytes - 1024 - kW8DqBytes) / stage_bytes_w8(mpad)
          : wq == WQ_4BIT ? (budget - kCtrlBytes - 1024) / stage_bytes_w4(mpad)
          : wq == WQ_FP8  ? (budget - kCtrlBytes - 1024) / stage_bytes_fp8(mpad)
                          : (budget - kCtrlBytes - 1024) / stage_bytes(mpad, epi);
  if (s > kMaxStages) s = kMaxStages;
  if (s < 2) s = 2;
  return s;
}
int gemm_stage_count(int mpad, int epi) { return stage_count_for(mpad, epi, 1 << 30); }

// ------------------------------------------------------------------------------------------------------------
// W8A16 dequantization: one warpgroup turns its 64 int8 weight rows of a stage (row-major, 64 B per row) into the model-dtype
// K-major SWIZZLE_128B layout wgmma reads (16-byte chunk c of row r at r * 128 + ((c ^ (r & 7)) * 16)).  Thread t handles the
// 16-element chunks t and t + 128, i.e. rows t / 4 and 32 + t / 4; sc[j] is the scale of its row j.  Arithmetic: transformers'
// dequantization T((q * SCB) * kInv127), two fp32 roundings and one cast, no FMA contraction.
// ------------------------------------------------------------------------------------------------------------
// exact int8 -> fp32 of byte b of w without a conversion instruction: with u = byte ^ 0x80 in [0, 255], the bit pattern
// 0x4B0000uu is the fp32 value 2^23 + u, and subtracting 2^23 + 128 leaves the signed byte exactly
__device__ __forceinline__ float i8_to_f32(uint32_t w_xor80, int b) {
  return __fsub_rn(__uint_as_float(__byte_perm(w_xor80, 0x4B000000u, 0x7540u + b)), 8388736.0f);
}
template <typename T> __device__ __forceinline__ uint32_t pack2_rn(float lo, float hi);
template <> __device__ __forceinline__ uint32_t pack2_rn<__nv_bfloat16>(float lo, float hi) {
  const __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&v);
}
template <> __device__ __forceinline__ uint32_t pack2_rn<__half>(float lo, float hi) {
  const __half2 v = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&v);
}
template <typename T> __device__ __forceinline__ uint32_t dq_pack2(uint32_t w_xor80, int b, float s) {
  const float lo = __fmul_rn(__fmul_rn(i8_to_f32(w_xor80, b), s), kInv127);
  const float hi = __fmul_rn(__fmul_rn(i8_to_f32(w_xor80, b + 1), s), kInv127);
  return pack2_rn<T>(lo, hi);
}
template <typename T> __device__ __forceinline__ void dequant_w8_rows(uint32_t src, uint32_t dst, const float (&sc)[2]) {
  const int t = threadIdx.x & 127;
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const int r = 32 * j + (t >> 2), c = t & 3;
    uint32_t w[4];
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]) : "r"(src + r * 64 + c * 16));
    uint32_t o[8];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      o[2 * i] = dq_pack2<T>(w[i] ^ 0x80808080u, 0, sc[j]);
      o[2 * i + 1] = dq_pack2<T>(w[i] ^ 0x80808080u, 2, sc[j]);
    }
    const uint32_t row = dst + r * 128;
    asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(row + (((2 * c) ^ (r & 7)) * 16)), "r"(o[0]), "r"(o[1]), "r"(o[2]), "r"(o[3])
                 : "memory");
    asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(row + (((2 * c + 1) ^ (r & 7)) * 16)), "r"(o[4]), "r"(o[5]), "r"(o[6]),
                 "r"(o[7])
                 : "memory");
  }
}
// W4A16: bitsandbytes' code tables (quant.py NF4_CODE / FP4_CODE, the constants of its dDequantizeNF4 / dDequantizeFP4Tree).  In global
// memory rather than a __constant__ bank: with a user constant bank in this module every GEMM launch of a replayed cycle graph measured
// slower on the H100, the model-dtype ones included.
__device__ const float kW4Codes[2][16] = {
    {-1.0f, -0.6961928009986877f, -0.5250730514526367f, -0.39491748809814453f, -0.28444138169288635f, -0.18477343022823334f,
     -0.09105003625154495f, 0.0f, 0.07958029955625534f, 0.16093020141458511f, 0.24611230194568634f, 0.33791524171829224f,
     0.44070982933044434f, 0.5626170039176941f, 0.7229568362236023f, 1.0f},
    {0.0f, 0.0052083333f, 0.66666667f, 1.0f, 0.33333333f, 0.5f, 0.16666667f, 0.25f, -0.0f, -0.0052083333f, -0.66666667f, -1.0f,
     -0.33333333f, -0.5f, -0.16666667f, -0.25f}};
// One k16 step of a thread's A fragment from its 4 repacked bytes w (byte i -> register i; the high nibble is the lower K column):
// T(code * absmax) with one __fmul_rn; s0 / s1 are the absmax of its rows r0 / r0 + 8 (registers 0, 2 / 1, 3).  The 16-entry table
// lives in shared memory: its entries fall in 16 distinct banks, so the lookups are conflict-free.
template <typename T>
__device__ __forceinline__ void w4_fragment(uint32_t w, uint32_t lut, float s0, float s1, uint32_t (&a)[4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float lo, hi;
    asm("ld.shared.f32 %0, [%1];" : "=f"(lo) : "r"(lut + ((w >> (8 * i + 2)) & 0x3Cu)));
    asm("ld.shared.f32 %0, [%1];" : "=f"(hi) : "r"(lut + ((w << 2 >> (8 * i)) & 0x3Cu)));
    const float sc = (i & 1) ? s1 : s0;
    a[i] = pack2_rn<T>(__fmul_rn(lo, sc), __fmul_rn(hi, sc));
  }
}

// W8A16 on FP8: one k16 step of a thread's A fragment from its 8 repacked e4m3 bytes (w0: registers 0, 1; w1: registers 2, 3; the
// low byte of each half-word is the lower K column): T(fp32(q) * scale) with one __fmul_rn.  e4m3 -> f16 -> f32 is exact, so this is
// transformers' `quantized.to(fp32) * scale_inv` followed by the model-dtype cast.  sc: the scale of the warpgroup's 64-row group.
template <typename T>
__device__ __forceinline__ void f8_fragment(uint32_t w0, uint32_t w1, float sc, uint32_t (&a)[4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    uint32_t h2;
    asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h2) : "h"(static_cast<unsigned short>((i < 2 ? w0 : w1) >> (16 * (i & 1)))));
    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&h2));
    a[i] = pack2_rn<T>(__fmul_rn(f.x, sc), __fmul_rn(f.y, sc));
  }
}

__device__ __forceinline__ float ld_global_f32(const float* p) {
  float v;
  asm volatile("ld.global.f32 %0, [%1];" : "=f"(v) : "l"(p) : "memory");
  return v;
}

// ------------------------------------------------------------------------------------------------------------
// wgmma + TMA kernel
// ------------------------------------------------------------------------------------------------------------
// Warps 0..7 are two MMA warpgroups: warpgroup g multiplies weight rows [64g, 64g + 64) of the tile with the X tile
// (wgmma m64 x MPAD x k16, fp32 accumulators in registers); warp 8 is the TMA producer.  After the main loop both
// warpgroups park their accumulators in the (then idle) stage memory as an fp32 [acc][MPAD][128] tile, and warpgroup 0
// runs the epilogue from there (thread <-> weight row).
// W8: tmW streams int8 weight tiles; the MMA warpgroups dequantize every stage into one model-dtype tile (an 8 KB half per
// warpgroup) and run the same k16 MMAs on it, so the accumulators equal those of the kernel on the dequantized W.  Each k-block's
// MMAs retire before the next dequantization (wgmma_wait<0>): ptxas serialises every wgmma of a kernel whose MMAs stay in flight
// across the conversion code.  The other warpgroup and the second resident CTA keep the tensor pipe and the TMA ring busy meanwhile.
// W4: tmW streams 4 KB nibble tiles in fragment order and tmW2 (unused by the single-matrix epilogues W4 serves) the tile's absmax.
// Each thread reads its 16 nibble bytes of a k-block with one shared load and converts one k16 step at a time straight into the A
// registers of a wgmma RS: step k + 1 is converted while step k's MMA runs (two fragment buffers, one commit group per step,
// wgmma_wait<1>), so neither a shared-memory round trip nor a proxy fence sits on the MMA chain.
// F8: the same register-A mainloop on e4m3 weights.  tmW streams the 8 KB tile (bytes permuted within the tile into fragment order,
// so each thread reads a k-block's 32 bytes with two conflict-free 16-byte shared loads) and tmW2 the tile's 16 B of block scales;
// warpgroup g's 64 rows share one scale per k-block.
template <typename T, int MPAD, int EPI, int WQ>
__global__ void __launch_bounds__(kGemmThreads, (MPAD >= 256 ? 1 : 2))
skinny_gemm_wgmma(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmW2,
                  const __grid_constant__ CUtensorMap tmX, const GemmParams p, const int stages, const __grid_constant__ L2Prefetch pf) {
  constexpr bool kDual = (EPI == EPI_SWIGLU);
  constexpr bool W8 = WQ == WQ_INT8, W4 = WQ == WQ_4BIT, F8 = WQ == WQ_FP8;
  static_assert(WQ == WQ_NONE || !kDual, "W8A16 / W4A16: single weight stream");
  // weight bytes of one stage (per weight matrix)
  constexpr int kWBytes = W8 ? kW8TileBytes : W4 ? kW4WBytes : F8 ? kF8WBytes : kWTileBytes;
  constexpr int kStageBytes = W8 ? stage_bytes_w8(MPAD) : W4 ? stage_bytes_w4(MPAD) : F8 ? stage_bytes_fp8(MPAD) : stage_bytes(MPAD, EPI);
  constexpr int kTxBytes = W4   ? kW4TileBytes + kW4AbsBytes + x_tile_bytes(MPAD)
                           : F8 ? kF8TileBytes + kF8ScaleBytes + x_tile_bytes(MPAD)
                                : kStageBytes;  // bytes TMA lands per stage
  constexpr int kPartBytes = acc_tile_bytes(MPAD, EPI);

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* wdq = smem + stages * kStageBytes;  // W8: the dequantized weight tile
  uint8_t* ctrl = wdq + (W8 ? kW8DqBytes : 0);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(ctrl);
  uint64_t* empty_bar = full_bar + kMaxStages;
  float* w4_lut = reinterpret_cast<float*>(ctrl + 512);  // W4: the code table

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int n_tile = blockIdx.x;
  const int split = blockIdx.y;
  const int num_kb = (p.K + kBlockK - 1) / kBlockK;
  const int kb_begin = static_cast<int>((static_cast<long>(num_kb) * split) / p.splitk);
  const int kb_end = static_cast<int>((static_cast<long>(num_kb) * (split + 1)) / p.splitk);
  pdl_launch_dependents();  // let the next kernel start its own (independent) prologue and weight prefetch
  // cluster = 1 x splitk x 1: the rank is this CTA's index among the split-K peers of its n-tile
  const uint32_t crank = p.splitk > 1 ? cluster_ctarank() : 0u;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmW);
    tma_prefetch_desc(&tmX);
    if (kDual) tma_prefetch_desc(&tmW2);
    for (int i = 0; i < stages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2);  // one arrival per MMA warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == kTmaWarp) {
    // ===== TMA producer =====
    if (lane == 0) {
      // The weight tiles do not depend on any earlier kernel: fill the whole ring with W before the programmatic
      // dependency wait, so this kernel's pipeline fill overlaps the tail of its predecessor.  Activation tiles
      // (written by the predecessor) follow after the wait; both land on the same full barrier (tx bytes add up).
      const int nkb = kb_end - kb_begin;
      const int pre = nkb < stages ? nkb : stages;
      auto load_w = [&](int stage, int kb) {
        uint8_t* st = smem + stage * kStageBytes;
        mbar_arrive_expect_tx(&full_bar[stage], kTxBytes);
        if constexpr (W4) {
          tma_load_2d(st, &tmW, &full_bar[stage], 0, (n_tile * num_kb + kb) * (kW4TileBytes / 256), kEvictFirst);
          tma_load_2d(st + kW4TileBytes, &tmW2, &full_bar[stage], n_tile * kBlockN, kb, kEvictFirst);
        } else {
          tma_load_2d(st, &tmW, &full_bar[stage], kb * kBlockK, n_tile * kBlockN, kEvictFirst);
          if (kDual) tma_load_2d(st + kWTileBytes, &tmW2, &full_bar[stage], kb * kBlockK, n_tile * kBlockN, kEvictFirst);
          if constexpr (F8) tma_load_2d(st + kF8TileBytes, &tmW2, &full_bar[stage], (kb / 2) * 4, n_tile, kEvictFirst);
        }
      };
      for (int j = 0; j < pre; ++j) load_w(j, kb_begin + j);
      pdl_wait();
      auto load_x = [&](int stage, int kb) {
        tma_load_2d(smem + stage * kStageBytes + kWBytes * (kDual ? 2 : 1), &tmX, &full_bar[stage], kb * kBlockK, 0, kEvictLast);
      };
      for (int j = 0; j < pre; ++j) load_x(j, kb_begin + j);
      int s = (pre == stages) ? 0 : pre;
      uint32_t ph = (pre == stages) ? 1 : 0;
      for (int kb = kb_begin + pre; kb < kb_end; ++kb) {
        mbar_wait_mma(&empty_bar[s], ph ^ 1);
        load_w(s, kb);
        load_x(s, kb);
        if (++s == stages) {
          s = 0;
          ph ^= 1;
        }
      }
      // every weight load of this CTA is issued: while the ring drains and the epilogue runs, stream this CTA's share of the
      // next GEMM's leading weight tiles into L2
      l2_prefetch_weights(pf, n_tile + static_cast<int>(gridDim.x) * split, static_cast<int>(gridDim.x * gridDim.y));
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
      if ((threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[st]);
    };
    float sc[2] = {0.f, 0.f};
    if constexpr (W8) {
      pdl_wait();  // the row scales are read with generic loads, which may not precede the dependency wait
      const int t = threadIdx.x & 127;
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int n = n_tile * kBlockN + wg * 64 + 32 * j + (t >> 2);  // the rows dequant_w8_rows gives this thread
        if (n < p.N) sc[j] = ld_global_f32(p.w_scale + n);
      }
    }
    int s = 0, prev = -1;
    uint32_t ph = 0;
    if constexpr (W4 || F8) {
      if constexpr (W4) {
        pdl_wait();  // the code table is read with a generic load, which may not precede the dependency wait (X tiles follow it anyway)
        if (threadIdx.x < 16)
          asm volatile("st.shared.f32 [%0], %1;" ::"r"(smem_u32(w4_lut + threadIdx.x)), "f"(ld_global_f32(&kW4Codes[p.w4_quant][threadIdx.x]))
                       : "memory");
        asm volatile("bar.sync 2, 256;" ::: "memory");  // both MMA warpgroups see the table
      }
      // W4: thread t of the warpgroup: its 16 bytes of every tile at (wg * 128 + t) * 16, word k = k16 step k; absmax of rows r0, r0 + 8.
      // F8: its 32 bytes at (wg * 128 + t) * 16 (steps 0, 1) and 4096 + (wg * 128 + t) * 16 (steps 2, 3), two words per step; s0 is
      // the scale of the warpgroup's 64-row group.
      const uint32_t lut = smem_u32(w4_lut);
      const int t = threadIdx.x & 127;
      const int r0 = wg * 64 + 16 * (t >> 5) + ((t & 31) >> 2);
      uint32_t q[F8 ? 8 : 4], a[2][4];
      float s0 = 0.f, s1 = 0.f;
      auto fetch = [&](int stage) {
        const uint32_t st = smem_u32(smem + stage * kStageBytes);
        asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(q[0]), "=r"(q[1]), "=r"(q[2]), "=r"(q[3]) : "r"(st + (threadIdx.x & 255) * 16)
                     : "memory");
        if constexpr (F8) {
          asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(q[4]), "=r"(q[5]), "=r"(q[6]), "=r"(q[7])
                       : "r"(st + kF8TileBytes / 2 + (threadIdx.x & 255) * 16)
                       : "memory");
          asm volatile("ld.shared.f32 %0, [%1];" : "=f"(s0) : "r"(st + kF8TileBytes + wg * 4) : "memory");
        } else {
          asm volatile("ld.shared.f32 %0, [%1];" : "=f"(s0) : "r"(st + kW4TileBytes + r0 * 4) : "memory");
          asm volatile("ld.shared.f32 %0, [%1];" : "=f"(s1) : "r"(st + kW4TileBytes + (r0 + 8) * 4) : "memory");
        }
      };
      auto fragment = [&](int k, uint32_t(&frag)[4]) {  // k16 step k of the fetched k-block
        if constexpr (F8) f8_fragment<T>(q[(k >> 1) * 4 + (k & 1) * 2], q[(k >> 1) * 4 + (k & 1) * 2 + 1], s0, frag);
        else w4_fragment<T>(q[k], lut, s0, s1, frag);
      };
      if (kb_begin < kb_end) {
        mbar_wait_mma(&full_bar[0], 0);
        fetch(0);
        fragment(0, a[0]);
      }
      for (int kb = kb_begin; kb < kb_end; ++kb) {
        const uint64_t b_desc = make_kmajor_sw128_desc(smem_u32(smem + s * kStageBytes) + kWBytes);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          wgmma_fence();
          WgmmaRS<T, MPAD>::mma(acc, a[k & 1], b_desc + 2 * k);
          wgmma_commit();
          wgmma_wait<1>();  // step k - 1 has retired: its fragment buffer a[(k + 1) & 1] may be rewritten
          if (k == 0 && prev >= 0) release(prev);  // ... and with it the previous k-block's last MMA
          if (k < 3) {
            fragment(k + 1, a[(k + 1) & 1]);
          } else if (kb + 1 < kb_end) {
            const int sn = s + 1 == stages ? 0 : s + 1;
            mbar_wait_mma(&full_bar[sn], sn == 0 ? ph ^ 1 : ph);
            fetch(sn);
            fragment(0, a[0]);
          }
        }
        prev = s;
        if (++s == stages) {
          s = 0;
          ph ^= 1;
        }
      }
    }
    for (int kb = kb_begin; kb < kb_end && !W4 && !F8; ++kb) {
      mbar_wait_mma(&full_bar[s], ph);
      const uint32_t st = smem_u32(smem + s * kStageBytes);
      uint32_t a_addr = st + wg * (kWTileBytes / 2);  // 64 weight rows = 8 KB = eight whole swizzle atoms
      if constexpr (W8) {
        a_addr = smem_u32(wdq) + wg * (kWTileBytes / 2);
        dequant_w8_rows<T>(st + wg * (kW8TileBytes / 2), a_addr, sc);
        fence_proxy_async();  // generic-proxy stores -> async-proxy (wgmma) reads
        asm volatile("bar.sync %0, 128;" ::"r"(3 + wg) : "memory");
      }
      const uint64_t b_desc = make_kmajor_sw128_desc(st + kWBytes * (kDual ? 2 : 1));
      wgmma_fence();
      wgmma_kblock<T, MPAD>(acc, make_kmajor_sw128_desc(a_addr), b_desc);
      if constexpr (kDual) wgmma_kblock<T, MPAD>(acc2, make_kmajor_sw128_desc(a_addr + kWTileBytes), b_desc);
      wgmma_commit();
      if constexpr (W8) {
        wgmma_wait<0>();  // this k-block's MMAs have retired: its slot and the dequantized tile can be rewritten
        release(s);
      } else {
        wgmma_wait<1>();  // the previous k-block's MMAs have retired: its slot can be refilled
        if (prev >= 0) release(prev);
        prev = s;
      }
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
      const int rank = static_cast<int>(crank);
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
          const uint32_t peer = dsmem_map(part_local, static_cast<uint32_t>(s));
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
template <typename T, int MPAD, int EPI, int WQ = WQ_NONE>
static int launch_one(const CUtensorMap* tmW, const CUtensorMap* tmW2, const CUtensorMap* tmX, const GemmParams& p, cudaStream_t s,
                      const L2Prefetch* pf) {
  auto kern = skinny_gemm_wgmma<T, MPAD, EPI, WQ>;
  dim3 grid((p.N + kBlockN - 1) / kBlockN, p.splitk);
  const int stages = stage_count_for(MPAD, EPI, static_cast<int>(grid.x * grid.y), WQ);
  const int sbytes = WQ == WQ_INT8   ? stage_bytes_w8(MPAD)
                     : WQ == WQ_4BIT ? stage_bytes_w4(MPAD)
                     : WQ == WQ_FP8  ? stage_bytes_fp8(MPAD)
                                     : stage_bytes(MPAD, EPI);
  const int smem = stages * sbytes + (WQ == WQ_INT8 ? kW8DqBytes : 0) + kCtrlBytes + 1024;
  if (p.splitk > 8) return static_cast<int>(cudaErrorInvalidValue);  // portable cluster size
  // the accumulators are parked as (1|2) x MPAD x 128 fp32 partials (+ a 4 KB exchange strip) in the stage memory
  if (stages * sbytes < acc_tile_bytes(MPAD, EPI) + 4096)
    return static_cast<int>(cudaErrorInvalidValue);
  static bool configured_dev[64] = {};  // per device (the attribute is per device) and per instantiation
  const int cur_dev = current_device_index();
  if (cur_dev < 0) return static_cast<int>(cudaErrorInvalidDevice);
  if (!configured_dev[cur_dev]) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024 + kCtrlBytes + 1024);
    if (e != cudaSuccess) return static_cast<int>(e);
    configured_dev[cur_dev] = true;
  }
  L2Prefetch none;
  memset(&none, 0, sizeof(none));
  return static_cast<int>(launch_kc(kern, grid, dim3(kGemmThreads), static_cast<size_t>(smem), s, dim3(1, p.splitk, 1), *tmW,
                                    tmW2 ? *tmW2 : *tmW, *tmX, p, stages, pf ? *pf : none));
}

template <typename T, int MPAD>
static int launch_epi(int epi, const CUtensorMap* a, const CUtensorMap* b, const CUtensorMap* c, const GemmParams& p,
                      cudaStream_t s, const L2Prefetch* pf) {
  switch (epi) {
    case EPI_STORE: return launch_one<T, MPAD, EPI_STORE>(a, b, c, p, s, pf);
    case EPI_RESIDUAL: return launch_one<T, MPAD, EPI_RESIDUAL>(a, b, c, p, s, pf);
    case EPI_SWIGLU: return launch_one<T, MPAD, EPI_SWIGLU>(a, b, c, p, s, pf);
    case EPI_QKV_ROPE: return launch_one<T, MPAD, EPI_QKV_ROPE>(a, b, c, p, s, pf);
    case EPI_PARTIAL_F32: return launch_one<T, MPAD, EPI_PARTIAL_F32>(a, b, c, p, s, pf);
    case EPI_SWIGLU_IL: return launch_one<T, MPAD, EPI_SWIGLU_IL>(a, b, c, p, s, pf);
  }
  return static_cast<int>(cudaErrorInvalidValue);
}

// 256 activation rows per launch (prompt prefill: wgmma N = 256, the weights are streamed once per 256 prompt tokens instead of
// once per 64): only the epilogues the target's decoder layer needs
template <typename T>
static int launch_epi256(int epi, const CUtensorMap* a, const CUtensorMap* c, const GemmParams& p, cudaStream_t s, const L2Prefetch* pf) {
  switch (epi) {
    case EPI_RESIDUAL: return launch_one<T, 256, EPI_RESIDUAL>(a, nullptr, c, p, s, pf);
    case EPI_QKV_ROPE: return launch_one<T, 256, EPI_QKV_ROPE>(a, nullptr, c, p, s, pf);
    case EPI_SWIGLU_IL: return launch_one<T, 256, EPI_SWIGLU_IL>(a, nullptr, c, p, s, pf);
  }
  return static_cast<int>(cudaErrorInvalidValue);
}

int launch_gemm(int dtype, int mpad, int epi, const CUtensorMap* tmW, const CUtensorMap* tmW2, const CUtensorMap* tmX,
                const GemmParams& p_in, cudaStream_t s, const L2Prefetch* pf) {
  GemmParams p = p_in;
  if (p.splitk < 1 || p.m_rows > mpad) return static_cast<int>(cudaErrorInvalidValue);
  if (epi == EPI_SWIGLU || epi == EPI_SWIGLU_IL) {
    p.silu_lut = silu_lut(dtype, s);
    if (!p.silu_lut) return static_cast<int>(cudaErrorNotReady);
  }
  if (dtype == DT_BF16) {
    if (mpad == 16) return launch_epi<__nv_bfloat16, 16>(epi, tmW, tmW2, tmX, p, s, pf);
    if (mpad == 64) return launch_epi<__nv_bfloat16, 64>(epi, tmW, tmW2, tmX, p, s, pf);
    if (mpad == 256) return launch_epi256<__nv_bfloat16>(epi, tmW, tmX, p, s, pf);
  } else if (dtype == DT_FP16) {
    if (mpad == 16) return launch_epi<__half, 16>(epi, tmW, tmW2, tmX, p, s, pf);
    if (mpad == 64) return launch_epi<__half, 64>(epi, tmW, tmW2, tmX, p, s, pf);
    if (mpad == 256) return launch_epi256<__half>(epi, tmW, tmX, p, s, pf);
  }
  return static_cast<int>(cudaErrorInvalidValue);
}

// W8A16 / W4A16: the epilogues of the target's decoder layer (+ EPI_STORE for mpad 16 / 64); w2: W4's absmax map, FP8's scale map
template <typename T, int MPAD, int WQ>
static int launch_wq_epi(int epi, const CUtensorMap* w, const CUtensorMap* w2, const CUtensorMap* x, const GemmParams& p, cudaStream_t s,
                         const L2Prefetch* pf) {
  switch (epi) {
    case EPI_STORE:
      if constexpr (MPAD < 256) return launch_one<T, MPAD, EPI_STORE, WQ>(w, w2, x, p, s, pf);
      break;
    case EPI_RESIDUAL: return launch_one<T, MPAD, EPI_RESIDUAL, WQ>(w, w2, x, p, s, pf);
    case EPI_QKV_ROPE: return launch_one<T, MPAD, EPI_QKV_ROPE, WQ>(w, w2, x, p, s, pf);
    case EPI_SWIGLU_IL: return launch_one<T, MPAD, EPI_SWIGLU_IL, WQ>(w, w2, x, p, s, pf);
  }
  return static_cast<int>(cudaErrorInvalidValue);
}
template <int WQ>
static int launch_wq(int dtype, int mpad, int epi, const CUtensorMap* tmW, const CUtensorMap* tmW2, const CUtensorMap* tmX, GemmParams& p,
                     cudaStream_t s, const L2Prefetch* pf) {
  if (epi == EPI_SWIGLU_IL) {
    p.silu_lut = silu_lut(dtype, s);
    if (!p.silu_lut) return static_cast<int>(cudaErrorNotReady);
  }
  if (dtype == DT_BF16) {
    if (mpad == 16) return launch_wq_epi<__nv_bfloat16, 16, WQ>(epi, tmW, tmW2, tmX, p, s, pf);
    if (mpad == 64) return launch_wq_epi<__nv_bfloat16, 64, WQ>(epi, tmW, tmW2, tmX, p, s, pf);
    if (mpad == 256) return launch_wq_epi<__nv_bfloat16, 256, WQ>(epi, tmW, tmW2, tmX, p, s, pf);
  } else if (dtype == DT_FP16) {
    if (mpad == 16) return launch_wq_epi<__half, 16, WQ>(epi, tmW, tmW2, tmX, p, s, pf);
    if (mpad == 64) return launch_wq_epi<__half, 64, WQ>(epi, tmW, tmW2, tmX, p, s, pf);
    if (mpad == 256) return launch_wq_epi<__half, 256, WQ>(epi, tmW, tmW2, tmX, p, s, pf);
  }
  return static_cast<int>(cudaErrorInvalidValue);
}

int launch_gemm_w8(int dtype, int mpad, int epi, const CUtensorMap* tmW, const CUtensorMap* tmX, const GemmParams& p_in, cudaStream_t s,
                   const L2Prefetch* pf) {
  GemmParams p = p_in;
  if (p.splitk < 1 || p.m_rows > mpad || !p.w_scale) return static_cast<int>(cudaErrorInvalidValue);
  return launch_wq<WQ_INT8>(dtype, mpad, epi, tmW, nullptr, tmX, p, s, pf);
}

int launch_gemm_w4(int dtype, int mpad, int epi, const CUtensorMap* tmW, const CUtensorMap* tmA, const CUtensorMap* tmX, const GemmParams& p_in,
                   cudaStream_t s, const L2Prefetch* pf) {
  GemmParams p = p_in;
  if (p.splitk < 1 || p.m_rows > mpad || !tmA || p.K % kBlockK || (p.w4_quant != W4_NF4 && p.w4_quant != W4_FP4))
    return static_cast<int>(cudaErrorInvalidValue);
  return launch_wq<WQ_4BIT>(dtype, mpad, epi, tmW, tmA, tmX, p, s, pf);
}

int launch_gemm_fp8(int dtype, int mpad, int epi, const CUtensorMap* tmW, const CUtensorMap* tmS, const CUtensorMap* tmX, const GemmParams& p_in,
                    cudaStream_t s, const L2Prefetch* pf) {
  GemmParams p = p_in;
  if (p.splitk < 1 || p.m_rows > mpad || !tmS || p.K % 128 || p.N % kBlockN) return static_cast<int>(cudaErrorInvalidValue);
  return launch_wq<WQ_FP8>(dtype, mpad, epi, tmW, tmS, tmX, p, s, pf);
}

// one thread per source byte and per source scale of a 64-row group; see kernels.h for the layouts
__global__ void fp8_repack_kernel(const uint8_t* __restrict__ src, const float* __restrict__ src_scale, int nr, int K, int row0, int half,
                                  uint8_t* __restrict__ dst, float* __restrict__ dst_scale, int n_rows) {
  const int kc_n = K / 128;
  const long n_bytes = src ? static_cast<long>(nr) * K : 0, n_sc = src_scale ? static_cast<long>(nr / 64) * kc_n : 0;
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < n_bytes + n_sc; i += static_cast<long>(gridDim.x) * blockDim.x) {
    if (i >= n_bytes) {
      const int g = static_cast<int>((i - n_bytes) / kc_n), kc = static_cast<int>((i - n_bytes) % kc_n);  // 64-row group, 128-column block
      const int d = half >= 0 ? g * 128 + half * 64 : row0 + g * 64;
      if (d >= n_rows) continue;  // the launcher checks the destination; this keeps a bad call inside the buffers
      dst_scale[(static_cast<long>(d / kBlockN) * kc_n + kc) * 4 + (d % kBlockN) / 64] = src_scale[static_cast<long>(g / 2) * kc_n + kc];
      continue;
    }
    const int row = static_cast<int>(i / K), col = static_cast<int>(i % K);
    const int d = half >= 0 ? (row / 64) * 128 + half * 64 + row % 64 : row0 + row;
    if (d >= n_rows) continue;
    // element (r, kk) of the 128 x 64 tile: k16 step kk / 16, column j of it; the thread and register that hold it in the A fragment
    const int r = d % kBlockN, kk = col % kBlockK, step = kk / 16, j = kk % 16;
    const int tidx = (r / 64) * 128 + ((r % 64) / 16) * 32 + (r % 8) * 4 + (j % 8) / 2;
    const int reg = (j / 8) * 2 + (r % 16) / 8;
    const int o = (step / 2) * (kF8TileBytes / 2) + tidx * 16 + (step % 2) * 8 + reg * 2 + (j & 1);  // byte offset in the stage
    dst[static_cast<long>(d - r + o / kBlockK) * K + (col - kk) + o % kBlockK] = src[i];
  }
}
int launch_fp8_repack(const uint8_t* src, const float* src_scale, int nr, int K, int row0, int half, uint8_t* dst, float* dst_scale,
                      int n_rows, cudaStream_t s) {
  if (nr < 0 || nr % 128 || K <= 0 || K % 128 || n_rows % kBlockN || (src && !dst) || (src_scale && !dst_scale))
    return static_cast<int>(cudaErrorInvalidValue);
  if (half >= 0 ? 2L * nr > n_rows : (row0 < 0 || row0 % 64 || static_cast<long>(row0) + nr > n_rows))
    return static_cast<int>(cudaErrorInvalidValue);  // destination rows beyond the buffers
  const long total = (src ? static_cast<long>(nr) * K : 0) + (src_scale ? static_cast<long>(nr / 64) * (K / 128) : 0);
  if (total == 0) return 0;
  const int blocks = static_cast<int>(std::min<long>((total + 255) / 256, 8192));
  fp8_repack_kernel<<<blocks, 256, 0, s>>>(src, src_scale, nr, K, row0, half, dst, dst_scale, n_rows);
  return static_cast<int>(cudaGetLastError());
}

// one thread per source byte (nibbles) and per source absmax; see kernels.h for the layouts
__global__ void w4_repack_kernel(const uint8_t* __restrict__ src, const float* __restrict__ src_absmax, int nr, int K, int row0, int half,
                                 uint8_t* __restrict__ dst, float* __restrict__ dst_absmax, int n_pad) {
  const int kbytes = K / 2, num_kb = K / kBlockK;
  const long n_bytes = src ? static_cast<long>(nr) * kbytes : 0, n_abs = src_absmax ? static_cast<long>(nr) * num_kb : 0;
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < n_bytes + n_abs; i += static_cast<long>(gridDim.x) * blockDim.x) {
    const bool is_abs = i >= n_bytes;
    const long j = is_abs ? i - n_bytes : i;
    const int row = static_cast<int>(j / (is_abs ? num_kb : kbytes)), col = static_cast<int>(j % (is_abs ? num_kb : kbytes));
    const int d = half >= 0 ? (row / 64) * 128 + half * 64 + row % 64 : row0 + row;
    if (d >= n_pad) continue;  // the launcher checks the destination; this keeps a bad call inside the buffers
    if (is_abs) {
      dst_absmax[static_cast<long>(col) * n_pad + d] = src_absmax[j];
      continue;
    }
    // byte b of the k-block holds K columns 2b, 2b + 1: k16 step b / 8, fragment column pair b % 4 of the low (b % 8 < 4) or high half
    const int r = d % kBlockN, kb = col / 32, b = col % 32;
    const int tidx = (r / 64) * 128 + ((r % 64) / 16) * 32 + (r % 8) * 4 + (b % 4);
    const int reg = ((b % 8) / 4) * 2 + (r % 16) / 8;
    dst[(static_cast<long>(d / kBlockN) * num_kb + kb) * kW4TileBytes + tidx * 16 + (b / 8) * 4 + reg] = src[j];
  }
}
int launch_w4_repack(const uint8_t* src, const float* src_absmax, int nr, int K, int row0, int half, uint8_t* dst, float* dst_absmax,
                     int n_pad, cudaStream_t s) {
  if (nr < 0 || K <= 0 || K % kBlockK || n_pad % kBlockN || (src && !dst) || (src_absmax && !dst_absmax)) return static_cast<int>(cudaErrorInvalidValue);
  if (half >= 0 ? (nr % 64 || 2L * nr > n_pad) : (row0 < 0 || static_cast<long>(row0) + nr > n_pad))
    return static_cast<int>(cudaErrorInvalidValue);  // destination rows beyond the buffers
  const long total = (src ? static_cast<long>(nr) * (K / 2) : 0) + (src_absmax ? static_cast<long>(nr) * (K / kBlockK) : 0);
  if (total == 0) return 0;
  const int blocks = static_cast<int>(std::min<long>((total + 255) / 256, 8192));
  w4_repack_kernel<<<blocks, 256, 0, s>>>(src, src_absmax, nr, K, row0, half, dst, dst_absmax, n_pad);
  return static_cast<int>(cudaGetLastError());
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
