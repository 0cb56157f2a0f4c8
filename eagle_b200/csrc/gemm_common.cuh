// Tile constants and the epilogue device functions shared by the wgmma GEMM kernel (cluster split-K, gemm.cu) and the SIMT
// bring-up kernel.
#pragma once
#include "common.cuh"
#include "kernels.h"

namespace eb {

constexpr int kBlockN = 128;  // weight rows per tile == two wgmma M = 64 halves
constexpr int kBlockK = 64;   // K elements per stage == one 128-byte swizzle row
constexpr int kGemmThreads = 288;  // warps 0..7: two MMA warpgroups; warp 8 TMA
constexpr int kTmaWarp = 8;
constexpr int kWTileBytes = kBlockN * kBlockK * 2;
constexpr int kMaxStages = 12;
constexpr int kCtrlBytes = 1024;

__host__ __device__ constexpr int x_tile_bytes(int mpad) { return mpad * kBlockK * 2; }
__host__ __device__ constexpr int stage_bytes(int mpad, int epi) {
  return kWTileBytes * (epi == EPI_SWIGLU ? 2 : 1) + x_tile_bytes(mpad);
}
// fp32 accumulator tile(s) of one CTA staged in shared memory: [acc][MPAD][128]
__host__ __device__ constexpr int acc_tile_bytes(int mpad, int epi) { return (epi == EPI_SWIGLU ? 2 : 1) * mpad * kBlockN * 4; }
// W8A16 (int8 weights + one fp32 scale per row): a stage holds the int8 weight tile (128 rows x 64 bytes, unswizzled) and the
// X tile; the MMA warpgroups dequantize each stage into the model-dtype SWIZZLE_128B tile that follows the ring
constexpr int kW8TileBytes = kBlockN * kBlockK;
constexpr int kW8DqBytes = kWTileBytes;
__host__ __device__ constexpr int stage_bytes_w8(int mpad) { return kW8TileBytes + x_tile_bytes(mpad); }
// transformers' bnb 8-bit dequantization factor (integrations/bitsandbytes.py), as the fp32 value torch multiplies by
constexpr float kInv127 = 7.874015718698502e-3f;
// W4A16 (bitsandbytes nf4 / fp4 codes, one fp32 absmax per 64-element block of a row): a stage holds the 4 KB nibble tile in
// the engine's fragment order (launch_w4_repack), the tile's 128 absmax values of the k-block, padding to 1 KB so the X tile
// stays 1024-byte aligned, and the X tile
constexpr int kW4TileBytes = kBlockN * kBlockK / 2;
constexpr int kW4AbsBytes = kBlockN * 4;
constexpr int kW4WBytes = 5 * 1024;
__host__ __device__ constexpr int stage_bytes_w4(int mpad) { return kW4WBytes + x_tile_bytes(mpad); }
// W8A16 on FP8 (transformers' fine-grained e4m3, one fp32 scale per 128 x 128 block): a stage holds the 8 KB e4m3 tile, its bytes
// permuted within the tile into fragment order (launch_fp8_repack), the tile's two 64-row-group scales of the k-block (16 B, two used),
// padding to 1 KB so the X tile stays 1024-byte aligned, and the X tile
constexpr int kF8TileBytes = kBlockN * kBlockK;
constexpr int kF8ScaleBytes = 16;
constexpr int kF8WBytes = 9 * 1024;
__host__ __device__ constexpr int stage_bytes_fp8(int mpad) { return kF8WBytes + x_tile_bytes(mpad); }
// weight modes of skinny_gemm_wgmma
enum WeightQuant : int { WQ_NONE = 0, WQ_INT8 = 1, WQ_4BIT = 2, WQ_FP8 = 3 };

// number of SMs of the current device (the grids are sized to fill it)
inline int device_sm_count() {
  static int n[64] = {};
  const int dev = current_device_index();
  if (dev < 0) return 1;
  if (!n[dev]) {
    int v = 0;
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v < 1) v = 1;
    n[dev] = v;
  }
  return n[dev];
}

// T(silu(g)) of an already-rounded g through the 64K-entry table (kernels.h: silu_lut)
template <typename T> __device__ __forceinline__ float silu_rounded(const GemmParams& p, float g) {
  const T gt = DT<T>::from_f(g);
  const unsigned short bits = *reinterpret_cast<const unsigned short*>(&gt);
  return DT<T>::to_f(__ldg(reinterpret_cast<const T*>(p.silu_lut) + bits));
}

__device__ __forceinline__ int dyn(const int* st, DynInt d) { return (d.idx >= 0 ? st[d.idx] : 0) + d.add; }
__device__ __forceinline__ void epi_bar() { asm volatile("bar.sync 1, 128;" ::: "memory"); }

// ------------------------------------------------------------------------------------------------------------
// Epilogue pieces shared by the wgmma kernels and the SIMT bring-up kernel.  They are called by exactly 128
// threads; thread `row` (0..127) owns weight row n = n_tile*128 + row and processes the activation rows in
// chunks of 16:  acc[j] is the fp32 accumulator of activation row m0 + j  (acc2: the `up` tile for SwiGLU).
// ------------------------------------------------------------------------------------------------------------
template <int MPAD, int EPI>
__device__ __forceinline__ void partial_store(const GemmParams& p, const float (&acc)[16], const float (&acc2)[16], int m0,
                                              int m_valid, int n, int split) {
  constexpr int kAcc = (EPI == EPI_SWIGLU) ? 2 : 1;
  const long n_ws = static_cast<long>(gridDim.x) * kBlockN;
  float* my = p.ws + (static_cast<long>(split) * kAcc * MPAD) * n_ws + n;
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int m = m0 + j;
    if (m < m_valid) {
      __stcg(my + static_cast<long>(m) * n_ws, acc[j]);
      if constexpr (EPI == EPI_SWIGLU) __stcg(my + static_cast<long>(MPAD + m) * n_ws, acc2[j]);
    }
  }
}
template <int MPAD, int EPI>
__device__ __forceinline__ void partial_reduce(const GemmParams& p, float (&acc)[16], float (&acc2)[16], int m0, int m_valid,
                                               int n) {
  constexpr int kAcc = (EPI == EPI_SWIGLU) ? 2 : 1;
  const long n_ws = static_cast<long>(gridDim.x) * kBlockN;
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int m = m0 + j;
    float a = 0.f, b = 0.f;
    if (m < m_valid) {
      for (int s = 0; s < p.splitk; ++s) {
        const float* src = p.ws + (static_cast<long>(s) * kAcc * MPAD) * n_ws + n;
        a += __ldcg(src + static_cast<long>(m) * n_ws);
        if constexpr (EPI == EPI_SWIGLU) b += __ldcg(src + static_cast<long>(MPAD + m) * n_ws);
      }
    }
    acc[j] = a;
    acc2[j] = b;
  }
}

template <typename T, int EPI>
__device__ __forceinline__ void final_chunk(const GemmParams& p, const float (&acc)[16], const float (&acc2)[16], int m0,
                                            int m_valid_in, int row, int n_tile, uint8_t* scratch, int nrows = 16) {
  const int m_valid = min(m_valid_in, m0 + nrows);  // rows [m0, m0 + nrows) of this pass
  using D = DT<T>;
  const int n = n_tile * kBlockN + row;
  if constexpr (EPI == EPI_STORE) {
    if (n < p.N) {
      T* out = reinterpret_cast<T*>(p.out) + n;
      const float bias = p.bias ? D::to_f(reinterpret_cast<const T*>(p.bias)[n]) : 0.f;
#pragma unroll
      for (int j = 0; j < 16; ++j)
        if (m0 + j < m_valid) out[static_cast<long>(m0 + j) * p.ld_out] = D::from_f(acc[j] + bias);
    }
  } else if constexpr (EPI == EPI_PARTIAL_F32) {
    if (n < p.N) {
      float* out = reinterpret_cast<float*>(p.out) + n;
#pragma unroll
      for (int j = 0; j < 16; ++j)
        if (m0 + j < m_valid) out[static_cast<long>(m0 + j) * p.ld_out] = acc[j];
    }
  } else if constexpr (EPI == EPI_RESIDUAL) {
    if (n < p.N) {
      T* out = reinterpret_cast<T*>(p.out) + n;
      const T* res = reinterpret_cast<const T*>(p.res) + n;
#pragma unroll
      for (int j = 0; j < 16; ++j)
        if (m0 + j < m_valid) {
          const float r = D::to_f(res[static_cast<long>(m0 + j) * p.ld_res]);
          out[static_cast<long>(m0 + j) * p.ld_out] = D::from_f(rnd<T>(acc[j]) + r);
        }
    }
  } else if constexpr (EPI == EPI_SWIGLU) {
    if (n < p.N) {
      T* out = reinterpret_cast<T*>(p.out) + n;
#pragma unroll
      for (int j = 0; j < 16; ++j)
        if (m0 + j < m_valid) {
          const float g = rnd<T>(acc[j]);
          const float sg = silu_rounded<T>(p, g);
          const float u = rnd<T>(acc2[j]);
          out[static_cast<long>(m0 + j) * p.ld_out] = D::from_f(sg * u);
        }
    }
  } else if constexpr (EPI == EPI_SWIGLU_IL) {
    // rows 0..63 of the tile are gate rows, rows 64..127 the up rows of the same 64 outputs: the up half hands its
    // accumulators to the gate half through shared memory; same rounding points as EPI_SWIGLU
    float* xch = reinterpret_cast<float*>(scratch);  // [16][64]
    if (row >= 64) {
#pragma unroll
      for (int j = 0; j < 16; ++j) xch[j * 64 + (row - 64)] = acc[j];
    }
    epi_bar();
    const int n_out = n_tile * 64 + row;
    if (row < 64 && 2 * n_out < p.N) {
      T* out = reinterpret_cast<T*>(p.out) + n_out;
#pragma unroll
      for (int j = 0; j < 16; ++j)
        if (m0 + j < m_valid) {
          const float g = rnd<T>(acc[j]);
          const float sg = silu_rounded<T>(p, g);
          const float u = rnd<T>(xch[j * 64 + row]);
          out[static_cast<long>(m0 + j) * p.ld_out] = D::from_f(sg * u);
        }
    }
    epi_bar();  // xch is rewritten by the next chunk
  } else {  // EPI_QKV_ROPE: tile == head (head_dim 128); rotate_half pairs d <-> d^64 live in other warps
    T* xch = reinterpret_cast<T*>(scratch);  // [16][128]
#pragma unroll
    for (int j = 0; j < 16; ++j) xch[j * kBlockN + row] = D::from_f(acc[j]);
    epi_bar();
    const int head = n_tile;
    const int d = row;
    const long kv0 = dyn(p.st, p.kv_base);
    if (head < p.n_q_heads + p.n_kv_heads) {  // q or k: apply rope
      const T* cosT = reinterpret_cast<const T*>(p.rope_cos);
      const T* sinT = reinterpret_cast<const T*>(p.rope_sin);
      const int pos0 = dyn(p.st, p.pos_base);
      T* dst;
      long ld;
      if (head < p.n_q_heads) {
        dst = reinterpret_cast<T*>(p.q_out) + static_cast<long>(head) * 128 + d;
        ld = static_cast<long>(p.n_q_heads) * 128;
      } else {
        dst = reinterpret_cast<T*>(p.k_cache) + (static_cast<long>(head - p.n_q_heads) * p.kv_cap + kv0) * 128 + d;
        ld = 128;
      }
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int m = m0 + j;
        if (m < m_valid) {
          const int pos = pos0 + (p.pos_arr ? p.pos_arr[m] : 0) + p.pos_mstride * m;
          const float c = D::to_f(cosT[static_cast<long>(pos) * 64 + (d & 63)]);
          const float sn = D::to_f(sinT[static_cast<long>(pos) * 64 + (d & 63)]);
          const float x = D::to_f(xch[j * kBlockN + d]);
          const float y = D::to_f(xch[j * kBlockN + (d ^ 64)]);
          const float rot = (d < 64) ? -y : y;
          dst[static_cast<long>(m) * ld] = D::from_f(rnd<T>(x * c) + rnd<T>(rot * sn));
        }
      }
    } else {
      T* dst = reinterpret_cast<T*>(p.v_cache) +
               (static_cast<long>(head - p.n_q_heads - p.n_kv_heads) * p.kv_cap + kv0) * 128 + d;
#pragma unroll
      for (int j = 0; j < 16; ++j)
        if (m0 + j < m_valid) dst[static_cast<long>(m0 + j) * 128] = xch[j * kBlockN + d];
    }
    epi_bar();  // xch is rewritten by the next chunk
  }
}

// returns true when this CTA must run the final epilogue (always for splitk == 1, else only the last arrival)
__device__ __forceinline__ bool splitk_arrive(const GemmParams& p, int n_tile, int row, uint8_t* scratch) {
  __threadfence();
  epi_bar();
  int* flag = reinterpret_cast<int*>(scratch);
  if (row == 0) {
    const int old = atomicAdd(p.counters + n_tile, 1);
    const int last = (old == p.splitk - 1);
    if (last) p.counters[n_tile] = 0;  // self-reset for the next launch on this stream
    *flag = last;
  }
  epi_bar();
  const int is_last = *reinterpret_cast<volatile int*>(flag);
  epi_bar();  // scratch is reused by the final epilogue
  if (is_last) __threadfence();
  return is_last != 0;
}

__device__ __forceinline__ int valid_rows(const GemmParams& p) {
  int m_valid = p.m_rows;
  if (p.m_idx >= 0) m_valid = min(m_valid, p.st[p.m_idx]);
  return m_valid;
}

}  // namespace eb
