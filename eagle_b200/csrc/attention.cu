// Tree-masked attention over a preallocated KV cache (target verify pass, draft stable pass, draft tree levels,
// chunked prefill).  Restates modeling_llama_kv.py:719-743 / cnets.py:292-312 with the reference's rounding points:
//     S = T(Q K^T); S = T(S / sqrt(d)); masked softmax in fp32; P = T(softmax); O = T(P V)
// so the result matches the eager reference up to fp32 summation order (no online-softmax rescaling).
//
// A query row r sees every cache row in the committed prefix [0, n_ctx) and tree column j (cache row n_ctx + j)
// iff bit j of its 128-bit ancestor mask is set -- the reference builds a dense fp32 [T, N+T] mask on the host
// each step (modeling_llama_kv.py:1010-1043); here the mask is two 64-bit words per row produced on device.
//
// KV split: for long contexts KS = 2 or 4 CTAs of a thread-block CLUSTER (1,1,KS) share one (head group, row tile); each
// sweeps 1/KS of the KV tiles, the row statistics (max, sum) and the partial outputs are exchanged through distributed
// shared memory (mapa + ld.shared::cluster), so both sweeps shrink KS-fold while P keeps the reference's rounding point.
// Work split: one CTA per (group of HPC query heads sharing a kv head, 16-row query tile), 8 warps; the 8/HPC warps
// of a head split each K tile's columns (phase 1) and the output dims (phase 3).  With GQA a K/V tile fetched once
// per CTA serves HPC heads.  The score strip S[HPC*16, kv] lives in shared memory (two-phase exact softmax).
// K tiles then V tiles stream through ONE 4-deep shared-memory ring filled by TMA (cp.async.bulk.tensor.2d, two 64x64-element
// SWIZZLE_128B boxes per 64-row tile, completion on an mbarrier) issued by a dedicated producer warp; the eight consumer
// warps release a slot through a second mbarrier, so there is no CTA-wide barrier per tile and the L2 latency of a tile is
// hidden behind the previous tiles' MMAs.  Both matmuls run on the
// tensor cores via mma.sync m16n8k16 + ldmatrix (the problem is ~1 GFLOP per layer and latency bound; the weight-streaming
// GEMMs are the wgmma kernels).
#include <stdlib.h>

#include "common.cuh"
#include "kernels.h"

namespace eb {

constexpr int kHd = 128;       // head_dim of every supported target
constexpr int kRowPad = 136;   // padded smem row (elements): conflict-free fragment loads
constexpr int kKvTile = 64;
constexpr int kRing = 5;       // tile buffers: tile i+3 is requested while tile i is consumed, into the slot tile i-2 left

template <typename T> struct MmaOp;
template <> struct MmaOp<__nv_bfloat16> {
  static __device__ __forceinline__ void run(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  }
};
template <> struct MmaOp<__half> {
  static __device__ __forceinline__ void run(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  }
};

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(src_bytes)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t (&r)[4], const void* smem_row) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_u32(smem_row)));
}

template <typename T> __device__ __forceinline__ uint32_t pack2(float lo, float hi) {
  typename DT<T>::type a = DT<T>::from_f(lo), b = DT<T>::from_f(hi);
  uint16_t ua = *reinterpret_cast<uint16_t*>(&a), ub = *reinterpret_cast<uint16_t*>(&b);
  return static_cast<uint32_t>(ua) | (static_cast<uint32_t>(ub) << 16);
}

template <typename T> __device__ __forceinline__ float2 ld2(const T* p);
template <> __device__ __forceinline__ float2 ld2<__nv_bfloat16>(const __nv_bfloat16* p) {
  return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p));
}
template <> __device__ __forceinline__ float2 ld2<__half>(const __half* p) { return __half22float2(*reinterpret_cast<const __half2*>(p)); }

__device__ __forceinline__ bool visible(int c, int n_ctx, uint64_t m0, uint64_t m1) {
  const int j = c - n_ctx;
  return (j < 0) || ((j < 64) ? ((m0 >> j) & 1ull) : ((m1 >> (j - 64)) & 1ull));
}

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ unsigned long long gtimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

constexpr int kWarps = 8;                 // consumer warps
constexpr int kThreads = kWarps * 32;
constexpr int kTileBytes = kKvTile * kHd * 2;  // 16 KB: [2 column halves][64 rows][128 B], each half one SWIZZLE_128B box
// byte offset of element (row r, column c) inside a ring tile
__device__ __forceinline__ int sw_off(int r, int c) {
  const int cc = c & 63;
  return (c >> 6) * (kKvTile * 128) + r * 128 + ((((cc >> 3) ^ (r & 7)) << 4) | ((cc & 7) << 1));
}

template <typename T, int HPC>
__global__ void __launch_bounds__(kThreads) tree_attention_kernel(const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                                                                  const AttnParams p, int kv_stride, int kvs) {
  using D = DT<T>;
  constexpr int CS = kWarps / HPC;         // warps sharing one query head (column / output-dim split)
  constexpr int NT1 = (kKvTile / CS) / 8;  // n8 score tiles per warp per kv tile
  constexpr int ND = (kHd / CS) / 8;       // n8 output tiles per warp (even)
  constexpr int RPW = (16 + CS - 1) / CS;  // softmax rows of the head handled by this warp
  static_assert(NT1 >= 1 && ND >= 2 && ND % 2 == 0, "bad split");
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[kRing], empty_bar[kRing];
  uint8_t* sRing = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));  // [kRing][kTileBytes]
  T* sQ = reinterpret_cast<T*>(sRing + kRing * kTileBytes);  // [HPC*16][kRowPad]
  T* sS = sQ + HPC * 16 * kRowPad;                      // [HPC*16][kv_stride]  (this CTA's slice of the KV columns)
  float* sStat = reinterpret_cast<float*>(sS + HPC * 16 * kv_stride);  // [2][HPC*16]: row max, row sum of this slice; then [kvs][2][HPC*16] peer copies
  float* sPO = reinterpret_cast<float*>(sRing);         // [HPC*16][128] partial outputs (aliases the ring after the sweeps)

  pdl_launch_dependents();
  if (threadIdx.x == 0) {
    // weights are immutable: prefetching them needs no dependency wait
    const unsigned long long n_cta = static_cast<unsigned long long>(gridDim.x) * gridDim.y * gridDim.z;
    const unsigned long long cta = blockIdx.x + static_cast<unsigned long long>(gridDim.x) * (blockIdx.y + static_cast<unsigned long long>(gridDim.y) * blockIdx.z);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      if (!p.pf_ptr[r] || !p.pf_bytes[r]) continue;
      const unsigned long long per = ((p.pf_bytes[r] + n_cta - 1) / n_cta + 4095ull) & ~4095ull;
      unsigned long long off = cta * per;
      const unsigned long long end = min(p.pf_bytes[r], off + per);
      for (; off < end; off += 16384ull) {
        const unsigned int sz = static_cast<unsigned int>(min(16384ull, end - off)) & ~15u;
        if (sz)
          asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(reinterpret_cast<const char*>(p.pf_ptr[r]) + off), "r"(sz) : "memory");
      }
    }
  }
  unsigned long long* tr = nullptr;
  unsigned long long t_launch = 0;
  if (p.trace && threadIdx.x == 0) {
    tr = p.trace + 16ull * (blockIdx.x + gridDim.x * (blockIdx.y + gridDim.y * blockIdx.z));
    t_launch = gtimer();
  }
  pdl_wait();  // Q, the K/V rows appended by the preceding GEMM and the device state all come from earlier kernels
  if (tr) {
    tr[0] = t_launch;  // nothing is written to global memory ahead of the wait
    tr[1] = gtimer();
  }
  const int head0 = blockIdx.x * HPC;
  const int kvh = head0 / (p.n_heads / p.n_kv_heads);
  const int row0 = blockIdx.y * 16;
  int rows_valid = p.rows;
  if (p.rows_idx >= 0) rows_valid = min(rows_valid, p.st[p.rows_idx]);
  if (row0 >= rows_valid) return;  // uniform over the whole cluster (same blockIdx.y)
  const int n_ctx = (p.n_ctx.idx >= 0 ? p.st[p.n_ctx.idx] : 0) + p.n_ctx.add;
  const int kv_len = min(n_ctx + p.n_tree, p.max_kv);
  const int n_tiles_all = (kv_len + kKvTile - 1) / kKvTile;
  const int rank = (kvs > 1) ? static_cast<int>(cluster_ctarank()) : 0;
  const int tiles_per = (n_tiles_all + kvs - 1) / kvs;
  const int t_begin = min(n_tiles_all, rank * tiles_per);
  const int n_tiles = min(n_tiles_all, t_begin + tiles_per) - t_begin;  // this CTA's KV tiles (may be 0)
  const int col0 = t_begin * kKvTile;                                    // global KV row of local column 0
  const int total = 2 * n_tiles;  // K tiles then V tiles through one ring

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int hl = warp % HPC;     // local head of this warp
  const int part = warp / HPC;   // which column / dim slice of that head
  const T* q = reinterpret_cast<const T*>(p.q);
  const T* kplane = reinterpret_cast<const T*>(p.k_cache) + static_cast<long>(kvh) * p.kv_cap * kHd;
  const T* vplane = reinterpret_cast<const T*>(p.v_cache) + static_cast<long>(kvh) * p.kv_cap * kHd;
  const long ldq = static_cast<long>(p.n_heads) * kHd;

  // ---- TMA producer (thread 0): K tiles then V tiles of this CTA's KV slice, one request = two 64x64 SWIZZLE_128B boxes.
  // Rows at or beyond kv_len hold whatever the cache holds (finite values): their score columns are masked out and their P is 0.
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    for (int i = 0; i < kRing; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], kWarps);
    }
    fence_barrier_init();
  }
  __syncthreads();
  const int plane_row0 = kvh * static_cast<int>(p.kv_cap);
  auto produce = [&](int j) {
    if (j >= total) return;
    const int slot = j % kRing;
    if (j >= kRing) mbar_wait(&empty_bar[slot], static_cast<uint32_t>((j / kRing) - 1) & 1u);
    const bool is_k = j < n_tiles;
    const int r0 = plane_row0 + (t_begin + (is_k ? j : j - n_tiles)) * kKvTile;
    uint8_t* dst = sRing + slot * kTileBytes;
    mbar_arrive_expect_tx(&full_bar[slot], kTileBytes);
    tma_load_2d(dst, is_k ? &tmK : &tmV, &full_bar[slot], 0, r0, kEvictNormal);
    tma_load_2d(dst + kKvTile * 128, is_k ? &tmK : &tmV, &full_bar[slot], 64, r0, kEvictNormal);
  };
  if (threadIdx.x == 0) {
#pragma unroll
    for (int j = 0; j < 3; ++j) produce(j);
  }

  // ---- Q tiles -> smem (rows beyond rows_valid are zero) ----
  for (int c = threadIdx.x; c < HPC * 16 * (kHd / 8); c += kThreads) {
    const int r = c >> 4, ch = c & 15;
    const int h = r >> 4, rr = r & 15;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (row0 + rr < rows_valid) v = *reinterpret_cast<const uint4*>(q + (row0 + rr) * ldq + (head0 + h) * kHd + ch * 8);
    *reinterpret_cast<uint4*>(sQ + r * kRowPad + ch * 8) = v;
  }
  __syncthreads();
  uint32_t qa[8][4];
  {
    const T* qb = sQ + hl * 16 * kRowPad;
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      qa[kk][0] = *reinterpret_cast<const uint32_t*>(qb + g * kRowPad + kk * 16 + t * 2);
      qa[kk][1] = *reinterpret_cast<const uint32_t*>(qb + (g + 8) * kRowPad + kk * 16 + t * 2);
      qa[kk][2] = *reinterpret_cast<const uint32_t*>(qb + g * kRowPad + kk * 16 + 8 + t * 2);
      qa[kk][3] = *reinterpret_cast<const uint32_t*>(qb + (g + 8) * kRowPad + kk * 16 + 8 + t * 2);
    }
  }
  T* sS_head = sS + hl * 16 * kv_stride;
  // S / sqrt(d) like the reference's `attn_weights / math.sqrt(head_dim)`: q = x*r, then one FMA residual correction.
  // For every bf16 and fp16 operand this three-instruction sequence is bit-identical to the IEEE fp32 division
  // (checked exhaustively over all mantissas, tools/check_div.py) and avoids four slow-path divisions per MMA tile.
  const float kSqrtD = 11.313708498984761f;
  const float kRcpSqrtD = 1.0f / 11.313708498984761f;
  auto div_sqrt_d = [&](float x) {
    const float q0 = x * kRcpSqrtD;
    return fmaf(fmaf(-q0, kSqrtD, x), kRcpSqrtD, q0);
  };

  if (tr) tr[2] = gtimer();
  // ================= sweep 1: S = T(T(Q K^T) / sqrt(d)) over this CTA's K tiles =================
  for (int i = 0; i < n_tiles; ++i) {
    if (threadIdx.x == 0) produce(i + 3);  // into the slot tile i-2 released two iterations ago
    mbar_wait(&full_bar[i % kRing], static_cast<uint32_t>(i / kRing) & 1u);
    const uint8_t* tile = sRing + (i % kRing) * kTileBytes;
    float c[NT1][4];
#pragma unroll
    for (int nt = 0; nt < NT1; ++nt) c[nt][0] = c[nt][1] = c[nt][2] = c[nt][3] = 0.f;
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {  // k outer: consecutive MMAs hit independent accumulators
#pragma unroll
      for (int nt = 0; nt < NT1; ++nt) {
        const int krow = part * (kKvTile / CS) + nt * 8 + g;
        const uint32_t b0 = *reinterpret_cast<const uint32_t*>(tile + sw_off(krow, kk * 16 + t * 2));
        const uint32_t b1 = *reinterpret_cast<const uint32_t*>(tile + sw_off(krow, kk * 16 + 8 + t * 2));
        MmaOp<T>::run(c[nt], qa[kk], b0, b1);
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[i % kRing]);  // this warp is done with the tile
#pragma unroll
    for (int nt = 0; nt < NT1; ++nt) {
      const int col = i * kKvTile + part * (kKvTile / CS) + nt * 8 + t * 2;
      *reinterpret_cast<uint32_t*>(sS_head + g * kv_stride + col) = pack2<T>(div_sqrt_d(rnd<T>(c[nt][0])), div_sqrt_d(rnd<T>(c[nt][1])));
      *reinterpret_cast<uint32_t*>(sS_head + (g + 8) * kv_stride + col) = pack2<T>(div_sqrt_d(rnd<T>(c[nt][2])), div_sqrt_d(rnd<T>(c[nt][3])));
    }
  }
  __syncthreads();
  if (tr) tr[3] = gtimer();

  // ================= softmax: row statistics of the local slice, exchanged over the cluster =================
  // exp(s - max) as ex2.approx((s - max) * log2e) and p = e * (1/sum): each within ~2 fp32 ulp of the reference's fp32
  // softmax (whose CPU and CUDA implementations differ from each other by as much); after the rounding of P to the model
  // dtype this moves ~1e-4 of the probabilities by one ulp.  With a KV split the row sum is assembled from the slices'
  // sums rescaled to the common maximum (again fp32-ulp-level).
  const float kLog2e = 1.4426950408889634f;
  static_assert(16 % CS == 0, "rows of a head must divide evenly over its warps");
  const int local_len = min(kv_len - col0, n_tiles * kKvTile);  // valid local columns (<= 0 when this CTA has no tiles)
  const int ctx_local = max(0, min(n_ctx - col0, local_len));   // local columns of the always-visible committed prefix
  const int kv_padded = n_tiles * kKvTile;
  const int nvec = kv_padded / 8;  // the strip is walked in 16-byte vectors of 8 columns; a warp's RPW rows are independent
                                   // chains issued back to back (latency hiding), one vector per lane and row per step
  uint64_t rm0[RPW], rm1[RPW];
  const T* srow0 = sS_head + part * RPW * kv_stride;
#pragma unroll
  for (int rr = 0; rr < RPW; ++rr) {
    const int grow = row0 + part * RPW + rr;
    uint64_t m0 = 0ull, m1 = 0ull;
    if (p.mask) {
      m0 = (grow < rows_valid) ? p.mask[grow * 2] : 0ull;
      m1 = (grow < rows_valid) ? p.mask[grow * 2 + 1] : 0ull;
    } else {  // causal inside the block of new rows
      m0 = (grow >= 63) ? ~0ull : ((1ull << (grow + 1)) - 1ull);
      m1 = (grow >= 127) ? ~0ull : (grow >= 64 ? ((1ull << (grow - 63)) - 1ull) : 0ull);
    }
    rm0[rr] = m0;
    rm1[rr] = m1;
  }
  // bit e set: local column c0 + e is a real column this row may attend to.  Tree column j = col0 + c - n_ctx; the eight
  // ancestor bits are one funnel shift of the 128-bit mask, columns of the committed prefix (j < 0) are always visible
  auto ok_bits = [&](int c0, uint64_t m0, uint64_t m1) -> uint32_t {
    if (c0 + 8 <= ctx_local) return 0xffu;
    if (c0 >= local_len) return 0u;
    const int j0 = col0 + c0 - n_ctx;
    uint32_t vis;
    if (j0 <= -8) {
      vis = 0xffu;
    } else if (j0 < 0) {
      vis = (static_cast<uint32_t>(m0 << (-j0)) | ((1u << (-j0)) - 1u)) & 0xffu;
    } else if (j0 < 64) {
      uint64_t w = m0 >> j0;
      if (j0 > 56) w |= m1 << (64 - j0);
      vis = static_cast<uint32_t>(w) & 0xffu;
    } else if (j0 < 128) {
      vis = static_cast<uint32_t>(m1 >> (j0 - 64)) & 0xffu;
    } else {
      vis = 0u;
    }
    const int nvalid = local_len - c0;
    if (nvalid < 8) vis &= (1u << nvalid) - 1u;
    return vis;
  };
  auto unpack8 = [&](const uint4& raw, float (&f)[8]) {
    const T* e2 = reinterpret_cast<const T*>(&raw);
#pragma unroll
    for (int j = 0; j < 8; j += 2) {
      const float2 v = ld2<T>(e2 + j);
      f[j] = v.x;
      f[j + 1] = v.y;
    }
  };
  float mx[RPW], sum[RPW];
#pragma unroll
  for (int rr = 0; rr < RPW; ++rr) {
    mx[rr] = -INFINITY;
    sum[rr] = 0.f;
  }
  for (int v = lane; v < nvec; v += 32) {
#pragma unroll
    for (int rr = 0; rr < RPW; ++rr) {
      const uint4 raw = *reinterpret_cast<const uint4*>(srow0 + rr * kv_stride + v * 8);
      const uint32_t ok = ok_bits(v * 8, rm0[rr], rm1[rr]);
      float f[8];
      unpack8(raw, f);
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if ((ok >> j) & 1u) mx[rr] = fmaxf(mx[rr], f[j]);
    }
  }
#pragma unroll
  for (int rr = 0; rr < RPW; ++rr) mx[rr] = warp_max(mx[rr]);
  for (int v = lane; v < nvec; v += 32) {
#pragma unroll
    for (int rr = 0; rr < RPW; ++rr) {
      if (mx[rr] == -INFINITY) continue;  // warp-uniform
      const uint4 raw = *reinterpret_cast<const uint4*>(srow0 + rr * kv_stride + v * 8);
      const uint32_t ok = ok_bits(v * 8, rm0[rr], rm1[rr]);
      const float mxs = mx[rr] * kLog2e;
      float f[8];
      unpack8(raw, f);
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if ((ok >> j) & 1u) sum[rr] += fast_exp2(fmaf(f[j], kLog2e, -mxs));
    }
  }
#pragma unroll
  for (int rr = 0; rr < RPW; ++rr) {
    sum[rr] = warp_sum(sum[rr]);
    if (lane == 0) {
      sStat[hl * 16 + part * RPW + rr] = mx[rr];
      sStat[HPC * 16 + hl * 16 + part * RPW + rr] = sum[rr];
    }
  }
  if (tr) tr[8] = gtimer();
  if (kvs > 1) cluster_sync_all(); else __syncthreads();
  if (tr) tr[4] = gtimer();
  if (kvs > 1) {
    // One remote round trip for the whole CTA: thread i fetches one peer statistic (kvs x 2 x HPC*16 floats <= 256) into
    // local shared memory; the per-row combination below then reads local memory only.
    float* sPeer = sStat + 2 * HPC * 16;  // [kvs][2][HPC*16]
    const int n_stat = kvs * 2 * HPC * 16;
    for (int i = threadIdx.x; i < n_stat; i += kThreads) {
      const int s2 = i / (2 * HPC * 16), w = i % (2 * HPC * 16);
      sPeer[i] = dsmem_ld_f32(dsmem_map(smem_u32(&sStat[w]), s2));
    }
    __syncthreads();
  }
  if (tr) tr[9] = gtimer();
  float inv[RPW], mxs[RPW];
#pragma unroll
  for (int rr = 0; rr < RPW; ++rr) {
    const int r = part * RPW + rr;
    float gmax = -INFINITY, gsum = 0.f;
    if (kvs > 1) {
      const float* sPeer = sStat + 2 * HPC * 16;
      for (int s2 = 0; s2 < kvs; ++s2) gmax = fmaxf(gmax, sPeer[s2 * 2 * HPC * 16 + hl * 16 + r]);
      for (int s2 = 0; s2 < kvs; ++s2) {
        const float ms = sPeer[s2 * 2 * HPC * 16 + hl * 16 + r];
        const float ls = sPeer[s2 * 2 * HPC * 16 + HPC * 16 + hl * 16 + r];
        if (ms > -INFINITY) gsum += ls * fast_exp2((ms - gmax) * kLog2e);
      }
    } else {
      gmax = sStat[hl * 16 + r];
      gsum = sStat[HPC * 16 + hl * 16 + r];
    }
    inv[rr] = (gmax > -INFINITY) ? __frcp_rn(gsum) : 0.f;
    mxs[rr] = (gmax > -INFINITY) ? gmax * kLog2e : 0.f;
  }
  T* prow0 = sS_head + part * RPW * kv_stride;
  for (int v = lane; v < nvec; v += 32) {
#pragma unroll
    for (int rr = 0; rr < RPW; ++rr) {
      T* ptr = prow0 + rr * kv_stride + v * 8;
      const uint4 raw = *reinterpret_cast<const uint4*>(ptr);
      const uint32_t ok = ok_bits(v * 8, rm0[rr], rm1[rr]);
      float f[8];
      unpack8(raw, f);
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = ((ok >> j) & 1u) ? fast_exp2(fmaf(f[j], kLog2e, -mxs[rr])) * inv[rr] : 0.f;
      uint4 outv;
      outv.x = pack2<T>(f[0], f[1]);
      outv.y = pack2<T>(f[2], f[3]);
      outv.z = pack2<T>(f[4], f[5]);
      outv.w = pack2<T>(f[6], f[7]);
      *reinterpret_cast<uint4*>(ptr) = outv;
    }
  }

  if (tr) tr[5] = gtimer();
  // ================= sweep 2: O += P V over this CTA's V tiles =================
  float o[ND][4];
#pragma unroll
  for (int i = 0; i < ND; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) o[i][j] = 0.f;
  __syncthreads();  // publishes P to the warps sharing this head
  for (int i = n_tiles; i < total; ++i) {
    if (threadIdx.x == 0) produce(i + 3);
    mbar_wait(&full_bar[i % kRing], static_cast<uint32_t>(i / kRing) & 1u);
    const uint8_t* tile = sRing + (i % kRing) * kTileBytes;
    const int vt = i - n_tiles;
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t pa[4];
      const int col = vt * kKvTile + kk * 16 + t * 2;
      pa[0] = *reinterpret_cast<const uint32_t*>(sS_head + g * kv_stride + col);
      pa[1] = *reinterpret_cast<const uint32_t*>(sS_head + (g + 8) * kv_stride + col);
      pa[2] = *reinterpret_cast<const uint32_t*>(sS_head + g * kv_stride + col + 8);
      pa[3] = *reinterpret_cast<const uint32_t*>(sS_head + (g + 8) * kv_stride + col + 8);
#pragma unroll
      for (int np = 0; np < ND / 2; ++np) {  // pairs of n8 tiles
        uint32_t vb[4];
        const int mrow = kk * 16 + ((lane >> 3) & 1) * 8 + (lane & 7);
        const int mcol = part * (kHd / CS) + np * 16 + (lane >> 4) * 8;
        ldmatrix_x4_trans(vb, tile + sw_off(mrow, mcol));
        MmaOp<T>::run(o[np * 2], pa, vb[0], vb[1]);
        MmaOp<T>::run(o[np * 2 + 1], pa, vb[2], vb[3]);
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[i % kRing]);
  }

  if (tr) tr[6] = gtimer();
  T* out = reinterpret_cast<T*>(p.out);
  if (kvs == 1) {
#pragma unroll
    for (int nt = 0; nt < ND; ++nt) {
      const int dcol = (head0 + hl) * kHd + part * (kHd / CS) + nt * 8 + t * 2;
      if (row0 + g < rows_valid)
        *reinterpret_cast<uint32_t*>(out + (row0 + g) * ldq + dcol) = pack2<T>(o[nt][0], o[nt][1]);
      if (row0 + g + 8 < rows_valid)
        *reinterpret_cast<uint32_t*>(out + (row0 + g + 8) * ldq + dcol) = pack2<T>(o[nt][2], o[nt][3]);
    }
    return;
  }
  // ================= KV split: reduce the partial outputs over the cluster through distributed shared memory =================
  __syncthreads();  // every requested tile has landed and was consumed: the ring becomes the partial-output buffer
#pragma unroll
  for (int nt = 0; nt < ND; ++nt) {
    const int dcol = part * (kHd / CS) + nt * 8 + t * 2;
    float* po = sPO + (hl * 16) * kHd + dcol;
    *reinterpret_cast<float2*>(po + g * kHd) = make_float2(o[nt][0], o[nt][1]);
    *reinterpret_cast<float2*>(po + (g + 8) * kHd) = make_float2(o[nt][2], o[nt][3]);
  }
  cluster_sync_all();
  {
    const int rows_per = 16 / kvs;  // kvs in {2, 4}
    const int n_pairs = HPC * rows_per * (kHd / 2);
    const uint32_t po_local = smem_u32(sPO);
    for (int e2 = threadIdx.x; e2 < n_pairs; e2 += kThreads) {
      const int dpair = e2 % (kHd / 2);
      const int rr = (e2 / (kHd / 2)) % rows_per;
      const int h = e2 / ((kHd / 2) * rows_per);
      const int r = rank * rows_per + rr;
      const uint32_t off = static_cast<uint32_t>(((h * 16 + r) * kHd + dpair * 2) * 4);
      float a0 = 0.f, a1 = 0.f;
      for (int s2 = 0; s2 < kvs; ++s2) {  // fixed rank order: deterministic
        const uint32_t peer = dsmem_map(po_local, s2) + off;
        a0 += dsmem_ld_f32(peer);
        a1 += dsmem_ld_f32(peer + 4);
      }
      if (row0 + r < rows_valid)
        *reinterpret_cast<uint32_t*>(out + (row0 + r) * ldq + (head0 + h) * kHd + dpair * 2) = pack2<T>(a0, a1);
    }
  }
  cluster_sync_all();  // no CTA may exit while a peer still reads its partial outputs
  if (tr) tr[7] = gtimer();
}

static size_t attn_smem(int hpc, int kv_stride) {
  return 1024 + static_cast<size_t>(kRing) * kTileBytes + (static_cast<size_t>(hpc) * 16 * kRowPad + static_cast<size_t>(hpc) * 16 * kv_stride) * 2 +
         static_cast<size_t>(2 + 2 * 4) * hpc * 16 * 4 + 16;
}

template <typename T, int HPC> static int launch_hpc(const AttnParams& p, int kv_stride, int kvs, size_t smem, cudaStream_t s) {
  auto kern = tree_attention_kernel<T, HPC>;
  static bool configured_dev[64] = {};  // per device (the attribute is per device) and per instantiation
  const int cur_dev = current_device_index();
  if (cur_dev < 0) return static_cast<int>(cudaErrorInvalidDevice);
  if (!configured_dev[cur_dev]) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 1024);
    if (e != cudaSuccess) return static_cast<int>(e);
    configured_dev[cur_dev] = true;
  }
  dim3 grid(p.n_heads / HPC, (p.rows + 15) / 16, kvs);
  return static_cast<int>(launch_kc(kern, grid, dim3(kThreads), smem, s, dim3(1, 1, kvs), *p.tmK, *p.tmV, p, kv_stride, kvs));
}

int launch_attention(int dtype, const AttnParams& p, cudaStream_t s) {
  if (p.rows <= 0 || p.n_tree > 128 || p.n_heads % p.n_kv_heads || p.max_kv < 1 || !p.tmK || !p.tmV) return static_cast<int>(cudaErrorInvalidValue);
  static int max_hpc = 0, max_kvs = 0;
  if (!max_hpc) {
    const char* e = getenv("EB200_ATTN_HPC");  // tuning knobs: cap on query heads per CTA, cap on the KV split
    max_hpc = e ? atoi(e) : 2;
    if (max_hpc != 1 && max_hpc != 2 && max_hpc != 4) max_hpc = 2;
    const char* k = getenv("EB200_ATTN_KVS");
    max_kvs = k ? atoi(k) : 4;
    if (max_kvs != 1 && max_kvs != 2 && max_kvs != 4) max_kvs = 4;
  }
  // KV split over a cluster: aim at ~3 tiles (192 KV rows) per CTA
  const int tiles_all = (p.max_kv + kKvTile - 1) / kKvTile;
  int kvs = 1;
  while (kvs < max_kvs && tiles_all > 3 * kvs) kvs *= 2;
  const int tiles_per = (tiles_all + kvs - 1) / kvs;
  const int kv_stride = tiles_per * kKvTile + 8;
  const int n_rep = p.n_heads / p.n_kv_heads;
  // most heads per CTA (fewest K/V re-reads) whose score strip still fits in shared memory
  int hpc = 1;
  const size_t limit = 220 * 1024;
  if (max_hpc >= 4 && n_rep % 4 == 0 && attn_smem(4, kv_stride) <= limit) hpc = 4;
  else if (max_hpc >= 2 && n_rep % 2 == 0 && attn_smem(2, kv_stride) <= limit) hpc = 2;
  const size_t smem = attn_smem(hpc, kv_stride);
  if (smem > limit) return static_cast<int>(cudaErrorInvalidValue);
  if (dtype == DT_BF16) {
    if (hpc == 4) return launch_hpc<__nv_bfloat16, 4>(p, kv_stride, kvs, smem, s);
    if (hpc == 2) return launch_hpc<__nv_bfloat16, 2>(p, kv_stride, kvs, smem, s);
    return launch_hpc<__nv_bfloat16, 1>(p, kv_stride, kvs, smem, s);
  }
  if (hpc == 4) return launch_hpc<__half, 4>(p, kv_stride, kvs, smem, s);
  if (hpc == 2) return launch_hpc<__half, 2>(p, kv_stride, kvs, smem, s);
  return launch_hpc<__half, 1>(p, kv_stride, kvs, smem, s);
}

}  // namespace eb
