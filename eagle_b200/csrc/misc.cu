// Row-wise kernels around the GEMMs: RMSNorm (with optional row gather / concatenated output), embedding gather,
// arg-max over the target vocabulary, log-softmax + top-k over the draft vocabulary, and device-state helpers.
// All are tiny (<= 64 rows) and latency bound: one CTA per row, 16-byte vector loads, fp32 math with the
// reference's rounding points (see oracle/eagle_oracle.py header).
#include "common.cuh"
#include "kernels.h"

namespace eb {

template <int kThreads> __device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) red[w] = v;
  __syncthreads();
  float t = (threadIdx.x < kThreads / 32) ? red[threadIdx.x] : 0.f;
  if (w == 0) {
    t = warp_sum(t);
    if (l == 0) red[0] = t;
  }
  __syncthreads();
  t = red[0];
  __syncthreads();
  return t;
}

// ---------------------------------------------------------------------------------------------------------
// RMSNorm: cnets.py:379-384 / modeling_llama_kv.py:128-132
//   h = x.float(); h = h * rsqrt(mean(h^2) + eps); y = w * h.to(T)
// ---------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) rmsnorm_kernel(const T* __restrict__ src, long ld_src,
                                                      const int64_t* __restrict__ ids64, const int* __restrict__ ids32,
                                                      const T* __restrict__ w, T* __restrict__ y, long ld_y, int col_off,
                                                      int H, float eps, const __grid_constant__ L2Prefetch pf) {
  pdl_launch_dependents();
  if (threadIdx.x < 32) l2_prefetch_weights(pf, blockIdx.x * 32 + threadIdx.x, gridDim.x * 32);  // weights: no dependency wait
  pdl_wait();
  using D = DT<T>;
  __shared__ float red[32];
  const int m = blockIdx.x;
  long r = m;
  if (ids64) r = ids64[m];
  if (ids32) r = ids32[m];
  const T* x = src + r * ld_src;
  T* o = y + static_cast<long>(m) * ld_y + col_off;
  float ss = 0.f;
  const int nv = H / 8;
  for (int i = threadIdx.x; i < nv; i += 256) {
    uint4 raw = *reinterpret_cast<const uint4*>(x + i * 8);
    const T* e = reinterpret_cast<const T*>(&raw);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float f = D::to_f(e[j]);
      ss = fmaf(f, f, ss);
    }
  }
  ss = block_sum<256>(ss, red);
  const float inv = rsqrtf(ss / static_cast<float>(H) + eps);
  for (int i = threadIdx.x; i < nv; i += 256) {
    uint4 raw = *reinterpret_cast<const uint4*>(x + i * 8);
    uint4 wr = *reinterpret_cast<const uint4*>(w + i * 8);
    const T* e = reinterpret_cast<const T*>(&raw);
    const T* we = reinterpret_cast<const T*>(&wr);
    uint4 outv;
    T* oe = reinterpret_cast<T*>(&outv);
#pragma unroll
    for (int j = 0; j < 8; ++j) oe[j] = D::from_f(D::to_f(we[j]) * rnd<T>(D::to_f(e[j]) * inv));
    *reinterpret_cast<uint4*>(o + i * 8) = outv;
  }
}

int launch_rmsnorm(int dtype, const void* src, long ld_src, const int64_t* ids64, const int* ids32, const void* w, void* y,
                   long ld_y, int col_off, int H, float eps, int rows, cudaStream_t s, const L2Prefetch* pf) {
  if (H % 8 || rows <= 0) return static_cast<int>(cudaErrorInvalidValue);
  L2Prefetch none;
  memset(&none, 0, sizeof(none));
  if (dtype == DT_BF16)
    launch_k(rmsnorm_kernel<__nv_bfloat16>, dim3(rows), dim3(256), 0, s, 1, reinterpret_cast<const __nv_bfloat16*>(src), ld_src, ids64, ids32,
                                                        reinterpret_cast<const __nv_bfloat16*>(w),
                                                        reinterpret_cast<__nv_bfloat16*>(y), ld_y, col_off, H, eps, pf ? *pf : none);
  else
    launch_k(rmsnorm_kernel<__half>, dim3(rows), dim3(256), 0, s, 1, reinterpret_cast<const __half*>(src), ld_src, ids64, ids32,
                                                 reinterpret_cast<const __half*>(w), reinterpret_cast<__half*>(y), ld_y,
                                                 col_off, H, eps, pf ? *pf : none);
  return static_cast<int>(cudaGetLastError());
}

// ---------------------------------------------------------------------------------------------------------
// EAGLE-3 draft input in ONE launch (cnets.py:427-430): cat(input_layernorm(embed(ids)), hidden_norm(hidden)).
// blockIdx.y == 0: the embedding half; blockIdx.y == 1: the hidden half, optionally gathering the hidden row from
// hsrc[src_rows[m]] (tree levels: the previous level's output rows picked by the frontier, cnets.py:716,:747) and keeping
// a copy in hdst (the layer's residual stream).  Same arithmetic and thread mapping as rmsnorm_kernel (bit-identical).
// ---------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) e3_input_kernel(const T* table, long ld_table, const int64_t* ids64, const int* ids32, const T* w_emb,
                                                       const T* hsrc, long ld_hsrc, const int* src_rows, T* hdst, long ld_hdst,
                                                       const T* w_hid, T* cat, long ld_cat, int H, float eps,
                                                       const __grid_constant__ L2Prefetch pf) {
  pdl_launch_dependents();
  if (threadIdx.x < 32) {  // weights: no dependency wait
    const int cta = blockIdx.x + gridDim.x * blockIdx.y;
    l2_prefetch_weights(pf, cta * 32 + threadIdx.x, gridDim.x * gridDim.y * 32);
  }
  pdl_wait();
  using D = DT<T>;
  __shared__ float red[32];
  const int m = blockIdx.x;
  const bool hid = blockIdx.y == 1;
  const T* x;
  const T* w;
  T* o = cat + static_cast<long>(m) * ld_cat + (hid ? H : 0);
  T* copy = nullptr;
  if (hid) {
    long r = m;
    if (src_rows) {
      r = ld_dep(src_rows + m);
      if (r < 0) r = 0;
      copy = hdst + static_cast<long>(m) * ld_hdst;
    }
    x = hsrc + r * ld_hsrc;
    w = w_hid;
  } else {
    long r = m;
    if (ids64) r = *reinterpret_cast<const volatile int64_t*>(ids64 + m);
    if (ids32) r = ld_dep(ids32 + m);
    if (r < 0) r = 0;
    x = table + r * ld_table;
    w = w_emb;
  }
  float ss = 0.f;
  const int nv = H / 8;
  for (int i = threadIdx.x; i < nv; i += 256) {
    uint4 raw = __ldcg(reinterpret_cast<const uint4*>(x + i * 8));
    const T* e = reinterpret_cast<const T*>(&raw);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float f = D::to_f(e[j]);
      ss = fmaf(f, f, ss);
    }
  }
  ss = block_sum<256>(ss, red);
  const float inv = rsqrtf(ss / static_cast<float>(H) + eps);
  for (int i = threadIdx.x; i < nv; i += 256) {
    uint4 raw = __ldcg(reinterpret_cast<const uint4*>(x + i * 8));
    uint4 wr = *reinterpret_cast<const uint4*>(w + i * 8);
    const T* e = reinterpret_cast<const T*>(&raw);
    const T* we = reinterpret_cast<const T*>(&wr);
    uint4 outv;
    T* oe = reinterpret_cast<T*>(&outv);
#pragma unroll
    for (int j = 0; j < 8; ++j) oe[j] = D::from_f(D::to_f(we[j]) * rnd<T>(D::to_f(e[j]) * inv));
    *reinterpret_cast<uint4*>(o + i * 8) = outv;
    if (copy) *reinterpret_cast<uint4*>(copy + i * 8) = raw;
  }
}

int launch_e3_input(int dtype, const void* table, long ld_table, const int64_t* ids64, const int* ids32, const void* w_emb, const void* hsrc,
                    long ld_hsrc, const int* src_rows, void* hdst, long ld_hdst, const void* w_hid, void* cat, long ld_cat, int H, float eps,
                    int rows, cudaStream_t s, const L2Prefetch* pf) {
  if (H % 8 || rows <= 0 || ld_table % 8 || ld_hsrc % 8 || ld_hdst % 8 || ld_cat % 8) return static_cast<int>(cudaErrorInvalidValue);
  if (src_rows && hsrc == hdst) return static_cast<int>(cudaErrorInvalidValue);  // a gather must not alias its destination
  L2Prefetch none;
  memset(&none, 0, sizeof(none));
  if (dtype == DT_BF16) {
    using T = __nv_bfloat16;
    launch_k(e3_input_kernel<T>, dim3(rows, 2), dim3(256), 0, s, 1, reinterpret_cast<const T*>(table), ld_table, ids64, ids32,
             reinterpret_cast<const T*>(w_emb), reinterpret_cast<const T*>(hsrc), ld_hsrc, src_rows, reinterpret_cast<T*>(hdst), ld_hdst,
             reinterpret_cast<const T*>(w_hid), reinterpret_cast<T*>(cat), ld_cat, H, eps, pf ? *pf : none);
  } else {
    using T = __half;
    launch_k(e3_input_kernel<T>, dim3(rows, 2), dim3(256), 0, s, 1, reinterpret_cast<const T*>(table), ld_table, ids64, ids32,
             reinterpret_cast<const T*>(w_emb), reinterpret_cast<const T*>(hsrc), ld_hsrc, src_rows, reinterpret_cast<T*>(hdst), ld_hdst,
             reinterpret_cast<const T*>(w_hid), reinterpret_cast<T*>(cat), ld_cat, H, eps, pf ? *pf : none);
  }
  return static_cast<int>(cudaGetLastError());
}

// ---------------------------------------------------------------------------------------------------------
// row gather (embedding lookup, feature-row gather by accepted path)
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) gather_rows_kernel(const uint4* __restrict__ table, long ld_table_v,
                                                          const int64_t* __restrict__ ids64,
                                                          const int* __restrict__ ids32, uint4* __restrict__ dst,
                                                          long ld_dst_v, int col_off_v, int nv) {
  pdl_launch_dependents();
  pdl_wait();
  const int m = blockIdx.x;
  long r = m;
  if (ids64) r = ids64[m];
  if (ids32) r = ids32[m];
  if (r < 0) r = 0;
  const uint4* x = table + r * ld_table_v;
  uint4* o = dst + static_cast<long>(m) * ld_dst_v + col_off_v;
  for (int i = threadIdx.x; i < nv; i += 256) o[i] = x[i];
}

int launch_gather_rows(int dtype, const void* table, long ld_table, const int64_t* ids64, const int* ids32, void* dst,
                       long ld_dst, int col_off, int H, int rows, cudaStream_t s) {
  (void)dtype;
  if (H % 8 || ld_table % 8 || ld_dst % 8 || col_off % 8 || rows <= 0) return static_cast<int>(cudaErrorInvalidValue);
  launch_k(gather_rows_kernel, dim3(rows), dim3(256), 0, s, 1, reinterpret_cast<const uint4*>(table), ld_table / 8, ids64, ids32,
                                          reinterpret_cast<uint4*>(dst), ld_dst / 8, col_off / 8, H / 8);
  return static_cast<int>(cudaGetLastError());
}

// ---------------------------------------------------------------------------------------------------------
// arg-max over the vocabulary (first maximal index, like torch.argmax on CPU): utils.py:243, :362, :463
// ---------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(1024) argmax_kernel(const T* __restrict__ logits, long ld, int V, int* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  using D = DT<T>;
  __shared__ float sv[32];
  __shared__ int si[32];
  const T* x = logits + static_cast<long>(blockIdx.x) * ld;
  float best = -INFINITY;
  int bi = 0x7fffffff;
  const int nv = V / 8;
  for (int i = threadIdx.x; i < nv; i += 1024) {
    uint4 raw = *reinterpret_cast<const uint4*>(x + i * 8);
    const T* e = reinterpret_cast<const T*>(&raw);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float f = D::to_f(e[j]);
      if (f > best) {  // strict: keeps the lowest index inside this thread's ascending scan
        best = f;
        bi = i * 8 + j;
      }
    }
  }
  for (int i = nv * 8 + threadIdx.x; i < V; i += 1024) {
    const float f = D::to_f(x[i]);
    if (f > best || (f == best && i < bi)) {
      best = f;
      bi = i;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > best || (ov == best && oi < bi)) {
      best = ov;
      bi = oi;
    }
  }
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) {
    sv[w] = best;
    si[w] = bi;
  }
  __syncthreads();
  if (w == 0) {
    best = sv[l];
    bi = si[l];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > best || (ov == best && oi < bi)) {
        best = ov;
        bi = oi;
      }
    }
    if (l == 0) out[blockIdx.x] = bi;
  }
}

int launch_argmax(int dtype, const void* logits, long ld, int V, int rows, int* out_idx, cudaStream_t s) {
  if (rows <= 0 || ld % 8) return static_cast<int>(cudaErrorInvalidValue);
  if (dtype == DT_BF16)
    launch_k(argmax_kernel<__nv_bfloat16>, dim3(rows), dim3(1024), 0, s, 1, reinterpret_cast<const __nv_bfloat16*>(logits), ld, V, out_idx);
  else
    launch_k(argmax_kernel<__half>, dim3(rows), dim3(1024), 0, s, 1, reinterpret_cast<const __half*>(logits), ld, V, out_idx);
  return static_cast<int>(cudaGetLastError());
}

// ---------------------------------------------------------------------------------------------------------
// log-softmax (fp32 math, result rounded to T like nn.LogSoftmax on a T tensor) + top-k, cnets.py:702-705, :735-738.
// Ties: value descending, then lowest index (torch.topk leaves tie order unspecified; we fix it).
// One CTA (1024 threads) per row.  k <= 32.
// ---------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(1024) logsoftmax_topk_kernel(const T* __restrict__ logits, long ld, int V,
                                                               const int* __restrict__ st, int row_idx, int k, int raw,
                                                               float* __restrict__ topk_p, int* __restrict__ topk_i) {
  pdl_launch_dependents();
  pdl_wait();
  using D = DT<T>;
  __shared__ float red[32];
  __shared__ float cand_v[32 * 32];
  __shared__ int cand_i[32 * 32];
  const int row = (row_idx >= 0 ? st[row_idx] : 0) + blockIdx.x;
  const T* x = logits + static_cast<long>(row) * ld;
  const int tid = threadIdx.x, w = tid >> 5, l = tid & 31;

  auto warp_pick = [&](float& v2, int& i2) {  // warp arg-max by (value desc, index asc)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, v2, o);
      const int oi = __shfl_xor_sync(0xffffffffu, i2, o);
      if (ov > v2 || (ov == v2 && oi < i2)) {
        v2 = ov;
        i2 = oi;
      }
    }
  };
  // ---- register-resident path: V <= 32768 (every draft vocabulary), rows 16-byte aligned.  Thread t owns the 16-byte
  // vectors t, t+1024, t+2048, t+3072 of the row (32 elements): ONE global read serves max, exp-sum and the k selection rounds.
  if (V % 8 == 0 && V <= 32768 && ld % 8 == 0) {
    float v[32];
    const uint4* xv = reinterpret_cast<const uint4*>(x);
    const int nvec = V / 8;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int vi = tid + 1024 * u;
      uint4 rawv = make_uint4(0, 0, 0, 0);
      if (vi < nvec) rawv = xv[vi];
      const T* e = reinterpret_cast<const T*>(&rawv);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[u * 8 + j] = (vi < nvec) ? D::to_f(e[j]) : -INFINITY;
    }
    if (!raw) {
      float mx = -INFINITY;
#pragma unroll
      for (int j = 0; j < 32; ++j) mx = fmaxf(mx, v[j]);
      mx = warp_max(mx);
      if (l == 0) red[w] = mx;
      __syncthreads();
      mx = red[l];
      mx = warp_max(mx);
      __syncthreads();
      float se = 0.f;
#pragma unroll
      for (int j = 0; j < 32; ++j) se += expf(v[j] - mx);  // exp(-inf) = 0 for the padding
      se = block_sum<1024>(se, red);
      const float lse = rnd<T>(logf(rnd<T>(se)));  // the reference's CPU roundings, see below
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = rnd<T>(v[j] - mx - lse);
    }
    uint32_t taken = 0;  // bit j: v[j] already selected
    for (int r = 0; r < k; ++r) {
      float bv = -INFINITY;
      int bj = -1;
#pragma unroll
      for (int j = 0; j < 32; ++j)  // ascending j == ascending vocabulary index inside a thread
        if (!((taken >> j) & 1u) && v[j] > bv) {
          bv = v[j];
          bj = j;
        }
      float v2 = bv;
      int i2 = bj >= 0 ? 8 * (tid + 1024 * (bj >> 3)) + (bj & 7) : 0x7fffffff;
      warp_pick(v2, i2);
      if (i2 != 0x7fffffff && ((i2 >> 3) & 1023) == tid) taken |= 1u << (((i2 >> 13) << 3) | (i2 & 7));
      if (l == 0) {
        cand_v[w * 32 + r] = v2;
        cand_i[w * 32 + r] = i2;
      }
    }
  } else {
    // raw != 0: rank the logits themselves (torch.topk(last_headout), static tree, modeling_eagle.py:900-903): the
    // log-softmax shift is the identity (x - 0 - 0 is exact in fp32 and already representable in T)
    float mx = 0.f, lse = 0.f;
    if (!raw) {
      // pass 1: max
      mx = -INFINITY;
      for (int i = tid; i < V; i += 1024) mx = fmaxf(mx, D::to_f(x[i]));
      mx = warp_max(mx);
      if (l == 0) red[w] = mx;
      __syncthreads();
      mx = red[l];
      mx = warp_max(mx);
      __syncthreads();
      // pass 2: sum exp
      float se = 0.f;
      for (int i = tid; i < V; i += 1024) se += expf(D::to_f(x[i]) - mx);
      se = block_sum<1024>(se, red);
      // The reference's CPU log_softmax on a model-dtype tensor (ATen vec_log_softmax_lastdim with scalar_t = T) keeps the
      // exp-sum and its log in T: out = T((x - max) - T(log(T(sum)))).  The oracle is pinned on that behaviour, so the
      // two extra roundings are reproduced here (they shift every log-prob of a row by the same amount).
      lse = rnd<T>(logf(rnd<T>(se)));
    }

    // pass 3: per-warp top-k over a contiguous slab (warp w owns [w*slab, (w+1)*slab)), k rounds of warp arg-max.
    const int slab = (V + 31) / 32;
    const int lo = w * slab, hi = min(V, lo + slab);
    const int per_lane = (slab + 31) / 32;
    {
      // bit j: element lo + l + 32*j of this lane already selected (per_lane <= 128  =>  V <= 131072)
      uint64_t taken0 = 0, taken1 = 0;
      for (int r = 0; r < k; ++r) {
        float bv = -INFINITY;
        int bi = 0x7fffffff;
        for (int j = 0; j < per_lane; ++j) {
          const int i = lo + l + 32 * j;
          const uint64_t tk = (j < 64) ? (taken0 >> j) : (taken1 >> (j - 64));
          if (i < hi && !(tk & 1ull)) {
            const float vv = rnd<T>(D::to_f(x[i]) - mx - lse);
            if (vv > bv) {
              bv = vv;
              bi = i;
            }
          }
        }
        float v2 = bv;
        int i2 = bi;
        warp_pick(v2, i2);
        if (i2 != 0x7fffffff && ((i2 - lo) & 31) == l) {
          const int j = (i2 - lo) >> 5;
          if (j < 64) taken0 |= 1ull << j; else taken1 |= 1ull << (j - 64);
        }
        if (l == 0) {
          cand_v[w * 32 + r] = v2;
          cand_i[w * 32 + r] = i2;
        }
      }
    }
  }
  __syncthreads();
  // pass 4: warp 0 merges 32 warps x k candidates
  if (w == 0) {
    float cv[32];
    int ci[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      cv[j] = (j < k) ? cand_v[l * 32 + j] : -INFINITY;  // lane l holds warp l's (sorted) list
      ci[j] = (j < k) ? cand_i[l * 32 + j] : 0x7fffffff;
    }
    int head = 0;  // lists are sorted (value desc, index asc): only the head of each list competes
    for (int r = 0; r < k; ++r) {
      float v = -INFINITY;
      int i = 0x7fffffff;
#pragma unroll
      for (int j = 0; j < 32; ++j)
        if (j == head) {
          v = cv[j];
          i = ci[j];
        }
      float v2 = v;
      int i2 = i;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, v2, o);
        const int oi = __shfl_xor_sync(0xffffffffu, i2, o);
        if (ov > v2 || (ov == v2 && oi < i2)) {
          v2 = ov;
          i2 = oi;
        }
      }
      if (i2 == i && i != 0x7fffffff) ++head;
      if (l == 0) {
        topk_p[blockIdx.x * k + r] = v2;
        topk_i[blockIdx.x * k + r] = i2;
      }
    }
  }
}

int launch_logsoftmax_topk(int dtype, const void* logits, long ld, int V, int rows, const int* st, int row_idx, int k, int raw,
                           float* topk_p, int* topk_i, cudaStream_t s) {
  if (k > 32 || k < 1 || V > 32 * 32 * 128 || rows <= 0) return static_cast<int>(cudaErrorInvalidValue);
  if (dtype == DT_BF16)
    launch_k(logsoftmax_topk_kernel<__nv_bfloat16>, dim3(rows), dim3(1024), 0, s, 1, reinterpret_cast<const __nv_bfloat16*>(logits), ld, V, st,
                                                                 row_idx, k, raw, topk_p, topk_i);
  else
    launch_k(logsoftmax_topk_kernel<__half>, dim3(rows), dim3(1024), 0, s, 1, reinterpret_cast<const __half*>(logits), ld, V, st, row_idx, k,
                                                          raw, topk_p, topk_i);
  return static_cast<int>(cudaGetLastError());
}

// ---------------------------------------------------------------------------------------------------------
// tensor-parallel helpers
// ---------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) residual_add_f32_kernel(const float* __restrict__ sum, T* __restrict__ x, long n) {
  pdl_launch_dependents();
  pdl_wait();
  const long i = (blockIdx.x * 256L + threadIdx.x) * 4;
  if (i + 3 < n) {
    const float4 v = *reinterpret_cast<const float4*>(sum + i);
    const float f[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) x[i + j] = DT<T>::from_f(rnd<T>(f[j]) + DT<T>::to_f(x[i + j]));
  }
}
int launch_residual_add_f32(int dtype, const float* sum, void* x, int rows, int H, cudaStream_t s) {
  const long n = static_cast<long>(rows) * H;
  if (n % 4) return static_cast<int>(cudaErrorInvalidValue);
  const unsigned blocks = static_cast<unsigned>((n / 4 + 255) / 256);
  if (dtype == DT_BF16) launch_k(residual_add_f32_kernel<__nv_bfloat16>, dim3(blocks), dim3(256), 0, s, 1, sum, reinterpret_cast<__nv_bfloat16*>(x), n);
  else launch_k(residual_add_f32_kernel<__half>, dim3(blocks), dim3(256), 0, s, 1, sum, reinterpret_cast<__half*>(x), n);
  return static_cast<int>(cudaGetLastError());
}

template <typename T>
__global__ void __launch_bounds__(1024) argmax_val_kernel(const T* __restrict__ logits, long ld, int V, int idx_offset,
                                                          float* __restrict__ out_val, int* __restrict__ out_idx) {
  using D = DT<T>;
  __shared__ float sv[32];
  __shared__ int si[32];
  pdl_launch_dependents();
  pdl_wait();
  const T* x = logits + static_cast<long>(blockIdx.x) * ld;
  float best = -INFINITY;
  int bi = 0x7fffffff;
  for (int i = threadIdx.x; i < V; i += 1024) {
    const float f = D::to_f(x[i]);
    if (f > best) {
      best = f;
      bi = i;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > best || (ov == best && oi < bi)) {
      best = ov;
      bi = oi;
    }
  }
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) {
    sv[w] = best;
    si[w] = bi;
  }
  __syncthreads();
  if (w == 0) {
    best = sv[l];
    bi = si[l];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > best || (ov == best && oi < bi)) {
        best = ov;
        bi = oi;
      }
    }
    if (l == 0) {
      out_val[blockIdx.x] = best;
      out_idx[blockIdx.x] = (bi == 0x7fffffff) ? bi : bi + idx_offset;
    }
  }
}
int launch_argmax_val(int dtype, const void* logits, long ld, int V_valid, int rows, int idx_offset, float* out_val, int* out_idx,
                      cudaStream_t s) {
  if (rows <= 0) return static_cast<int>(cudaErrorInvalidValue);
  if (dtype == DT_BF16)
    launch_k(argmax_val_kernel<__nv_bfloat16>, dim3(rows), dim3(1024), 0, s, 1, reinterpret_cast<const __nv_bfloat16*>(logits), ld, V_valid,
             idx_offset, out_val, out_idx);
  else
    launch_k(argmax_val_kernel<__half>, dim3(rows), dim3(1024), 0, s, 1, reinterpret_cast<const __half*>(logits), ld, V_valid, idx_offset,
             out_val, out_idx);
  return static_cast<int>(cudaGetLastError());
}

__global__ void argmax_merge_kernel(const float* __restrict__ vals, const int* __restrict__ idxs, int n_ranks, int rows,
                                    int stride, int* __restrict__ out_idx) {
  pdl_launch_dependents();
  pdl_wait();
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= rows) return;
  float best = -INFINITY;
  int bi = 0x7fffffff;
  for (int r = 0; r < n_ranks; ++r) {
    const float v = vals[r * stride + m];
    const int i = idxs[r * stride + m];
    if (v > best || (v == best && i < bi)) {
      best = v;
      bi = i;
    }
  }
  out_idx[m] = bi;
}
int launch_argmax_merge(const float* vals, const int* idxs, int n_ranks, int rows, int stride, int* out_idx, cudaStream_t s) {
  launch_k(argmax_merge_kernel, dim3((rows + 63) / 64), dim3(64), 0, s, 1, vals, idxs, n_ranks, rows, stride, out_idx);
  return static_cast<int>(cudaGetLastError());
}

// ---------------------------------------------------------------------------------------------------------
// device-state helpers
// ---------------------------------------------------------------------------------------------------------
__global__ void set_state_kernel(int* st, int idx, int value) {
  pdl_launch_dependents();
  pdl_wait();
  st[idx] = value;
}
__global__ void copy_state_kernel(int* st, int dst, int src, int add) {
  pdl_launch_dependents();
  pdl_wait();
  st[dst] = st[src] + add;
}
__global__ void state_to_kernel(int* dst, const int* st, int idx) {
  pdl_launch_dependents();
  pdl_wait();
  *dst = st[idx];
}
int launch_state_to(int* dst, const int* st, int idx, cudaStream_t s) {
  launch_k(state_to_kernel, dim3(1), dim3(1), 0, s, 1, dst, st, idx);
  return static_cast<int>(cudaGetLastError());
}
// [ranks][rows][cols] -> [rows][ranks*cols]  (2-byte elements): vocab-parallel logits gathered for the sampling posterior
__global__ void __launch_bounds__(256) unshard_rows_kernel(const uint16_t* __restrict__ in, uint16_t* __restrict__ out, int ranks, int rows,
                                                          int cols) {
  pdl_launch_dependents();
  pdl_wait();
  const long n = static_cast<long>(ranks) * rows * cols;
  for (long i = blockIdx.x * 256L + threadIdx.x; i < n; i += static_cast<long>(gridDim.x) * 256) {
    const int j = static_cast<int>(i % cols);
    const int m = static_cast<int>((i / cols) % rows);
    const int r = static_cast<int>(i / (static_cast<long>(cols) * rows));
    out[(static_cast<long>(m) * ranks + r) * cols + j] = in[i];
  }
}
int launch_unshard_rows(const void* in, void* out, int ranks, int rows, int cols, cudaStream_t s) {
  launch_k(unshard_rows_kernel, dim3(592), dim3(256), 0, s, 1, reinterpret_cast<const uint16_t*>(in), reinterpret_cast<uint16_t*>(out), ranks,
           rows, cols);
  return static_cast<int>(cudaGetLastError());
}
int launch_set_state(int* st, int idx, int value, cudaStream_t s) {
  launch_k(set_state_kernel, dim3(1), dim3(1), 0, s, 1, st, idx, value);
  return static_cast<int>(cudaGetLastError());
}
int launch_copy_state(int* st, int dst_idx, int src_idx, int add, cudaStream_t s) {
  launch_k(copy_state_kernel, dim3(1), dim3(1), 0, s, 1, st, dst_idx, src_idx, add);
  return static_cast<int>(cudaGetLastError());
}

}  // namespace eb
