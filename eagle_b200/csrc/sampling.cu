// Sampling posterior (temperature > 0): the reference's sequential multi-candidate speculative sampling
// (utils.py:375-415, q(x) == 1) with its logits warpers (temperature -> top-p -> top-k, utils.py:38-54), on device.
// The reference drives this with Python loops, `.item()` per candidate, host `random.random()` and `torch.multinomial`.
// Here: one pass computes the softmax statistics (max, normaliser, keep-threshold) of every tree node's logits row,
// one single-CTA kernel walks the tree exactly like the reference, one kernel draws the bonus token by inverse CDF.
//
// Differences from the reference, by design: probabilities are kept in fp32 (the reference's CPU path rounds the
// softmax to the model dtype, a ~0.4 % relative quantisation of p), repeated renormalisation after a rejection is
// carried as the removed mass (mathematically identical), the bonus token is drawn by inverse CDF from a counter-based
// RNG (torch.multinomial uses exponential races): identical distribution, different stream -- parity for this path is
// statistical (losslessness) plus exact decisions for injected uniforms away from the thresholds.
#include "tree_common.cuh"

namespace eb {

template <typename T> __device__ __forceinline__ uint32_t order_key(T v);
template <> __device__ __forceinline__ uint32_t order_key<__nv_bfloat16>(__nv_bfloat16 v) {
  const uint16_t b = *reinterpret_cast<const uint16_t*>(&v);
  return (b & 0x8000u) ? static_cast<uint16_t>(~b) : static_cast<uint16_t>(b | 0x8000u);
}
template <> __device__ __forceinline__ uint32_t order_key<__half>(__half v) {
  const uint16_t b = *reinterpret_cast<const uint16_t*>(&v);
  return (b & 0x8000u) ? static_cast<uint16_t>(~b) : static_cast<uint16_t>(b | 0x8000u);
}
template <typename T> __device__ __forceinline__ T key_to_value(uint32_t k) {
  const uint16_t b = (k & 0x8000u) ? static_cast<uint16_t>(k & 0x7fffu) : static_cast<uint16_t>(~k);
  return *reinterpret_cast<const T*>(&b);
}
// TemperatureLogitsWarper: scores / temperature evaluated in the model dtype
template <typename T> __device__ __forceinline__ float warp_temp(T l, float temperature) {
  const float f = DT<T>::to_f(l);
  return (temperature != 1.0f) ? rnd<T>(__fdiv_rn(f, temperature)) : f;
}

__device__ __forceinline__ float block_sum_1024(float v, float* red) {
  v = warp_sum(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) red[w] = v;
  __syncthreads();
  float t = (threadIdx.x < 32) ? red[threadIdx.x] : 0.f;
  if (w == 0) {
    t = warp_sum(t);
    if (l == 0) red[0] = t;
  }
  __syncthreads();
  return red[0];
}
__device__ __forceinline__ float block_max_1024(float v, float* red) {
  v = warp_max(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) red[w] = v;
  __syncthreads();
  float t = (threadIdx.x < 32) ? red[threadIdx.x] : -INFINITY;
  if (w == 0) {
    t = warp_max(t);
    if (l == 0) red[0] = t;
  }
  __syncthreads();
  return red[0];
}

template <typename T>
__global__ void __launch_bounds__(1024) row_softmax_stats_kernel(const T* __restrict__ logits, long ld, int V, SampleParams sp,
                                                                 RowStats* __restrict__ stats) {
  __shared__ float red[32];
  pdl_launch_dependents();
  pdl_wait();
  const T* x = logits + static_cast<long>(blockIdx.x) * ld;
  const float temp = sp.temperature;
  float mx = -INFINITY;
  for (int i = threadIdx.x; i < V; i += 1024) mx = fmaxf(mx, warp_temp<T>(x[i], temp));
  mx = block_max_1024(mx, red);
  float z = 0.f;
  for (int i = threadIdx.x; i < V; i += 1024) z += expf(warp_temp<T>(x[i], temp) - mx);
  z = block_sum_1024(z, red);
  float thr = -INFINITY;
  if (sp.top_p >= 1e-8f && sp.top_p < 1.0f) {
    // TopPLogitsWarper: ascending cumulative probability; tokens with cumulative mass <= 1 - top_p are removed.
    // Keep v iff mass(l <= l_v) > 1 - top_p  ->  bisect the smallest model-dtype value with that property (16 steps).
    // The row maximum is always kept (min_tokens_to_keep = 1): the search ends at it even where no mass exceeds the cut,
    // which happens when 1 - top_p rounds to 1 in fp32 (top_p below 2^-25).
    const float cut = (1.0f - sp.top_p) * z;
    uint32_t lo = 0, hi = order_key<T>(DT<T>::from_f(mx));  // keys; answer in [lo, hi]
    while (lo < hi) {
      const uint32_t mid = (lo + hi) >> 1;
      float m = 0.f;
      for (int i = threadIdx.x; i < V; i += 1024) {
        const float lt = warp_temp<T>(x[i], temp);
        if (order_key<T>(DT<T>::from_f(lt)) <= mid) m += expf(lt - mx);
      }
      m = block_sum_1024(m, red);
      if (m > cut) hi = mid; else lo = mid + 1;
    }
    thr = DT<T>::to_f(key_to_value<T>(lo));
  }
  if (sp.top_k > 0 && sp.top_k < V) {
    // TopKLogitsWarper: remove scores < k-th largest  ->  largest key with count(l >= key) >= k
    uint32_t lo = 0, hi = 0xffffu;
    while (lo < hi) {
      const uint32_t mid = (lo + hi + 1) >> 1;
      float c = 0.f;
      for (int i = threadIdx.x; i < V; i += 1024) {
        const float lt = warp_temp<T>(x[i], temp);
        if (lt >= thr && order_key<T>(DT<T>::from_f(lt)) >= mid) c += 1.f;
      }
      c = block_sum_1024(c, red);
      if (c >= static_cast<float>(sp.top_k)) lo = mid; else hi = mid - 1;
    }
    const float kth = DT<T>::to_f(key_to_value<T>(lo));
    thr = fmaxf(thr, kth);
  }
  float sum = z;
  if (thr > -INFINITY) {
    sum = 0.f;
    for (int i = threadIdx.x; i < V; i += 1024) {
      const float lt = warp_temp<T>(x[i], temp);
      if (lt >= thr) sum += expf(lt - mx);
    }
    sum = block_sum_1024(sum, red);
  }
  if (threadIdx.x == 0) stats[blockIdx.x] = RowStats{mx, sum, thr, 0.f};
}

int launch_row_softmax_stats(int dtype, const void* logits, long ld, int V, int rows, SampleParams sp, RowStats* stats, cudaStream_t s) {
  if (rows <= 0) return static_cast<int>(cudaErrorInvalidValue);
  if (dtype == DT_BF16) launch_k(row_softmax_stats_kernel<__nv_bfloat16>, dim3(rows), dim3(1024), 0, s, 1, reinterpret_cast<const __nv_bfloat16*>(logits), ld, V, sp, stats);
  else launch_k(row_softmax_stats_kernel<__half>, dim3(rows), dim3(1024), 0, s, 1, reinterpret_cast<const __half*>(logits), ld, V, sp, stats);
  return static_cast<int>(cudaGetLastError());
}

// counter-based uniform in (0, 1): splitmix64 of (seed, counter)
__device__ __forceinline__ float counter_uniform(unsigned long long seed, int counter) {
  unsigned long long z = seed + 0x9E3779B97F4A7C15ull * (static_cast<unsigned long long>(counter) + 1ull);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  return (static_cast<float>(z >> 40) + 0.5f) * (1.0f / 16777216.0f);
}
__device__ __forceinline__ float next_uniform(const SampleParams& sp, int* st) {
  const int c = st[S_UCOUNT];
  st[S_UCOUNT] = c + 1;
  return (sp.uniforms && c < sp.n_uniforms) ? sp.uniforms[c] : counter_uniform(sp.seed, c);
}
template <typename T>
__device__ __forceinline__ float row_prob(const T* __restrict__ logits, long ld, const RowStats* __restrict__ stats, int node, int tok,
                                          float temperature) {
  const RowStats rs = stats[node];
  const float lt = warp_temp<T>(logits[static_cast<long>(node) * ld + tok], temperature);
  return (lt >= rs.thr) ? expf(lt - rs.max) / rs.sum : 0.f;
}

// utils.py:375-415, one thread (the work is a handful of probability look-ups per level)
template <typename T>
__global__ void posterior_sample_kernel(const T* __restrict__ logits, long ld, int V, const RowStats* __restrict__ stats, TreeBuffers tb,
                                        int depth, SampleParams sp, int* __restrict__ rej_tokens, int* __restrict__ st) {
  pdl_launch_dependents();
  pdl_wait();
  if (threadIdx.x != 0) return;
  const int D = depth + 2;
  const int n_leaf = st[S_NLEAF], maxd = st[S_MAXDEPTH];
  int accept_length = 1, best = 0;
  int prefix[16];
  prefix[0] = tb.retrieve[0];  // node ids of the accepted path (row 0, column 0 == root)
  bool adjust = false;
  int n_rej = 0, last_node = prefix[0];
  for (int i = 1; i < maxd; ++i) {
    if (i != accept_length) break;
    adjust = false;
    n_rej = 0;
    // first row sharing the accepted prefix; its node at depth i-1 carries the target distribution
    int fi = -1;
    for (int r = 0; r < n_leaf && fi < 0; ++r) {
      bool eq = true;
      for (int j = 0; j < accept_length && eq; ++j) eq = (tb.retrieve[r * D + j] == prefix[j]);
      if (eq) fi = r;
    }
    if (fi < 0) break;
    last_node = tb.retrieve[fi * D + i - 1];
    float removed = 0.f;
    bool accepted = false;
    for (int r = 0; r < n_leaf; ++r) {
      bool eq = true;
      for (int j = 0; j < accept_length && eq; ++j) eq = (tb.retrieve[r * D + j] == prefix[j]);
      if (!eq) continue;
      const int node = tb.retrieve[r * D + i];
      if (node < 0) continue;  // padding (candidate token -1)
      const int xi = tb.draft_tokens[node];
      bool seen = false;
      for (int q = 0; q < n_rej && !seen; ++q) seen = (rej_tokens[q] == xi);
      if (seen) continue;
      const float u = next_uniform(sp, st);
      const float px = row_prob<T>(logits, ld, stats, last_node, xi, sp.temperature);
      const float acp = px / fmaxf(1.0f - removed, 1e-30f);  // p after zeroing the rejected tokens and renormalising
      if (u <= acp) {
        prefix[accept_length] = node;
        ++accept_length;
        best = r;
        accepted = true;
        break;
      }
      if (n_rej < 64) rej_tokens[n_rej++] = xi;
      removed += px;
      adjust = true;
    }
    if (!accepted) break;
  }
  const int a = accept_length - 1;
  // distribution of the bonus token: the residual of the last examined level if it ended in rejections, else a fresh
  // softmax at the last accepted node (utils.py:409-414)
  if (adjust && accept_length != maxd) {
    st[S_SNODE] = last_node;
    st[S_SNREJ] = n_rej;
  } else {
    st[S_SNODE] = tb.retrieve[best * D + a];
    st[S_SNREJ] = 0;
  }
  st[S_BEST] = best;
  st[S_ACC] = a + 1;
}

int launch_sample_posterior(int dtype, const void* logits, long ld, int V, const RowStats* stats, TreeBuffers tb, int depth, SampleParams sp,
                            int* rej_tokens, int* st, cudaStream_t s) {
  if (depth + 2 > 16) return static_cast<int>(cudaErrorInvalidValue);
  if (dtype == DT_BF16) launch_k(posterior_sample_kernel<__nv_bfloat16>, dim3(1), dim3(32), 0, s, 1, reinterpret_cast<const __nv_bfloat16*>(logits), ld, V, stats, tb, depth, sp, rej_tokens, st);
  else launch_k(posterior_sample_kernel<__half>, dim3(1), dim3(32), 0, s, 1, reinterpret_cast<const __half*>(logits), ld, V, stats, tb, depth, sp, rej_tokens, st);
  return static_cast<int>(cudaGetLastError());
}

// inverse CDF over one row (minus rejected tokens): token = min{ v : cumsum_{w<=v} p'(w) >= u * total }
template <typename T>
__global__ void __launch_bounds__(1024) sample_commit_kernel(const T* __restrict__ logits, long ld, int V, const RowStats* __restrict__ stats,
                                                             TreeBuffers tb, int depth, SampleParams sp, const int* __restrict__ rej_tokens,
                                                             AcceptOut out, int* __restrict__ st, int64_t* __restrict__ out_ids, int out_cap,
                                                             int first_token) {
  __shared__ float part[1024];
  __shared__ float s_u;
  __shared__ int s_tok;
  pdl_launch_dependents();
  pdl_wait();
  const int node = first_token ? 0 : st[S_SNODE];
  const int n_rej = first_token ? 0 : st[S_SNREJ];
  const RowStats rs = stats[node];
  const T* x = logits + static_cast<long>(node) * ld;
  const int per = (V + 1023) / 1024;
  const int lo = threadIdx.x * per, hi = min(V, lo + per);
  auto weight = [&](int v) {
    const float lt = warp_temp<T>(x[v], sp.temperature);
    if (lt < rs.thr) return 0.f;
    for (int q = 0; q < n_rej; ++q)
      if (rej_tokens[q] == v) return 0.f;
    return expf(lt - rs.max);
  };
  float mine = 0.f;
  for (int v = lo; v < hi; ++v) mine += weight(v);
  part[threadIdx.x] = mine;
  if (threadIdx.x == 0) {
    s_u = next_uniform(sp, st);
    s_tok = -1;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float total = 0.f;
    for (int i = 0; i < 1024; ++i) total += part[i];
    const float target = s_u * total;
    float run = 0.f;
    int chunk = 1023;
    for (int i = 0; i < 1024; ++i) {
      if (run + part[i] >= target && part[i] > 0.f) {
        chunk = i;
        break;
      }
      run += part[i];
    }
    int tok = -1;
    const int clo = chunk * per, chi = min(V, clo + per);
    for (int v = clo; v < chi; ++v) {
      const float w = weight(v);
      if (w > 0.f) {
        tok = v;  // last positive-weight token of the chunk is the fallback for rounding at the chunk's end
        run += w;
        if (run >= target) break;
      }
    }
    if (tok < 0) {  // degenerate row: fall back to the first kept token
      for (int v = 0; v < V && tok < 0; ++v)
        if (weight(v) > 0.f) tok = v;
      if (tok < 0) tok = 0;
    }
    s_tok = tok;
    if (first_token) {
      st[S_BONUS] = tok;
    } else {
      const int D = depth + 2;
      const int best = st[S_BEST], a = st[S_ACC] - 1;
      commit_accept(tb, tb.retrieve + best * D, best, a, tok, D, out, st, out_ids, out_cap);
    }
  }
}

int launch_sample_commit(int dtype, const void* logits, long ld, int V, const RowStats* stats, TreeBuffers tb, int depth, SampleParams sp,
                         const int* rej_tokens, AcceptOut out, int* st, int64_t* out_ids, int out_cap, int first_token, cudaStream_t s) {
  if (dtype == DT_BF16) launch_k(sample_commit_kernel<__nv_bfloat16>, dim3(1), dim3(1024), 0, s, 1, reinterpret_cast<const __nv_bfloat16*>(logits), ld, V, stats, tb, depth, sp, rej_tokens, out, st, out_ids, out_cap, first_token);
  else launch_k(sample_commit_kernel<__half>, dim3(1), dim3(1024), 0, s, 1, reinterpret_cast<const __half*>(logits), ld, V, stats, tb, depth, sp, rej_tokens, out, st, out_ids, out_cap, first_token);
  return static_cast<int>(cudaGetLastError());
}

}  // namespace eb
