// Integer kernels of the cycle: draft-tree growth (top-k expand), global rerank + tree buffers, greedy posterior
// acceptance and KV compaction.  The reference runs these as ~12 tiny torch ops per level plus host-side Python
// loops with .tolist()/.item() syncs (cnets.py:728-827, utils.py:360-373, :435-452); here each is one small kernel
// whose inputs and outputs stay on the device, so the cycle has no host round trip.
//
// Tie policy: torch.topk leaves the order of equal values unspecified; these kernels use (value desc, flat index
// asc).  With that policy a parent is always selected before its equal-score child, so the "parent not selected"
// mis-link the reference can hit through ties (cnets.py:771, commented-out guard) cannot occur.
#include "tree_common.cuh"

namespace eb {

// a beats b in the descending (value, -index) order
__device__ __forceinline__ bool beats(float va, int ia, float vb, int ib) { return va > vb || (va == vb && ia < ib); }

// --------------------------------------------------------------------------------------------------------------
// level 0 seed: cnets.py:703-716
// --------------------------------------------------------------------------------------------------------------
__global__ void tree_seed_kernel(const float* __restrict__ topk_p, const int* __restrict__ topk_i,
                                 const int64_t* __restrict__ d2t, int k, TreeBuffers tb, const int* __restrict__ st) {
  pdl_launch_dependents();
  pdl_wait();
  const int j = threadIdx.x;
  if (j == 0) tb.parents[0] = 0;
  if (j < k) {
    int di = topk_i[j];
    if (di < 0 || di == 0x7fffffff) di = 0;  // only reachable with non-finite logits; stay in bounds
    const int tok = di + (d2t ? static_cast<int>(d2t[di]) : 0);
    tb.scores[j] = topk_p[j];
    tb.tokens[j] = tok;
    tb.front_scores[j] = topk_p[j];
    tb.front_ids[j] = tok;
    tb.front_src[j] = st[S_LASTROW];  // input_hidden = last_hidden repeated k times
    tb.front_cs[j] = j;
    tb.front_mask[2 * j] = (j < 64) ? (1ull << j) : 0ull;
    tb.front_mask[2 * j + 1] = (j >= 64) ? (1ull << (j - 64)) : 0ull;
  }
}
int launch_tree_seed(const float* topk_p, const int* topk_i, const int64_t* d2t, int k, TreeBuffers tb, int* st,
                     cudaStream_t s) {
  launch_k(tree_seed_kernel, dim3(1), dim3(32), 0, s, 1, topk_p, topk_i, d2t, k, tb, st);
  return static_cast<int>(cudaGetLastError());
}

// --------------------------------------------------------------------------------------------------------------
// level expansion: cnets.py:728-757.  One CTA, one thread per (frontier slot j, child c).
// --------------------------------------------------------------------------------------------------------------
constexpr int kExpandMaxK = 32;  // largest top_k of tree_expand_kernel: k * k candidates, one per thread of a 1024-thread CTA
static_assert(kExpandMaxK * kExpandMaxK <= 1024, "tree_expand_kernel runs one thread per candidate in a single CTA");

template <typename T>
__global__ void __launch_bounds__(1024) tree_expand_kernel(const float* __restrict__ topk_p, const int* __restrict__ topk_i,
                                                           const int64_t* __restrict__ d2t, int k, int level,
                                                           TreeBuffers tb) {
  pdl_launch_dependents();
  pdl_wait();
  // one thread per candidate and two mask words per frontier slot: all four arrays are sized by kExpandMaxK, the bound
  // launch_tree_expand enforces (eb200_create accepts top_k <= 16, well inside it)
  __shared__ float cu[kExpandMaxK * kExpandMaxK];
  __shared__ int tok[kExpandMaxK * kExpandMaxK];
  __shared__ uint64_t old_mask[2 * kExpandMaxK];
  __shared__ int new_cs[kExpandMaxK];
  const int e = threadIdx.x;
  const int kk = k * k;
  const int base = k + level * kk;
  if (e < k) {
    old_mask[2 * e] = tb.front_mask[2 * e];
    old_mask[2 * e + 1] = tb.front_mask[2 * e + 1];
    const int bias = 1 + kk * max(0, level - 1) + (level > 0 ? k : 0);
    tb.parents[1 + level * k + e] = tb.front_cs[e] + bias;
  }
  float my = -INFINITY;
  if (e < kk) {
    const int j = e / k;
    // cu_scores = topk_p + scores[:, None] evaluated in the model dtype (cnets.py:740)
    my = rnd<T>(topk_p[e] + tb.front_scores[j]);
    int di = topk_i[e];
    if (di < 0 || di == 0x7fffffff) di = 0;
    const int t = di + (d2t ? static_cast<int>(d2t[di]) : 0);
    cu[e] = my;
    tok[e] = t;
    tb.scores[base + e] = my;
    tb.tokens[base + e] = t;
  }
  __syncthreads();
  if (e < kk) {
    int rank = 0;
    for (int o = 0; o < kk; ++o) rank += beats(cu[o], o, my, e) ? 1 : 0;
    if (rank < k) new_cs[rank] = e;
  }
  __syncthreads();
  if (e < k) {
    const int f = new_cs[e];
    const int src = f / k;
    const int col = (level + 1) * k + e;
    tb.front_scores[e] = cu[f];
    tb.front_cs[e] = f;
    tb.front_src[e] = src;
    tb.front_ids[e] = tok[f];
    uint64_t m0 = old_mask[2 * src], m1 = old_mask[2 * src + 1];
    // the last level's own columns can lie beyond the two mask words (depth * k <= 128 bounds the columns a draft forward
    // attends over, and nothing attends over the frontier the last level leaves): drop them rather than shift by >= 64
    if (col < 64) m0 |= 1ull << col; else if (col < 128) m1 |= 1ull << (col - 64);
    tb.front_mask[2 * e] = m0;
    tb.front_mask[2 * e + 1] = m1;
  }
}
int launch_tree_expand(int dtype, const float* topk_p, const int* topk_i, const int64_t* d2t, int k, int level,
                       TreeBuffers tb, cudaStream_t s) {
  if (k > kExpandMaxK) return static_cast<int>(cudaErrorInvalidValue);
  if (dtype == DT_BF16) launch_k(tree_expand_kernel<__nv_bfloat16>, dim3(1), dim3(1024), 0, s, 1, topk_p, topk_i, d2t, k, level, tb);
  else launch_k(tree_expand_kernel<__half>, dim3(1), dim3(1024), 0, s, 1, topk_p, topk_i, d2t, k, level, tb);
  return static_cast<int>(cudaGetLastError());
}

// --------------------------------------------------------------------------------------------------------------
// global rerank + tree buffers: cnets.py:760-827
// --------------------------------------------------------------------------------------------------------------
constexpr int kMaxPool = 4096;
constexpr int kMaxNodes = 128;

__global__ void __launch_bounds__(1024) tree_finalize_kernel(int k, int depth, int total, int sort_rows, TreeBuffers tb,
                                                             int* __restrict__ st) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float sc[kMaxPool];
  __shared__ unsigned char selected[kMaxPool];
  __shared__ int top_idx[kMaxNodes];     // ascending flat indices of the selected candidates
  __shared__ int parent[kMaxNodes + 1];  // node -> parent node
  __shared__ int posn[kMaxNodes + 1];
  __shared__ unsigned char is_parent[kMaxNodes + 1];
  __shared__ int leaf_rank[kMaxNodes + 1];
  __shared__ int s_nleaf, s_maxd;
  const int n = k + depth * k * k;
  const int T = total + 1;
  const int D = depth + 2;
  const int tid = threadIdx.x;

  for (int i = tid; i < n; i += 1024) {
    sc[i] = tb.scores[i];
    selected[i] = 0;
  }
  if (tid <= T) is_parent[tid] = 0;
  __syncthreads();
  // top-`total` by rank counting
  for (int i = tid; i < n; i += 1024) {
    const float v = sc[i];
    int rank = 0;
    for (int o = 0; o < n; ++o) rank += beats(sc[o], o, v, i) ? 1 : 0;
    if (rank < total) selected[i] = 1;
  }
  __syncthreads();
  // ascending index order == position among the selected (torch.sort of the indices, cnets.py:764)
  for (int i = tid; i < n; i += 1024) {
    if (selected[i]) {
      int pos = 0;
      for (int o = 0; o < i; ++o) pos += selected[o];
      top_idx[pos] = i;
    }
  }
  __syncthreads();
  // parents: searchsorted(top_idx, draft_parent - 1) + 1, root where draft_parent == 0 (cnets.py:769-773)
  if (tid == 0) {
    parent[0] = 0;
    tb.draft_tokens[0] = st[S_BONUS];  // node 0 = the token sampled from the target (sample_token)
  }
  if (tid < total) {
    const int flat = top_idx[tid];
    tb.draft_tokens[tid + 1] = tb.tokens[flat];
    const int dp = tb.parents[flat / k];
    int pn = 0;
    if (dp != 0) {
      const int target = dp - 1;
      int lo = 0, hi = total;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (top_idx[mid] < target) lo = mid + 1; else hi = mid;
      }
      pn = lo + 1;
    }
    parent[tid + 1] = pn;
    tb.parent_node[tid + 1] = pn;
    is_parent[pn] = 1;  // benign race: all writers store 1
  }
  if (tid == 0) {
    tb.parent_node[0] = 0;
    is_parent[0] = 1;
  }
  __syncthreads();
  // ancestor masks (tree_mask[i+1] = onehot | tree_mask[parent], column 0 all ones) and depth = popcount - 1
  if (tid < T) {
    uint64_t m0 = 1ull, m1 = 0ull;
    int p = tid, guard = 0;
    while (p != 0 && guard++ < kMaxNodes) {
      if (p < 64) m0 |= 1ull << p; else m1 |= 1ull << (p - 64);
      p = parent[p];
    }
    tb.tree_mask[2 * tid] = m0;
    tb.tree_mask[2 * tid + 1] = m1;
    const int d = __popcll(m0) + __popcll(m1) - 1;
    posn[tid] = d;
    tb.tree_pos[tid] = d;
  }
  __syncthreads();
  if (tid == 0) {
    int nl = 0, md = 0;
    for (int i = 0; i < T; ++i) {
      leaf_rank[i] = is_parent[i] ? -1 : nl;
      nl += is_parent[i] ? 0 : 1;
      md = max(md, posn[i]);
    }
    s_nleaf = nl;
    s_maxd = md + 1;
    st[S_NLEAF] = nl;
    st[S_MAXDEPTH] = md + 1;
  }
  __syncthreads();
  // retrieve_indices: root->leaf node paths, -1 padded, leaves in ascending node id (cnets.py:791-809)
  for (int i = tid; i < T * D; i += 1024) tb.retrieve[i] = -1;
  __syncthreads();
  if (tid < T && leaf_rank[tid] >= 0) {
    int cid = tid;
    int* row = tb.retrieve + leaf_rank[tid] * D;
    for (int j = posn[tid]; j >= 0; --j) {
      row[j] = cid;
      cid = parent[cid];
    }
  }
  if (sort_rows) {  // cnets.py:811-821: lexicographic row order with -1 -> large (sampling only)
    __syncthreads();
    __threadfence_block();
    __shared__ int rows_tmp[kMaxNodes * 16];
    const int nl = s_nleaf;
    if (D <= 16) {
      for (int i = tid; i < nl * D; i += 1024) rows_tmp[i] = tb.retrieve[i];
      __syncthreads();
      if (tid < nl) {
        int rank = 0;
        for (int o = 0; o < nl; ++o) {
          if (o == tid) continue;
          int cmp = 0;  // <0: o before tid
          for (int j = 0; j < D && cmp == 0; ++j) {
            const int a = rows_tmp[o * D + j] < 0 ? (total + 5) : rows_tmp[o * D + j];
            const int b = rows_tmp[tid * D + j] < 0 ? (total + 5) : rows_tmp[tid * D + j];
            cmp = (a < b) ? -1 : (a > b ? 1 : 0);
          }
          if (cmp < 0 || (cmp == 0 && o < tid)) ++rank;
        }
        for (int j = 0; j < D; ++j) tb.retrieve[rank * D + j] = rows_tmp[tid * D + j];
      }
    }
  }
}
int launch_tree_finalize(int dtype, int k, int depth, int total, int sort_rows, TreeBuffers tb, int* st, cudaStream_t s) {
  (void)dtype;
  const int n = k + depth * k * k;
  if (n > kMaxPool || total + 1 > kMaxNodes || total > n || (sort_rows && depth + 2 > 16))
    return static_cast<int>(cudaErrorInvalidValue);
  launch_k(tree_finalize_kernel, dim3(1), dim3(1024), 0, s, 1, k, depth, total, sort_rows, tb, st);
  return static_cast<int>(cudaGetLastError());
}

// --------------------------------------------------------------------------------------------------------------
// greedy posterior + commit bookkeeping: utils.py:360-373, :435-441, :458-464
// --------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) greedy_accept_kernel(const int* __restrict__ node_argmax, TreeBuffers tb, int T,
                                                            int depth, AcceptOut out, int* __restrict__ st,
                                                            int64_t* __restrict__ out_ids, int out_cap) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ int acc_len[kMaxNodes];
  __shared__ int s_best, s_acc;
  const int D = depth + 2;
  const int n_leaf = st[S_NLEAF];
  const int maxd = st[S_MAXDEPTH];
  const int r = threadIdx.x;
  if (r < n_leaf) {
    const int* row = tb.retrieve + r * D;
    int a = 0;
    for (int j = 1; j < maxd; ++j) {
      const int node = row[j];
      if (node < 0) break;  // candidate token -1 never equals an arg-max
      if (tb.draft_tokens[node] != node_argmax[row[j - 1]]) break;
      ++a;
    }
    acc_len[r] = a;
  }
  __syncthreads();
  if (r == 0) {
    int best = 0, a = acc_len[0];
    for (int i = 1; i < n_leaf; ++i)
      if (acc_len[i] > a) {
        a = acc_len[i];
        best = i;
      }
    s_best = best;
    s_acc = a;
    const int* row = tb.retrieve + best * D;
    commit_accept(tb, row, best, a, node_argmax[row[a]], D, out, st, out_ids, out_cap);
  }
}
int launch_greedy_accept(const int* node_argmax, TreeBuffers tb, int T, int depth, AcceptOut out, int* st,
                         int64_t* out_ids, int out_cap, cudaStream_t s) {
  if (T > 128) return static_cast<int>(cudaErrorInvalidValue);
  launch_k(greedy_accept_kernel, dim3(1), dim3(128), 0, s, 1, node_argmax, tb, T, depth, out, st, out_ids, out_cap);
  return static_cast<int>(cudaGetLastError());
}

// --------------------------------------------------------------------------------------------------------------
// KV compaction: utils.py:444-452.  Rows NPREV + sel[j] -> NPREV + j of every [kv_cap][128] plane.
// Gather into registers first (the reference gathers into a temporary), then store: sources and destinations overlap.
// --------------------------------------------------------------------------------------------------------------
// One CTA moves at most kCompactRows rows (row j = threadIdx.x >> 4; rows beyond would be silently left in place).  A cycle
// commits accept_length + 1 <= depth + 2 rows -- the root's token plus one per draft level, a whole retrieve row -- and
// eb200_create keeps depth + 2 <= kMaxRetrieveWidth, so st[S_ACC] never reaches past the CTA's rows.  Raise both together.
constexpr int kCompactRows = 16;
constexpr int kMaxRetrieveWidth = 16;  // depth + 2 of the deepest accepted tree (eb200_create: depth <= 14)
static_assert(kMaxRetrieveWidth <= kCompactRows, "kv_compact_kernel must cover a full-depth commit (depth + 2 rows)");
__global__ void __launch_bounds__(kCompactRows * 16) kv_compact_kernel(uint4* kv, long plane_stride_v, long kv_cap, const int* sel, const int* st) {
  pdl_launch_dependents();
  pdl_wait();
  // sel / st are written by the accept kernel right before this one: dependent loads (see common.cuh:ld_dep)
  const int n = ld_dep(st + S_ACC);
  const int base = ld_dep(st + S_NPREV);
  uint4* plane = kv + static_cast<long>(blockIdx.x) * plane_stride_v;
  const int j = threadIdx.x >> 4, ch = threadIdx.x & 15;  // 16 rows x 16 chunks of 16 B (128 x 2-byte elements)
  uint4 v = make_uint4(0, 0, 0, 0);
  const bool act = (j < n) && (j > 0);
  if (act) v = plane[static_cast<long>(base + ld_dep(sel + j)) * 16 + ch];
  __syncthreads();
  if (act) plane[static_cast<long>(base + j) * 16 + ch] = v;
}
int launch_kv_compact(int dtype, void* kv_base, long plane_stride, int n_planes, long kv_cap, const int* sel, const int* st,
                      cudaStream_t s) {
  (void)dtype;
  launch_k(kv_compact_kernel, dim3(n_planes), dim3(kCompactRows * 16), 0, s, 1, reinterpret_cast<uint4*>(kv_base), plane_stride / 8, kv_cap, sel, st);
  return static_cast<int>(cudaGetLastError());
}

}  // namespace eb
