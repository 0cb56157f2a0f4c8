// eagle_b200 engine: device-resident state of one EaModel (target weights, draft head, both KV caches, the
// current draft tree) and the host-side launch sequences for prefill / one draft->verify->accept cycle.
// Implements the C ABI declared in include/eagle_b200.h.  Host code only enqueues kernels on one stream; every
// per-cycle quantity (committed length, accepted rows, tree shape) lives in a device int array (kernels.h StateIdx).
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <string>
#include <vector>

#include "../../include/eagle_b200.h"
#include "kernels.h"

using namespace eb;

struct eb200_nccl_id {
  char internal[128];
};

// ------------------------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------------------------
static thread_local char g_err[1024] = "";
static int fail(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return 1;
}
#define CK(call)                                                                                         \
  do {                                                                                                   \
    cudaError_t _e = (call);                                                                             \
    if (_e != cudaSuccess) return fail("%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(_e)); \
  } while (0)
#define CKL(call)                                                                                        \
  do {                                                                                                   \
    int _e = (call);                                                                                     \
    if (_e != 0) return fail("%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString((cudaError_t)_e)); \
  } while (0)
#define TRY(call)            \
  do {                       \
    int _r = (call);         \
    if (_r != 0) return _r;  \
  } while (0)

extern "C" const char* eb200_last_error(void) { return g_err; }
extern "C" int eb200_abi_version(void) { return EB200_ABI_VERSION; }

// ------------------------------------------------------------------------------------------------------------
// TMA descriptors (driver entry point resolved at run time: no link-time libcuda dependency)
// ------------------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn g_encode = nullptr;
static int resolve_encode() {
  if (g_encode) return 0;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult q;
  CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q));
  if (!fn || q != cudaDriverEntryPointSuccess) return fail("cuTensorMapEncodeTiled not available from the driver");
  g_encode = reinterpret_cast<EncodeTiledFn>(fn);
  return 0;
}
// row-major [rows][cols] 2-byte elements; box = box_rows x 64 columns (128 B), SWIZZLE_128B
static int make_tmap(CUtensorMap* m, int dtype, const void* ptr, uint64_t rows, uint64_t cols, uint32_t box_rows) {
  TRY(resolve_encode());
  if ((cols * 2) % 16) return fail("tensor map: row pitch %llu B is not a multiple of 16", (unsigned long long)cols * 2);
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {cols * 2};
  cuuint32_t box[2] = {64, box_rows};
  cuuint32_t es[2] = {1, 1};
  CUresult r = g_encode(m, dtype == DT_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2,
                        const_cast<void*>(ptr), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail("cuTensorMapEncodeTiled failed (%d) rows=%llu cols=%llu box_rows=%u", (int)r,
                                     (unsigned long long)rows, (unsigned long long)cols, box_rows);
  return 0;
}
// row-major [rows][cols] int8 weights of the W8A16 GEMM; box = 128 rows x 64 columns (64 B), unswizzled (the MMA warpgroups read
// it with generic loads and write the swizzled model-dtype tile themselves)
static int make_tmap_w8(CUtensorMap* m, const void* ptr, uint64_t rows, uint64_t cols) {
  TRY(resolve_encode());
  if (cols % 16) return fail("int8 tensor map: row pitch %llu B is not a multiple of 16", (unsigned long long)cols);
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {cols};
  cuuint32_t box[2] = {64, 128};
  cuuint32_t es[2] = {1, 1};
  CUresult r = g_encode(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(ptr), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail("cuTensorMapEncodeTiled (int8) failed (%d) rows=%llu cols=%llu", (int)r, (unsigned long long)rows,
                                     (unsigned long long)cols);
  return 0;
}
// W4A16 (launch_gemm_w4): the repacked nibble tiles [n_pad / 128][K / 64][4096 B] as rows of 256 B, box = one tile; the transposed
// absmax [K / 64][n_pad] fp32, box = the 128 values of one tile
static int make_tmap_w4(CUtensorMap* w, CUtensorMap* a, const void* tiles, const float* absmax, uint64_t n_pad, uint64_t K) {
  TRY(resolve_encode());
  const cuuint64_t wdims[2] = {256, n_pad * K / 2 / 256}, wstrides[1] = {256}, adims[2] = {n_pad, K / 64}, astrides[1] = {n_pad * 4};
  const cuuint32_t wbox[2] = {256, 16}, abox[2] = {128, 1}, es[2] = {1, 1};
  CUresult r = g_encode(w, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(tiles), wdims, wstrides, wbox, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r == CUDA_SUCCESS)
    r = g_encode(a, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(absmax), adims, astrides, abox, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                 CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail("cuTensorMapEncodeTiled (4-bit) failed (%d) n_pad=%llu K=%llu", (int)r, (unsigned long long)n_pad,
                                     (unsigned long long)K);
  return 0;
}
// FP8 (launch_gemm_fp8): the repacked e4m3 [N][K] maps like an int8 weight; the block scales [N / 128][K / 128][4] fp32, box = the
// 16 B of one tile and 128-column block
static int make_tmap_fp8(CUtensorMap* w, CUtensorMap* sc, const void* q, const float* scales, uint64_t N, uint64_t K) {
  TRY(make_tmap_w8(w, q, N, K));
  const cuuint64_t dims[2] = {K / 128 * 4, N / 128}, strides[1] = {K / 128 * 16};
  const cuuint32_t box[2] = {4, 1}, es[2] = {1, 1};
  const CUresult r = g_encode(sc, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(scales), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                              CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail("cuTensorMapEncodeTiled (fp8 scales) failed (%d) N=%llu K=%llu", (int)r, (unsigned long long)N,
                                     (unsigned long long)K);
  return 0;
}

// ------------------------------------------------------------------------------------------------------------
// engine data
// ------------------------------------------------------------------------------------------------------------
// the flags that store the target's decoder projections quantized (one at a time)
constexpr int kTargetQuantFlags = EB200_FLAG_TARGET_INT8 | EB200_FLAG_TARGET_NF4 | EB200_FLAG_TARGET_FP4 | EB200_FLAG_TARGET_FP8;
struct Linear {
  void* w = nullptr;
  int N = 0, K = 0;
  int esize = 2;              // bytes per weight: 2 (model dtype) or 1 (int8 / FP8, EB200_FLAG_TARGET_INT8 / _FP8)
  float* scale = nullptr;     // int8 only: fp32 scale of each row (SCB)
  float* absmax = nullptr;    // 4-bit only: w holds the repacked nibble tiles, absmax [K/64][n_pad] (launch_w4_repack)
  int w4_quant = -1;          // 4-bit only: W4_NF4 / W4_FP4
  int n_pad = 0;              // 4-bit only: N rounded up to whole 128-row tiles
  float* scale_inv = nullptr; // FP8 only: w holds the repacked e4m3 [N][K], scale_inv the block scales [N/128][K/128][4] (launch_fp8_repack)
  CUtensorMap tm, tm_abs;     // tm_abs: the 4-bit absmax / FP8 block scales
  uint64_t loaded_rows = 0;   // bookkeeping for fused / sharded loads
  uint64_t loaded_scales = 0; // int8 SCB / 4-bit absmax / FP8 weight_scale_inv
};
struct ActBuf {  // an activation buffer usable as the X operand of the GEMM (64 rows; 256 where the prompt prefill runs through it)
  void* p = nullptr;
  int cols = 0, rows = 64;
  CUtensorMap tm16, tm64, tm256;
};
struct Layer {
  Linear qkv, o, gu, down;  // gu: gate_proj and up_proj interleaved in 64-row groups (EPI_SWIGLU_IL)
  void* ln1 = nullptr;  // input_layernorm (null for EAGLE-1 layer 0)
  void* ln2 = nullptr;  // post_attention_layernorm
  bool ln1_loaded = false, ln2_loaded = false;
};
struct RowCtx {
  int kv_bound = 0;  // host-known upper bound of n_ctx + n_tree (sizes the attention score strip)
  int mpad, rows, rows_idx;
  DynInt n_ctx;
  int n_tree;
  const uint64_t* mask;
  DynInt pos_base;
  const int* pos_arr;
  int pos_mstride;
  DynInt kv_base;
};

struct ProfRec {
  cudaEvent_t a, b;
  int cat;  // 0 gemm, 1 attention, 2 other
  double bytes;
  int verify;
};

struct eb200_engine {
  eb200_config c;
  int dtype;
  cudaStream_t stream = nullptr;
  std::vector<void*> allocs;
  bool finalized = false;
  // dims (local to this TP rank where sharded)
  int H, I_l, L, nh_l, nkv_l, V, V_l;
  int Hh, Ih, hL, hnh, hnkv, Vd, F;  // F = feature width fed to the head (3H for EAGLE-3, H for EAGLE-1)
  int T, k, depth, D;                 // tree nodes, top-k, depth, D = depth + 2
  long cap, dcap;                     // KV rows: target, draft
  int act_rows = 64;                  // rows of the target's activation buffers: 256 when the prompt prefill runs 256-row GEMMs
  // target weights
  void* t_embed = nullptr;
  bool t_embed_loaded = false;
  std::vector<Layer> tl;
  void* t_norm = nullptr;
  bool t_norm_loaded = false;
  Linear t_head;
  void *t_cos = nullptr, *t_sin = nullptr;
  int t_npos = 0;
  // head weights
  void* h_embed = nullptr;
  bool h_embed_own = false;
  Linear h_fc;
  void* h_fc_bias = nullptr;
  bool h_fc_bias_loaded = false;
  std::vector<Layer> hl;
  void *h_hidden_norm = nullptr, *h_norm = nullptr;  // EAGLE-3
  bool h_hidden_norm_loaded = false, h_norm_loaded = false;
  Linear h_head;  // EAGLE-3 draft lm_head
  int64_t* d2t = nullptr;
  bool d2t_loaded = false;
  void *h_cos = nullptr, *h_sin = nullptr;
  int h_npos = 0;
  // KV caches: [layer][k|v][kv_head][cap][128]
  void *t_kv = nullptr, *d_kv = nullptr;
  // activations
  void *x = nullptr, *q = nullptr, *logits = nullptr, *feat = nullptr, *feat_all = nullptr;
  ActBuf xn, attn, act, xn_last;
  void *d_q = nullptr, *d_h2 = nullptr, *d_logits = nullptr;
  ActBuf d_feat, d_cat, d_h, d_attn, d_xn, d_act, d_out;
  // split-K
  float* ws = nullptr;
  size_t ws_bytes = 0;
  size_t l2_bytes = 0;  // device L2 size: caps the weight bytes prefetched ahead of a GEMM
  int* counters = nullptr;
  // tree + cycle state
  int* st = nullptr;
  TreeBuffers tb;
  float* topk_p = nullptr;
  int* topk_i = nullptr;
  int* node_argmax = nullptr;
  int* accepted = nullptr;  // [2*D]: committed tokens, then next stable-pass token inputs
  int* sel_nodes = nullptr;
  int* ident = nullptr;     // 0..63
  int64_t* ids_dev = nullptr;  // prompt / shifted ids
  int64_t* out_ids_dev = nullptr;
  int64_t* pinned = nullptr;   // host-visible mirror of the last accept
  cudaEvent_t ev_done = nullptr;
  cudaEvent_t ev_slot[2] = {nullptr, nullptr};  // completion of the cycle whose results sit in read-back slot 0 / 1
  unsigned launch_seq = 0, collect_seq = 0;     // cycles launched / collected (eb200_generate keeps one cycle in flight)
  // counters / profiling
  eb200_stats stats;
  bool profiling = false;
  bool in_verify = false;
  std::vector<ProfRec> prof;
  std::vector<cudaEvent_t> ev_pool;
  int last_best = 0, last_acc = 0;
  long committed = 0;  // host mirror of S_N
  int naive_tok = 0;   // vanilla decoding: the token the next eb200_naive_step feeds
  // sampling posterior (temperature > 0)
  bool sampling = false;
  SampleParams sp;
  RowStats* row_stats = nullptr;  // [128]
  int* rej_tokens = nullptr;      // [64]
  float* uniforms = nullptr;      // injected uniforms (tests)
  int n_uniforms = 0;
  void* lg_recv = nullptr;        // TP: gathered logits shards [tp][64][V_l]
  void* logits_full = nullptr;    // TP: [64][tp*V_l]
  // CUDA graph of one cycle (captured after the first eager cycle; all per-cycle values live in device state)
  cudaGraph_t graph = nullptr;
  cudaGraphExec_t graph_exec = nullptr;
  uint64_t launches_per_cycle = 0;
  int eager_cycles = 0;
  bool capturing = false;
  int kv_bucket = 0;  // attention score-strip capacity baked into the launches (and the captured graph)
  // static draft tree (eb200_set_static_tree): host tables + their device copies
  bool static_tree = false;
  StaticTreeHost stree;
  int *st_tree_indices = nullptr, *st_sel = nullptr, *st_src = nullptr, *ss_tokens = nullptr;
  uint64_t* st_lmask = nullptr;
  unsigned long long* attn_trace = nullptr;  // EB200_ATTN_TRACE=<file>: phase stamps of the last verify attention launch
  // TP
  void* nccl_comm = nullptr;
  float* f32buf = nullptr;      // [64][H] fp32 partial sums of the row-parallel projections (all-reduced in place)
  uint32_t* am_send = nullptr;  // [2*128] local (value, index) arg-max pairs
  uint32_t* am_recv = nullptr;  // [tp][2*128]
  Linear t_head_full;           // EAGLE-1 + TP: the draft needs the whole target lm_head
  // TP over NVLink peer memory (ChainTP, kernels.h): one window per rank, opened on the peers through CUDA IPC
  char* tp_win = nullptr;
  size_t tp_win_bytes = 0;
  char* tp_peer[kMaxTp] = {};
  bool tp_fused = false;        // peers opened: row-parallel projections finish over peer memory (tp_fused.cu), not through NCCL
  long tp_inbox_off = 0, tp_flag_off = 0, tp_ready_off = 0, tp_am_off = 0;
  int* tp_epoch = nullptr;
  // lm_head launch (mega.cu)
  int* chain_sync = nullptr;    // [2] self-resetting counters
  unsigned long long* chain_timing = nullptr;  // [4] in-kernel %globaltimer accounting (ns sum, launches, scratch)
  double chain_bytes_cycle = 0;  // algorithmic bytes of the chain launches captured in the cycle graph
  double chain_bytes_pending = 0;
  float* tile_val = nullptr;    // [lm_head tiles][64] per-tile row maxima of the fused arg-max
  int* tile_idx = nullptr;
  bool chain_head = false;      // the target lm_head runs as one mega.cu launch (fused arg-max / direct store)
  bool fused_e3_input = true;   // EAGLE-3 draft input (gather + two RMSNorms + concat) as one launch
  std::map<const void*, CUtensorMap> kv_maps;  // TMA descriptors of the K/V cache planes (attention.cu), built on first use
};


static int dalloc(eb200_engine* e, void** p, size_t bytes, bool zero = true) {
  if (bytes == 0) bytes = 16;
  CK(cudaMalloc(p, bytes));
  e->allocs.push_back(*p);
  if (zero) CK(cudaMemsetAsync(*p, 0, bytes, e->stream));
  return 0;
}
// wq: 0 model dtype, EB200_FLAG_TARGET_INT8 / _NF4 / _FP4 / _FP8
static int alloc_linear(eb200_engine* e, Linear& l, int N, int K, int wq = 0) {
  l.N = N;
  l.K = K;
  if (wq == EB200_FLAG_TARGET_FP8) {
    if (N % 128 || K % 128) return fail("FP8 target weights need out- and in-features divisible by 128 (128 x 128 scale blocks), got [%d, %d]", N, K);
    l.esize = 1;
    TRY(dalloc(e, reinterpret_cast<void**>(&l.scale_inv), static_cast<size_t>(N / 128) * (K / 128) * 16));
    return dalloc(e, &l.w, static_cast<size_t>(N) * K, false);
  }
  if (wq == EB200_FLAG_TARGET_NF4 || wq == EB200_FLAG_TARGET_FP4) {
    if (K % 64) return fail("4-bit target weights need in-features divisible by 64 (blocksize 64 blocks must not straddle rows), got %d", K);
    l.w4_quant = wq == EB200_FLAG_TARGET_NF4 ? W4_NF4 : W4_FP4;
    l.n_pad = (N + 127) / 128 * 128;
    l.esize = 1;  // per two weights
    TRY(dalloc(e, reinterpret_cast<void**>(&l.absmax), static_cast<size_t>(l.n_pad) * (K / 64) * 4));
    return dalloc(e, &l.w, static_cast<size_t>(l.n_pad) * K / 2);
  }
  const bool int8 = wq == EB200_FLAG_TARGET_INT8;
  l.esize = int8 ? 1 : 2;
  if (int8) TRY(dalloc(e, reinterpret_cast<void**>(&l.scale), static_cast<size_t>(N) * 4, false));
  return dalloc(e, &l.w, static_cast<size_t>(N) * K * l.esize, false);
}
static int alloc_act(eb200_engine* e, ActBuf& a, int cols, int rows = 64) {
  a.cols = cols;
  a.rows = rows;
  TRY(dalloc(e, &a.p, static_cast<size_t>(rows) * cols * 2));
  TRY(make_tmap(&a.tm16, e->dtype, a.p, rows, cols, 16));
  TRY(make_tmap(&a.tm64, e->dtype, a.p, rows, cols, 64));
  if (rows >= 256) TRY(make_tmap(&a.tm256, e->dtype, a.p, rows, cols, 256));
  return 0;
}

extern "C" int eb200_create(const eb200_config* cfg, eb200_engine** out) {
  if (!cfg || !out) return fail("eb200_create: null argument");
  if (cfg->abi_version != EB200_ABI_VERSION) return fail("ABI version mismatch: header %d, library %d", cfg->abi_version, EB200_ABI_VERSION);
  const eb200_config& c = *cfg;
  {
    int n_dev = 0;
    if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev == 0)
      return fail("no CUDA device visible: eagle_b200 has no CPU path (the engine is sm_90a CUDA only)");
  }
  if (c.dtype != EB200_BF16 && c.dtype != EB200_FP16) return fail("dtype must be bf16 or fp16");
  if (c.vocab_size < 1 || c.hidden_size < 128 || c.intermediate_size < 64 || c.num_layers < 1 || c.num_heads < 1 ||
      c.num_kv_heads < 1 || c.head_hidden_size < 128 || c.head_intermediate_size < 64 || c.head_num_heads < 1 ||
      c.head_num_kv_heads < 1 || c.max_length < 64)
    return fail("eb200_create: non-positive model dimensions");
  if (c.num_heads % c.num_kv_heads || c.head_num_heads % c.head_num_kv_heads) return fail("heads must be a multiple of kv heads");
  if (c.hidden_size % 64 || c.intermediate_size % 64 || c.head_hidden_size % 64 || c.head_intermediate_size % 64)
    return fail("hidden / intermediate sizes must be multiples of 64");
  if (c.hidden_size % c.num_heads || c.hidden_size / c.num_heads != 128) return fail("target head_dim must be 128");
  if (c.head_hidden_size / std::max(1, c.head_num_heads) != 128) return fail("draft head_dim must be 128");
  if (c.tp_size < 1 || c.tp_rank < 0 || c.tp_rank >= c.tp_size) return fail("bad tp rank/size");
  if (c.num_heads % c.tp_size || c.num_kv_heads % c.tp_size || c.intermediate_size % c.tp_size)
    return fail("heads / kv heads / intermediate size must divide by tp_size");
  {
    const int wq = c.flags & kTargetQuantFlags;
    if (wq & (wq - 1))
      return fail("EB200_FLAG_TARGET_INT8, EB200_FLAG_TARGET_NF4, EB200_FLAG_TARGET_FP4 and EB200_FLAG_TARGET_FP8 exclude each other");
    // the 4-bit and FP8 loaders place whole checkpoint tensors (no tensor-parallel sharding of codes, absmax or block scales)
    if ((wq & (EB200_FLAG_TARGET_NF4 | EB200_FLAG_TARGET_FP4)) && c.tp_size > 1)
      return fail("4-bit target weights (EB200_FLAG_TARGET_NF4 / _FP4) are not supported with tensor parallelism (tp_size %d); "
                  "they run on one GPU", c.tp_size);
    if ((wq & EB200_FLAG_TARGET_FP8) && c.tp_size > 1)
      return fail("FP8 target weights (EB200_FLAG_TARGET_FP8) are not supported with tensor parallelism (tp_size %d); they run on one GPU",
                  c.tp_size);
  }
  if (c.total_token < 2 || c.total_token > 64) return fail("total_token must be in [2, 64]");
  if (c.top_k < 1 || c.top_k > 16) return fail("top_k must be in [1, 16]");
  if (c.depth < 1 || c.depth + 2 > 16) return fail("depth must be in [1, 14]");
  if (c.top_k * (c.depth) > 128) return fail("depth * top_k must be <= 128 (draft tree columns)");
  if (c.top_k + c.depth * c.top_k * c.top_k < c.total_token - 1) return fail("candidate pool smaller than total_token - 1");
  {
    // the draft planes hold max_length + 128 + depth * top_k rows, and the attention score strip must be able to span them all
    const long dcap = static_cast<long>(c.max_length) + 64 + c.depth * c.top_k + 64;
    const int lim = attention_max_kv();
    if (dcap > lim)
      return fail("max_length %d too large: the draft KV needs %ld rows, tree attention holds at most %d (max_length <= %d at "
                  "depth %d, top_k %d)", c.max_length, dcap, lim, lim - 128 - c.depth * c.top_k, c.depth, c.top_k);
  }
  int dev_count = 0;
  CK(cudaGetDeviceCount(&dev_count));
  if (dev_count == 0) return fail("no CUDA device: eagle_b200 has no CPU path");
  CK(cudaSetDevice(c.device));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, c.device));
  if (prop.major != 9 || prop.minor != 0)
    return fail("device %d is sm_%d%d; eagle_b200 kernels are sm_90a (H100) only", c.device, prop.major, prop.minor);

  eb200_engine* e = new eb200_engine();
  e->c = c;
  e->dtype = c.dtype;
  e->l2_bytes = static_cast<size_t>(prop.l2CacheSize);
  memset(&e->stats, 0, sizeof(e->stats));
  {
    cudaError_t se = cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking);
    if (se != cudaSuccess) {
      delete e;
      return fail("cudaStreamCreate failed: %s", cudaGetErrorString(se));
    }
  }
  e->H = c.hidden_size;
  e->L = c.num_layers;
  e->V = c.vocab_size;
  e->nh_l = c.num_heads / c.tp_size;
  e->nkv_l = c.num_kv_heads / c.tp_size;
  e->I_l = c.intermediate_size / c.tp_size;
  e->V_l = c.tp_size == 1 ? c.vocab_size : (c.vocab_size + c.tp_size - 1) / c.tp_size;
  e->Hh = c.head_hidden_size;
  e->Ih = c.head_intermediate_size;
  e->hL = c.eagle3 ? 1 : std::max(1, c.head_num_layers);
  e->hnh = c.head_num_heads;
  e->hnkv = c.head_num_kv_heads;
  e->Vd = c.eagle3 ? c.draft_vocab_size : c.vocab_size;
  e->F = c.eagle3 ? 3 * c.hidden_size : c.hidden_size;
  e->T = c.total_token;
  e->k = c.top_k;
  e->depth = c.depth;
  e->D = c.depth + 2;
  e->cap = c.max_length + 64;
  {
    const char* pe = getenv("EB200_PREFILL_ROWS");  // 64 = weights streamed once per 64 prompt tokens instead of 256
    const int want = pe ? atoi(pe) : 256;
    e->act_rows = (want >= 256 && c.tp_size == 1 && !(c.flags & EB200_FLAG_SIMT_GEMM)) ? 256 : 64;
  }
  e->dcap = c.max_length + 64 + c.depth * c.top_k + 64;
  if (!c.eagle3 && c.head_hidden_size != c.hidden_size) return fail("EAGLE-1 head hidden size must equal the target's");

  int rc = 0;
  auto body = [&]() -> int {
    const int H = e->H, Hh = e->Hh;
    // ---- target weights
    TRY(dalloc(e, &e->t_embed, static_cast<size_t>(e->V) * H * 2, false));
    e->tl.resize(e->L);
    const int wq = c.flags & kTargetQuantFlags;
    for (auto& l : e->tl) {
      TRY(alloc_linear(e, l.qkv, (e->nh_l + 2 * e->nkv_l) * 128, H, wq));
      TRY(alloc_linear(e, l.o, H, e->nh_l * 128, wq));
      TRY(alloc_linear(e, l.gu, 2 * e->I_l, H, wq));
      TRY(alloc_linear(e, l.down, H, e->I_l, wq));
      TRY(dalloc(e, &l.ln1, H * 2, false));
      TRY(dalloc(e, &l.ln2, H * 2, false));
    }
    TRY(dalloc(e, &e->t_norm, H * 2, false));
    TRY(alloc_linear(e, e->t_head, e->V_l, H));
    // ---- head weights
    e->hl.resize(e->hL);
    const int qk_in = c.eagle3 ? 2 * Hh : Hh;
    for (int i = 0; i < e->hL; ++i) {
      Layer& l = e->hl[i];
      TRY(alloc_linear(e, l.qkv, (e->hnh + 2 * e->hnkv) * 128, qk_in));
      TRY(alloc_linear(e, l.o, Hh, e->hnh * 128));
      TRY(alloc_linear(e, l.gu, 2 * e->Ih, Hh));
      TRY(alloc_linear(e, l.down, Hh, e->Ih));
      if (c.eagle3 || i > 0) TRY(dalloc(e, &l.ln1, Hh * 2, false));
      TRY(dalloc(e, &l.ln2, Hh * 2, false));
    }
    if (c.eagle3) {
      TRY(alloc_linear(e, e->h_fc, Hh, 3 * H));
      TRY(dalloc(e, &e->h_hidden_norm, Hh * 2, false));
      TRY(dalloc(e, &e->h_norm, Hh * 2, false));
      TRY(alloc_linear(e, e->h_head, e->Vd, Hh));
      if (e->Vd != e->V) TRY(dalloc(e, reinterpret_cast<void**>(&e->d2t), static_cast<size_t>(e->Vd) * 8, false));
    } else {
      TRY(alloc_linear(e, e->h_fc, Hh, 2 * Hh));
      if (c.head_fc_bias) TRY(dalloc(e, &e->h_fc_bias, Hh * 2, false));
    }
    // ---- KV
    TRY(dalloc(e, &e->t_kv, static_cast<size_t>(e->L) * 2 * e->nkv_l * e->cap * 128 * 2));
    TRY(dalloc(e, &e->d_kv, static_cast<size_t>(e->hL) * 2 * e->hnkv * e->dcap * 128 * 2));
    // ---- activations
    if (c.tp_size > 1) {
      // replicated activations live in the peer-visible window so that row owners can push finished rows into every rank
      auto up = [](size_t v) { return (v + 1023) & ~static_cast<size_t>(1023); };
      size_t off = 0;
      const size_t off_x = off; off += up(static_cast<size_t>(64) * H * 2);
      const size_t off_xn = off; off += up(static_cast<size_t>(64) * H * 2);
      const size_t off_feat = off; off += up(static_cast<size_t>(64) * e->F * 2);
      const size_t off_fall = off; off += up(static_cast<size_t>(c.max_length + 64) * e->F * 2);
      e->tp_inbox_off = static_cast<long>(off); off += up(static_cast<size_t>(2) * c.tp_size * 64 * H * 4);  // double-buffered by epoch parity
      e->tp_flag_off = static_cast<long>(off); off += up(static_cast<size_t>(kMaxTp) * 64 * 4);
      e->tp_ready_off = static_cast<long>(off); off += 1024;
      e->tp_am_off = static_cast<long>(off); off += up(static_cast<size_t>(kMaxTp) * 64 * 12);
      e->tp_win_bytes = off;
      void* w = nullptr;
      TRY(dalloc(e, &w, off));
      e->tp_win = reinterpret_cast<char*>(w);
      e->tp_peer[c.tp_rank] = e->tp_win;
      e->x = e->tp_win + off_x;
      e->feat = e->tp_win + off_feat;
      e->feat_all = e->tp_win + off_fall;
      e->xn.p = e->tp_win + off_xn;
      e->xn.cols = H;
      TRY(make_tmap(&e->xn.tm16, e->dtype, e->xn.p, 64, H, 16));
      TRY(make_tmap(&e->xn.tm64, e->dtype, e->xn.p, 64, H, 64));
      TRY(dalloc(e, reinterpret_cast<void**>(&e->tp_epoch), 64));
    } else {
      TRY(dalloc(e, &e->x, static_cast<size_t>(e->act_rows) * H * 2));
      TRY(dalloc(e, &e->feat, static_cast<size_t>(64) * e->F * 2));
      TRY(dalloc(e, &e->feat_all, static_cast<size_t>(c.max_length + 256) * e->F * 2));
      TRY(alloc_act(e, e->xn, H, e->act_rows));
    }
    TRY(dalloc(e, &e->q, static_cast<size_t>(e->act_rows) * e->nh_l * 128 * 2));
    TRY(dalloc(e, &e->logits, static_cast<size_t>(64) * e->V_l * 2));
    TRY(alloc_act(e, e->attn, e->nh_l * 128, e->act_rows));
    TRY(alloc_act(e, e->act, e->I_l, e->act_rows));
    TRY(alloc_act(e, e->xn_last, H));
    TRY(dalloc(e, &e->d_q, 64 * e->hnh * 128 * 2));
    TRY(dalloc(e, &e->d_h2, 64 * Hh * 2));
    TRY(dalloc(e, &e->d_logits, static_cast<size_t>(64) * e->Vd * 2));
    TRY(alloc_act(e, e->d_feat, e->F));
    TRY(alloc_act(e, e->d_cat, 2 * Hh));
    TRY(alloc_act(e, e->d_h, Hh));
    TRY(alloc_act(e, e->d_attn, e->hnh * 128));
    TRY(alloc_act(e, e->d_xn, Hh));
    TRY(alloc_act(e, e->d_act, e->Ih));
    TRY(alloc_act(e, e->d_out, Hh));
    // ---- split-K workspace: worst case = 2 accumulators x 64 rows x padded N x splits
    e->ws_bytes = static_cast<size_t>(96) << 20;
    TRY(dalloc(e, reinterpret_cast<void**>(&e->ws), e->ws_bytes, false));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->counters), 8192 * sizeof(int)));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->chain_sync), 2 * sizeof(int)));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->chain_timing), 4 * sizeof(unsigned long long)));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->tile_val), static_cast<size_t>((e->V_l + 127) / 128) * 64 * sizeof(float)));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->tile_idx), static_cast<size_t>((e->V_l + 127) / 128) * 64 * sizeof(int)));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->row_stats), 128 * sizeof(RowStats)));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->rej_tokens), 64 * sizeof(int)));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->uniforms), 4096 * sizeof(float)));
    if (c.tp_size > 1) {
      TRY(dalloc(e, &e->lg_recv, static_cast<size_t>(c.tp_size) * 64 * e->V_l * 2));
      TRY(dalloc(e, &e->logits_full, static_cast<size_t>(c.tp_size) * 64 * e->V_l * 2));
      TRY(dalloc(e, reinterpret_cast<void**>(&e->f32buf), static_cast<size_t>(64) * H * 4));
      TRY(dalloc(e, reinterpret_cast<void**>(&e->am_send), 2 * 128 * 4));
      TRY(dalloc(e, reinterpret_cast<void**>(&e->am_recv), static_cast<size_t>(c.tp_size) * 2 * 128 * 4));
      if (!c.eagle3) TRY(alloc_linear(e, e->t_head_full, e->V, H));
    }
    // ---- tree / state
    const int pool = e->k + e->depth * e->k * e->k;
    TRY(dalloc(e, reinterpret_cast<void**>(&e->st), S_COUNT * sizeof(int)));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->tb.scores), pool * sizeof(float)));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->tb.tokens), pool * sizeof(int)));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->tb.parents), (1 + e->depth * e->k) * sizeof(int)));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->tb.front_scores), 64 * sizeof(float)));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->tb.front_ids), 64 * sizeof(int)));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->tb.front_src), 64 * sizeof(int)));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->tb.front_mask), 64 * 2 * sizeof(uint64_t)));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->tb.front_cs), 64 * sizeof(int)));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->tb.draft_tokens), 128 * sizeof(int)));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->tb.tree_mask), 128 * 2 * sizeof(uint64_t)));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->tb.tree_pos), 128 * sizeof(int)));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->tb.retrieve), 128 * 16 * sizeof(int)));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->tb.parent_node), 128 * sizeof(int)));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->topk_p), 64 * 32 * sizeof(float)));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->topk_i), 64 * 32 * sizeof(int)));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->node_argmax), 128 * sizeof(int)));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->accepted), 64 * sizeof(int)));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->sel_nodes), 64 * sizeof(int)));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->ident), 256 * sizeof(int)));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->st_tree_indices), kStaticMaxNodes * sizeof(int)));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->st_sel), kStaticMaxNodes * sizeof(int)));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->st_src), kStaticMaxNodes * sizeof(int)));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->st_lmask), kStaticMaxNodes * 2 * sizeof(uint64_t)));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->ss_tokens), (kStaticMaxNodes + 1) * 32 * sizeof(int)));
    if (getenv("EB200_ATTN_TRACE")) TRY(dalloc(e, reinterpret_cast<void**>(&e->attn_trace), 8192 * 16 * sizeof(unsigned long long)));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->ids_dev), static_cast<size_t>(c.max_length + 128) * 8));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->out_ids_dev), static_cast<size_t>(c.max_length + 128) * 8));
    int ident[256];
    for (int i = 0; i < 256; ++i) ident[i] = i;
    CK(cudaMemcpyAsync(e->ident, ident, sizeof(ident), cudaMemcpyHostToDevice, e->stream));
    CK(cudaHostAlloc(reinterpret_cast<void**>(&e->pinned), 2 * 64 * sizeof(int64_t), cudaHostAllocDefault));  // two read-back slots
    memset(e->pinned, 0, 2 * 64 * sizeof(int64_t));
    CK(cudaEventCreateWithFlags(&e->ev_done, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&e->ev_slot[0], cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&e->ev_slot[1], cudaEventDisableTiming));
    CK(cudaStreamSynchronize(e->stream));
    return 0;
  };
  rc = body();
  if (rc != 0) {
    eb200_destroy(e);
    return rc;
  }
  *out = e;
  return 0;
}

static void tp_destroy_comm(void* comm);
extern "C" void eb200_destroy(eb200_engine* e) {
  if (!e) return;
  cudaSetDevice(e->c.device);
  if (e->stream) cudaStreamSynchronize(e->stream);
  if (e->attn_trace) {  // debugging aid: dump the stamps of the last traced launch
    std::vector<unsigned long long> h(8192 * 16);
    if (cudaMemcpy(h.data(), e->attn_trace, h.size() * 8, cudaMemcpyDeviceToHost) == cudaSuccess) {
      if (FILE* f = fopen(getenv("EB200_ATTN_TRACE"), "w")) {
        for (size_t c = 0; c < 8192; ++c) {
          if (!h[c * 16]) continue;
          fprintf(f, "%zu", c);
          for (int j = 0; j < 16; ++j) fprintf(f, " %llu", h[c * 16 + j]);
          fprintf(f, "\n");
        }
        fclose(f);
      }
    }
  }
  for (int r = 0; r < kMaxTp; ++r)
    if (e->tp_peer[r] && e->tp_peer[r] != e->tp_win) cudaIpcCloseMemHandle(e->tp_peer[r]);
  for (void* p : e->allocs) cudaFree(p);
  if (e->nccl_comm) tp_destroy_comm(e->nccl_comm);
  if (e->graph_exec) cudaGraphExecDestroy(e->graph_exec);
  if (e->graph) cudaGraphDestroy(e->graph);
  if (e->pinned) cudaFreeHost(e->pinned);
  if (e->ev_done) cudaEventDestroy(e->ev_done);
  for (auto ev : e->ev_slot)
    if (ev) cudaEventDestroy(ev);
  for (auto ev : e->ev_pool) cudaEventDestroy(ev);
  for (auto& r : e->prof) {
    cudaEventDestroy(r.a);
    cudaEventDestroy(r.b);
  }
  if (e->stream) cudaStreamDestroy(e->stream);
  delete e;
}

// ------------------------------------------------------------------------------------------------------------
// weight loading
// ------------------------------------------------------------------------------------------------------------
// copy rows [r0, r0+nr) x cols [c0, c0+nc) of a row-major [R][C] source of `es`-byte elements into dst rows [dr0, ...) of pitch nc
static int copy_block(eb200_engine* e, void* dst, long dst_row0, const void* src, long C, long r0, long nr, long c0, long nc, long es = 2) {
  const char* s = reinterpret_cast<const char*>(src) + (r0 * C + c0) * es;
  char* d = reinterpret_cast<char*>(dst) + dst_row0 * nc * es;
  CK(cudaMemcpy2DAsync(d, nc * es, s, C * es, nc * es, nr, cudaMemcpyDefault, e->stream));
  return 0;
}
static bool shape_is(const int64_t* s, int nd, int64_t a, int64_t b = -1) {
  if (b < 0) return nd == 1 && s[0] == a;
  return nd == 2 && s[0] == a && s[1] == b;
}

// Megatron-style shard of a target tensor for tensor-parallel rank `rk` of `tp`:
//   column-parallel (q/k/v by heads, gate/up, lm_head): a contiguous block of ROWS;  row-parallel (o_proj, down_proj): a
//   contiguous block of COLUMNS;  everything else replicated.  The same function backs eb200_tp_shard (CPU-testable).
struct Shard {
  long r0, nr, c0, nc;
};
static Shard shard_of(const std::string& name, long R, long C, int rk, int tp) {
  auto ends = [&](const char* suf) {
    const size_t n = strlen(suf);
    return name.size() >= n && name.compare(name.size() - n, n, suf) == 0;
  };
  if (tp <= 1) return Shard{0, R, 0, C};
  if (ends("q_proj.weight") || ends("k_proj.weight") || ends("v_proj.weight") || ends("gate_proj.weight") || ends("up_proj.weight"))
    return Shard{rk * (R / tp), R / tp, 0, C};
  if (ends("o_proj.weight") || ends("down_proj.weight")) return Shard{0, R, rk * (C / tp), C / tp};
  if (name == "lm_head.weight") {
    const long per = (R + tp - 1) / tp;
    const long r0 = std::min<long>(R, rk * per);
    return Shard{r0, std::max<long>(0, std::min<long>(per, R - r0)), 0, C};
  }
  return Shard{0, R, 0, C};
}
extern "C" int eb200_tp_shard(const char* name, int64_t rows, int64_t cols, int32_t tp_rank, int32_t tp_size, int64_t* out4) {
  if (!name || !out4 || tp_size < 1 || tp_rank < 0 || tp_rank >= tp_size) return fail("eb200_tp_shard: bad argument");
  const Shard sh = shard_of(name, rows, cols, tp_rank, tp_size);
  out4[0] = sh.r0;
  out4[1] = sh.nr;
  out4[2] = sh.c0;
  out4[3] = sh.nc;
  return 0;
}

// gate_proj (half 0) / up_proj (half 1) rows land interleaved in 64-row groups: source row i of the shard goes to row
// (i / 64) * 128 + half * 64 + i % 64, so that every 128-row GEMM tile holds the gate AND up rows of the same 64 outputs
// (row scales of int8 weights follow their rows: C = 1, es = 4)
static int copy_interleaved64(eb200_engine* e, void* dst, int half, const void* src, long C, const Shard& sh, long es = 2) {
  if (sh.nr % 64 || sh.c0 != 0 || sh.nc != C) return fail("gate/up shard must be whole rows in multiples of 64");
  const char* s = reinterpret_cast<const char*>(src) + sh.r0 * C * es;
  char* d = reinterpret_cast<char*>(dst) + static_cast<size_t>(half) * 64 * C * es;
  CK(cudaMemcpy2DAsync(d, static_cast<size_t>(128) * C * es, s, static_cast<size_t>(64) * C * es, static_cast<size_t>(64) * C * es, sh.nr / 64,
                       cudaMemcpyDefault, e->stream));
  return 0;
}

static bool ends_with(const std::string& s, const char* suf) {
  const size_t n = strlen(suf);
  return s.size() >= n && s.compare(s.size() - n, n, suf) == 0;
}
// the seven decoder-layer projections: weight "<proj>.weight"; int8 row scales "<proj>.SCB" (EB200_FLAG_TARGET_INT8); 4-bit block
// absmax "<proj>.weight.absmax" (EB200_FLAG_TARGET_NF4 / _FP4); FP8 block scales "<proj>.weight_scale_inv" (EB200_FLAG_TARGET_FP8)
static const char* const kProjNames[7] = {"self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj", "self_attn.o_proj",
                                          "mlp.gate_proj",    "mlp.up_proj",      "mlp.down_proj"};
enum ProjPart { PART_WEIGHT = 0, PART_SCB = 1, PART_ABSMAX = 2, PART_SCALE_INV = 3 };
static int proj_index(const std::string& sub, int* part) {
  for (int i = 0; i < 7; ++i) {
    const std::string p(kProjNames[i]);
    if (sub == p + ".weight" || sub == p + ".SCB" || sub == p + ".weight.absmax" || sub == p + ".weight_scale_inv") {
      *part = sub == p + ".weight" ? PART_WEIGHT : sub == p + ".SCB" ? PART_SCB : sub == p + ".weight.absmax" ? PART_ABSMAX : PART_SCALE_INV;
      return i;
    }
  }
  return -1;
}
// FP8: copy the e4m3 [nr][K] tensor (or its [nr / 128][K / 128] fp32 scales) to the device and repack it into the engine's layout
static int load_fp8(eb200_engine* e, Linear& L, bool scales, const void* data, long nr, long row0, int half) {
  const long rows_needed = half >= 0 ? nr * 2 : row0 + nr;  // gate/up: the two halves interleave over 2 * nr rows
  if (nr < 0 || nr % 128 || row0 < 0 || row0 % 64 || rows_needed > L.N)
    return fail("FP8 load: %ld source rows at destination row %ld do not fit the %d rows of the projection in 128-row blocks", nr, row0, L.N);
  const size_t bytes = scales ? static_cast<size_t>(nr / 128) * (L.K / 128) * 4 : static_cast<size_t>(nr) * L.K;
  void* tmp = nullptr;
  CK(cudaMalloc(&tmp, bytes));
  int rc = 0;
  if (cudaMemcpyAsync(tmp, data, bytes, cudaMemcpyDefault, e->stream) != cudaSuccess) rc = fail("FP8 load: copy failed");
  else if (launch_fp8_repack(scales ? nullptr : static_cast<const uint8_t*>(tmp), scales ? static_cast<const float*>(tmp) : nullptr,
                             static_cast<int>(nr), L.K, static_cast<int>(row0), half, static_cast<uint8_t*>(L.w), L.scale_inv, L.N,
                             e->stream) != 0 ||
           cudaStreamSynchronize(e->stream) != cudaSuccess)
    rc = fail("FP8 load: repack failed");
  cudaFree(tmp);
  return rc;
}
// 4-bit: copy the [nr][C] tensor (nibbles, or absmax with C = K / 64) to the device and repack its rows into the engine's layout
static int load_w4(eb200_engine* e, Linear& L, bool absmax, const void* data, long nr, long row0, int half) {
  const long rows_needed = half >= 0 ? nr * 2 : row0 + nr;  // gate/up: the two halves interleave over 2 * nr rows
  if (nr < 0 || row0 < 0 || (half >= 0 && nr % 64) || rows_needed > L.N)
    return fail("4-bit load: %ld source rows at destination row %ld do not fit the %d rows of the projection", nr, row0, L.N);
  const size_t bytes = absmax ? static_cast<size_t>(nr) * (L.K / 64) * 4 : static_cast<size_t>(nr) * L.K / 2;
  void* tmp = nullptr;
  CK(cudaMalloc(&tmp, bytes));
  int rc = 0;
  if (cudaMemcpyAsync(tmp, data, bytes, cudaMemcpyDefault, e->stream) != cudaSuccess) rc = fail("4-bit load: copy failed");
  else if (launch_w4_repack(absmax ? nullptr : static_cast<const uint8_t*>(tmp), absmax ? static_cast<const float*>(tmp) : nullptr,
                            static_cast<int>(nr), L.K, static_cast<int>(row0), half, static_cast<uint8_t*>(L.w), L.absmax, L.n_pad,
                            e->stream) != 0 ||
           cudaStreamSynchronize(e->stream) != cudaSuccess)
    rc = fail("4-bit load: repack failed");
  cudaFree(tmp);
  return rc;
}

static int load_layer_tensor(eb200_engine* e, Layer& l, const std::string& sub, const void* data, const int64_t* shape,
                             int nd, bool is_target, int Hin_qkv, int Hm, int nh_full, int nkv_full, int I_full) {
  const int tp = is_target ? e->c.tp_size : 1, rk = is_target ? e->c.tp_rank : 0;
  const int nh_l = nh_full / tp, nkv_l = nkv_full / tp;
  int part = PART_WEIGHT;
  const int pi = proj_index(sub, &part);
  const bool scb = part == PART_SCB;
  if (pi >= 0) {
    // destination matrix, full [rows, cols] of the checkpoint tensor, first destination row, gate/up half, loaded bit
    struct Slot {
      Linear* lin;
      long rows, cols, row0;
      int half, bit;
    };
    const Slot slots[7] = {{&l.qkv, nh_full * 128L, Hin_qkv, 0, -1, 1},
                           {&l.qkv, nkv_full * 128L, Hin_qkv, nh_l * 128L, -1, 2},
                           {&l.qkv, nkv_full * 128L, Hin_qkv, (nh_l + nkv_l) * 128L, -1, 4},
                           {&l.o, Hm, nh_full * 128L, 0, -1, 1},
                           {&l.gu, I_full, Hm, 0, 0, 1},
                           {&l.gu, I_full, Hm, 0, 1, 2},
                           {&l.down, Hm, I_full, 0, -1, 1}};
    const Slot& sl = slots[pi];
    const char* short_name = strchr(kProjNames[pi], '.') + 1;
    const std::string wname = std::string(kProjNames[pi]) + ".weight";
    const Shard sh = shard_of(wname, sl.rows, sl.cols, rk, tp);
    Linear& L = *sl.lin;
    if (L.scale_inv) {  // FP8 (one GPU: the shard is the whole tensor)
      if (part == PART_SCB || part == PART_ABSMAX)
        return fail("%s%s: belongs to int8 / 4-bit projections; this engine stores FP8 weights", short_name, part == PART_SCB ? ".SCB" : ".weight.absmax");
      const bool si = part == PART_SCALE_INV;
      if (sl.rows % 128 || sl.cols % 128)
        return fail("%s: FP8 weights need out- and in-features divisible by 128, got [%ld, %ld]", short_name, sl.rows, sl.cols);
      if (!shape_is(shape, nd, si ? sl.rows / 128 : sl.rows, si ? sl.cols / 128 : sl.cols))
        return fail("%s%s shape mismatch (want [%ld, %ld] %s)", short_name, si ? ".weight_scale_inv" : ".weight", si ? sl.rows / 128 : sl.rows,
                    si ? sl.cols / 128 : sl.cols, si ? "fp32: one scale per 128 x 128 block" : "float8_e4m3fn");
      TRY(load_fp8(e, L, si, data, sl.rows, sl.row0, sl.half));
      (si ? L.loaded_scales : L.loaded_rows) |= sl.bit;
    } else if (part == PART_SCALE_INV) {
      return fail("%s.weight_scale_inv: block scales belong to FP8 projections (EB200_FLAG_TARGET_FP8)", short_name);
    } else if (L.absmax) {  // 4-bit (one GPU: the shard is the whole tensor)
      if (part == PART_SCB) return fail("%s.SCB: row scales belong to int8 projections; this engine stores 4-bit weights", short_name);
      const bool am = part == PART_ABSMAX;
      if (!shape_is(shape, nd, sl.rows, am ? sl.cols / 64 : sl.cols / 2))
        return fail("%s%s shape mismatch (want [%ld, %ld] %s)", short_name, am ? ".weight.absmax" : ".weight", sl.rows,
                    am ? sl.cols / 64 : sl.cols / 2, am ? "fp32" : "uint8: two 4-bit codes per byte");
      TRY(load_w4(e, L, am, data, sl.rows, sl.row0, sl.half));
      (am ? L.loaded_scales : L.loaded_rows) |= sl.bit;
    } else if (part == PART_ABSMAX) {
      return fail("%s.weight.absmax: block absmax belongs to 4-bit projections (EB200_FLAG_TARGET_NF4 / _FP4)", short_name);
    } else if (!scb) {
      if (!shape_is(shape, nd, sl.rows, sl.cols)) return fail("%s shape mismatch", short_name);
      if (sl.half >= 0) TRY(copy_interleaved64(e, L.w, sl.half, data, sl.cols, sh, L.esize));
      else TRY(copy_block(e, L.w, sl.row0, data, sl.cols, sh.r0, sh.nr, sh.c0, sh.nc, L.esize));
      L.loaded_rows |= sl.bit;
    } else {
      if (!L.scale) return fail("%s.SCB: row scales belong to int8 projections (EB200_FLAG_TARGET_INT8)", short_name);
      if (!shape_is(shape, nd, sl.rows)) return fail("%s.SCB shape mismatch (want [%ld] fp32)", short_name, sl.rows);
      const Shard rs{sh.r0, sh.nr, 0, 1};  // the scales shard with their rows
      if (sl.half >= 0) TRY(copy_interleaved64(e, L.scale, sl.half, data, 1, rs, 4));
      else TRY(copy_block(e, L.scale, sl.row0, data, 1, rs.r0, rs.nr, 0, 1, 4));
      L.loaded_scales |= sl.bit;
    }
  } else if (sub == "input_layernorm.weight") {
    if (!l.ln1) return 0;  // EAGLE-1 layer 0 has no input norm (cnets1.py:399-401): ignore like strict=False
    if (!shape_is(shape, nd, Hm)) return fail("input_layernorm shape mismatch");
    CK(cudaMemcpyAsync(l.ln1, data, Hm * 2, cudaMemcpyDefault, e->stream));
    l.ln1_loaded = true;
  } else if (sub == "post_attention_layernorm.weight") {
    if (!shape_is(shape, nd, Hm)) return fail("post_attention_layernorm shape mismatch");
    CK(cudaMemcpyAsync(l.ln2, data, Hm * 2, cudaMemcpyDefault, e->stream));
    l.ln2_loaded = true;
  } else if (sub.find("rotary_emb") != std::string::npos) {
    return 0;
  } else {
    return fail("unknown layer tensor '%s'", sub.c_str());
  }
  return 0;
}

extern "C" int eb200_load_tensor(eb200_engine* e, const char* name_c, const void* data, const int64_t* shape, int32_t ndim,
                                 int32_t dtype) {
  if (!e || !name_c || !data || !shape) return fail("eb200_load_tensor: null argument");
  if (e->finalized) return fail("eb200_load_tensor after eb200_finalize");
  CK(cudaSetDevice(e->c.device));
  std::string name(name_c);
  const bool is_head = name.rfind("head.", 0) == 0;
  const bool want_model_dtype = !(name == "head.d2t" || name == "head.t2d");
  const eb200_config& c = e->c;
  // int8 target projections: "<proj>.weight" int8 + "<proj>.SCB" fp32, only on an engine created with EB200_FLAG_TARGET_INT8
  int part = PART_WEIGHT;
  const bool target_proj = !is_head && name.rfind("model.layers.", 0) == 0 && name.find('.', strlen("model.layers.")) != std::string::npos &&
                           proj_index(name.substr(name.find('.', strlen("model.layers.")) + 1), &part) >= 0;
  const bool scb = part == PART_SCB;
  const bool w8 = (c.flags & EB200_FLAG_TARGET_INT8) != 0;
  const bool w4 = (c.flags & (EB200_FLAG_TARGET_NF4 | EB200_FLAG_TARGET_FP4)) != 0;
  const bool f8 = (c.flags & EB200_FLAG_TARGET_FP8) != 0;
  if (dtype == EB200_DT_FP8_E4M3 || ends_with(name, ".weight_scale_inv")) {
    // FP8 target projections: "<proj>.weight" float8_e4m3fn + "<proj>.weight_scale_inv" fp32 (transformers' FineGrainedFP8Config keys)
    if (!target_proj)
      return fail("tensor '%s': FP8 weights and weight_scale_inv are accepted only for the target decoder projections "
                  "(q/k/v/o/gate/up/down_proj); embeddings, norms, lm_head and the draft head stay in the model dtype", name_c);
    if (!f8) return fail("tensor '%s': FP8 data for an engine created without EB200_FLAG_TARGET_FP8", name_c);
    if (part == PART_SCALE_INV && dtype != EB200_DT_FP32) return fail("tensor '%s': FP8 weight_scale_inv must be fp32", name_c);
    if (part != PART_SCALE_INV && (part != PART_WEIGHT || dtype != EB200_DT_FP8_E4M3))
      return fail("tensor '%s': FP8 data is accepted as '<proj>.weight' (float8_e4m3fn) and '<proj>.weight_scale_inv' (fp32)", name_c);
  } else if (f8 && target_proj) {
    return fail("tensor '%s': this engine stores the target projections in FP8 (EB200_FLAG_TARGET_FP8): pass the float8_e4m3fn weight and "
                "its fp32 weight_scale_inv (eagle_b200.quant.quantize_fp8_block)", name_c);
  } else if (dtype == EB200_DT_UINT8 || ends_with(name, ".absmax")) {
    // 4-bit target projections: "<proj>.weight" uint8 + "<proj>.weight.absmax" fp32
    if (!target_proj)
      return fail("tensor '%s': 4-bit codes and absmax are accepted only for the target decoder projections (q/k/v/o/gate/up/down_proj); "
                  "embeddings, norms, lm_head and the draft head stay in the model dtype", name_c);
    if (!w4) return fail("tensor '%s': 4-bit data for an engine created without EB200_FLAG_TARGET_NF4 / _FP4 (load_in_4bit)", name_c);
    if (part == PART_ABSMAX && dtype != EB200_DT_FP32) return fail("tensor '%s': 4-bit block absmax must be fp32", name_c);
    if (part == PART_WEIGHT && dtype != EB200_DT_UINT8) return fail("tensor '%s': 4-bit weights must be uint8 (two codes per byte)", name_c);
  } else if (w4 && target_proj && (dtype == EB200_DT_INT8 || scb)) {
    return fail("tensor '%s': int8 data (load_in_8bit format) for an engine that stores the target projections in 4 bits "
                "(EB200_FLAG_TARGET_NF4 / _FP4)", name_c);
  } else if (w4 && target_proj) {
    return fail("tensor '%s': this engine stores the target projections in 4 bits (EB200_FLAG_TARGET_NF4 / _FP4): pass the uint8 codes and "
                "their fp32 block absmax (eagle_b200.quant.quantize_4bit)", name_c);
  } else if (dtype == EB200_DT_INT8 || ends_with(name, ".SCB")) {
    if (!target_proj)
      return fail("tensor '%s': int8 weights and SCB row scales are accepted only for the target decoder projections "
                  "(q/k/v/o/gate/up/down_proj); embeddings, norms, lm_head and the draft head stay in the model dtype", name_c);
    if (!w8) return fail("tensor '%s': int8 data for an engine created without EB200_FLAG_TARGET_INT8 (load_in_8bit)", name_c);
    if (scb && dtype != EB200_DT_FP32) return fail("tensor '%s': SCB row scales must be fp32", name_c);
  } else if (w8 && target_proj) {
    return fail("tensor '%s': this engine stores the target projections in int8 (EB200_FLAG_TARGET_INT8): pass the int8 weight and "
                "its fp32 SCB row scales (eagle_b200.quant.quantize_int8_rowwise)", name_c);
  } else if (want_model_dtype && dtype != e->dtype) {
    return fail("tensor '%s': dtype %d does not match the engine's model dtype %d (cast it like `.to(base_model.dtype)`, ea_model.py:77)",
                name_c, dtype, e->dtype);
  }
  if (!is_head) {
    if (name == "model.embed_tokens.weight") {
      if (!shape_is(shape, ndim, e->V, e->H)) return fail("embed_tokens shape mismatch");
      CK(cudaMemcpyAsync(e->t_embed, data, static_cast<size_t>(e->V) * e->H * 2, cudaMemcpyDefault, e->stream));
      e->t_embed_loaded = true;
    } else if (name == "model.norm.weight") {
      if (!shape_is(shape, ndim, e->H)) return fail("model.norm shape mismatch");
      CK(cudaMemcpyAsync(e->t_norm, data, e->H * 2, cudaMemcpyDefault, e->stream));
      e->t_norm_loaded = true;
    } else if (name == "lm_head.weight") {
      if (!shape_is(shape, ndim, e->V, e->H)) return fail("lm_head shape mismatch");
      const Shard sh = shard_of(name, e->V, e->H, c.tp_rank, c.tp_size);
      if (sh.nr < e->V_l) CK(cudaMemsetAsync(e->t_head.w, 0, static_cast<size_t>(e->V_l) * e->H * 2, e->stream));
      TRY(copy_block(e, e->t_head.w, 0, data, e->H, sh.r0, sh.nr, sh.c0, sh.nc));
      e->t_head.loaded_rows = 1;
      if (e->t_head_full.w) {
        CK(cudaMemcpyAsync(e->t_head_full.w, data, static_cast<size_t>(e->V) * e->H * 2, cudaMemcpyDefault, e->stream));
        e->t_head_full.loaded_rows = 1;
      }
    } else if (name.rfind("model.layers.", 0) == 0) {
      const size_t p0 = strlen("model.layers.");
      const size_t p1 = name.find('.', p0);
      if (p1 == std::string::npos) return fail("bad tensor name '%s'", name_c);
      const int li = atoi(name.substr(p0, p1 - p0).c_str());
      if (li < 0 || li >= e->L) return fail("layer index out of range in '%s'", name_c);
      TRY(load_layer_tensor(e, e->tl[li], name.substr(p1 + 1), data, shape, ndim, true, e->H, e->H, c.num_heads,
                            c.num_kv_heads, c.intermediate_size));
    } else {
      return fail("unknown target tensor '%s'", name_c);
    }
  } else {
    const std::string sub = name.substr(5);
    const int Hh = e->Hh;
    if (sub == "embed_tokens.weight") {
      if (!shape_is(shape, ndim, e->V, Hh)) return fail("head embed_tokens shape mismatch");
      if (!e->h_embed_own) {
        TRY(dalloc(e, &e->h_embed, static_cast<size_t>(e->V) * Hh * 2, false));
        e->h_embed_own = true;
      }
      CK(cudaMemcpyAsync(e->h_embed, data, static_cast<size_t>(e->V) * Hh * 2, cudaMemcpyDefault, e->stream));
    } else if (sub == "fc.weight") {
      if (!shape_is(shape, ndim, e->h_fc.N, e->h_fc.K)) return fail("head fc.weight shape mismatch");
      CK(cudaMemcpyAsync(e->h_fc.w, data, static_cast<size_t>(e->h_fc.N) * e->h_fc.K * 2, cudaMemcpyDefault, e->stream));
      e->h_fc.loaded_rows = 1;
    } else if (sub == "fc.bias") {
      if (!e->h_fc_bias) return 0;  // config says no bias: ignore (strict=False)
      if (!shape_is(shape, ndim, Hh)) return fail("head fc.bias shape mismatch");
      CK(cudaMemcpyAsync(e->h_fc_bias, data, Hh * 2, cudaMemcpyDefault, e->stream));
      e->h_fc_bias_loaded = true;
    } else if (sub == "d2t") {
      if (!e->d2t) return 0;  // vocab == draft vocab: the reference deletes the buffer (ea_model.py:74-75)
      if (dtype != EB200_DT_INT64 || !shape_is(shape, ndim, e->Vd)) return fail("head d2t must be int64[draft_vocab]");
      CK(cudaMemcpyAsync(e->d2t, data, static_cast<size_t>(e->Vd) * 8, cudaMemcpyDefault, e->stream));
      e->d2t_loaded = true;
    } else if (sub == "t2d") {
      return 0;  // only used by training
    } else if (c.eagle3 && sub == "norm.weight") {
      CK(cudaMemcpyAsync(e->h_norm, data, Hh * 2, cudaMemcpyDefault, e->stream));
      e->h_norm_loaded = true;
    } else if (c.eagle3 && sub == "lm_head.weight") {
      if (!shape_is(shape, ndim, e->Vd, Hh)) return fail("head lm_head shape mismatch");
      CK(cudaMemcpyAsync(e->h_head.w, data, static_cast<size_t>(e->Vd) * Hh * 2, cudaMemcpyDefault, e->stream));
      e->h_head.loaded_rows = 1;
    } else if (c.eagle3 && sub == "midlayer.hidden_norm.weight") {
      CK(cudaMemcpyAsync(e->h_hidden_norm, data, Hh * 2, cudaMemcpyDefault, e->stream));
      e->h_hidden_norm_loaded = true;
    } else if (c.eagle3 && sub.rfind("midlayer.", 0) == 0) {
      TRY(load_layer_tensor(e, e->hl[0], sub.substr(9), data, shape, ndim, false, 2 * Hh, Hh, e->hnh, e->hnkv, e->Ih));
    } else if (!c.eagle3 && sub.rfind("layers.", 0) == 0) {
      const size_t p1 = sub.find('.', 7);
      if (p1 == std::string::npos) return fail("bad tensor name '%s'", name_c);
      const int li = atoi(sub.substr(7, p1 - 7).c_str());
      if (li < 0 || li >= e->hL) return fail("head layer index out of range in '%s'", name_c);
      TRY(load_layer_tensor(e, e->hl[li], sub.substr(p1 + 1), data, shape, ndim, false, Hh, Hh, e->hnh, e->hnkv, e->Ih));
    } else {
      return fail("unknown head tensor '%s'", name_c);
    }
  }
  CK(cudaStreamSynchronize(e->stream));  // the caller may free `data` on return
  return 0;
}

extern "C" int eb200_set_rope_table(eb200_engine* e, int32_t which, const void* cosp, const void* sinp, int32_t n_pos) {
  if (!e || !cosp || !sinp || n_pos <= 0) return fail("eb200_set_rope_table: bad argument");
  CK(cudaSetDevice(e->c.device));
  void** c = which == 0 ? &e->t_cos : &e->h_cos;
  void** s = which == 0 ? &e->t_sin : &e->h_sin;
  TRY(dalloc(e, c, static_cast<size_t>(n_pos) * 64 * 2, false));
  TRY(dalloc(e, s, static_cast<size_t>(n_pos) * 64 * 2, false));
  CK(cudaMemcpyAsync(*c, cosp, static_cast<size_t>(n_pos) * 64 * 2, cudaMemcpyDefault, e->stream));
  CK(cudaMemcpyAsync(*s, sinp, static_cast<size_t>(n_pos) * 64 * 2, cudaMemcpyDefault, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  (which == 0 ? e->t_npos : e->h_npos) = n_pos;
  return 0;
}

static int finalize_linear(eb200_engine* e, Linear& l, const char* what, uint64_t need) {
  if (l.loaded_rows != need) return fail("weights missing for %s", what);
  if (l.scale_inv) {
    if (l.loaded_scales != need) return fail("block scales missing for %s (FP8 weights need their fp32 .weight_scale_inv)", what);
    return make_tmap_fp8(&l.tm, &l.tm_abs, l.w, l.scale_inv, l.N, l.K);
  }
  if (l.absmax) {
    if (l.loaded_scales != need) return fail("block absmax missing for %s (4-bit weights need their fp32 .weight.absmax)", what);
    return make_tmap_w4(&l.tm, &l.tm_abs, l.w, l.absmax, l.n_pad, l.K);
  }
  if (l.scale) {
    if (l.loaded_scales != need) return fail("SCB row scales missing for %s (int8 weights need their fp32 row scales)", what);
    return make_tmap_w8(&l.tm, l.w, l.N, l.K);
  }
  return make_tmap(&l.tm, e->dtype, l.w, l.N, l.K, 128);
}

extern "C" int eb200_finalize(eb200_engine* e) {
  if (!e) return fail("eb200_finalize: null engine");
  CK(cudaSetDevice(e->c.device));
  if (e->c.flags & kTargetQuantFlags) {
    // the W8A16 / W4A16 GEMMs exist as the cluster split-K kernel of one GPU only
    const char* fmt = (e->c.flags & EB200_FLAG_TARGET_INT8)  ? "int8 target weights (EB200_FLAG_TARGET_INT8)"
                      : (e->c.flags & EB200_FLAG_TARGET_FP8) ? "FP8 target weights (EB200_FLAG_TARGET_FP8)"
                                                             : "4-bit target weights (EB200_FLAG_TARGET_NF4 / _FP4)";
    const char* what = nullptr;
    if (e->c.tp_size > 1) what = "tensor parallelism (tp_size > 1)";
    else if (e->c.flags & EB200_FLAG_SIMT_GEMM) what = "EB200_FLAG_SIMT_GEMM";
    if (what)
      return fail("%s are not supported with %s; they run on one GPU with the default cluster split-K GEMM", fmt, what);
  }
  char nm[128];
  if (!e->t_embed_loaded || !e->t_norm_loaded) return fail("target embed/norm weights missing");
  for (int i = 0; i < e->L; ++i) {
    Layer& l = e->tl[i];
    snprintf(nm, sizeof(nm), "model.layers.%d", i);
    TRY(finalize_linear(e, l.qkv, nm, 7));
    TRY(finalize_linear(e, l.o, nm, 1));
    TRY(finalize_linear(e, l.gu, nm, 3));
    TRY(finalize_linear(e, l.down, nm, 1));
    if (!l.ln1_loaded || !l.ln2_loaded) return fail("layernorm weights missing for %s", nm);
  }
  TRY(finalize_linear(e, e->t_head, "lm_head", 1));
  if (e->t_head_full.w) TRY(finalize_linear(e, e->t_head_full, "lm_head (full copy for the EAGLE-1 draft)", 1));
  if (e->c.tp_size > 1 && !e->nccl_comm) return fail("tp_size > 1: call eb200_tp_init before eb200_finalize");
  for (int i = 0; i < e->hL; ++i) {
    Layer& l = e->hl[i];
    snprintf(nm, sizeof(nm), "head layer %d", i);
    TRY(finalize_linear(e, l.qkv, nm, 7));
    TRY(finalize_linear(e, l.o, nm, 1));
    TRY(finalize_linear(e, l.gu, nm, 3));
    TRY(finalize_linear(e, l.down, nm, 1));
    if ((l.ln1 && !l.ln1_loaded) || !l.ln2_loaded) return fail("layernorm weights missing for %s", nm);
  }
  TRY(finalize_linear(e, e->h_fc, "head fc", 1));
  if (e->h_fc_bias && !e->h_fc_bias_loaded) return fail("head fc.bias missing");
  if (e->c.eagle3) {
    TRY(finalize_linear(e, e->h_head, "head lm_head", 1));
    if (!e->h_norm_loaded || !e->h_hidden_norm_loaded) return fail("head norm weights missing");
    if (e->d2t && !e->d2t_loaded) return fail("head d2t missing (draft_vocab_size != vocab_size)");
  }
  {
    // The target lm_head runs as one launch of whole vocabulary tiles per CTA (mega.cu) with the arg-max fused (no 15 MB logits
    // round trip).  It needs the peer windows under tensor parallelism (vocabulary-parallel arg-max exchange); without them, and
    // with EB200_FLAG_SIMT_GEMM / EB200_FLAG_NO_CHAIN, the lm_head is a GEMM launch followed by vocab_argmax.
    e->chain_head = !(e->c.flags & (EB200_FLAG_SIMT_GEMM | EB200_FLAG_NO_CHAIN)) && (e->c.tp_size == 1 || e->tp_fused) &&
                    chain_phase_ok(e->t_head.N, e->t_head.K);
    const char* fenv = getenv("EB200_FUSED_E3_INPUT");
    e->fused_e3_input = !(fenv && atoi(fenv) == 0);
  }
  if (!e->h_embed) e->h_embed = e->t_embed;  // load_emb: the head embeds with the target's table (cnets.py:488-519)
  if (!e->t_cos || !e->h_cos) return fail("rope tables missing (eb200_set_rope_table)");
  if (e->t_npos < e->c.max_length + 64 || e->h_npos < e->c.max_length + 64) return fail("rope tables shorter than max_length + 64");
  e->finalized = true;
  return 0;
}

// ------------------------------------------------------------------------------------------------------------
// launch helpers (profiling + counters)
// ------------------------------------------------------------------------------------------------------------
static cudaEvent_t get_event(eb200_engine* e) {
  if (!e->ev_pool.empty()) {
    cudaEvent_t ev = e->ev_pool.back();
    e->ev_pool.pop_back();
    return ev;
  }
  cudaEvent_t ev;
  cudaEventCreate(&ev);
  return ev;
}
static int g_debug_sync = -1;
template <typename T> __global__ void count_nonfinite_kernel(const T* p, long n, int* out) {
  long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x;
  if (i < n) {
    const float v = static_cast<float>(p[i]);
    if (!(v == v) || v > 3.0e38f || v < -3.0e38f) atomicAdd(out, 1);
  }
}
static void debug_scan(eb200_engine* e, const char* label);
struct ProfScope {
  eb200_engine* e;
  ProfRec r;
  bool on;
  const char* label;
  ProfScope(eb200_engine* e_, int cat, double bytes, const char* label_ = "") : e(e_), on(e_->profiling), label(label_) {
    if (g_debug_sync < 0) {
      const char* s = getenv("EB200_DEBUG_SYNC");  // bring-up: synchronize after every launch and name the faulting kernel
      g_debug_sync = s ? atoi(s) : 0;
    }
    e->stats.kernel_launches++;
    if (on) {
      r.a = get_event(e);
      r.b = get_event(e);
      r.cat = cat;
      r.bytes = bytes;
      r.verify = e->in_verify ? 1 : 0;
      cudaEventRecord(r.a, e->stream);
    }
  }
  ~ProfScope() {
    if (on) {
      cudaEventRecord(r.b, e->stream);
      e->prof.push_back(r);
    }
    if (g_debug_sync) {
      cudaError_t err = cudaStreamSynchronize(e->stream);
      if (err != cudaSuccess) {
        fprintf(stderr, "eagle_b200[debug-sync]: launch #%llu '%s' failed: %s\n", (unsigned long long)e->stats.kernel_launches, label,
                cudaGetErrorString(err));
        fflush(stderr);
      } else if (g_debug_sync >= 2) {
        debug_scan(e, label);
      }
    }
  }
};

// EB200_DEBUG_SYNC=2: after every launch count non-finite values in the live activation buffers and report the first hit
static void debug_scan(eb200_engine* e, const char* label) {
  static int* d_cnt = nullptr;
  static bool reported = false;
  if (reported) return;
  if (!d_cnt) cudaMalloc(&d_cnt, sizeof(int));
  struct B { const char* name; const void* p; long n; };
  const B bufs[] = {{"x", e->x, 64L * e->H}, {"xn", e->xn.p, 64L * e->H}, {"q", e->q, 64L * e->nh_l * 128},
                    {"attn", e->attn.p, 64L * e->nh_l * 128}, {"act", e->act.p, 64L * e->I_l},
                    {"d_h", e->d_h.p, 64L * e->Hh}, {"d_cat", e->d_cat.p, 128L * e->Hh}, {"d_out", e->d_out.p, 64L * e->Hh}};
  for (const B& b : bufs) {
    cudaMemsetAsync(d_cnt, 0, sizeof(int), e->stream);
    const int blocks = static_cast<int>((b.n + 255) / 256);
    if (e->dtype == DT_BF16) count_nonfinite_kernel<<<blocks, 256, 0, e->stream>>>(reinterpret_cast<const __nv_bfloat16*>(b.p), b.n, d_cnt);
    else count_nonfinite_kernel<<<blocks, 256, 0, e->stream>>>(reinterpret_cast<const __half*>(b.p), b.n, d_cnt);
    int h = 0;
    cudaMemcpyAsync(&h, d_cnt, sizeof(int), cudaMemcpyDeviceToHost, e->stream);
    cudaStreamSynchronize(e->stream);
    if (h > 0) {
      fprintf(stderr, "eagle_b200[debug-scan]: after launch #%llu '%s': buffer %s holds %d non-finite values\n",
              (unsigned long long)e->stats.kernel_launches, label, b.name, h);
      fflush(stderr);
      reported = true;
      return;
    }
  }
}

// split-K factor (== cluster size) of the cluster GEMM: the smallest power of two that gives the launch >= ~100 CTAs
// (one per SM on most SMs) with >= 4 k-blocks each.  Powers of two only: odd cluster sizes schedule badly, and a grid a
// little below the SM count leaves room for the next kernel's programmatic-dependent-launch prologue.
static int pick_splitk(int N, int K, int mpad, int epi, size_t ws_bytes) {
  (void)mpad; (void)epi; (void)ws_bytes;
  static int forced = -1, target = 0;
  if (forced < 0) {
    const char* s = getenv("EB200_SPLITK");
    forced = s ? atoi(s) : 0;
    const char* t = getenv("EB200_GEMM_TARGET_CTAS");
    target = t ? atoi(t) : 100;
  }
  const int tiles = (N + 127) / 128;
  const int num_kb = (K + 63) / 64;
  int sk = 1;
  if (forced > 0) sk = forced;
  else while (sk < 8 && tiles * sk < target) sk *= 2;
  while (sk > 1 && num_kb / sk < 4) sk /= 2;
  return std::min(sk, 8);
}

// EB200_L2_PREFETCH=1 turns the L2 weight prefetch on; read once.  Off by default: on the H100 every window measured slower with
// it (DESIGN.md §5), so it stays an experiment.
static bool l2_prefetch_on() {
  static int v = -1;
  if (v < 0) {
    const char* s = getenv("EB200_L2_PREFETCH");
    v = (s && atoi(s) == 1) ? 1 : 0;
  }
  return v == 1;
}
// Bytes a GEMM's drain and an RMSNorm / e3_input window prefetch of the GEMM that follows (about their idle time x HBM rate), and
// the cap on what is prefetched ahead of one GEMM in all, as a share of L2 (the live working set besides is a few MB).
static double pf_tail_bytes() { return 8.0 * (1 << 20); }
static double pf_norm_bytes() { return 8.0 * (1 << 20); }
static double pf_cap_share() { return 0.5; }
// Plan (kernels.h L2Prefetch) over the weight of `next`, the GEMM launched next over it at `mpad` rows: its k-block rows
// [j0, j0 + about `bytes`), with the same grid (pick_splitk) as that launch.  The plan ends at the matrix, and at the L2 cap
// counted from row 0; pf.j1 is where a later window's plan over the same GEMM continues.
static int pick_splitk(int N, int K, int mpad, int epi, size_t ws_bytes);
static L2Prefetch l2_plan(const eb200_engine* e, const Linear& next, int mpad, int j0, double bytes) {
  L2Prefetch pf;
  memset(&pf, 0, sizeof(pf));
  pf.j0 = pf.j1 = j0;
  // 4-bit weights are not prefetched: their tiles and absmax are two maps with other boxes than the plan's.  FP8 weights are: their
  // map has the int8 box (128 rows x 64 bytes, esize 1); their block scales (1/512 of the bytes) are not.
  if (!l2_prefetch_on() || !next.w || next.absmax || next.N <= 0 || next.K <= 0 || bytes <= 0) return pf;
  pf.tm = next.tm;
  pf.n_tiles = (next.N + 127) / 128;
  pf.splitk = pick_splitk(next.N, next.K, mpad, 0, e->ws_bytes);
  pf.num_kb = (next.K + 63) / 64;
  const double row = static_cast<double>(pf.n_tiles) * pf.splitk * 128 * 64 * next.esize;  // one k-block of every (n-tile, split)
  const int rows_all = (pf.num_kb + pf.splitk - 1) / pf.splitk;
  const int rows_cap = static_cast<int>(static_cast<double>(e->l2_bytes) * pf_cap_share() / row);
  const int rows = std::max(1, static_cast<int>(bytes / row));
  pf.j1 = std::max(j0, std::min({rows_all, rows_cap, j0 + rows}));
  return pf;
}
// the rest of the L2 cap over the same GEMM, after `prev`
static L2Prefetch l2_plan_rest(const eb200_engine* e, const Linear& next, int mpad, const L2Prefetch& prev) {
  return l2_plan(e, next, mpad, prev.j1, static_cast<double>(e->l2_bytes));
}

struct GemmCall {
  const Linear* W;
  const Linear* W2;
  const ActBuf* X;
  int epi;
  GemmParams p;
  const L2Prefetch* pf;  // optional: the next GEMM's leading weight tiles, prefetched by this launch's producers after their last load
};
static bool skip_kernel(const char* name);
static int run_gemm(eb200_engine* e, const RowCtx& cx, GemmCall& g) {
  GemmParams& p = g.p;
  p.N = g.W->N;
  p.K = g.W->K;
  p.m_rows = cx.rows;
  p.m_idx = cx.rows_idx;
  p.st = e->st;
  p.ws = e->ws;
  p.counters = e->counters;
  p.splitk = pick_splitk(p.N, p.K, cx.mpad, g.epi, e->ws_bytes);
  if ((p.N + 127) / 128 > 8192) return fail("too many n tiles");
  p.w_scale = g.W->scale;
  p.w4_quant = g.W->w4_quant;
  // algorithmic weight bytes: int8 weights stream N*K bytes plus the N fp32 row scales; 4-bit ones N*K/2 plus N*K/64 fp32 absmax;
  // FP8 ones N*K plus 16 B of block scales per 128 x 128 block
  const double nk = static_cast<double>(p.N) * p.K;
  const double bytes = g.W->absmax ? nk / 2 + 4.0 * nk / 64 : p.w_scale ? nk + 4.0 * p.N : g.W->scale_inv ? nk + 16.0 * nk / (128 * 128)
                                                                                                          : nk * 2 * (g.epi == EPI_SWIGLU ? 2 : 1);
  const char* kname = g.epi == EPI_STORE ? "gemm_store" : g.epi == EPI_RESIDUAL ? "gemm_residual" :
                      (g.epi == EPI_SWIGLU || g.epi == EPI_SWIGLU_IL) ? "gemm_swiglu" : "gemm_qkv_rope";
  {
    char kk[64];
    snprintf(kk, sizeof(kk), "%s@%d", kname, p.K);  // e.g. gemm_residual@14336 = down_proj only
    if (skip_kernel(kname) || skip_kernel(kk)) return 0;
  }
  ProfScope ps(e, 0, bytes, kname);
  if (g.W->scale_inv) {
    if (cx.mpad == 256 && g.X->rows < 256) return fail("256-row GEMM on a 64-row activation buffer");
    CKL(launch_gemm_fp8(e->dtype, cx.mpad, g.epi, &g.W->tm, &g.W->tm_abs, cx.mpad == 16 ? &g.X->tm16 : (cx.mpad == 64 ? &g.X->tm64 : &g.X->tm256),
                        p, e->stream, g.pf));
  } else if (g.W->absmax) {
    if (cx.mpad == 256 && g.X->rows < 256) return fail("256-row GEMM on a 64-row activation buffer");
    CKL(launch_gemm_w4(e->dtype, cx.mpad, g.epi, &g.W->tm, &g.W->tm_abs, cx.mpad == 16 ? &g.X->tm16 : (cx.mpad == 64 ? &g.X->tm64 : &g.X->tm256),
                       p, e->stream, g.pf));
  } else if (p.w_scale) {
    if (cx.mpad == 256 && g.X->rows < 256) return fail("256-row GEMM on a 64-row activation buffer");
    CKL(launch_gemm_w8(e->dtype, cx.mpad, g.epi, &g.W->tm, cx.mpad == 16 ? &g.X->tm16 : (cx.mpad == 64 ? &g.X->tm64 : &g.X->tm256), p,
                       e->stream, g.pf));
  } else if (e->c.flags & EB200_FLAG_SIMT_GEMM) {
    const size_t per_split = static_cast<size_t>(g.epi == EPI_SWIGLU ? 2 : 1) * cx.mpad * ((p.N + 127) / 128) * 128 * 4;
    while (p.splitk > 1 && per_split * p.splitk > e->ws_bytes) --p.splitk;
    CKL(launch_gemm_simt(e->dtype, cx.mpad, g.epi, g.W->w, g.W2 ? g.W2->w : nullptr, g.X->p, g.X->cols, p, e->stream));
  } else {
    if (cx.mpad == 256 && g.X->rows < 256) return fail("256-row GEMM on a 64-row activation buffer");
    CKL(launch_gemm(e->dtype, cx.mpad, g.epi, &g.W->tm, g.W2 ? &g.W2->tm : nullptr,
                    cx.mpad == 16 ? &g.X->tm16 : (cx.mpad == 64 ? &g.X->tm64 : &g.X->tm256), p, e->stream, g.pf));
  }
  return 0;
}
static int gemm_store(eb200_engine* e, const RowCtx& cx, const Linear& W, const ActBuf& X, void* out, long ld, const void* bias,
                      const L2Prefetch* pf = nullptr) {
  GemmCall g{&W, nullptr, &X, EPI_STORE, {}, pf};
  memset(&g.p, 0, sizeof(g.p));
  g.p.out = out;
  g.p.ld_out = ld;
  g.p.bias = bias;
  return run_gemm(e, cx, g);
}
static int gemm_residual(eb200_engine* e, const RowCtx& cx, const Linear& W, const ActBuf& X, const void* res, void* out, long ld,
                         const L2Prefetch* pf = nullptr) {
  GemmCall g{&W, nullptr, &X, EPI_RESIDUAL, {}, pf};
  memset(&g.p, 0, sizeof(g.p));
  g.p.out = out;
  g.p.ld_out = ld;
  g.p.res = res;
  g.p.ld_res = ld;
  return run_gemm(e, cx, g);
}
static int gemm_swiglu(eb200_engine* e, const RowCtx& cx, const Linear& Wgu, const ActBuf& X, void* out, long ld,
                       const L2Prefetch* pf = nullptr) {
  GemmCall g{&Wgu, nullptr, &X, EPI_SWIGLU_IL, {}, pf};
  memset(&g.p, 0, sizeof(g.p));
  g.p.out = out;
  g.p.ld_out = ld;
  return run_gemm(e, cx, g);
}
static int gemm_qkv(eb200_engine* e, const RowCtx& cx, const Linear& W, const ActBuf& X, void* q_out, void* kc, void* vc, long cap,
                    int nq, int nkv, const void* cosp, const void* sinp, const L2Prefetch* pf = nullptr) {
  GemmCall g{&W, nullptr, &X, EPI_QKV_ROPE, {}, pf};
  memset(&g.p, 0, sizeof(g.p));
  g.p.q_out = q_out;
  g.p.k_cache = kc;
  g.p.v_cache = vc;
  g.p.kv_cap = cap;
  g.p.n_q_heads = nq;
  g.p.n_kv_heads = nkv;
  g.p.rope_cos = cosp;
  g.p.rope_sin = sinp;
  g.p.pos_base = cx.pos_base;
  g.p.pos_arr = cx.pos_arr;
  g.p.pos_mstride = cx.pos_mstride;
  g.p.kv_base = cx.kv_base;
  return run_gemm(e, cx, g);
}
static int gemm_partial_f32(eb200_engine* e, const RowCtx& cx, const Linear& W, const ActBuf& X, float* out, long ld,
                            const L2Prefetch* pf = nullptr) {
  GemmCall g{&W, nullptr, &X, EPI_PARTIAL_F32, {}, pf};
  memset(&g.p, 0, sizeof(g.p));
  g.p.out = out;
  g.p.ld_out = ld;
  return run_gemm(e, cx, g);
}
static int tp_allreduce_f32(eb200_engine* e, float* buf, size_t count);
static int tp_allgather_u32(eb200_engine* e, const void* send, void* recv, size_t count);
static void chain_fill_tp(eb200_engine* e, ChainTP& tp);
// x += W . X  for a row-parallel projection (o_proj, down_proj).  Single GPU: fused residual epilogue.  Tensor parallel: every
// rank produces an unrounded fp32 partial over its slice of the reduction dim; then either
//   * NVLink peer windows (default): ONE kernel pushes the partial rows to their owners, reduces them in rank order, applies the
//     reference's two roundings (modeling_llama_kv.py:768, :838-845) AND the following RMSNorm, and publishes x / xn (/ tap) on
//     every rank (tp_fused.cu) -- *did_norm tells the caller that xn is already there; or
//   * NCCL: all-reduce, then the residual add; the caller runs the RMSNorm.
static int row_parallel_residual(eb200_engine* e, const RowCtx& cx, const Linear& W, const ActBuf& X, void* x, int H, const void* norm_w = nullptr,
                                 void* tap = nullptr, bool* did_norm = nullptr, const L2Prefetch* pf = nullptr) {
  if (did_norm) *did_norm = false;
  if (e->c.tp_size == 1) return gemm_residual(e, cx, W, X, x, x, H, pf);
  TRY(gemm_partial_f32(e, cx, W, X, e->f32buf, H, pf));
  if (e->tp_fused && cx.rows_idx < 0) {
    TpResidParams p;
    memset(&p, 0, sizeof(p));
    chain_fill_tp(e, p.tp);
    p.partial = e->f32buf;
    p.ld_partial = H;
    p.N = H;
    p.x = x;
    p.ld_x = H;
    p.tap = tap;
    p.ld_tap = e->F;
    p.norm_w = norm_w;
    p.xn = e->xn.p;
    p.ld_xn = H;
    p.eps = e->c.rms_norm_eps;
    ProfScope ps(e, 2, 0, "tp_resid_norm");
    CKL(launch_tp_resid_norm(e->dtype, p, cx.rows, e->stream));
    if (did_norm) *did_norm = norm_w != nullptr;
    return 0;
  }
  TRY(tp_allreduce_f32(e, e->f32buf, static_cast<size_t>(cx.rows) * H));
  ProfScope ps(e, 2, 0, "residual_add_f32");
  CKL(launch_residual_add_f32(e->dtype, e->f32buf, x, cx.rows, H, e->stream));
  return 0;
}
// arg-max over the (vocab-parallel) target logits of `rows` rows -> e->node_argmax (global token ids)
static int vocab_argmax(eb200_engine* e, int rows) {
  if (e->c.tp_size == 1) {
    ProfScope ps(e, 2, 0, "argmax");
    CKL(launch_argmax(e->dtype, e->logits, e->V_l, e->V_l, rows, e->node_argmax, e->stream));
    return 0;
  }
  const int r0 = e->c.tp_rank * e->V_l;
  const int valid = std::max(0, std::min(e->V_l, e->V - r0));
  {
    ProfScope ps(e, 2, 0, "argmax_val");
    CKL(launch_argmax_val(e->dtype, e->logits, e->V_l, valid, rows, r0, reinterpret_cast<float*>(e->am_send),
                          reinterpret_cast<int*>(e->am_send) + 128, e->stream));
  }
  TRY(tp_allgather_u32(e, e->am_send, e->am_recv, 256));
  ProfScope ps(e, 2, 0, "argmax_merge");
  CKL(launch_argmax_merge(reinterpret_cast<const float*>(e->am_recv), reinterpret_cast<const int*>(e->am_recv) + 128, e->c.tp_size, rows, 256,
                          e->node_argmax, e->stream));
  return 0;
}
static int tp_allgather_bytes(eb200_engine* e, const void* send, void* recv, size_t bytes);
// full-vocabulary logits rows for the sampling posterior: the local buffer on one GPU, an all-gather + unshard under TP
static int full_logits(eb200_engine* e, int rows, const void** out, long* ld, int* V) {
  if (e->c.tp_size == 1) {
    *out = e->logits;
    *ld = e->V_l;
    *V = e->V;
    return 0;
  }
  TRY(tp_allgather_bytes(e, e->logits, e->lg_recv, static_cast<size_t>(64) * e->V_l * 2));
  ProfScope ps(e, 2, 0, "unshard_rows");
  CKL(launch_unshard_rows(e->lg_recv, e->logits_full, e->c.tp_size, 64, e->V_l, e->stream));
  (void)rows;
  *out = e->logits_full;
  *ld = static_cast<long>(e->c.tp_size) * e->V_l;
  *V = e->V;
  return 0;
}
// sample one token from logits row 0 (first token after prefill, vanilla sampling): leaves it in st[S_BONUS]
static int sample_row0(eb200_engine* e) {
  const void* lg;
  long ld;
  int V;
  TRY(full_logits(e, 1, &lg, &ld, &V));
  {
    ProfScope ps(e, 2, 0, "row_softmax_stats");
    CKL(launch_row_softmax_stats(e->dtype, lg, ld, V, 1, e->sp, e->row_stats, e->stream));
  }
  AcceptOut ao;
  ao.accepted_tokens = e->accepted;
  ao.sel_nodes = e->sel_nodes;
  ao.host_visible = nullptr;
  ProfScope ps(e, 2, 0, "sample_commit");
  CKL(launch_sample_commit(e->dtype, lg, ld, V, e->row_stats, e->tb, e->depth, e->sp, e->rej_tokens, ao, e->st, nullptr, 0, 1, e->stream));
  return 0;
}
static void set_sampling(eb200_engine* e, const eb200_gen_params* gp) {
  e->sampling = gp && gp->temperature > 1e-5f;
  e->sp.temperature = gp ? gp->temperature : 0.f;
  e->sp.top_p = gp ? gp->top_p : 0.f;
  e->sp.top_k = gp ? gp->top_k : 0;
  e->sp.seed = gp ? gp->seed : 0;
  e->sp.uniforms = e->n_uniforms > 0 ? e->uniforms : nullptr;
  e->sp.n_uniforms = e->n_uniforms;
}
extern "C" int eb200_set_uniforms(eb200_engine* e, const float* host_uniforms, int32_t n) {
  if (!e || n < 0 || n > 4096 || (n > 0 && !host_uniforms)) return fail("eb200_set_uniforms: bad argument (at most 4096 values)");
  CK(cudaSetDevice(e->c.device));
  if (n > 0) CK(cudaMemcpy(e->uniforms, host_uniforms, n * sizeof(float), cudaMemcpyHostToDevice));
  e->n_uniforms = n;
  return 0;
}
// EB200_SKIP=name[,name...]: TIMING EXPERIMENTS ONLY -- drop every launch of the named kind (results become garbage) to
// read a kernel's marginal cost inside the captured cycle.  Names: rmsnorm, attention, gemm_store, gemm_residual,
// gemm_swiglu, gemm_qkv_rope.
static bool skip_kernel(const char* name) {
  static std::string list = [] {
    const char* s = getenv("EB200_SKIP");
    return std::string(s ? s : "");
  }();
  if (list.empty()) return false;
  const std::string key(name);
  size_t pos = 0;
  while (pos <= list.size()) {
    const size_t end = list.find(',', pos);
    if (list.compare(pos, (end == std::string::npos ? list.size() : end) - pos, key) == 0) return true;
    if (end == std::string::npos) break;
    pos = end + 1;
  }
  return false;
}

static int rmsnorm(eb200_engine* e, const void* src, long ld_src, const int64_t* ids64, const int* ids32, const void* w, void* y,
                   long ld_y, int col_off, int H, float eps, int rows, const L2Prefetch* pf = nullptr) {
  if (skip_kernel("rmsnorm")) return 0;
  ProfScope ps(e, 2, 0, "rmsnorm");
  CKL(launch_rmsnorm(e->dtype, src, ld_src, ids64, ids32, w, y, ld_y, col_off, H, eps, rows, e->stream, pf));
  return 0;
}
static int gather(eb200_engine* e, const void* table, long ld_table, const int64_t* ids64, const int* ids32, void* dst, long ld_dst,
                  int col_off, int H, int rows) {
  ProfScope ps(e, 2, 0, "gather_rows");
  CKL(launch_gather_rows(e->dtype, table, ld_table, ids64, ids32, dst, ld_dst, col_off, H, rows, e->stream));
  return 0;
}
static int attention(eb200_engine* e, const RowCtx& cx, const void* q, void* kc, void* vc, void* out, long cap, int nh, int nkv,
                     const L2Prefetch* pf = nullptr) {
  if (skip_kernel("attention")) return 0;
  if (cx.rows > 64) {
    // a causal prompt chunk of up to 256 rows: the kernel's ancestor mask covers 128 new columns, so the chunk is attended in
    // blocks of 64 query rows; block j sees the committed prefix + the earlier blocks of the chunk + itself causally
    if (cx.mask != nullptr || cx.rows_idx >= 0) return fail("attention: more than 64 rows only for causal prefill chunks");
    for (int r0 = 0; r0 < cx.rows; r0 += 64) {
      RowCtx sub = cx;
      sub.rows = std::min(64, cx.rows - r0);
      sub.mpad = 64;
      sub.n_ctx = DynInt{cx.n_ctx.idx, cx.n_ctx.add + r0};
      sub.n_tree = sub.rows;
      sub.kv_bound = cx.kv_bound > 0 ? std::min(cx.kv_bound, cx.kv_bound - cx.rows + r0 + sub.rows) : 0;
      const size_t off = static_cast<size_t>(r0) * nh * 128 * 2;
      TRY(attention(e, sub, reinterpret_cast<const char*>(q) + off, kc, vc, reinterpret_cast<char*>(out) + off, cap, nh, nkv, r0 == 0 ? pf : nullptr));
    }
    return 0;
  }
  AttnParams a;
  memset(&a, 0, sizeof(a));
  a.pf = pf;
  a.trace = e->in_verify ? e->attn_trace : nullptr;
  a.q = q;
  a.k_cache = kc;
  a.v_cache = vc;
  for (const void* plane : {static_cast<const void*>(kc), static_cast<const void*>(vc)}) {
    if (!e->kv_maps.count(plane)) {
      CUtensorMap m;
      TRY(make_tmap(&m, e->dtype, plane, static_cast<uint64_t>(nkv) * cap, 128, 64));
      e->kv_maps[plane] = m;
    }
  }
  a.tmK = &e->kv_maps[kc];
  a.tmV = &e->kv_maps[vc];
  a.out = out;
  a.kv_cap = cap;
  a.n_heads = nh;
  a.n_kv_heads = nkv;
  a.rows = cx.rows;
  a.rows_idx = cx.rows_idx;
  a.st = e->st;
  a.n_ctx = cx.n_ctx;
  a.n_tree = cx.n_tree;
  a.mask = cx.mask;
  a.max_kv = static_cast<int>(std::min<long>(cap, cx.kv_bound > 0 ? cx.kv_bound : e->c.max_length + 64 + 128));
  ProfScope ps(e, 1, 0, "attention");
  CKL(launch_attention(e->dtype, a, e->stream));
  return 0;
}
static int set_state(eb200_engine* e, int idx, int v) {
  ProfScope ps(e, 2, 0, "set_state");
  CKL(launch_set_state(e->st, idx, v, e->stream));
  return 0;
}

// ------------------------------------------------------------------------------------------------------------
// tensor parallel plumbing: NCCL over NVLink, resolved at run time (the library has no link-time NCCL dependency;
// in a torch process libnccl.so.2 is already mapped).  Only used when tp_size > 1.
// ------------------------------------------------------------------------------------------------------------
struct NcclApi {
  void* lib = nullptr;
  int (*GetUniqueId)(void*) = nullptr;
  int (*CommInitRank)(void**, int, eb200_nccl_id, int) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
  int (*CommDestroy)(void*) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};
static NcclApi g_nccl;
static int load_nccl() {
  if (g_nccl.lib) return 0;
  void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
  const char* env = getenv("EB200_NCCL_LIB");
  if (!h && env) h = dlopen(env, RTLD_NOW | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!h) return fail("cannot load libnccl.so.2 (set EB200_NCCL_LIB): %s", dlerror());
  g_nccl.GetUniqueId = reinterpret_cast<int (*)(void*)>(dlsym(h, "ncclGetUniqueId"));
  g_nccl.CommInitRank = reinterpret_cast<int (*)(void**, int, eb200_nccl_id, int)>(dlsym(h, "ncclCommInitRank"));
  g_nccl.AllReduce = reinterpret_cast<int (*)(const void*, void*, size_t, int, int, void*, cudaStream_t)>(dlsym(h, "ncclAllReduce"));
  g_nccl.AllGather = reinterpret_cast<int (*)(const void*, void*, size_t, int, void*, cudaStream_t)>(dlsym(h, "ncclAllGather"));
  g_nccl.CommDestroy = reinterpret_cast<int (*)(void*)>(dlsym(h, "ncclCommDestroy"));
  g_nccl.GetErrorString = reinterpret_cast<const char* (*)(int)>(dlsym(h, "ncclGetErrorString"));
  if (!g_nccl.GetUniqueId || !g_nccl.CommInitRank || !g_nccl.AllReduce || !g_nccl.AllGather) return fail("libnccl lacks required symbols");
  g_nccl.lib = h;
  return 0;
}
#define NCCLCK(call)                                                                                                \
  do {                                                                                                              \
    int _r = (call);                                                                                                \
    if (_r != 0) return fail("%s:%d %s -> NCCL error %d (%s)", __FILE__, __LINE__, #call, _r,                       \
                             g_nccl.GetErrorString ? g_nccl.GetErrorString(_r) : "?");                              \
  } while (0)

extern "C" int eb200_tp_unique_id(void* out_id128) {
  if (!out_id128) return fail("null id buffer");
  TRY(load_nccl());
  NCCLCK(g_nccl.GetUniqueId(out_id128));
  return 0;
}
extern "C" int eb200_tp_init(eb200_engine* e, const void* id128) {
  if (!e || !id128) return fail("null argument");
  if (e->c.tp_size <= 1) return 0;
  CK(cudaSetDevice(e->c.device));
  TRY(load_nccl());
  eb200_nccl_id id;
  memcpy(&id, id128, sizeof(id));
  NCCLCK(g_nccl.CommInitRank(&e->nccl_comm, e->c.tp_size, id, e->c.tp_rank));
  return 0;
}
// Peer windows: every rank exports the CUDA IPC handle of its window; after the launcher has exchanged them, each rank maps the
// others' windows.  From then on the row-parallel projections finish over peer memory (tp_fused.cu) instead of through NCCL, and
// the lm_head's vocabulary-parallel arg-max exchanges its (value, index) pairs through the same windows.
extern "C" int eb200_tp_ipc_handle(eb200_engine* e, void* out64) {
  if (!e || !out64) return fail("null argument");
  if (e->c.tp_size <= 1 || !e->tp_win) return fail("eb200_tp_ipc_handle: engine is not tensor parallel");
  CK(cudaSetDevice(e->c.device));
  cudaIpcMemHandle_t h;
  CK(cudaIpcGetMemHandle(&h, e->tp_win));
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handle size");
  memcpy(out64, &h, 64);
  return 0;
}
extern "C" int eb200_tp_open_peers(eb200_engine* e, const void* handles, int32_t n) {
  if (!e || !handles) return fail("null argument");
  if (e->c.tp_size <= 1) return 0;
  if (n != e->c.tp_size || n > kMaxTp) return fail("eb200_tp_open_peers: expected %d handles (at most %d ranks)", e->c.tp_size, kMaxTp);
  if (e->finalized) return fail("eb200_tp_open_peers after eb200_finalize");
  const char* off = getenv("EB200_TP_FUSED");
  if (off && atoi(off) == 0) return 0;  // A/B: keep the NCCL path
  CK(cudaSetDevice(e->c.device));
  CK(cudaStreamSynchronize(e->stream));
  for (int r = 0; r < n; ++r) {
    if (r == e->c.tp_rank) continue;
    cudaIpcMemHandle_t h;
    memcpy(&h, reinterpret_cast<const char*>(handles) + static_cast<size_t>(r) * 64, 64);
    void* p = nullptr;
    cudaError_t ce = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
    if (ce != cudaSuccess) {
      for (int q = 0; q < r; ++q)
        if (q != e->c.tp_rank && e->tp_peer[q]) {
          cudaIpcCloseMemHandle(e->tp_peer[q]);
          e->tp_peer[q] = nullptr;
        }
      cudaGetLastError();
      return fail("cudaIpcOpenMemHandle(rank %d) failed: %s -- no peer access between the GPUs of this job", r, cudaGetErrorString(ce));
    }
    e->tp_peer[r] = reinterpret_cast<char*>(p);
  }
  e->tp_fused = true;
  return 0;
}
static void tp_destroy_comm(void* comm) {
  if (g_nccl.CommDestroy) g_nccl.CommDestroy(comm);
}
static int tp_allreduce_f32(eb200_engine* e, float* buf, size_t count) {
  if (!e->nccl_comm) return fail("tensor parallel engine used before eb200_tp_init");
  e->stats.kernel_launches++;
  NCCLCK(g_nccl.AllReduce(buf, buf, count, 7 /* ncclFloat32 */, 0 /* ncclSum */, e->nccl_comm, e->stream));
  return 0;
}
static int tp_allgather_bytes(eb200_engine* e, const void* send, void* recv, size_t bytes) {
  if (!e->nccl_comm) return fail("tensor parallel engine used before eb200_tp_init");
  e->stats.kernel_launches++;
  NCCLCK(g_nccl.AllGather(send, recv, bytes, 0 /* ncclInt8 */, e->nccl_comm, e->stream));
  return 0;
}
static int tp_allgather_u32(eb200_engine* e, const void* send, void* recv, size_t count) {
  if (!e->nccl_comm) return fail("tensor parallel engine used before eb200_tp_init");
  e->stats.kernel_launches++;
  NCCLCK(g_nccl.AllGather(send, recv, count, 3 /* ncclUint32 */, e->nccl_comm, e->stream));
  return 0;
}

// ------------------------------------------------------------------------------------------------------------
// model passes
// ------------------------------------------------------------------------------------------------------------
static int update_kv_bucket(eb200_engine* e);
static void* kv_plane(void* base, int layer, int kv, int n_kv_heads, long cap) {
  return reinterpret_cast<char*>(base) + (static_cast<size_t>(layer) * 2 + kv) * n_kv_heads * cap * 128 * 2;
}

enum HeadMode : int { HEAD_NONE = 0, HEAD_ARGMAX = 1, HEAD_LOGITS = 2 };
static bool is_tap_layer(const eb200_engine* e, int i) { return i == e->L - 3 || i == e->L / 2 || i == 2; }
static int vocab_argmax(eb200_engine* e, int rows);

static void chain_fill_tp(eb200_engine* e, ChainTP& tp) {
  if (e->c.tp_size <= 1) return;
  tp.size = e->c.tp_size;
  tp.rank = e->c.tp_rank;
  for (int r = 0; r < e->c.tp_size; ++r) tp.win[r] = e->tp_peer[r];
  tp.inbox_off = e->tp_inbox_off;
  tp.ld_inbox = e->H;
  tp.flag_off = e->tp_flag_off;
  tp.ready_off = e->tp_ready_off;
  tp.am_off = e->tp_am_off;
  tp.epoch = e->tp_epoch;
}

// lm_head over the rows in e->xn (ea_model.py:190): one launch of whole 128-row vocabulary tiles per CTA (mega.cu), with the
// per-row arg-max taken straight from the staged accumulator tile and merged per row or, for the sampling path, the logits of
// this rank's shard.
static int target_head(eb200_engine* e, const RowCtx& cx, int head_mode) {
  if (head_mode == HEAD_NONE) return 0;
  if (!e->chain_head) {
    TRY(gemm_store(e, cx, e->t_head, e->xn, e->logits, e->V_l, nullptr));
    if (head_mode == HEAD_ARGMAX) TRY(vocab_argmax(e, cx.rows));
    return 0;
  }
  ChainArgs a;
  ChainMaps m;
  memset(&a, 0, sizeof(a));
  memset(&m, 0, sizeof(m));
  a.m_rows = cx.rows;
  a.m_idx = cx.rows_idx;
  a.st = e->st;
  a.sync = e->chain_sync;
  a.timing = e->chain_timing;
  chain_fill_tp(e, a.tp);
  ChainPhase& h = a.ph;
  h.N = e->t_head.N;
  h.K = e->t_head.K;
  m.w = e->t_head.tm;
  m.x = cx.mpad == 16 ? e->xn.tm16 : e->xn.tm64;
  if (head_mode == HEAD_ARGMAX) {
    h.fin = FIN_ARGMAX;
    h.tile_val = e->tile_val;
    h.tile_idx = e->tile_idx;
    h.out_idx = e->node_argmax;
    if (e->c.tp_size > 1) {  // vocabulary-parallel shard: only the real rows compete, indices are global
      h.idx_offset = e->c.tp_rank * e->V_l;
      h.N = std::max(0, std::min(e->V_l, e->V - h.idx_offset));
    }
  } else {
    h.fin = FIN_STORE_DIRECT;
    h.out = e->logits;
    h.ld_out = e->V_l;
  }
  const double bytes = static_cast<double>(e->t_head.N) * e->t_head.K * 2;
  if (skip_kernel("chain")) return 0;
  ProfScope ps(e, 0, bytes, "gemm_chain_head");
  CKL(launch_gemm_chain(e->dtype, cx.mpad, m, a, e->stream));
  e->stats.chain_bytes += bytes;
  return 0;
}

// LlamaModel.forward over <= 64 rows (modeling_llama_kv.py:1046-1200).  feat_dst receives the head's input features:
// EAGLE-3: hidden states entering layers 2, L/2, L-3 concatenated (:1138-1139, utils.py:248-252); EAGLE-1: the final
// normed hidden state.  Leaves the final-norm output in e->xn.  head_mode: also run the lm_head over the rows
// (ea_model.py:190) -> e->node_argmax (HEAD_ARGMAX: global token ids) or e->logits (HEAD_LOGITS: this rank's vocabulary shard).
static int target_forward(eb200_engine* e, const RowCtx& cx, const int64_t* ids64, const int* ids32, void* feat_dst, int head_mode) {
  const int H = e->H, L = e->L;
  const float eps = e->c.rms_norm_eps;
  TRY(gather(e, e->t_embed, H, ids64, ids32, e->x, H, 0, H, cx.rows));
  int slot = 0;
  bool have_xn = false;   // xn already holds this layer's input_layernorm(x) (written by the previous down_proj's fused TP kernel)
  bool tap_done = false;  // ... and the EAGLE-3 tap of this layer was written there too
  // L2 prefetch: every GEMM's producers fetch the leading weight tiles of the next GEMM after their last load, and the latency-bound
  // kernel in between (RMSNorm, attention) continues where that plan ends
  L2Prefetch pf_qkv_head;  // the part of this layer's qkv the previous down_proj prefetched
  memset(&pf_qkv_head, 0, sizeof(pf_qkv_head));
  for (int i = 0; i < L; ++i) {
    Layer& l = e->tl[i];
    if (e->c.eagle3 && feat_dst && is_tap_layer(e, i)) {
      if (!tap_done) TRY(gather(e, e->x, H, nullptr, e->ident, feat_dst, e->F, slot * H, H, cx.rows));
      ++slot;
    }
    if (!have_xn) {
      const L2Prefetch pf = l2_plan(e, l.qkv, cx.mpad, pf_qkv_head.j1, pf_norm_bytes());
      TRY(rmsnorm(e, e->x, H, nullptr, nullptr, l.ln1, e->xn.p, H, 0, H, eps, cx.rows, &pf));
    }
    void* kc = kv_plane(e->t_kv, i, 0, e->nkv_l, e->cap);
    void* vc = kv_plane(e->t_kv, i, 1, e->nkv_l, e->cap);
    const L2Prefetch pf_o = l2_plan(e, l.o, cx.mpad, 0, pf_tail_bytes());
    TRY(gemm_qkv(e, cx, l.qkv, e->xn, e->q, kc, vc, e->cap, e->nh_l, e->nkv_l, e->t_cos, e->t_sin, &pf_o));
    const L2Prefetch pf_o_rest = l2_plan_rest(e, l.o, cx.mpad, pf_o);
    TRY(attention(e, cx, e->q, kc, vc, e->attn.p, e->cap, e->nh_l, e->nkv_l, &pf_o_rest));
    bool did = false;
    const L2Prefetch pf_gu = l2_plan(e, l.gu, cx.mpad, 0, pf_tail_bytes());
    TRY(row_parallel_residual(e, cx, l.o, e->attn, e->x, H, l.ln2, nullptr, &did, &pf_gu));
    if (!did) {
      const L2Prefetch pf = l2_plan(e, l.gu, cx.mpad, pf_gu.j1, pf_norm_bytes());
      TRY(rmsnorm(e, e->x, H, nullptr, nullptr, l.ln2, e->xn.p, H, 0, H, eps, cx.rows, &pf));
    }
    const L2Prefetch pf_down = l2_plan(e, l.down, cx.mpad, 0, pf_tail_bytes());
    TRY(gemm_swiglu(e, cx, l.gu, e->xn, e->act.p, e->I_l, &pf_down));
    const void* next_norm = (i + 1 < L) ? e->tl[i + 1].ln1 : e->t_norm;
    void* tap = nullptr;
    if (e->c.eagle3 && feat_dst && i + 1 < L && is_tap_layer(e, i + 1)) tap = reinterpret_cast<char*>(feat_dst) + static_cast<size_t>(slot) * H * 2;
    pf_qkv_head = i + 1 < L ? l2_plan(e, e->tl[i + 1].qkv, cx.mpad, 0, pf_tail_bytes()) : l2_plan(e, l.qkv, cx.mpad, 0, 0);
    TRY(row_parallel_residual(e, cx, l.down, e->act, e->x, H, next_norm, tap, &did, &pf_qkv_head));
    have_xn = did;
    tap_done = did && tap != nullptr;
  }
  if (!have_xn) TRY(rmsnorm(e, e->x, H, nullptr, nullptr, e->t_norm, e->xn.p, H, 0, H, eps, cx.rows));
  if (!e->c.eagle3 && feat_dst) TRY(gather(e, e->xn.p, H, nullptr, e->ident, feat_dst, e->F, 0, H, cx.rows));
  TRY(target_head(e, cx, head_mode));  // lm_head on all rows (ea_model.py:190)
  return 0;
}

// Draft head forward over <= 64 rows.  first_pass: the rows' features are in e->d_feat (EAGLE-3: 3H taps -> fc).  Tree levels
// (src_rows != nullptr): the hidden input of row m is row src_rows[m] of the previous pass' output e->d_out (cnets.py:716,
// :747).  Ends with the draft logits of all rows in e->d_logits.
static int draft_forward(eb200_engine* e, const RowCtx& cx, const int64_t* ids64, const int* ids32, bool first_pass, const int* src_rows) {
  const int Hh = e->Hh;
  const float eps = e->c.head_rms_norm_eps;
  if (e->c.eagle3) {
    Layer& l = e->hl[0];
    // L2 prefetch as in target_forward.  The qkv's head is prefetched by the fc (first pass) or by the previous pass' lm_head.
    const L2Prefetch pf_qkv_head = l2_plan(e, l.qkv, cx.mpad, 0, pf_tail_bytes());
    if (first_pass) TRY(gemm_store(e, cx, e->h_fc, e->d_feat, e->d_h.p, Hh, nullptr, &pf_qkv_head));  // cnets.py:639-640
    // cat(norm(emb(ids)), norm(hidden))  cnets.py:427-430
    if (e->fused_e3_input) {
      ProfScope ps(e, 2, 0, "e3_input");
      const L2Prefetch pf = l2_plan(e, l.qkv, cx.mpad, pf_qkv_head.j1, pf_norm_bytes());
      CKL(launch_e3_input(e->dtype, e->h_embed, Hh, ids64, ids32, l.ln1, src_rows ? e->d_out.p : e->d_h.p, Hh, src_rows, e->d_h.p, Hh,
                          e->h_hidden_norm, e->d_cat.p, 2 * Hh, Hh, eps, cx.rows, e->stream, &pf));
    } else {
      if (src_rows) TRY(gather(e, e->d_out.p, Hh, nullptr, src_rows, e->d_h.p, Hh, 0, Hh, cx.rows));
      TRY(rmsnorm(e, e->h_embed, Hh, ids64, ids32, l.ln1, e->d_cat.p, 2 * Hh, 0, Hh, eps, cx.rows));
      TRY(rmsnorm(e, e->d_h.p, Hh, nullptr, nullptr, e->h_hidden_norm, e->d_cat.p, 2 * Hh, Hh, Hh, eps, cx.rows));
    }
    void* kc = kv_plane(e->d_kv, 0, 0, e->hnkv, e->dcap);
    void* vc = kv_plane(e->d_kv, 0, 1, e->hnkv, e->dcap);
    const L2Prefetch pf_o = l2_plan(e, l.o, cx.mpad, 0, pf_tail_bytes());
    TRY(gemm_qkv(e, cx, l.qkv, e->d_cat, e->d_q, kc, vc, e->dcap, e->hnh, e->hnkv, e->h_cos, e->h_sin, &pf_o));
    const L2Prefetch pf_o_rest = l2_plan_rest(e, l.o, cx.mpad, pf_o);
    TRY(attention(e, cx, e->d_q, kc, vc, e->d_attn.p, e->dcap, e->hnh, e->hnkv, &pf_o_rest));
    const L2Prefetch pf_gu = l2_plan(e, l.gu, cx.mpad, 0, pf_tail_bytes());
    TRY(gemm_residual(e, cx, l.o, e->d_attn, e->d_h.p, e->d_h2, Hh, &pf_gu));
    const L2Prefetch pf_gu_rest = l2_plan(e, l.gu, cx.mpad, pf_gu.j1, pf_norm_bytes());
    TRY(rmsnorm(e, e->d_h2, Hh, nullptr, nullptr, l.ln2, e->d_xn.p, Hh, 0, Hh, eps, cx.rows, &pf_gu_rest));
    const L2Prefetch pf_down = l2_plan(e, l.down, cx.mpad, 0, pf_tail_bytes());
    TRY(gemm_swiglu(e, cx, l.gu, e->d_xn, e->d_act.p, e->Ih, &pf_down));
    const L2Prefetch pf_head = l2_plan(e, e->h_head, cx.mpad, 0, pf_tail_bytes());
    TRY(gemm_residual(e, cx, l.down, e->d_act, e->d_h2, e->d_out.p, Hh, &pf_head));
    // lm_head(norm(out))  cnets.py:700, :734
    const L2Prefetch pf_head_rest = l2_plan(e, e->h_head, cx.mpad, pf_head.j1, pf_norm_bytes());
    TRY(rmsnorm(e, e->d_out.p, Hh, nullptr, nullptr, e->h_norm, e->d_xn.p, Hh, 0, Hh, eps, cx.rows, &pf_head_rest));
    // the next draft pass starts with the same qkv (after the level's top-k / tree kernels and e3_input)
    TRY(gemm_store(e, cx, e->h_head, e->d_xn, e->d_logits, e->Vd, nullptr, &pf_qkv_head));
    return 0;
  }
  // EAGLE-1/2: fc(cat(emb, hidden)) (cnets1.py:623), layer 0 without input norm (:428-429), target lm_head (:702,:732)
  TRY(gather(e, e->h_embed, Hh, ids64, ids32, e->d_cat.p, 2 * Hh, 0, Hh, cx.rows));
  if (first_pass) TRY(gather(e, e->d_feat.p, e->F, nullptr, e->ident, e->d_cat.p, 2 * Hh, Hh, Hh, cx.rows));
  else if (src_rows) TRY(gather(e, e->d_out.p, Hh, nullptr, src_rows, e->d_cat.p, 2 * Hh, Hh, Hh, cx.rows));
  TRY(gemm_store(e, cx, e->h_fc, e->d_cat, e->d_h.p, Hh, e->h_fc_bias));
  for (int i = 0; i < e->hL; ++i) {
    Layer& l = e->hl[i];
    const ActBuf* xin = &e->d_h;
    if (i > 0) {
      TRY(rmsnorm(e, e->d_h.p, Hh, nullptr, nullptr, l.ln1, e->d_xn.p, Hh, 0, Hh, eps, cx.rows));
      xin = &e->d_xn;
    }
    void* kc = kv_plane(e->d_kv, i, 0, e->hnkv, e->dcap);
    void* vc = kv_plane(e->d_kv, i, 1, e->hnkv, e->dcap);
    TRY(gemm_qkv(e, cx, l.qkv, *xin, e->d_q, kc, vc, e->dcap, e->hnh, e->hnkv, e->h_cos, e->h_sin));
    TRY(attention(e, cx, e->d_q, kc, vc, e->d_attn.p, e->dcap, e->hnh, e->hnkv));
    TRY(gemm_residual(e, cx, l.o, e->d_attn, e->d_h.p, e->d_h2, Hh));
    TRY(rmsnorm(e, e->d_h2, Hh, nullptr, nullptr, l.ln2, e->d_xn.p, Hh, 0, Hh, eps, cx.rows));
    TRY(gemm_swiglu(e, cx, l.gu, e->d_xn, e->d_act.p, e->Ih));
    void* dst = (i == e->hL - 1) ? e->d_out.p : e->d_h.p;
    TRY(gemm_residual(e, cx, l.down, e->d_act, e->d_h2, dst, Hh));
  }
  TRY(gemm_store(e, cx, e->t_head_full.w ? e->t_head_full : e->t_head, e->d_out, e->d_logits, e->Vd, nullptr));
  return 0;
}

// Tree growth after a stable pass whose last valid row index is st[S_LASTROW] (cnets.py:697-827)
static int grow_tree_static(eb200_engine* e);
static int grow_tree(eb200_engine* e, bool sampling) {
  if (e->static_tree) return grow_tree_static(e);
  const int k = e->k;
  {
    ProfScope ps(e, 2, 0, "logsoftmax_topk");
    CKL(launch_logsoftmax_topk(e->dtype, e->d_logits, e->Vd, e->Vd, 1, e->st, S_LASTROW, k, 0, e->topk_p, e->topk_i, e->stream));
  }
  {
    ProfScope ps(e, 2, 0, "tree_seed");
    CKL(launch_tree_seed(e->topk_p, e->topk_i, e->d2t, k, e->tb, e->st, e->stream));
  }
  const int mpad = k <= 16 ? 16 : 64;
  for (int i = 0; i < e->depth; ++i) {
    RowCtx cx;
    cx.kv_bound = e->kv_bucket;
    cx.mpad = mpad;
    cx.rows = k;
    cx.rows_idx = -1;
    cx.n_ctx = DynInt{S_N, 0};
    cx.n_tree = (i + 1) * k;
    cx.mask = e->tb.front_mask;
    cx.pos_base = DynInt{S_N, i};  // every node of a level shares one position (cnets.py:721)
    cx.pos_arr = nullptr;
    cx.pos_mstride = 0;
    cx.kv_base = DynInt{S_N, i * k};
    // inputs: rows of the previous output picked by the frontier (cnets.py:716, :747)
    TRY(draft_forward(e, cx, nullptr, e->tb.front_ids, false, e->tb.front_src));
    {
      ProfScope ps(e, 2, 0, "logsoftmax_topk");
      CKL(launch_logsoftmax_topk(e->dtype, e->d_logits, e->Vd, e->Vd, k, e->st, -1, k, 0, e->topk_p, e->topk_i, e->stream));
    }
    {
      ProfScope ps(e, 2, 0, "tree_expand");
      CKL(launch_tree_expand(e->dtype, e->topk_p, e->topk_i, e->d2t, k, i, e->tb, e->stream));
    }
  }
  {
    ProfScope ps(e, 2, 0, "tree_finalize");
    CKL(launch_tree_finalize(e->dtype, k, e->depth, e->T - 1, sampling ? 1 : 0, e->tb, e->st, e->stream));
  }
  return 0;
}

// Fixed-tree growth (modeling_eagle.py:863-957, greedy branch): level l feeds the stree.count[l] nodes that have children,
// each picked from its parent's top-k row; the last call gathers the T candidate tokens (utils.py:284-303).  The tree
// mask / positions / retrieve paths never change and were uploaded by eb200_set_static_tree.
static int grow_tree_static(eb200_engine* e) {
  const StaticTreeHost& t = e->stree;
  const int k = e->k;
  {
    ProfScope ps(e, 2, 0, "topk_raw");
    CKL(launch_logsoftmax_topk(e->dtype, e->d_logits, e->Vd, e->Vd, 1, e->st, S_LASTROW, k, 1, e->topk_p, e->topk_i, e->stream));
  }
  int off = 0;
  for (int l = 0; l <= t.n_levels; ++l) {
    const bool last = (l == t.n_levels);
    StaticLevelArgs a;
    a.topk_i = e->topk_i;
    a.d2t = e->d2t;
    a.k = k;
    a.rows_prev = l == 0 ? 1 : t.count[l - 1];
    a.ss_row0 = l == 0 ? 0 : 1 + (l >= 2 ? t.cum[l - 2] : 0);
    a.ss_tokens = e->ss_tokens;
    a.count = last ? 0 : t.count[l];
    a.sel = e->st_sel + off;
    a.src = e->st_src + off;
    a.lmask = e->st_lmask + 2 * off;
    a.first = l == 0 ? 1 : 0;
    a.final_T = last ? t.T : 0;
    a.tree_indices = e->st_tree_indices;
    a.n_leaf = t.n_leaf;
    a.width = t.width;
    {
      ProfScope ps(e, 2, 0, "static_level");
      CKL(launch_static_level(a, e->tb, e->st, e->stream));
    }
    if (last) break;
    const int rows = t.count[l];
    RowCtx cx;
    cx.kv_bound = e->kv_bucket;
    cx.mpad = rows <= 16 ? 16 : 64;
    cx.rows = rows;
    cx.rows_idx = -1;
    cx.n_ctx = DynInt{S_N, 0};
    cx.n_tree = t.cum[l];
    cx.mask = e->tb.front_mask;
    cx.pos_base = DynInt{S_N, l};  // len_posi advances by one per level (modeling_eagle.py:921-925)
    cx.pos_arr = nullptr;
    cx.pos_mstride = 0;
    cx.kv_base = DynInt{S_N, t.cum[l] - rows};
    TRY(draft_forward(e, cx, nullptr, e->tb.front_ids, false, e->tb.front_src));
    {
      ProfScope ps(e, 2, 0, "topk_raw");
      CKL(launch_logsoftmax_topk(e->dtype, e->d_logits, e->Vd, e->Vd, rows, e->st, -1, k, 1, e->topk_p, e->topk_i, e->stream));
    }
    off += rows;
  }
  return 0;
}

static RowCtx chunk_ctx(int rows, int base_idx, int kv_bound) {
  RowCtx cx;
  cx.kv_bound = kv_bound;
  cx.mpad = rows <= 16 ? 16 : (rows <= 64 ? 64 : 256);
  cx.rows = rows;
  cx.rows_idx = -1;
  cx.n_ctx = DynInt{base_idx, 0};
  cx.n_tree = rows;
  cx.mask = nullptr;  // causal inside the chunk
  cx.pos_base = DynInt{base_idx, 0};
  cx.pos_arr = nullptr;
  cx.pos_mstride = 1;
  cx.kv_base = DynInt{base_idx, 0};
  return cx;
}

static int check_ready(eb200_engine* e) {
  if (!e) return fail("null engine");
  if (!e->finalized) return fail("engine not finalized (eb200_finalize)");
  CK(cudaSetDevice(e->c.device));
  return 0;
}

// target prefill over P prompt rows in causal chunks of 64; returns the arg-max of the last row (utils.py:233-245)
static int target_prefill(eb200_engine* e, const int64_t* prompt, int P, int* first_token) {
  if (P < 1 || P > e->c.max_length - e->T) return fail("prompt length %d out of range", P);
  CK(cudaMemcpyAsync(e->ids_dev, prompt, static_cast<size_t>(P) * 8, cudaMemcpyDefault, e->stream));
  CK(cudaMemcpyAsync(e->out_ids_dev, e->ids_dev, static_cast<size_t>(P) * 8, cudaMemcpyDeviceToDevice, e->stream));
  int last_rows = 0;
  // 256 prompt rows per pass where the activation buffers allow it (one GPU, wgmma path): the weights are streamed
  // ceil(P / 256) times instead of ceil(P / 64) times (utils.py:232-254 runs the whole prompt in one forward)
  const int chunk = e->act_rows >= 256 ? 256 : 64;
  for (int base = 0; base < P; base += chunk) {
    const int rows = std::min(chunk, P - base);
    TRY(set_state(e, S_TMP0, base));
    RowCtx cx = chunk_ctx(rows, S_TMP0, base + rows);
    TRY(target_forward(e, cx, e->ids_dev + base, nullptr, reinterpret_cast<char*>(e->feat_all) + static_cast<size_t>(base) * e->F * 2, HEAD_NONE));
    last_rows = rows;
  }
  // lm_head on the last row only (the reference computes all P rows and uses the last, utils.py:243)
  TRY(gather(e, reinterpret_cast<char*>(e->xn.p) + static_cast<size_t>(last_rows - 1) * e->H * 2, e->H, nullptr, e->ident, e->xn_last.p,
             e->H, 0, e->H, 1));
  RowCtx one = chunk_ctx(1, S_TMP0, 0);
  TRY(gemm_store(e, one, e->t_head, e->xn_last, e->logits, e->V_l, nullptr));
  if (e->sampling) {  // utils.py:237-241: multinomial(softmax(processor(logits[:, -1])))
    TRY(set_state(e, S_UCOUNT, 0));
    TRY(sample_row0(e));
    ProfScope ps(e, 2, 0, "state_to");
    CKL(launch_state_to(e->node_argmax, e->st, S_BONUS, e->stream));
  } else {
    TRY(vocab_argmax(e, 1));
  }
  CK(cudaMemcpyAsync(first_token, e->node_argmax, sizeof(int), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  return 0;
}

extern "C" int eb200_prefill(eb200_engine* e, const int64_t* prompt, int32_t P, const eb200_gen_params* gp, int64_t* first_token) {
  TRY(check_ready(e));
  if (!prompt) return fail("eb200_prefill: null prompt");
  set_sampling(e, gp);
  int tok = 0;
  e->kv_bucket = 0;  // new sequence: size the attention strips (and re-capture the cycle graph) from scratch
  e->committed = 0;
  TRY(target_prefill(e, prompt, P, &tok));
  // draft stable pass over the P (feature_j, token_{j+1}) pairs (cnets.py:677-696)
  const int64_t tok64 = tok;
  if (P > 1) CK(cudaMemcpyAsync(e->ids_dev, prompt + 1, static_cast<size_t>(P - 1) * 8, cudaMemcpyDefault, e->stream));
  CK(cudaMemcpyAsync(e->ids_dev + (P - 1), &tok64, 8, cudaMemcpyHostToDevice, e->stream));
  int last_rows = 0;
  for (int base = 0; base < P; base += 64) {
    const int rows = std::min(64, P - base);
    TRY(set_state(e, S_TMP0, base));
    RowCtx cx = chunk_ctx(rows, S_TMP0, base + rows);
    TRY(gather(e, reinterpret_cast<char*>(e->feat_all) + static_cast<size_t>(base) * e->F * 2, e->F, nullptr, e->ident, e->d_feat.p, e->F,
               0, e->F, rows));
    TRY(draft_forward(e, cx, e->ids_dev + base, nullptr, true, nullptr));
    last_rows = rows;
  }
  TRY(set_state(e, S_N, P));
  TRY(set_state(e, S_NPREV, 0));
  TRY(set_state(e, S_ACC, 0));
  TRY(set_state(e, S_NEWTOK, 0));
  TRY(set_state(e, S_LASTROW, last_rows - 1));
  TRY(set_state(e, S_BONUS, tok));
  e->committed = P;
  TRY(update_kv_bucket(e));
  TRY(grow_tree(e, e->sampling));
  CK(cudaStreamSynchronize(e->stream));
  e->committed = P;
  if (first_token) *first_token = tok;
  return 0;
}

// The attention kernels size their shared-memory score strip from a host-known bound on the KV length.  The bound
// moves in buckets of 256 rows; crossing a bucket invalidates the captured cycle graph (re-captured on the next step).
static int update_kv_bucket(eb200_engine* e) {
  // e->committed mirrors the last COLLECTED cycle; a cycle still in flight may add up to D rows
  const long in_flight = static_cast<long>(e->launch_seq - e->collect_seq);
  const long committed = e->committed + in_flight * e->D;
  const long need = committed + e->T + e->D + static_cast<long>(e->depth) * e->k + 8;
  if (need > e->kv_bucket) {
    e->kv_bucket = static_cast<int>(std::min<long>(((need + 64 + 255) / 256) * 256, e->dcap));
    if (e->graph_exec) {
      cudaGraphExecDestroy(e->graph_exec);
      e->graph_exec = nullptr;
    }
    if (e->graph) {
      cudaGraphDestroy(e->graph);
      e->graph = nullptr;
    }
  }
  // the verify pass appends T tree rows to the TARGET planes (cap rows each), the draft levels up to depth*k (or the static
  // tree's inner nodes) rows behind the D stable rows of the DRAFT planes (dcap rows)
  const long draft_tree_rows = e->static_tree ? static_cast<long>(e->stree.sel.size()) : static_cast<long>(e->depth) * e->k;
  if (need > e->dcap || committed + e->T > e->cap || committed + e->D + draft_tree_rows > e->dcap)
    return fail("KV capacity exceeded: committed %ld of max_length %d", committed, e->c.max_length);
  return 0;
}

// one draft->verify->accept cycle (ea_model.py:251-288)
static int enqueue_cycle(eb200_engine* e) {
  const int T = e->T;
  RowCtx cx;
  cx.kv_bound = e->kv_bucket;
  cx.mpad = T <= 16 ? 16 : 64;
  cx.rows = T;
  cx.rows_idx = -1;
  cx.n_ctx = DynInt{S_N, 0};
  cx.n_tree = T;
  cx.mask = e->tb.tree_mask;
  cx.pos_base = DynInt{S_N, 0};  // position_ids = tree_position_ids + input_ids.shape[1]  (utils.py:314)
  cx.pos_arr = e->tb.tree_pos;
  cx.pos_mstride = 0;
  cx.kv_base = DynInt{S_N, 0};
  e->in_verify = true;
  TRY(target_forward(e, cx, nullptr, e->tb.draft_tokens, e->feat, e->sampling ? HEAD_LOGITS : HEAD_ARGMAX));  // + lm_head on all T rows (ea_model.py:190)
  e->in_verify = false;
  AcceptOut ao;
  ao.accepted_tokens = e->accepted;
  ao.sel_nodes = e->sel_nodes;
  ao.host_visible = nullptr;
  if (e->sampling) {
    const void* lg;
    long ld;
    int V;
    TRY(full_logits(e, T, &lg, &ld, &V));
    {
      ProfScope ps(e, 2, 0, "row_softmax_stats");
      CKL(launch_row_softmax_stats(e->dtype, lg, ld, V, T, e->sp, e->row_stats, e->stream));
    }
    {
      ProfScope ps(e, 2, 0, "sample_posterior");
      CKL(launch_sample_posterior(e->dtype, lg, ld, V, e->row_stats, e->tb, e->depth, e->sp, e->rej_tokens, e->st, e->stream));
    }
    ProfScope ps(e, 2, 0, "sample_commit");
    CKL(launch_sample_commit(e->dtype, lg, ld, V, e->row_stats, e->tb, e->depth, e->sp, e->rej_tokens, ao, e->st, e->out_ids_dev,
                             e->c.max_length + 128, 0, e->stream));
  } else {
    ProfScope ps(e, 2, 0, "greedy_accept");
    CKL(launch_greedy_accept(e->node_argmax, e->tb, T, e->depth, ao, e->st, e->out_ids_dev, e->c.max_length + 128, e->stream));
  }
  {
    ProfScope ps(e, 2, 0, "kv_compact");
    CKL(launch_kv_compact(e->dtype, e->t_kv, e->cap * 128, e->L * 2 * e->nkv_l, e->cap, e->sel_nodes, e->st, e->stream));
  }
  // draft stable pass over the accepted (feature, next-token) pairs (utils.py:454-468, cnets.py:690-696)
  TRY(gather(e, e->feat, e->F, nullptr, e->sel_nodes, e->d_feat.p, e->F, 0, e->F, e->D));
  RowCtx sx;
  sx.kv_bound = e->kv_bucket;
  sx.mpad = 16;
  sx.rows = e->D;
  sx.rows_idx = S_ACC;
  sx.n_ctx = DynInt{S_NPREV, 0};
  sx.n_tree = e->D;
  sx.mask = nullptr;
  sx.pos_base = DynInt{S_NPREV, 0};
  sx.pos_arr = nullptr;
  sx.pos_mstride = 1;
  sx.kv_base = DynInt{S_NPREV, 0};
  TRY(draft_forward(e, sx, nullptr, e->accepted + e->D, true, nullptr));
  TRY(grow_tree(e, e->sampling));
  return 0;
}

// One cycle = launch (graph replay / capture / eager) + read-back of the 16-int state and the committed tokens into one of two
// pinned slots + an event.  eb200_step launches and collects; eb200_generate keeps the NEXT cycle in flight while the host
// looks at the previous one (no GPU idle gap for the host round trip; the speculative cycle is drained and dropped at a stop).
static int launch_cycle(eb200_engine* e) {
  TRY(update_kv_bucket(e));
  const bool use_graph = !(e->c.flags & EB200_FLAG_NO_GRAPH) && !e->profiling && g_debug_sync <= 0;
  if (use_graph && e->graph_exec) {
    CK(cudaGraphLaunch(e->graph_exec, e->stream));
    e->stats.kernel_launches += e->launches_per_cycle;
    e->stats.chain_bytes += e->chain_bytes_cycle;
  } else if (use_graph && e->eager_cycles >= 1) {
    // capture the (static) launch sequence of one cycle once, then replay it every cycle
    const uint64_t before = e->stats.kernel_launches;
    const double bytes_before = e->stats.chain_bytes;
    CK(cudaStreamBeginCapture(e->stream, cudaStreamCaptureModeThreadLocal));
    e->capturing = true;
    const int rc = enqueue_cycle(e);
    e->capturing = false;
    cudaGraph_t g = nullptr;
    cudaError_t ce = cudaStreamEndCapture(e->stream, &g);
    if (rc != 0) {
      if (g) cudaGraphDestroy(g);
      return rc;
    }
    if (ce != cudaSuccess) return fail("cudaStreamEndCapture: %s", cudaGetErrorString(ce));
    e->graph = g;
    e->launches_per_cycle = e->stats.kernel_launches - before;
    e->chain_bytes_cycle = e->stats.chain_bytes - bytes_before;
    CK(cudaGraphInstantiate(&e->graph_exec, e->graph, 0));
    CK(cudaGraphLaunch(e->graph_exec, e->stream));
  } else {
    TRY(enqueue_cycle(e));
    e->eager_cycles++;
  }
  // host-visible mirror of this cycle: device state (accept rows, bonus token, lengths) and the committed tokens
  const unsigned slot = e->launch_seq & 1u;
  int64_t* pin = e->pinned + slot * 64;
  CK(cudaMemcpyAsync(pin + 8, e->st, S_COUNT * sizeof(int), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaMemcpyAsync(pin + 32, e->accepted, e->D * sizeof(int), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaEventRecord(e->ev_slot[slot], e->stream));
  e->launch_seq++;
  return 0;
}
static int collect_cycle(eb200_engine* e, int64_t* out_tokens, int32_t* out_n, int64_t* next_token) {
  if (e->collect_seq == e->launch_seq) return fail("collect_cycle: no cycle in flight");
  const unsigned slot = e->collect_seq & 1u;
  CK(cudaEventSynchronize(e->ev_slot[slot]));
  e->collect_seq++;
  const int64_t* pin = e->pinned + slot * 64;
  const int* st = reinterpret_cast<const int*>(pin + 8);
  const int* acc = reinterpret_cast<const int*>(pin + 32);
  const int n = st[S_ACC];
  if (n < 1 || n > e->D) return fail("engine state corrupt: accepted rows = %d", n);
  for (int j = 0; j < n; ++j)
    if (out_tokens) out_tokens[j] = acc[j];
  if (out_n) *out_n = n;
  if (next_token) *next_token = st[S_BONUS];
  e->last_best = st[S_BEST];
  e->last_acc = n - 1;
  e->committed = st[S_N];
  e->stats.cycles++;
  e->stats.tokens_committed += n;
  return 0;
}
// may the next cycle be launched before the previous one has been looked at?  Not while a KV bucket (and with it the captured
// graph) must change, not in the eager / profiled modes (their launch sequences are enqueued from host state).
static bool can_speculate(eb200_engine* e) {
  if ((e->c.flags & EB200_FLAG_NO_GRAPH) || e->profiling || g_debug_sync > 0 || !e->graph_exec) return false;
  static int on = -1;
  if (on < 0) {
    const char* s = getenv("EB200_ASYNC_CYCLES");
    on = (s && atoi(s) == 0) ? 0 : 1;
  }
  if (!on) return false;
  const long committed = e->committed + static_cast<long>(e->launch_seq - e->collect_seq + 1) * e->D;
  const long need = committed + e->T + e->D + static_cast<long>(e->depth) * e->k + 8;
  return need <= e->kv_bucket && committed + e->T <= e->cap;
}

extern "C" int eb200_step(eb200_engine* e, int64_t* out_tokens, int32_t* out_n, int64_t* next_token) {
  TRY(check_ready(e));
  if (e->launch_seq != e->collect_seq) return fail("eb200_step while a cycle is in flight");
  TRY(launch_cycle(e));
  return collect_cycle(e, out_tokens, out_n, next_token);
}

extern "C" int eb200_generate(eb200_engine* e, const int64_t* prompt, int32_t P, const eb200_gen_params* gp, int64_t* out_ids,
                              int32_t out_cap, int32_t* out_len, int32_t* out_new_token, int32_t* out_steps) {
  TRY(check_ready(e));
  if (!prompt || !gp || !out_ids) return fail("eb200_generate: null argument");
  if (out_cap < P) return fail("out_ids capacity too small");
  int64_t first = 0;
  TRY(eb200_prefill(e, prompt, P, gp, &first));
  CK(cudaMemcpy(out_ids, prompt, static_cast<size_t>(P) * 8, cudaMemcpyDefault));
  int len = P, new_token = 0, idx = 0;
  const int max_len = (gp->max_length > 0 && gp->max_length <= e->c.max_length) ? gp->max_length : e->c.max_length;
  const int limit = max_len - (e->T - 1) - 10;  // ea_model.py:250
  int64_t toks[16];
  if (limit > 0) TRY(launch_cycle(e));
  for (idx = 0; idx < limit; ++idx) {
    int n = 0;
    int64_t nxt = 0;
    // keep the GPU busy across the host round trip: cycle idx+1 is queued before cycle idx is inspected
    const bool spec = idx + 1 < limit && can_speculate(e);
    if (spec) TRY(launch_cycle(e));
    TRY(collect_cycle(e, toks, &n, &nxt));
    bool stop = false;
    for (int j = 0; j < n; ++j) {
      if (len < out_cap) out_ids[len] = toks[j];
      ++len;
      if (gp->stop_token_id >= 0 && toks[j] == gp->stop_token_id) stop = true;
      if (gp->eos_token_id >= 0 && toks[j] == gp->eos_token_id) stop = true;
    }
    new_token += n;
    if (stop) break;
    if (new_token > gp->max_new_tokens) break;
    if (len > limit) break;
    if (!spec && idx + 1 < limit) TRY(launch_cycle(e));
  }
  while (e->collect_seq != e->launch_seq) {  // a speculative cycle past the stop: let it finish, drop its tokens
    int n = 0;
    int64_t nxt = 0;
    TRY(collect_cycle(e, toks, &n, &nxt));
  }
  if (idx == limit) idx = limit - 1;  // python's `for idx in range(limit)` leaves idx at the last value
  if (out_len) *out_len = std::min(len, out_cap);
  if (out_new_token) *out_new_token = new_token;
  if (out_steps) *out_steps = idx;
  return 0;
}

// Vanilla decoding (ea_model.py:305-380 / :485-558) in two calls so that a generator can stream: begin = prefill + first
// token; step = feed the pending token, return it (`fed`) and the next one.
extern "C" int eb200_naive_begin(eb200_engine* e, const int64_t* prompt, int32_t P, const eb200_gen_params* gp, int64_t* first_token) {
  TRY(check_ready(e));
  if (!prompt) return fail("eb200_naive_begin: null prompt");
  set_sampling(e, gp);
  int tok = 0;
  e->kv_bucket = 0;
  e->committed = 0;
  TRY(target_prefill(e, prompt, P, &tok));
  TRY(set_state(e, S_N, P));
  e->committed = P;
  e->naive_tok = tok;
  if (first_token) *first_token = tok;
  return 0;
}
extern "C" int eb200_naive_step(eb200_engine* e, int64_t* fed_token, int64_t* next_token) {
  TRY(check_ready(e));
  if (e->committed + 2 > e->cap) return fail("KV capacity exceeded: committed %ld of max_length %d", e->committed, e->c.max_length);
  // feed the token, get the next arg-max / sample (ea_model.py:353-362)
  RowCtx cx = chunk_ctx(1, S_N, static_cast<int>(e->committed) + 2);
  TRY(target_forward(e, cx, nullptr, e->node_argmax, nullptr, e->sampling ? HEAD_LOGITS : HEAD_ARGMAX));
  const int fed = e->naive_tok;
  if (e->sampling) {
    TRY(sample_row0(e));
    ProfScope ps(e, 2, 0, "state_to");
    CKL(launch_state_to(e->node_argmax, e->st, S_BONUS, e->stream));
  }
  {
    ProfScope ps(e, 2, 0, "copy_state");
    CKL(launch_copy_state(e->st, S_N, S_N, 1, e->stream));
  }
  int tok = 0;
  CK(cudaMemcpyAsync(&tok, e->node_argmax, sizeof(int), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  e->committed += 1;
  e->naive_tok = tok;
  if (fed_token) *fed_token = fed;
  if (next_token) *next_token = tok;
  return 0;
}

extern "C" int eb200_naive_generate(eb200_engine* e, const int64_t* prompt, int32_t P, const eb200_gen_params* gp, int64_t* out_ids,
                                    int32_t out_cap, int32_t* out_len, int32_t* out_new_token, int32_t* out_steps) {
  TRY(check_ready(e));
  if (!prompt || !gp || !out_ids) return fail("eb200_naive_generate: null argument");
  if (out_cap < P) return fail("out_ids capacity too small");
  int64_t first = 0;
  TRY(eb200_naive_begin(e, prompt, P, gp, &first));
  CK(cudaMemcpy(out_ids, prompt, static_cast<size_t>(P) * 8, cudaMemcpyDefault));
  int len = P, new_token = 0, idx = 0;
  const int max_len = (gp->max_length > 0 && gp->max_length <= e->c.max_length) ? gp->max_length : e->c.max_length;
  const int limit = max_len - (e->T - 1) - 10;
  for (idx = 0; idx < limit; ++idx) {
    int64_t fed = 0, nxt = 0;
    TRY(eb200_naive_step(e, &fed, &nxt));
    if (len < out_cap) out_ids[len] = fed;
    ++len;
    ++new_token;
    if (gp->eos_token_id >= 0 && fed == gp->eos_token_id) break;
    if (gp->stop_token_id >= 0 && fed == gp->stop_token_id) break;
    if (new_token > gp->max_new_tokens) break;
    if (len > limit) break;
  }
  if (idx == limit) idx = limit - 1;
  if (out_len) *out_len = std::min(len, out_cap);
  if (out_new_token) *out_new_token = new_token;
  if (out_steps) *out_steps = idx;
  return 0;
}

// total_token = -1 support (ea_model.py:148-168): the timed quantity is the target forward (incl. lm_head) over `rows` fresh
// rows, `iters` times; the caller compares candidates and then fixes the tree size with eb200_set_total_token.
extern "C" int eb200_time_target_forward(eb200_engine* e, int32_t rows, int32_t iters, double* ms_total) {
  TRY(check_ready(e));
  if (rows < 1 || rows > 64 || iters < 1 || !ms_total) return fail("eb200_time_target_forward: bad arguments");
  TRY(set_state(e, S_TMP0, 0));
  CK(cudaMemsetAsync(e->ids_dev, 0, 64 * 8, e->stream));
  RowCtx cx = chunk_ctx(rows, S_TMP0, rows);
  TRY(target_forward(e, cx, e->ids_dev, nullptr, nullptr, HEAD_ARGMAX));  // warm-up (function attributes, SiLU table)
  cudaEvent_t a, b;
  CK(cudaEventCreate(&a));
  CK(cudaEventCreate(&b));
  CK(cudaEventRecord(a, e->stream));
  int rc = 0;
  for (int i = 0; i < iters && rc == 0; ++i) rc = target_forward(e, cx, e->ids_dev, nullptr, nullptr, HEAD_ARGMAX);
  cudaEventRecord(b, e->stream);
  cudaError_t se = cudaStreamSynchronize(e->stream);
  float ms = 0.f;
  if (rc == 0 && se == cudaSuccess) cudaEventElapsedTime(&ms, a, b);
  cudaEventDestroy(a);
  cudaEventDestroy(b);
  if (rc != 0) return rc;
  if (se != cudaSuccess) return fail("eb200_time_target_forward: %s", cudaGetErrorString(se));
  *ms_total = ms;
  return 0;
}
static void drop_graph(eb200_engine* e);
extern "C" int eb200_set_total_token(eb200_engine* e, int32_t total_token) {
  if (!e) return fail("null engine");
  if (e->static_tree) return fail("eb200_set_total_token: the static tree fixes total_token");
  if (total_token < 2 || total_token > e->c.total_token) return fail("total_token must be in [2, %d] (the capacity the engine was created with)", e->c.total_token);
  if (e->k + e->depth * e->k * e->k < total_token - 1) return fail("candidate pool smaller than total_token - 1");
  CK(cudaSetDevice(e->c.device));
  CK(cudaStreamSynchronize(e->stream));
  e->T = total_token;
  drop_graph(e);
  return 0;
}

// ------------------------------------------------------------------------------------------------------------
// static draft tree (SURVEY.md 8 row a11)
// ------------------------------------------------------------------------------------------------------------
static void drop_graph(eb200_engine* e) {
  if (e->graph_exec) {
    cudaGraphExecDestroy(e->graph_exec);
    e->graph_exec = nullptr;
  }
  if (e->graph) {
    cudaGraphDestroy(e->graph);
    e->graph = nullptr;
  }
  e->eager_cycles = 0;
}

extern "C" int eb200_set_static_tree(eb200_engine* e, const int32_t* choices, const int32_t* choice_len, int32_t n_choices) {
  if (!e) return fail("eb200_set_static_tree: null engine");
  CK(cudaSetDevice(e->c.device));
  CK(cudaStreamSynchronize(e->stream));
  if (n_choices == 0) {  // back to the dynamic tree
    e->static_tree = false;
    drop_graph(e);
    return 0;
  }
  StaticTreeHost t;
  std::string err;
  if (build_static_tree(choices, choice_len, n_choices, e->k, t, err)) return fail("%s", err.c_str());
  if (t.T != e->T) return fail("static tree has %d nodes but the engine was created with total_token = %d", t.T, e->T);
  if (t.width != e->D) return fail("static tree depth: longest choice has %d entries, the engine needs depth = %d", t.width - 1, t.width - 2);
  CK(cudaMemcpy(e->tb.tree_mask, t.mask.data(), t.mask.size() * sizeof(uint64_t), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(e->tb.tree_pos, t.pos.data(), t.T * sizeof(int), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(e->tb.parent_node, t.parent.data(), t.T * sizeof(int), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(e->tb.retrieve, t.retrieve.data(), t.retrieve.size() * sizeof(int), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(e->st_tree_indices, t.tree_indices.data(), t.T * sizeof(int), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(e->st_sel, t.sel.data(), t.sel.size() * sizeof(int), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(e->st_src, t.src.data(), t.src.size() * sizeof(int), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(e->st_lmask, t.lmask.data(), t.lmask.size() * sizeof(uint64_t), cudaMemcpyHostToDevice));
  e->stree = t;
  e->static_tree = true;
  drop_graph(e);
  return 0;
}

// Host-only: the integer tables of a fixed tree in the reference's own formats (generate_tree_buffers, utils.py:89-207;
// generate_tree_buffers_for_eagle, modeling_eagle.py:625-692).  Caller sizes every output for n = n_choices:
// tree_indices / tree_position_ids [n+1], tree_attn_mask [(n+1)^2], retrieve_indices [(n+1)^2] (n_leaf x width used),
// level_count [n], level_sel / level_src [n], level_mask [n*n] (n_inner x n_inner used, row r = r-th node with children).
extern "C" int eb200_static_tree_buffers(const int32_t* choices, const int32_t* choice_len, int32_t n_choices, int32_t top_k,
                                         int32_t* tree_indices, int32_t* tree_position_ids, float* tree_attn_mask,
                                         int32_t* retrieve_indices, int32_t* n_leaf, int32_t* width, int32_t* n_levels,
                                         int32_t* level_count, int32_t* level_sel, int32_t* level_src, float* level_mask,
                                         int32_t* n_inner) {
  StaticTreeHost t;
  std::string err;
  if (build_static_tree(choices, choice_len, n_choices, top_k, t, err)) return fail("%s", err.c_str());
  auto bit = [](const std::vector<uint64_t>& m, int row, int col) { return (m[2 * row + (col >> 6)] >> (col & 63)) & 1ull; };
  for (int i = 0; i < t.T; ++i) {
    if (tree_indices) tree_indices[i] = t.tree_indices[i];
    if (tree_position_ids) tree_position_ids[i] = t.pos[i];
    if (tree_attn_mask)
      for (int j = 0; j < t.T; ++j) tree_attn_mask[i * t.T + j] = bit(t.mask, i, j) ? 1.f : 0.f;
  }
  if (retrieve_indices) std::copy(t.retrieve.begin(), t.retrieve.end(), retrieve_indices);
  if (n_leaf) *n_leaf = t.n_leaf;
  if (width) *width = t.width;
  if (n_levels) *n_levels = t.n_levels;
  const int ni = static_cast<int>(t.sel.size());
  if (n_inner) *n_inner = ni;
  for (int l = 0; l < t.n_levels; ++l)
    if (level_count) level_count[l] = t.count[l];
  for (int r = 0; r < ni; ++r) {
    if (level_sel) level_sel[r] = t.sel[r];
    if (level_src) level_src[r] = t.src[r];
    if (level_mask)
      for (int j = 0; j < ni; ++j) level_mask[r * ni + j] = bit(t.lmask, r, j) ? 1.f : 0.f;
  }
  return 0;
}


// ------------------------------------------------------------------------------------------------------------
// inspection
// ------------------------------------------------------------------------------------------------------------
extern "C" int eb200_get_tree(eb200_engine* e, int64_t* draft_tokens, float* tree_mask, int64_t* tree_position_ids,
                              int64_t* retrieve_indices, int32_t* n_leaf, int32_t* max_depth) {
  TRY(check_ready(e));
  CK(cudaStreamSynchronize(e->stream));
  const int T = e->T, D = e->D;
  std::vector<int> tok(128), pos(128), ret(128 * 16), st(S_COUNT);
  std::vector<uint64_t> mask(256);
  CK(cudaMemcpy(tok.data(), e->tb.draft_tokens, 128 * 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(pos.data(), e->tb.tree_pos, 128 * 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(ret.data(), e->tb.retrieve, 128 * 16 * 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(mask.data(), e->tb.tree_mask, 256 * 8, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(st.data(), e->st, S_COUNT * 4, cudaMemcpyDeviceToHost));
  const int nl = st[S_NLEAF], md = st[S_MAXDEPTH];
  for (int i = 0; i < T; ++i) {
    if (draft_tokens) draft_tokens[i] = tok[i];
    if (tree_position_ids) tree_position_ids[i] = pos[i];
    if (tree_mask)
      for (int j = 0; j < T; ++j) tree_mask[i * T + j] = ((j < 64 ? (mask[2 * i] >> j) : (mask[2 * i + 1] >> (j - 64))) & 1ull) ? 1.f : 0.f;
  }
  if (retrieve_indices)
    for (int r = 0; r < nl; ++r)
      for (int j = 0; j < md; ++j) retrieve_indices[r * md + j] = ret[r * D + j];
  if (n_leaf) *n_leaf = nl;
  if (max_depth) *max_depth = md;
  return 0;
}

extern "C" int eb200_get_verify(eb200_engine* e, int64_t* node_argmax, int32_t* best, int32_t* accept_length, int32_t* committed_len) {
  TRY(check_ready(e));
  CK(cudaStreamSynchronize(e->stream));
  if (node_argmax) {
    std::vector<int> a(128);
    CK(cudaMemcpy(a.data(), e->node_argmax, 128 * 4, cudaMemcpyDeviceToHost));
    for (int i = 0; i < e->T; ++i) node_argmax[i] = a[i];
  }
  if (best) *best = e->last_best;
  if (accept_length) *accept_length = e->last_acc;
  if (committed_len) *committed_len = static_cast<int>(e->committed);
  return 0;
}

template <typename T> __global__ void to_float_kernel(const T* src, float* dst, long n) {
  long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x;
  if (i < n) dst[i] = static_cast<float>(src[i]);
}

extern "C" int eb200_debug_read(eb200_engine* e, const char* what, float* out, int64_t cap, int32_t* rows, int32_t* cols) {
  TRY(check_ready(e));
  CK(cudaStreamSynchronize(e->stream));
  std::string w(what ? what : "");
  const void* src = nullptr;
  int r = 0, c = 0;
  if (w == "verify_features") { src = e->feat; r = e->T; c = e->F; }
  else if (w == "verify_logits") { src = e->logits; r = e->T; c = e->V_l; }
  else if (w == "verify_hidden") { src = e->xn.p; r = e->T; c = e->H; }
  else if (w == "draft_out") { src = e->d_out.p; r = 16; c = e->Hh; }
  else if (w == "draft_logits") { src = e->d_logits; r = 16; c = e->Vd; }
  else if (w == "target_kv") { src = e->t_kv; r = e->L * 2 * e->nkv_l; c = static_cast<int>(e->cap * 128); }
  else if (w == "draft_kv") { src = e->d_kv; r = e->hL * 2 * e->hnkv; c = static_cast<int>(e->dcap * 128); }
  else return fail("eb200_debug_read: unknown buffer '%s'", what);
  const long n = static_cast<long>(r) * c;
  if (rows) *rows = r;
  if (cols) *cols = c;
  if (!out) return 0;
  if (n > cap) return fail("eb200_debug_read: need %ld floats, capacity %ld", n, (long)cap);
  float* tmp = nullptr;
  CK(cudaMalloc(&tmp, n * sizeof(float)));
  const int blocks = static_cast<int>((n + 255) / 256);
  if (e->dtype == DT_BF16) to_float_kernel<<<blocks, 256, 0, e->stream>>>(reinterpret_cast<const __nv_bfloat16*>(src), tmp, n);
  else to_float_kernel<<<blocks, 256, 0, e->stream>>>(reinterpret_cast<const __half*>(src), tmp, n);
  cudaError_t err = cudaMemcpyAsync(out, tmp, n * sizeof(float), cudaMemcpyDeviceToHost, e->stream);
  if (err == cudaSuccess) err = cudaStreamSynchronize(e->stream);
  cudaFree(tmp);
  if (err != cudaSuccess) return fail("eb200_debug_read copy failed: %s", cudaGetErrorString(err));
  return 0;
}

// ------------------------------------------------------------------------------------------------------------
// stats / profiling
// ------------------------------------------------------------------------------------------------------------
static void drain_prof(eb200_engine* e) {
  if (e->prof.empty()) return;
  cudaStreamSynchronize(e->stream);
  for (auto& r : e->prof) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, r.a, r.b) == cudaSuccess) {
      if (r.cat == 0) {
        e->stats.gemm_ms += ms;
        e->stats.gemm_bytes += r.bytes;
        e->stats.gemm_launches++;
        if (r.verify) {
          e->stats.verify_gemm_ms += ms;
          e->stats.verify_gemm_bytes += r.bytes;
        }
      } else if (r.cat == 1) {
        e->stats.attn_ms += ms;
      } else {
        e->stats.other_ms += ms;
      }
    }
    e->ev_pool.push_back(r.a);
    e->ev_pool.push_back(r.b);
  }
  e->prof.clear();
}
extern "C" void* eb200_get_stream(eb200_engine* e) { return e ? reinterpret_cast<void*>(e->stream) : nullptr; }
extern "C" int eb200_set_profiling(eb200_engine* e, int32_t on) {
  if (!e) return fail("null engine");
  drain_prof(e);
  e->profiling = on != 0;
  return 0;
}
extern "C" int eb200_get_stats(eb200_engine* e, eb200_stats* out) {
  if (!e || !out) return fail("null argument");
  drain_prof(e);
  CK(cudaSetDevice(e->c.device));
  CK(cudaStreamSynchronize(e->stream));
  unsigned long long tm[4] = {0, 0, 0, 0};
  CK(cudaMemcpy(tm, e->chain_timing, sizeof(tm), cudaMemcpyDeviceToHost));
  e->stats.chain_ms = static_cast<double>(tm[0]) * 1e-6;
  e->stats.chain_launches = tm[1];
  *out = e->stats;
  return 0;
}
extern "C" int eb200_reset_stats(eb200_engine* e) {
  if (!e) return fail("null engine");
  drain_prof(e);
  CK(cudaSetDevice(e->c.device));
  CK(cudaStreamSynchronize(e->stream));
  CK(cudaMemset(e->chain_timing, 0, 4 * sizeof(unsigned long long)));
  memset(&e->stats, 0, sizeof(e->stats));
  return 0;
}



// ------------------------------------------------------------------------------------------------------------
// per-kernel entry points (parity tests).  Scratch is allocated per call: these are test paths, not hot paths.
// ------------------------------------------------------------------------------------------------------------
struct Scratch {
  std::vector<void*> ptrs;
  ~Scratch() {
    for (void* p : ptrs) cudaFree(p);
  }
  template <typename T> T* get(size_t n, bool zero = true) {
    void* p = nullptr;
    if (cudaMalloc(&p, std::max<size_t>(16, n * sizeof(T))) != cudaSuccess) return nullptr;
    ptrs.push_back(p);
    if (zero) cudaMemset(p, 0, std::max<size_t>(16, n * sizeof(T)));
    return reinterpret_cast<T*>(p);
  }
};

// Activation rows a test entry point launches for M rows: 16 or 64 like the cycle, or 256 like the prompt prefill (X is then a
// [256, K] buffer).  Above 64 rows only what target_prefill runs is accepted -- the wgmma kernel with the residual, interleaved
// SwiGLU or QKV + RoPE epilogue -- and anything else is refused before an allocation or a launch.
static int entry_mpad(const char* who, int M, int epilogue, bool simt, int* mpad) {
  if (M < 1 || M > 256) return fail("%s: M = %d is outside [1, 256]", who, M);
  if (M <= 64) {
    *mpad = M <= 16 ? 16 : 64;
    return 0;
  }
  if (simt) return fail("%s: the SIMT kernel runs at most 64 rows (M = %d)", who, M);
  if (epilogue != EPI_RESIDUAL && epilogue != EPI_SWIGLU_IL && epilogue != EPI_QKV_ROPE)
    return fail("%s: epilogue %d is not run at 256 rows (M = %d): only residual, interleaved SwiGLU and QKV + RoPE are", who, epilogue, M);
  *mpad = 256;
  return 0;
}

extern "C" int eb200_k_gemm(int32_t dtype, int32_t simt, int32_t epilogue, const void* W, const void* W2, const void* X, void* out,
                            const void* res, const void* bias, int32_t M, int32_t N, int32_t K, int32_t splitk, void* stream) {
  if (epilogue < EPI_STORE || (epilogue > EPI_SWIGLU && epilogue != EPI_SWIGLU_IL)) return fail("eb200_k_gemm: bad arguments");
  int mpad = 0;
  TRY(entry_mpad("eb200_k_gemm", M, epilogue, simt == 1, &mpad));
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  Scratch sc;
  const int n_out = N;  // EPI_SWIGLU_IL: W is the [2N, K] interleaved gate/up matrix, out is [M, N]
  if (epilogue == EPI_SWIGLU_IL) {
    if (N % 64) return fail("eb200_k_gemm: interleaved SwiGLU needs N % 64 == 0");
    N *= 2;
  }
  const int tiles = (N + 127) / 128;
  float* ws = sc.get<float>(static_cast<size_t>(std::max(1, splitk)) * 2 * mpad * tiles * 128, false);
  int* counters = sc.get<int>(tiles);
  if (!ws || !counters) return fail("eb200_k_gemm: scratch allocation failed");
  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.N = N;
  p.K = K;
  p.m_rows = M;
  p.m_idx = -1;
  p.splitk = std::max(1, splitk);
  p.ws = ws;
  p.counters = counters;
  p.out = out;
  p.ld_out = n_out;
  p.res = res;
  p.ld_res = n_out;
  p.bias = bias;
  if (simt == 1) {
    CKL(launch_gemm_simt(dtype, mpad, epilogue, W, W2, X, K, p, s));
  } else {
    CUtensorMap tw, tw2, tx;
    TRY(make_tmap(&tw, dtype, W, N, K, 128));
    if (W2) TRY(make_tmap(&tw2, dtype, W2, N, K, 128));
    TRY(make_tmap(&tx, dtype, X, std::max(64, mpad), K, mpad));
    if (p.splitk > 8) p.splitk = 8;
    CKL(launch_gemm(dtype, mpad, epilogue, &tw, W2 ? &tw2 : nullptr, &tx, p, s));
  }
  CK(cudaStreamSynchronize(s));
  return 0;
}

extern "C" int eb200_k_prefetch(int32_t dtype, int32_t kernel, int32_t epilogue, const void* W, const void* X, void* out, const void* res,
                                int32_t M, int32_t N, int32_t K, int32_t splitk, float eps, const void* P, int32_t PN, int32_t PK,
                                int32_t p_splitk, int32_t j0, int32_t j1, void* stream) {
  if (M < 1 || M > 64 || N < 1 || !P || PN < 1 || PK < 1 || p_splitk < 1 || p_splitk > 8 || kernel < 0 || kernel > 1 ||
      (kernel == 0 && (K < 1 || splitk < 1 || splitk > 8 || (epilogue != EPI_STORE && epilogue != EPI_RESIDUAL))))
    return fail("eb200_k_prefetch: bad arguments");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  L2Prefetch pf;
  memset(&pf, 0, sizeof(pf));
  TRY(make_tmap(&pf.tm, dtype, P, PN, PK, 128));
  pf.n_tiles = (PN + 127) / 128;
  pf.splitk = p_splitk;
  pf.num_kb = (PK + 63) / 64;
  pf.j0 = j0;
  pf.j1 = j1;
  if (kernel == 1) {
    CKL(launch_rmsnorm(dtype, X, N, nullptr, nullptr, W, out, N, 0, N, eps, M, s, &pf));
  } else {
    const int mpad = M <= 16 ? 16 : 64;
    GemmParams p;
    memset(&p, 0, sizeof(p));
    p.N = N;
    p.K = K;
    p.m_rows = M;
    p.m_idx = -1;
    p.splitk = splitk;
    p.out = out;
    p.ld_out = N;
    p.res = res;
    p.ld_res = N;
    CUtensorMap tw, tx;
    TRY(make_tmap(&tw, dtype, W, N, K, 128));
    TRY(make_tmap(&tx, dtype, X, 64, K, mpad));
    CKL(launch_gemm(dtype, mpad, epilogue, &tw, nullptr, &tx, p, s, &pf));
  }
  CK(cudaStreamSynchronize(s));
  return 0;
}

extern "C" int eb200_k_gemm_w8(int32_t dtype, int32_t epilogue, const void* Wq, const void* scb, const void* X, void* out, const void* res,
                               const void* bias, int32_t M, int32_t N, int32_t K, int32_t splitk, void* stream) {
  if ((epilogue != EPI_STORE && epilogue != EPI_RESIDUAL && epilogue != EPI_SWIGLU_IL) || !Wq || !scb || splitk < 1 || splitk > 8)
    return fail("eb200_k_gemm_w8: bad arguments");
  int mpad = 0;
  TRY(entry_mpad("eb200_k_gemm_w8", M, epilogue, false, &mpad));
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int n_out = N;  // EPI_SWIGLU_IL: Wq is the [2N, K] interleaved gate/up matrix, out is [M, N]
  if (epilogue == EPI_SWIGLU_IL) {
    if (N % 64) return fail("eb200_k_gemm_w8: interleaved SwiGLU needs N % 64 == 0");
    N *= 2;
  }
  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.N = N;
  p.K = K;
  p.m_rows = M;
  p.m_idx = -1;
  p.splitk = splitk;
  p.out = out;
  p.ld_out = n_out;
  p.res = res;
  p.ld_res = n_out;
  p.bias = bias;
  p.w_scale = reinterpret_cast<const float*>(scb);
  CUtensorMap tw, tx;
  TRY(make_tmap_w8(&tw, Wq, N, K));
  TRY(make_tmap(&tx, dtype, X, std::max(64, mpad), K, mpad));
  CKL(launch_gemm_w8(dtype, mpad, epilogue, &tw, &tx, p, s));
  CK(cudaStreamSynchronize(s));
  return 0;
}

extern "C" int eb200_k_gemm_w4(int32_t dtype, int32_t quant_type, int32_t epilogue, const void* Wq, const void* absmax, const void* X, void* out,
                               const void* res, const void* bias, int32_t M, int32_t N, int32_t K, int32_t splitk, void* stream) {
  if ((epilogue != EPI_STORE && epilogue != EPI_RESIDUAL && epilogue != EPI_SWIGLU_IL) || !Wq || !absmax || splitk < 1 || splitk > 8 ||
      N < 1 || K < 64 || K % 64 || (quant_type != W4_NF4 && quant_type != W4_FP4))
    return fail("eb200_k_gemm_w4: bad arguments");
  int mpad = 0;
  TRY(entry_mpad("eb200_k_gemm_w4", M, epilogue, false, &mpad));
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int n_out = N;  // EPI_SWIGLU_IL: Wq is the [2N, K/2] interleaved gate/up matrix, out is [M, N]
  if (epilogue == EPI_SWIGLU_IL) {
    if (N % 64) return fail("eb200_k_gemm_w4: interleaved SwiGLU needs N % 64 == 0");
    N *= 2;
  }
  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.N = N;
  p.K = K;
  p.m_rows = M;
  p.m_idx = -1;
  p.splitk = splitk;
  p.out = out;
  p.ld_out = n_out;
  p.res = res;
  p.ld_res = n_out;
  p.bias = bias;
  p.w4_quant = quant_type;
  const int n_pad = (N + 127) / 128 * 128;
  const size_t tile_bytes = static_cast<size_t>(n_pad) * K / 2, abs_bytes = static_cast<size_t>(n_pad) * (K / 64) * 4;
  void* buf = nullptr;
  CK(cudaMalloc(&buf, tile_bytes + abs_bytes));
  uint8_t* tiles = static_cast<uint8_t*>(buf);
  float* am = reinterpret_cast<float*>(tiles + tile_bytes);
  int rc = 0;
  CUtensorMap tw, ta, tx;
  if (cudaMemsetAsync(buf, 0, tile_bytes + abs_bytes, s) != cudaSuccess ||
      launch_w4_repack(static_cast<const uint8_t*>(Wq), static_cast<const float*>(absmax), N, K, 0, -1, tiles, am, n_pad, s) != 0)
    rc = fail("eb200_k_gemm_w4: repack failed");
  if (!rc) rc = make_tmap_w4(&tw, &ta, tiles, am, n_pad, K);
  if (!rc) rc = make_tmap(&tx, dtype, X, std::max(64, mpad), K, mpad);
  if (!rc) {
    const int r = launch_gemm_w4(dtype, mpad, epilogue, &tw, &ta, &tx, p, s);
    if (r != 0) rc = fail("eb200_k_gemm_w4: launch failed (%d)", r);
  }
  if (cudaStreamSynchronize(s) != cudaSuccess && !rc) rc = fail("eb200_k_gemm_w4: %s", cudaGetErrorString(cudaGetLastError()));
  cudaFree(buf);
  return rc;
}

extern "C" int eb200_k_gemm_fp8(int32_t dtype, int32_t epilogue, const void* Wq, const void* scale_inv, const void* X, void* out,
                                const void* res, const void* bias, int32_t M, int32_t N, int32_t K, int32_t splitk, void* stream) {
  if ((epilogue != EPI_STORE && epilogue != EPI_RESIDUAL && epilogue != EPI_SWIGLU_IL) || !Wq || !scale_inv || splitk < 1 || splitk > 8 ||
      N < 1 || K < 128 || K % 128)
    return fail("eb200_k_gemm_fp8: bad arguments");
  int mpad = 0;
  TRY(entry_mpad("eb200_k_gemm_fp8", M, epilogue, false, &mpad));
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int n_out = N;  // EPI_SWIGLU_IL: Wq is the [2N, K] interleaved gate/up matrix, out is [M, N]
  if (epilogue == EPI_SWIGLU_IL) N *= 2;
  if (N % 128) return fail("eb200_k_gemm_fp8: the weight's rows (%d) must be a multiple of 128", N);
  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.N = N;
  p.K = K;
  p.m_rows = M;
  p.m_idx = -1;
  p.splitk = splitk;
  p.out = out;
  p.ld_out = n_out;
  p.res = res;
  p.ld_res = n_out;
  p.bias = bias;
  const size_t w_bytes = static_cast<size_t>(N) * K, s_bytes = static_cast<size_t>(N / 128) * (K / 128) * 16;
  void* buf = nullptr;
  CK(cudaMalloc(&buf, w_bytes + s_bytes));
  uint8_t* q = static_cast<uint8_t*>(buf);
  float* sc = reinterpret_cast<float*>(q + w_bytes);
  int rc = 0;
  CUtensorMap tw, ts, tx;
  if (cudaMemsetAsync(sc, 0, s_bytes, s) != cudaSuccess ||
      launch_fp8_repack(static_cast<const uint8_t*>(Wq), static_cast<const float*>(scale_inv), N, K, 0, -1, q, sc, N, s) != 0)
    rc = fail("eb200_k_gemm_fp8: repack failed");
  if (!rc) rc = make_tmap_fp8(&tw, &ts, q, sc, N, K);
  if (!rc) rc = make_tmap(&tx, dtype, X, std::max(64, mpad), K, mpad);
  if (!rc) {
    const int r = launch_gemm_fp8(dtype, mpad, epilogue, &tw, &ts, &tx, p, s);
    if (r != 0) rc = fail("eb200_k_gemm_fp8: launch failed (%d)", r);
  }
  if (cudaStreamSynchronize(s) != cudaSuccess && !rc) rc = fail("eb200_k_gemm_fp8: %s", cudaGetErrorString(cudaGetLastError()));
  cudaFree(buf);
  return rc;
}

// A single GEMM through the lm_head launch (mega.cu).  mode 1: direct store, out = T(X . W^T [+ bias]); mode 2: fused arg-max ->
// out_idx[M] (int32).  `repeat` launches back to back (exercises the self-resetting counters).
extern "C" int eb200_k_chain_gemm(int32_t dtype, int32_t mode, const void* W, const void* X, void* out, const void* bias, int32_t* out_idx,
                                  int32_t M, int32_t N, int32_t K, int32_t repeat, void* stream) {
  if (M < 1 || M > 64 || mode < 1 || mode > 2 || repeat < 1) return fail("eb200_k_chain_gemm: bad arguments");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int mpad = M <= 16 ? 16 : 64;
  if (!chain_phase_ok(N, K)) return fail("eb200_k_chain_gemm: shape not supported by the chain kernel");
  Scratch sc;
  int* sync = sc.get<int>(2);
  const int tiles = (N + 127) / 128;
  float* tv = sc.get<float>(static_cast<size_t>(tiles) * 64);
  int* ti = sc.get<int>(static_cast<size_t>(tiles) * 64);
  if (!sync || !tv || !ti) return fail("scratch allocation failed");
  ChainArgs a;
  ChainMaps m;
  memset(&a, 0, sizeof(a));
  memset(&m, 0, sizeof(m));
  a.m_rows = M;
  a.m_idx = -1;
  a.sync = sync;
  ChainPhase& ph = a.ph;
  ph.N = N; ph.K = K; ph.fin = mode == 1 ? FIN_STORE_DIRECT : FIN_ARGMAX;
  ph.out = out; ph.ld_out = N; ph.bias = bias;
  ph.tile_val = tv; ph.tile_idx = ti; ph.out_idx = out_idx;
  TRY(make_tmap(&m.w, dtype, W, N, K, 128));
  TRY(make_tmap(&m.x, dtype, X, 64, K, mpad));
  for (int r = 0; r < repeat; ++r) CKL(launch_gemm_chain(dtype, mpad, m, a, s));
  CK(cudaStreamSynchronize(s));
  return 0;
}

extern "C" int eb200_k_gemm_bench(int32_t dtype, int32_t epilogue, int32_t M, int32_t N, int32_t K, int32_t splitk, int32_t n_weights,
                                  int32_t iters, int32_t use_graph, double* us_per_launch) {
  if (M < 1 || M > 64 || epilogue < EPI_STORE || (epilogue > EPI_SWIGLU && epilogue != EPI_SWIGLU_IL) || n_weights < 1 || iters < 1)
    return fail("bad arguments");
  const int mpad = M <= 16 ? 16 : 64;
  const int n_out = N;
  if (epilogue == EPI_SWIGLU_IL) N *= 2;  // interleaved gate/up rows
  Scratch sc;
  std::vector<CUtensorMap> tw(n_weights), tw2(n_weights);
  for (int i = 0; i < n_weights; ++i) {
    void* w = sc.get<uint16_t>(static_cast<size_t>(N) * K, true);
    if (!w) return fail("weight allocation failed");
    TRY(make_tmap(&tw[i], dtype, w, N, K, 128));
    if (epilogue == EPI_SWIGLU) {
      void* w2 = sc.get<uint16_t>(static_cast<size_t>(N) * K, true);
      if (!w2) return fail("weight allocation failed");
      TRY(make_tmap(&tw2[i], dtype, w2, N, K, 128));
    }
  }
  void* X = sc.get<uint16_t>(static_cast<size_t>(64) * K, true);
  void* out = sc.get<uint16_t>(static_cast<size_t>(64) * N, true);
  if (!X || !out) return fail("allocation failed");
  (void)n_out;
  CUtensorMap tx;
  TRY(make_tmap(&tx, dtype, X, 64, K, mpad));
  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.N = N;
  p.K = K;
  p.m_rows = M;
  p.m_idx = -1;
  p.splitk = std::max(1, splitk);
  p.out = out;
  p.ld_out = N;
  p.res = out;
  p.ld_res = N;
  cudaStream_t s;
  CK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
  auto run_all = [&]() -> int {
    for (int i = 0; i < iters; ++i) {
      const int wi = i % n_weights;
      CKL(launch_gemm(dtype, mpad, epilogue, &tw[wi], epilogue == EPI_SWIGLU ? &tw2[wi] : nullptr, &tx, p, s));
    }
    return 0;
  };
  TRY(run_all());  // warm-up (also sets function attributes outside any capture)
  CK(cudaStreamSynchronize(s));
  cudaGraphExec_t exec = nullptr;
  cudaGraph_t graph = nullptr;
  if (use_graph) {
    CK(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
    const int rc = run_all();
    cudaError_t ce = cudaStreamEndCapture(s, &graph);
    if (rc != 0) return rc;
    if (ce != cudaSuccess) return fail("capture failed: %s", cudaGetErrorString(ce));
    CK(cudaGraphInstantiate(&exec, graph, 0));
    CK(cudaGraphLaunch(exec, s));
    CK(cudaStreamSynchronize(s));
  }
  cudaEvent_t a, b;
  CK(cudaEventCreate(&a));
  CK(cudaEventCreate(&b));
  CK(cudaEventRecord(a, s));
  if (use_graph) CK(cudaGraphLaunch(exec, s));
  else TRY(run_all());
  CK(cudaEventRecord(b, s));
  CK(cudaStreamSynchronize(s));
  float ms = 0.f;
  CK(cudaEventElapsedTime(&ms, a, b));
  if (us_per_launch) *us_per_launch = 1000.0 * ms / iters;
  cudaEventDestroy(a);
  cudaEventDestroy(b);
  if (exec) cudaGraphExecDestroy(exec);
  if (graph) cudaGraphDestroy(graph);
  cudaStreamDestroy(s);
  return 0;
}

extern "C" int eb200_k_qkv_rope(int32_t dtype, int32_t simt, const void* Wqkv, const void* X, void* q_out, void* k_cache, void* v_cache,
                                const void* cosp, const void* sinp, const int32_t* pos, int32_t M, int32_t n_heads, int32_t n_kv_heads,
                                int32_t K, int64_t kv_cap, int32_t kv_base, int32_t splitk, void* stream) {
  int mpad = 0;
  TRY(entry_mpad("eb200_k_qkv_rope", M, EPI_QKV_ROPE, simt == 1, &mpad));
  if (kv_base < 0 || kv_base + M > kv_cap) return fail("eb200_k_qkv_rope: cache rows [%d, %d) outside [0, %lld)", kv_base, kv_base + M, (long long)kv_cap);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int N = (n_heads + 2 * n_kv_heads) * 128;
  Scratch sc;
  const int tiles = N / 128;
  float* ws = sc.get<float>(static_cast<size_t>(std::max(1, splitk)) * mpad * tiles * 128, false);
  int* counters = sc.get<int>(tiles);
  if (!ws || !counters) return fail("scratch allocation failed");
  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.N = N;
  p.K = K;
  p.m_rows = M;
  p.m_idx = -1;
  p.splitk = std::max(1, splitk);
  p.ws = ws;
  p.counters = counters;
  p.q_out = q_out;
  p.k_cache = k_cache;
  p.v_cache = v_cache;
  p.kv_cap = kv_cap;
  p.n_q_heads = n_heads;
  p.n_kv_heads = n_kv_heads;
  p.rope_cos = cosp;
  p.rope_sin = sinp;
  // pos[m]: the cycle's form (tree positions); no pos: the prefill's (chunk_ctx), row m at position kv_base + m
  p.pos_base = DynInt{-1, pos ? 0 : kv_base};
  p.pos_arr = pos;
  p.pos_mstride = pos ? 0 : 1;
  p.kv_base = DynInt{-1, kv_base};
  if (simt == 1) {
    CKL(launch_gemm_simt(dtype, mpad, EPI_QKV_ROPE, Wqkv, nullptr, X, K, p, s));
  } else {
    CUtensorMap tw, tx;
    TRY(make_tmap(&tw, dtype, Wqkv, N, K, 128));
    TRY(make_tmap(&tx, dtype, X, std::max(64, mpad), K, mpad));
    if (p.splitk > 8) p.splitk = 8;
    CKL(launch_gemm(dtype, mpad, EPI_QKV_ROPE, &tw, nullptr, &tx, p, s));
  }
  CK(cudaStreamSynchronize(s));
  return 0;
}

extern "C" int eb200_k_rmsnorm(int32_t dtype, const void* x, const void* w, void* y, int32_t rows, int32_t H, float eps, void* stream) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  CKL(launch_rmsnorm(dtype, x, H, nullptr, nullptr, w, y, H, 0, H, eps, rows, s));
  CK(cudaStreamSynchronize(s));
  return 0;
}

extern "C" int eb200_k_attention(int32_t dtype, const void* q, const void* k_cache, const void* v_cache, void* out, int32_t rows,
                                 int32_t n_heads, int32_t n_kv_heads, int64_t kv_cap, int32_t n_ctx, int32_t n_tree,
                                 const uint64_t* mask, void* stream) {
  return eb200_k_attention_ex(dtype, q, k_cache, v_cache, out, rows, n_heads, n_kv_heads, kv_cap, n_ctx + n_tree, nullptr, -1, -1,
                              n_ctx, n_tree, mask, 0, 0, stream);
}

extern "C" int eb200_k_attention_plan(int32_t max_kv, int32_t n_heads, int32_t n_kv_heads, int32_t hpc_cap, int32_t kvs_cap,
                                      int32_t* hpc, int32_t* kvs, int32_t* kv_stride, int64_t* smem) {
  AttnGeometry g;
  if (attention_geometry(max_kv, n_heads, n_kv_heads, hpc_cap, kvs_cap, &g))
    return fail("attention: no launch geometry for max_kv %d, %d / %d heads, caps hpc %d kvs %d (max_kv <= %d under the default "
                "caps; caps must be 0, 1, 2 or 4)", max_kv, n_heads, n_kv_heads, hpc_cap, kvs_cap, attention_max_kv());
  if (hpc) *hpc = g.hpc;
  if (kvs) *kvs = g.kvs;
  if (kv_stride) *kv_stride = g.kv_stride;
  if (smem) *smem = static_cast<int64_t>(g.smem);
  return 0;
}

extern "C" int eb200_k_attention_ex(int32_t dtype, const void* q, const void* k_cache, const void* v_cache, void* out, int32_t rows,
                                    int32_t n_heads, int32_t n_kv_heads, int64_t kv_cap, int32_t max_kv, const int32_t* st,
                                    int32_t rows_idx, int32_t n_ctx_idx, int32_t n_ctx_add, int32_t n_tree, const uint64_t* mask,
                                    int32_t hpc_cap, int32_t kvs_cap, void* stream) {
  TRY(eb200_k_attention_plan(max_kv, n_heads, n_kv_heads, hpc_cap, kvs_cap, nullptr, nullptr, nullptr, nullptr));
  if (rows < 1 || n_tree < 0 || n_tree > 128) return fail("eb200_k_attention_ex: rows must be >= 1 and n_tree in [0, 128]");
  if ((rows_idx >= 0 || n_ctx_idx >= 0) && !st) return fail("eb200_k_attention_ex: a state index needs the state pointer");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  AttnParams a;
  memset(&a, 0, sizeof(a));
  a.trace = nullptr;
  a.q = q;
  a.k_cache = k_cache;
  a.v_cache = v_cache;
  a.out = out;
  a.kv_cap = kv_cap;
  a.n_heads = n_heads;
  a.n_kv_heads = n_kv_heads;
  a.rows = rows;
  a.rows_idx = rows_idx;
  a.st = st;
  a.n_ctx = DynInt{n_ctx_idx, n_ctx_add};
  a.n_tree = n_tree;
  a.mask = mask;
  a.max_kv = max_kv;
  a.hpc_cap = hpc_cap;
  a.kvs_cap = kvs_cap;
  CUtensorMap mk, mv;
  TRY(make_tmap(&mk, dtype, k_cache, static_cast<uint64_t>(n_kv_heads) * kv_cap, 128, 64));
  TRY(make_tmap(&mv, dtype, v_cache, static_cast<uint64_t>(n_kv_heads) * kv_cap, 128, 64));
  a.tmK = &mk;
  a.tmV = &mv;
  CKL(launch_attention(dtype, a, s));
  CK(cudaStreamSynchronize(s));
  return 0;
}

extern "C" int eb200_k_argmax(int32_t dtype, const void* logits, int32_t rows, int32_t V, int32_t* out, void* stream) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  CKL(launch_argmax(dtype, logits, V, V, rows, out, s));
  CK(cudaStreamSynchronize(s));
  return 0;
}

extern "C" int eb200_k_logsoftmax_topk(int32_t dtype, const void* logits, int32_t rows, int32_t V, int32_t k, float* topk_p,
                                       int32_t* topk_i, void* stream) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  CKL(launch_logsoftmax_topk(dtype, logits, V, V, rows, nullptr, -1, k, 0, topk_p, topk_i, s));
  CK(cudaStreamSynchronize(s));
  return 0;
}

extern "C" int eb200_k_topk_raw(int32_t dtype, const void* logits, int32_t rows, int32_t V, int32_t k, float* topk_v,
                                int32_t* topk_i, void* stream) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  CKL(launch_logsoftmax_topk(dtype, logits, V, V, rows, nullptr, -1, k, 1, topk_v, topk_i, s));
  CK(cudaStreamSynchronize(s));
  return 0;
}

// generate_candidates (utils.py:284-303) on device: table = the draft's [rows][k] top-k table (host, draft-vocab ids),
// d2t optional (host, [d2t_len]); out tree_candidates [T] (host)
extern "C" int eb200_k_generate_candidates(const int32_t* table, int32_t rows, int32_t k, const int64_t* d2t, int32_t d2t_len,
                                           const int32_t* tree_indices, int32_t T, int32_t sample_token, int64_t* tree_candidates) {
  if (rows < 1 || rows > 64 || k < 1 || k > 32 || T < 1 || T > 128 || !table || !tree_indices || !tree_candidates)
    return fail("eb200_k_generate_candidates: bad arguments");
  for (int i = 1; i < T; ++i)
    if (tree_indices[i] < 1 || tree_indices[i] > rows * k) return fail("eb200_k_generate_candidates: tree index outside the table");
  Scratch sc;
  TreeBuffers tb;
  memset(&tb, 0, sizeof(tb));
  tb.draft_tokens = sc.get<int>(128);
  tb.front_ids = sc.get<int>(64);
  tb.front_src = sc.get<int>(64);
  tb.front_mask = sc.get<uint64_t>(128);
  int* st = sc.get<int>(S_COUNT);
  int* d_table = sc.get<int>(rows * k);
  int* d_ss = sc.get<int>(rows * k);
  int* d_ti = sc.get<int>(128);
  int64_t* d_d2t = d2t ? sc.get<int64_t>(d2t_len) : nullptr;
  if (!d_ti || (d2t && !d_d2t)) return fail("scratch allocation failed");
  CK(cudaMemcpy(d_table, table, rows * k * sizeof(int), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(d_ti, tree_indices, T * sizeof(int), cudaMemcpyHostToDevice));
  if (d2t) CK(cudaMemcpy(d_d2t, d2t, d2t_len * sizeof(int64_t), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(st + S_BONUS, &sample_token, sizeof(int), cudaMemcpyHostToDevice));
  StaticLevelArgs a;
  memset(&a, 0, sizeof(a));
  a.topk_i = d_table;
  a.d2t = d_d2t;
  a.k = k;
  a.rows_prev = rows;
  a.ss_row0 = 0;
  a.ss_tokens = d_ss;
  a.final_T = T;
  a.tree_indices = d_ti;
  CKL(launch_static_level(a, tb, st, 0));
  CK(cudaDeviceSynchronize());
  std::vector<int> tok(T);
  CK(cudaMemcpy(tok.data(), tb.draft_tokens, T * sizeof(int), cudaMemcpyDeviceToHost));
  for (int i = 0; i < T; ++i) tree_candidates[i] = tok[i];
  return 0;
}

extern "C" int eb200_k_tree_finalize(int32_t dtype, const float* scores, const int32_t* tokens, const int32_t* parents, int32_t k,
                                     int32_t depth, int32_t total_token, int32_t sample_token, int32_t sort_rows,
                                     int64_t* draft_tokens, float* tree_mask, int64_t* tree_position_ids, int64_t* retrieve_indices,
                                     int32_t* n_leaf, int32_t* max_depth) {
  if (total_token < 2 || total_token > 128 || depth + 2 > 16) return fail("eb200_k_tree_finalize: bad arguments");
  const int pool = k + depth * k * k;
  const int T = total_token, D = depth + 2;
  Scratch sc;
  TreeBuffers tb;
  memset(&tb, 0, sizeof(tb));
  tb.scores = sc.get<float>(pool);
  tb.tokens = sc.get<int>(pool);
  tb.parents = sc.get<int>(1 + depth * k);
  tb.draft_tokens = sc.get<int>(128);
  tb.tree_mask = sc.get<uint64_t>(256);
  tb.tree_pos = sc.get<int>(128);
  tb.retrieve = sc.get<int>(128 * 16);
  tb.parent_node = sc.get<int>(128);
  int* st = sc.get<int>(S_COUNT);
  if (!st) return fail("scratch allocation failed");
  CK(cudaMemcpy(tb.scores, scores, pool * sizeof(float), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(tb.tokens, tokens, pool * sizeof(int), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(tb.parents, parents, (1 + depth * k) * sizeof(int), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(st + S_BONUS, &sample_token, sizeof(int), cudaMemcpyHostToDevice));
  CKL(launch_tree_finalize(dtype, k, depth, T - 1, sort_rows, tb, st, 0));
  CK(cudaDeviceSynchronize());
  std::vector<int> tok(128), pos(128), ret(128 * 16), hst(S_COUNT);
  std::vector<uint64_t> mask(256);
  CK(cudaMemcpy(tok.data(), tb.draft_tokens, 128 * 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(pos.data(), tb.tree_pos, 128 * 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(ret.data(), tb.retrieve, 128 * 16 * 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(mask.data(), tb.tree_mask, 256 * 8, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(hst.data(), st, S_COUNT * 4, cudaMemcpyDeviceToHost));
  const int nl = hst[S_NLEAF], md = hst[S_MAXDEPTH];
  for (int i = 0; i < T; ++i) {
    if (draft_tokens) draft_tokens[i] = tok[i];
    if (tree_position_ids) tree_position_ids[i] = pos[i];
    if (tree_mask)
      for (int j = 0; j < T; ++j) tree_mask[i * T + j] = ((j < 64 ? (mask[2 * i] >> j) : (mask[2 * i + 1] >> (j - 64))) & 1ull) ? 1.f : 0.f;
  }
  if (retrieve_indices)
    for (int r = 0; r < nl; ++r)
      for (int j = 0; j < md; ++j) retrieve_indices[r * md + j] = ret[r * D + j];
  if (n_leaf) *n_leaf = nl;
  if (max_depth) *max_depth = md;
  return 0;
}

// draft-tree growth on host-supplied per-level top-k tables: tree_seed then tree_expand for level 0..depth-1, the frontier
// copied out after the seed and after every level.  The tables do not depend on what the kernels produce, so a plain
// transcription of cnets.py:703-757 driven by the same tables must give the same integers and the same rounded scores.
extern "C" int eb200_k_tree_grow(int32_t dtype, const float* topk_p, const int32_t* topk_i, const int64_t* d2t, int32_t d2t_len,
                                 int32_t k, int32_t depth, int32_t last_row, float* scores, int32_t* tokens, int32_t* parents,
                                 int32_t* front_ids, int32_t* front_src, int32_t* front_cs, float* front_scores,
                                 uint64_t* front_mask) {
  if (dtype != EB200_BF16 && dtype != EB200_FP16) return fail("eb200_k_tree_grow: dtype must be bf16 or fp16");
  if (!topk_p || !topk_i) return fail("eb200_k_tree_grow: null top-k table");
  if (k < 1 || k > 32) return fail("eb200_k_tree_grow: top_k must be in [1, 32]");
  if (depth < 1 || depth + 2 > 16) return fail("eb200_k_tree_grow: depth must be in [1, 14]");
  if (depth * k > 128) return fail("eb200_k_tree_grow: depth * top_k must be <= 128 (draft tree columns)");
  if (last_row < 0) return fail("eb200_k_tree_grow: last_row must be >= 0");
  if (d2t && d2t_len < 1) return fail("eb200_k_tree_grow: empty d2t");
  const int kk = k * k, pool = k + depth * kk, rows = 1 + depth * k;
  for (int i = 0; i < rows * k; ++i) {
    if (topk_i[i] < 0 || (d2t && topk_i[i] >= d2t_len)) return fail("eb200_k_tree_grow: top-k index %d out of range at %d", topk_i[i], i);
  }
  Scratch sc;
  TreeBuffers tb;
  memset(&tb, 0, sizeof(tb));
  tb.scores = sc.get<float>(pool);
  tb.tokens = sc.get<int>(pool);
  tb.parents = sc.get<int>(rows);
  tb.front_scores = sc.get<float>(k);
  tb.front_ids = sc.get<int>(k);
  tb.front_src = sc.get<int>(k);
  tb.front_cs = sc.get<int>(k);
  tb.front_mask = sc.get<uint64_t>(2 * k);
  int* st = sc.get<int>(S_COUNT);
  float* d_p = sc.get<float>(rows * k);
  int* d_i = sc.get<int>(rows * k);
  int64_t* d_d2t = d2t ? sc.get<int64_t>(d2t_len) : nullptr;
  if (!d_i || (d2t && !d_d2t)) return fail("scratch allocation failed");
  CK(cudaMemcpy(d_p, topk_p, rows * k * sizeof(float), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(d_i, topk_i, rows * k * sizeof(int), cudaMemcpyHostToDevice));
  if (d2t) CK(cudaMemcpy(d_d2t, d2t, d2t_len * sizeof(int64_t), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(st + S_LASTROW, &last_row, sizeof(int), cudaMemcpyHostToDevice));
  auto snapshot = [&](int slot) -> int {
    CK(cudaDeviceSynchronize());
    if (front_ids) CK(cudaMemcpy(front_ids + slot * k, tb.front_ids, k * sizeof(int), cudaMemcpyDeviceToHost));
    if (front_src) CK(cudaMemcpy(front_src + slot * k, tb.front_src, k * sizeof(int), cudaMemcpyDeviceToHost));
    if (front_cs) CK(cudaMemcpy(front_cs + slot * k, tb.front_cs, k * sizeof(int), cudaMemcpyDeviceToHost));
    if (front_scores) CK(cudaMemcpy(front_scores + slot * k, tb.front_scores, k * sizeof(float), cudaMemcpyDeviceToHost));
    if (front_mask) CK(cudaMemcpy(front_mask + slot * 2 * k, tb.front_mask, 2 * k * sizeof(uint64_t), cudaMemcpyDeviceToHost));
    return 0;
  };
  CKL(launch_tree_seed(d_p, d_i, d_d2t, k, tb, st, 0));
  TRY(snapshot(0));
  for (int level = 0; level < depth; ++level) {
    CKL(launch_tree_expand(dtype, d_p + (1 + level * k) * k, d_i + (1 + level * k) * k, d_d2t, k, level, tb, 0));
    TRY(snapshot(level + 1));
  }
  if (scores) CK(cudaMemcpy(scores, tb.scores, pool * sizeof(float), cudaMemcpyDeviceToHost));
  if (tokens) CK(cudaMemcpy(tokens, tb.tokens, pool * sizeof(int), cudaMemcpyDeviceToHost));
  if (parents) CK(cudaMemcpy(parents, tb.parents, rows * sizeof(int), cudaMemcpyDeviceToHost));
  return 0;
}

extern "C" int eb200_k_greedy_accept(const int32_t* node_argmax, const int32_t* draft_tokens, const int32_t* retrieve, int32_t T,
                                     int32_t n_leaf, int32_t max_depth, int32_t* best, int32_t* accept_length, int32_t* bonus) {
  if (T < 1 || T > 128 || max_depth > 16 || n_leaf > 128) return fail("eb200_k_greedy_accept: bad arguments");
  const int depth = 14, D = 16;  // widest row layout
  Scratch sc;
  TreeBuffers tb;
  memset(&tb, 0, sizeof(tb));
  tb.draft_tokens = sc.get<int>(128);
  tb.retrieve = sc.get<int>(128 * 16);
  int* st = sc.get<int>(S_COUNT);
  int* am = sc.get<int>(128);
  int* acc = sc.get<int>(64);
  int* sel = sc.get<int>(64);
  if (!sel) return fail("scratch allocation failed");
  std::vector<int> ret(128 * 16, -1);
  for (int r = 0; r < n_leaf; ++r)
    for (int j = 0; j < max_depth; ++j) ret[r * D + j] = retrieve[r * max_depth + j];
  std::vector<int> hst(S_COUNT, 0);
  hst[S_NLEAF] = n_leaf;
  hst[S_MAXDEPTH] = max_depth;
  CK(cudaMemcpy(tb.draft_tokens, draft_tokens, T * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(tb.retrieve, ret.data(), 128 * 16 * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(st, hst.data(), S_COUNT * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(am, node_argmax, T * 4, cudaMemcpyHostToDevice));
  AcceptOut ao;
  ao.accepted_tokens = acc;
  ao.sel_nodes = sel;
  ao.host_visible = nullptr;
  CKL(launch_greedy_accept(am, tb, T, depth, ao, st, nullptr, 0, 0));
  CK(cudaDeviceSynchronize());
  CK(cudaMemcpy(hst.data(), st, S_COUNT * 4, cudaMemcpyDeviceToHost));
  if (best) *best = hst[S_BEST];
  if (accept_length) *accept_length = hst[S_ACC] - 1;
  if (bonus) *bonus = hst[S_BONUS];
  return 0;
}

// sampling posterior on a host-described tree (utils.py:375-415): logits is a DEVICE [T][V] model-dtype tensor.
extern "C" int eb200_k_sample_posterior(int32_t dtype, const void* logits, int32_t V, const int32_t* draft_tokens, const int32_t* retrieve,
                                        int32_t T, int32_t n_leaf, int32_t max_depth, float temperature, float top_p, int32_t top_k,
                                        const float* uniforms, int32_t n_uniforms, int32_t* best, int32_t* accept_length, int32_t* bonus,
                                        int32_t* uniforms_used) {
  if (T < 1 || T > 128 || max_depth > 16 || n_leaf > 128 || n_uniforms > 4096) return fail("eb200_k_sample_posterior: bad arguments");
  const int depth = 14, D = 16;
  Scratch sc;
  TreeBuffers tb;
  memset(&tb, 0, sizeof(tb));
  tb.draft_tokens = sc.get<int>(128);
  tb.retrieve = sc.get<int>(128 * 16);
  int* st = sc.get<int>(S_COUNT);
  int* acc = sc.get<int>(64);
  int* sel = sc.get<int>(64);
  int* rej = sc.get<int>(64);
  RowStats* stats = sc.get<RowStats>(128);
  float* un = sc.get<float>(4096);
  if (!un) return fail("scratch allocation failed");
  std::vector<int> ret(128 * 16, -1);
  for (int r = 0; r < n_leaf; ++r)
    for (int j = 0; j < max_depth; ++j) ret[r * D + j] = retrieve[r * max_depth + j];
  std::vector<int> hst(S_COUNT, 0);
  hst[S_NLEAF] = n_leaf;
  hst[S_MAXDEPTH] = max_depth;
  CK(cudaMemcpy(tb.draft_tokens, draft_tokens, T * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(tb.retrieve, ret.data(), 128 * 16 * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(st, hst.data(), S_COUNT * 4, cudaMemcpyHostToDevice));
  if (n_uniforms > 0) CK(cudaMemcpy(un, uniforms, n_uniforms * 4, cudaMemcpyHostToDevice));
  SampleParams sp;
  sp.temperature = temperature;
  sp.top_p = top_p;
  sp.top_k = top_k;
  sp.seed = 12345;
  sp.uniforms = n_uniforms > 0 ? un : nullptr;
  sp.n_uniforms = n_uniforms;
  AcceptOut ao;
  ao.accepted_tokens = acc;
  ao.sel_nodes = sel;
  ao.host_visible = nullptr;
  CKL(launch_row_softmax_stats(dtype, logits, V, V, T, sp, stats, 0));
  CKL(launch_sample_posterior(dtype, logits, V, V, stats, tb, depth, sp, rej, st, 0));
  CKL(launch_sample_commit(dtype, logits, V, V, stats, tb, depth, sp, rej, ao, st, nullptr, 0, 0, 0));
  CK(cudaDeviceSynchronize());
  CK(cudaMemcpy(hst.data(), st, S_COUNT * 4, cudaMemcpyDeviceToHost));
  if (best) *best = hst[S_BEST];
  if (accept_length) *accept_length = hst[S_ACC] - 1;
  if (bonus) *bonus = hst[S_BONUS];
  if (uniforms_used) *uniforms_used = hst[S_UCOUNT];
  return 0;
}

// softmax statistics of the warped rows (row_softmax_stats_kernel): logits is a DEVICE [rows][V] model-dtype tensor,
// stats (HOST) [rows][3] = max, sum, thr
extern "C" int eb200_k_sample_stats(int32_t dtype, const void* logits, int32_t rows, int32_t V, float temperature, float top_p,
                                    int32_t top_k, float* stats) {
  if (dtype != EB200_BF16 && dtype != EB200_FP16) return fail("eb200_k_sample_stats: dtype must be bf16 or fp16");
  if (!logits || !stats || rows < 1 || V < 1) return fail("eb200_k_sample_stats: bad arguments");
  Scratch sc;
  RowStats* d = sc.get<RowStats>(rows);
  if (!d) return fail("scratch allocation failed");
  SampleParams sp;
  memset(&sp, 0, sizeof(sp));
  sp.temperature = temperature;
  sp.top_p = top_p;
  sp.top_k = top_k;
  CKL(launch_row_softmax_stats(dtype, logits, V, V, rows, sp, d, 0));
  CK(cudaDeviceSynchronize());
  std::vector<RowStats> h(rows);
  CK(cudaMemcpy(h.data(), d, rows * sizeof(RowStats), cudaMemcpyDeviceToHost));
  for (int r = 0; r < rows; ++r) {
    stats[3 * r] = h[r].max;
    stats[3 * r + 1] = h[r].sum;
    stats[3 * r + 2] = h[r].thr;
  }
  return 0;
}

// one token drawn from logits row 0 exactly as sample_row0 draws the first token after prefill: the row's statistics, then
// the inverse CDF (sample_commit_kernel, first_token = 1) with `u` as its uniform
extern "C" int eb200_k_sample_token(int32_t dtype, const void* logits, int32_t V, float temperature, float top_p, int32_t top_k, float u,
                                    int32_t* token) {
  if (dtype != EB200_BF16 && dtype != EB200_FP16) return fail("eb200_k_sample_token: dtype must be bf16 or fp16");
  if (!logits || !token || V < 1) return fail("eb200_k_sample_token: bad arguments");
  Scratch sc;
  TreeBuffers tb;
  memset(&tb, 0, sizeof(tb));
  RowStats* stats = sc.get<RowStats>(1);
  int* st = sc.get<int>(S_COUNT);
  float* un = sc.get<float>(1);
  if (!un) return fail("scratch allocation failed");
  CK(cudaMemcpy(un, &u, sizeof(float), cudaMemcpyHostToDevice));
  SampleParams sp;
  memset(&sp, 0, sizeof(sp));
  sp.temperature = temperature;
  sp.top_p = top_p;
  sp.top_k = top_k;
  sp.uniforms = un;
  sp.n_uniforms = 1;
  AcceptOut ao;
  memset(&ao, 0, sizeof(ao));
  CKL(launch_row_softmax_stats(dtype, logits, V, V, 1, sp, stats, 0));
  CKL(launch_sample_commit(dtype, logits, V, V, stats, tb, 0, sp, nullptr, ao, st, nullptr, 0, 1, 0));
  CK(cudaDeviceSynchronize());
  CK(cudaMemcpy(token, st + S_BONUS, sizeof(int), cudaMemcpyDeviceToHost));
  return 0;
}
