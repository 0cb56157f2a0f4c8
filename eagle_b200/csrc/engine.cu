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

// ------------------------------------------------------------------------------------------------------------
// engine data
// ------------------------------------------------------------------------------------------------------------
struct Linear {
  void* w = nullptr;
  int N = 0, K = 0;
  CUtensorMap tm;
  uint64_t loaded_rows = 0;  // bookkeeping for fused / sharded loads
};
struct ActBuf {  // an activation buffer usable as the X operand of the GEMM (64 rows; 256 where the prompt prefill runs through it)
  void* p = nullptr;
  int cols = 0, rows = 64;
  CUtensorMap tm16, tm32, tm64, tm256;  // tm32: half of a 64-row X tile (TMA multicast between neighbouring n-tiles)
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
  float* sk_ws = nullptr;  // stream-K partial slots
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
  bool tp_fused = false;        // peers opened: row-parallel projections finish inside the chain launch
  long tp_inbox_off = 0, tp_flag_off = 0, tp_ready_off = 0, tp_am_off = 0;
  int* tp_epoch = nullptr;
  int* tp_ready_base = nullptr;
  // persistent GEMM chain (mega.cu)
  int* chain_sync = nullptr;    // [16] self-resetting phase counters
  unsigned long long* chain_timing = nullptr;  // [4] in-kernel %globaltimer accounting (ns sum, launches, scratch)
  unsigned long long* chain_trace = nullptr;   // EB200_CHAIN_TRACE=<file>: phase stamps of the verify pass' layer-5 chain launch
  double chain_bytes_cycle = 0;  // algorithmic bytes of the chain launches captured in the cycle graph
  double chain_bytes_pending = 0;
  float* tile_val = nullptr;    // [lm_head tiles][64] per-tile row maxima of the fused arg-max
  int* tile_idx = nullptr;
  bool chain_target = false;    // the target's layer segments run as chain launches
  bool chain_head = false;      // ... including the lm_head (fused arg-max / direct store)
  bool chain_draft = false;     // the draft head's layer tail + lm_head run as one chain launch per pass
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
static int alloc_linear(eb200_engine* e, Linear& l, int N, int K) {
  l.N = N;
  l.K = K;
  return dalloc(e, &l.w, static_cast<size_t>(N) * K * 2, false);
}
static int alloc_act(eb200_engine* e, ActBuf& a, int cols, int rows = 64) {
  a.cols = cols;
  a.rows = rows;
  TRY(dalloc(e, &a.p, static_cast<size_t>(rows) * cols * 2));
  TRY(make_tmap(&a.tm16, e->dtype, a.p, rows, cols, 16));
  TRY(make_tmap(&a.tm64, e->dtype, a.p, rows, cols, 64));
  TRY(make_tmap(&a.tm32, e->dtype, a.p, rows, cols, 32));
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
  if (c.total_token < 2 || c.total_token > 64) return fail("total_token must be in [2, 64]");
  if (c.top_k < 1 || c.top_k > 16) return fail("top_k must be in [1, 16]");
  if (c.depth < 1 || c.depth + 2 > 16) return fail("depth must be in [1, 14]");
  if (c.top_k * (c.depth) > 128) return fail("depth * top_k must be <= 128 (draft tree columns)");
  if (c.top_k + c.depth * c.top_k * c.top_k < c.total_token - 1) return fail("candidate pool smaller than total_token - 1");
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
    for (auto& l : e->tl) {
      TRY(alloc_linear(e, l.qkv, (e->nh_l + 2 * e->nkv_l) * 128, H));
      TRY(alloc_linear(e, l.o, H, e->nh_l * 128));
      TRY(alloc_linear(e, l.gu, 2 * e->I_l, H));
      TRY(alloc_linear(e, l.down, H, e->I_l));
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
      TRY(make_tmap(&e->xn.tm32, e->dtype, e->xn.p, 64, H, 32));
      TRY(dalloc(e, reinterpret_cast<void**>(&e->tp_epoch), 64));
      TRY(dalloc(e, reinterpret_cast<void**>(&e->tp_ready_base), 64));
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
    TRY(dalloc(e, reinterpret_cast<void**>(&e->sk_ws), streamk_ws_bytes(), false));
    TRY(dalloc(e, reinterpret_cast<void**>(&e->chain_sync), 16 * sizeof(int)));
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
    if (getenv("EB200_CHAIN_TRACE")) TRY(dalloc(e, reinterpret_cast<void**>(&e->chain_trace), 256 * 32 * sizeof(unsigned long long)));
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
  if (e->chain_trace) {
    std::vector<unsigned long long> h(256 * 32);
    if (cudaMemcpy(h.data(), e->chain_trace, h.size() * 8, cudaMemcpyDeviceToHost) == cudaSuccess) {
      if (FILE* f = fopen(getenv("EB200_CHAIN_TRACE"), "w")) {
        for (size_t c = 0; c < 256; ++c) {
          if (!h[c * 32]) continue;
          fprintf(f, "%zu", c);
          for (int j = 0; j < 32; ++j) fprintf(f, " %llu", h[c * 32 + j]);
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
// copy rows [r0, r0+nr) x cols [c0, c0+nc) of a row-major [R][C] 2-byte source into dst rows [dr0, ...) of pitch nc
static int copy_block(eb200_engine* e, void* dst, long dst_row0, const void* src, long C, long r0, long nr, long c0, long nc) {
  const char* s = reinterpret_cast<const char*>(src) + (r0 * C + c0) * 2;
  char* d = reinterpret_cast<char*>(dst) + dst_row0 * nc * 2;
  CK(cudaMemcpy2DAsync(d, nc * 2, s, C * 2, nc * 2, nr, cudaMemcpyDefault, e->stream));
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
static int copy_interleaved64(eb200_engine* e, void* dst, int half, const void* src, long C, const Shard& sh) {
  if (sh.nr % 64 || sh.c0 != 0 || sh.nc != C) return fail("gate/up shard must be whole rows in multiples of 64");
  const char* s = reinterpret_cast<const char*>(src) + sh.r0 * C * 2;
  char* d = reinterpret_cast<char*>(dst) + static_cast<size_t>(half) * 64 * C * 2;
  CK(cudaMemcpy2DAsync(d, static_cast<size_t>(128) * C * 2, s, static_cast<size_t>(64) * C * 2, static_cast<size_t>(64) * C * 2, sh.nr / 64,
                       cudaMemcpyDefault, e->stream));
  return 0;
}

static int load_layer_tensor(eb200_engine* e, Layer& l, const std::string& sub, const void* data, const int64_t* shape,
                             int nd, bool is_target, int Hin_qkv, int Hm, int nh_full, int nkv_full, int I_full) {
  const int tp = is_target ? e->c.tp_size : 1, rk = is_target ? e->c.tp_rank : 0;
  const int nh_l = nh_full / tp, nkv_l = nkv_full / tp;
  if (sub == "self_attn.q_proj.weight") {
    if (!shape_is(shape, nd, nh_full * 128, Hin_qkv)) return fail("q_proj shape mismatch");
    const Shard sh = shard_of(sub, nh_full * 128, Hin_qkv, rk, tp);
    TRY(copy_block(e, l.qkv.w, 0, data, Hin_qkv, sh.r0, sh.nr, sh.c0, sh.nc));
    l.qkv.loaded_rows |= 1;
  } else if (sub == "self_attn.k_proj.weight") {
    if (!shape_is(shape, nd, nkv_full * 128, Hin_qkv)) return fail("k_proj shape mismatch");
    const Shard sh = shard_of(sub, nkv_full * 128, Hin_qkv, rk, tp);
    TRY(copy_block(e, l.qkv.w, nh_l * 128, data, Hin_qkv, sh.r0, sh.nr, sh.c0, sh.nc));
    l.qkv.loaded_rows |= 2;
  } else if (sub == "self_attn.v_proj.weight") {
    if (!shape_is(shape, nd, nkv_full * 128, Hin_qkv)) return fail("v_proj shape mismatch");
    const Shard sh = shard_of(sub, nkv_full * 128, Hin_qkv, rk, tp);
    TRY(copy_block(e, l.qkv.w, (nh_l + nkv_l) * 128, data, Hin_qkv, sh.r0, sh.nr, sh.c0, sh.nc));
    l.qkv.loaded_rows |= 4;
  } else if (sub == "self_attn.o_proj.weight") {
    if (!shape_is(shape, nd, Hm, nh_full * 128)) return fail("o_proj shape mismatch");
    const Shard sh = shard_of(sub, Hm, nh_full * 128, rk, tp);
    TRY(copy_block(e, l.o.w, 0, data, nh_full * 128, sh.r0, sh.nr, sh.c0, sh.nc));
    l.o.loaded_rows = 1;
  } else if (sub == "mlp.gate_proj.weight") {
    if (!shape_is(shape, nd, I_full, Hm)) return fail("gate_proj shape mismatch");
    const Shard sh = shard_of(sub, I_full, Hm, rk, tp);
    TRY(copy_interleaved64(e, l.gu.w, 0, data, Hm, sh));
    l.gu.loaded_rows |= 1;
  } else if (sub == "mlp.up_proj.weight") {
    if (!shape_is(shape, nd, I_full, Hm)) return fail("up_proj shape mismatch");
    const Shard sh = shard_of(sub, I_full, Hm, rk, tp);
    TRY(copy_interleaved64(e, l.gu.w, 1, data, Hm, sh));
    l.gu.loaded_rows |= 2;
  } else if (sub == "mlp.down_proj.weight") {
    if (!shape_is(shape, nd, Hm, I_full)) return fail("down_proj shape mismatch");
    const Shard sh = shard_of(sub, Hm, I_full, rk, tp);
    TRY(copy_block(e, l.down.w, 0, data, I_full, sh.r0, sh.nr, sh.c0, sh.nc));
    l.down.loaded_rows = 1;
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
  if (want_model_dtype && dtype != e->dtype)
    return fail("tensor '%s': dtype %d does not match the engine's model dtype %d (cast it like `.to(base_model.dtype)`, ea_model.py:77)",
                name_c, dtype, e->dtype);
  const eb200_config& c = e->c;
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
  return make_tmap(&l.tm, e->dtype, l.w, l.N, l.K, 128);
}

extern "C" int eb200_finalize(eb200_engine* e) {
  if (!e) return fail("eb200_finalize: null engine");
  CK(cudaSetDevice(e->c.device));
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
    // Persistent chain launches (mega.cu).  The layer segment as ONE launch is slower than the per-projection cluster split-K
    // kernels (its global-memory split-K reduction is bounded by the LSU path of the finishing SMs), so on one GPU only the
    // lm_head runs as a (single-phase, reduction-free) chain launch with the fused arg-max (no 15 MB logits round trip).
    // Under tensor parallelism the chain segment is slower as well, so the peer-window exchange runs as its own kernel behind
    // the per-projection GEMMs (tp_fused.cu) and the chain segment stays opt-in.
    //   EB200_CHAIN=0 : never;  EB200_CHAIN=1 : layer segments as chain launches (A/B);  EB200_CHAIN_DRAFT=1 : draft head tail too
    const char* env = getenv("EB200_CHAIN");
    const int mode = env ? atoi(env) : -1;  // -1 = default policy
    const bool allowed = mode != 0 && !(e->c.flags & (EB200_FLAG_SIMT_GEMM | EB200_FLAG_NO_CHAIN));
    const Layer& l0 = e->tl[0];
    const bool shapes_ok = e->ws_bytes >= chain_ws_bytes(64) && chain_phase_ok(l0.o.N, l0.o.K, FIN_RESID_NORM) &&
                           chain_phase_ok(l0.gu.N, l0.gu.K, FIN_SWIGLU_IL) && chain_phase_ok(l0.down.N, l0.down.K, FIN_RESID_NORM) &&
                           chain_phase_ok(l0.qkv.N, l0.qkv.K, FIN_QKV_ROPE);
    e->chain_target = allowed && shapes_ok && mode == 1 && (e->c.tp_size == 1 || e->tp_fused);
    e->chain_head = allowed && e->ws_bytes >= chain_ws_bytes(64) && (e->c.tp_size == 1 || e->tp_fused) &&
                    chain_phase_ok(e->t_head.N, e->t_head.K, FIN_ARGMAX);
    const Layer& h0 = e->hl[0];
    const char* denv = getenv("EB200_CHAIN_DRAFT");
    e->chain_draft = allowed && denv && atoi(denv) == 1 && e->ws_bytes >= chain_ws_bytes(64) && chain_phase_ok(h0.o.N, h0.o.K, FIN_RESID_NORM) &&
                     chain_phase_ok(h0.gu.N, h0.gu.K, FIN_SWIGLU_IL) && chain_phase_ok(h0.down.N, h0.down.K, FIN_RESID_NORM);
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

// 0 = persistent stream-K, 1 = cluster split-K (default)
static int gemm_mode() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("EB200_GEMM_MODE");
    v = (e && !strcmp(e, "streamk")) ? 0 : 1;  // cluster split-K is the faster one on the benchmark shapes (DESIGN.md)
  }
  return v;
}

struct GemmCall {
  const Linear* W;
  const Linear* W2;
  const ActBuf* X;
  int epi;
  GemmParams p;
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
  const double bytes = static_cast<double>(p.N) * p.K * 2 * (g.epi == EPI_SWIGLU ? 2 : 1);
  const char* kname = g.epi == EPI_STORE ? "gemm_store" : g.epi == EPI_RESIDUAL ? "gemm_residual" :
                      (g.epi == EPI_SWIGLU || g.epi == EPI_SWIGLU_IL) ? "gemm_swiglu" : "gemm_qkv_rope";
  {
    char kk[64];
    snprintf(kk, sizeof(kk), "%s@%d", kname, p.K);  // e.g. gemm_residual@14336 = down_proj only
    if (skip_kernel(kname) || skip_kernel(kk)) return 0;
  }
  ProfScope ps(e, 0, bytes, kname);
  if (e->c.flags & EB200_FLAG_SIMT_GEMM) {
    const size_t per_split = static_cast<size_t>(g.epi == EPI_SWIGLU ? 2 : 1) * cx.mpad * ((p.N + 127) / 128) * 128 * 4;
    while (p.splitk > 1 && per_split * p.splitk > e->ws_bytes) --p.splitk;
    CKL(launch_gemm_simt(e->dtype, cx.mpad, g.epi, g.W->w, g.W2 ? g.W2->w : nullptr, g.X->p, g.X->cols, p, e->stream));
  } else if (gemm_mode() == 1) {
    if (cx.mpad == 256 && g.X->rows < 256) return fail("256-row GEMM on a 64-row activation buffer");
    CKL(launch_gemm(e->dtype, cx.mpad, g.epi, &g.W->tm, g.W2 ? &g.W2->tm : nullptr,
                    cx.mpad == 16 ? &g.X->tm16 : (cx.mpad == 64 ? &g.X->tm64 : &g.X->tm256), p, e->stream, cx.mpad == 64 ? &g.X->tm32 : nullptr));
  } else {
    CKL(launch_gemm_streamk(e->dtype, cx.mpad, g.epi, &g.W->tm, g.W2 ? &g.W2->tm : nullptr, cx.mpad == 16 ? &g.X->tm16 : &g.X->tm64, p,
                            e->sk_ws, e->counters, e->stream));
  }
  return 0;
}
static int gemm_store(eb200_engine* e, const RowCtx& cx, const Linear& W, const ActBuf& X, void* out, long ld, const void* bias) {
  GemmCall g{&W, nullptr, &X, EPI_STORE, {}};
  memset(&g.p, 0, sizeof(g.p));
  g.p.out = out;
  g.p.ld_out = ld;
  g.p.bias = bias;
  return run_gemm(e, cx, g);
}
static int gemm_residual(eb200_engine* e, const RowCtx& cx, const Linear& W, const ActBuf& X, const void* res, void* out, long ld) {
  GemmCall g{&W, nullptr, &X, EPI_RESIDUAL, {}};
  memset(&g.p, 0, sizeof(g.p));
  g.p.out = out;
  g.p.ld_out = ld;
  g.p.res = res;
  g.p.ld_res = ld;
  return run_gemm(e, cx, g);
}
static int gemm_swiglu(eb200_engine* e, const RowCtx& cx, const Linear& Wgu, const ActBuf& X, void* out, long ld) {
  GemmCall g{&Wgu, nullptr, &X, EPI_SWIGLU_IL, {}};
  memset(&g.p, 0, sizeof(g.p));
  g.p.out = out;
  g.p.ld_out = ld;
  return run_gemm(e, cx, g);
}
static int gemm_qkv(eb200_engine* e, const RowCtx& cx, const Linear& W, const ActBuf& X, void* q_out, void* kc, void* vc, long cap,
                    int nq, int nkv, const void* cosp, const void* sinp) {
  GemmCall g{&W, nullptr, &X, EPI_QKV_ROPE, {}};
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
static int gemm_partial_f32(eb200_engine* e, const RowCtx& cx, const Linear& W, const ActBuf& X, float* out, long ld) {
  GemmCall g{&W, nullptr, &X, EPI_PARTIAL_F32, {}};
  memset(&g.p, 0, sizeof(g.p));
  g.p.out = out;
  g.p.ld_out = ld;
  return run_gemm(e, cx, g);
}
static int tp_allreduce_f32(eb200_engine* e, float* buf, size_t count);
static int tp_allgather_u32(eb200_engine* e, const void* send, void* recv, size_t count);
static void chain_fill_tp(eb200_engine* e, ChainArgs& a);
// x += W . X  for a row-parallel projection (o_proj, down_proj).  Single GPU: fused residual epilogue.  Tensor parallel: every
// rank produces an unrounded fp32 partial over its slice of the reduction dim; then either
//   * NVLink peer windows (default): ONE kernel pushes the partial rows to their owners, reduces them in rank order, applies the
//     reference's two roundings (modeling_llama_kv.py:768, :838-845) AND the following RMSNorm, and publishes x / xn (/ tap) on
//     every rank (tp_fused.cu) -- *did_norm tells the caller that xn is already there; or
//   * NCCL: all-reduce, then the residual add; the caller runs the RMSNorm.
static int row_parallel_residual(eb200_engine* e, const RowCtx& cx, const Linear& W, const ActBuf& X, void* x, int H, const void* norm_w = nullptr,
                                 void* tap = nullptr, bool* did_norm = nullptr) {
  if (did_norm) *did_norm = false;
  if (e->c.tp_size == 1) return gemm_residual(e, cx, W, X, x, x, H);
  TRY(gemm_partial_f32(e, cx, W, X, e->f32buf, H));
  if (e->tp_fused && cx.rows_idx < 0) {
    TpResidParams p;
    memset(&p, 0, sizeof(p));
    ChainArgs tmp;
    memset(&tmp, 0, sizeof(tmp));
    chain_fill_tp(e, tmp);
    p.tp = tmp.tp;
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
                   long ld_y, int col_off, int H, float eps, int rows) {
  if (skip_kernel("rmsnorm")) return 0;
  ProfScope ps(e, 2, 0, "rmsnorm");
  CKL(launch_rmsnorm(e->dtype, src, ld_src, ids64, ids32, w, y, ld_y, col_off, H, eps, rows, e->stream));
  return 0;
}
static int gather(eb200_engine* e, const void* table, long ld_table, const int64_t* ids64, const int* ids32, void* dst, long ld_dst,
                  int col_off, int H, int rows) {
  ProfScope ps(e, 2, 0, "gather_rows");
  CKL(launch_gather_rows(e->dtype, table, ld_table, ids64, ids32, dst, ld_dst, col_off, H, rows, e->stream));
  return 0;
}
static int attention(eb200_engine* e, const RowCtx& cx, const void* q, void* kc, void* vc, void* out, long cap, int nh, int nkv,
                     const Linear* next0 = nullptr, const Linear* next1 = nullptr) {
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
      TRY(attention(e, sub, reinterpret_cast<const char*>(q) + off, kc, vc, reinterpret_cast<char*>(out) + off, cap, nh, nkv, nullptr, nullptr));
    }
    return 0;
  }
  AttnParams a;
  memset(&a, 0, sizeof(a));
  {
    // L2 prefetch budget for the weights the following chain launch streams first (EB200_ATTN_PREFETCH_MB, 0 = off)
    static long budget = -1;
    if (budget < 0) {
      const char* s = getenv("EB200_ATTN_PREFETCH_MB");
      budget = (s ? atol(s) : 0) << 20;  // off by default (an experiment knob)
    }
    long left = budget;
    const Linear* nx[2] = {next0, next1};
    for (int r = 0; r < 2; ++r) {
      if (!nx[r] || left <= 0) continue;
      const long bytes = std::min<long>(left, static_cast<long>(nx[r]->N) * nx[r]->K * 2);
      a.pf_ptr[r] = nx[r]->w;
      a.pf_bytes[r] = static_cast<unsigned long long>(bytes);
      left -= bytes;
    }
  }
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
// others' windows.  From then on the row-parallel projections finish inside the chain launch (ChainTP) instead of through NCCL.
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

// finish items per activation row: spread the row-wise finish over the CTAs that are not needed for other rows
static int chain_chunks(int passes, int rows) {
  const int G = std::max(1, chain_grid());
  return std::max(1, std::min(passes, G / std::max(1, rows)));
}
static void chain_phase_gemm(ChainArgs& a, ChainMaps& m, int p, const RowCtx& cx, const Linear& W, const ActBuf& X) {
  a.ph[p].N = W.N;
  a.ph[p].K = W.K;
  m.w[p] = W.tm;
  m.x[p] = cx.mpad == 16 ? X.tm16 : X.tm64;
}

static void chain_fill_tp(eb200_engine* e, ChainArgs& a) {
  if (e->c.tp_size <= 1) return;
  a.tp.size = e->c.tp_size;
  a.tp.rank = e->c.tp_rank;
  for (int r = 0; r < e->c.tp_size; ++r) a.tp.win[r] = e->tp_peer[r];
  a.tp.inbox_off = e->tp_inbox_off;
  a.tp.ld_inbox = e->H;
  a.tp.flag_off = e->tp_flag_off;
  a.tp.ready_off = e->tp_ready_off;
  a.tp.am_off = e->tp_am_off;
  a.tp.epoch = e->tp_epoch;
  a.tp.ready_base = e->tp_ready_base;
}
static void chain_head_phase(eb200_engine* e, ChainArgs& a, ChainMaps& m, int p, const RowCtx& cx, int head_mode) {
  chain_phase_gemm(a, m, p, cx, e->t_head, e->xn);
  ChainPhase& h = a.ph[p];
  h.chunks = 1;
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
}
// One chain launch = o_proj(+residual, RMSNorm) -> gate/up(SwiGLU) -> down_proj(+residual, RMSNorm) -> the NEXT block's
// qkv(+RoPE, KV append) or, after the last layer, the lm_head (fused arg-max, or logits for the sampling path).
static int target_segment_chain(eb200_engine* e, const RowCtx& cx, int i, void* feat_dst, int* slot, int head_mode) {
  const int H = e->H, L = e->L;
  Layer& l = e->tl[i];
  ChainArgs a;
  ChainMaps m;
  memset(&a, 0, sizeof(a));
  memset(&m, 0, sizeof(m));
  a.m_rows = cx.rows;
  a.m_idx = cx.rows_idx;
  a.st = e->st;
  a.ws = e->ws;
  a.sync = e->chain_sync;
  a.timing = e->chain_timing;
  chain_fill_tp(e, a);
  double bytes = 0;
  int p = 0;
  // o_proj: x += attn . Wo^T ; xn = post_attention_layernorm(x)      (modeling_llama_kv.py:838-845, :128-132)
  chain_phase_gemm(a, m, p, cx, l.o, e->attn);
  a.ph[p].fin = FIN_RESID_NORM;
  a.ph[p].chunks = 1;
  a.ph[p].x = e->x;
  a.ph[p].ld_x = H;
  a.ph[p].norm_w = l.ln2;
  a.ph[p].xn = e->xn.p;
  a.ph[p].ld_xn = H;
  a.ph[p].eps = e->c.rms_norm_eps;
  bytes += static_cast<double>(l.o.N) * l.o.K * 2;
  ++p;
  // gate/up + SwiGLU (modeling_llama_kv.py:501-535)
  chain_phase_gemm(a, m, p, cx, l.gu, e->xn);
  a.ph[p].fin = FIN_SWIGLU_IL;
  a.ph[p].chunks = chain_chunks((e->I_l + 511) / 512, cx.rows);
  a.ph[p].out = e->act.p;
  a.ph[p].ld_out = e->I_l;
  a.ph[p].silu_lut = silu_lut(e->dtype, e->stream);
  if (!a.ph[p].silu_lut) return fail("SiLU table not ready (first use inside stream capture)");
  bytes += static_cast<double>(l.gu.N) * l.gu.K * 2;
  ++p;
  // down_proj: x += act . Wd^T ; xn = the next block's input_layernorm(x) (or the final norm)
  chain_phase_gemm(a, m, p, cx, l.down, e->act);
  a.ph[p].fin = FIN_RESID_NORM;
  a.ph[p].chunks = 1;
  a.ph[p].x = e->x;
  a.ph[p].ld_x = H;
  if (e->c.eagle3 && feat_dst && i + 1 < L && is_tap_layer(e, i + 1)) {  // hidden state entering layer i+1 (utils.py:248-252)
    a.ph[p].tap = reinterpret_cast<char*>(feat_dst) + static_cast<size_t>(*slot) * H * 2;
    a.ph[p].ld_tap = e->F;
    ++*slot;
  }
  a.ph[p].norm_w = (i + 1 < L) ? e->tl[i + 1].ln1 : e->t_norm;
  a.ph[p].xn = e->xn.p;
  a.ph[p].ld_xn = H;
  a.ph[p].eps = e->c.rms_norm_eps;
  bytes += static_cast<double>(l.down.N) * l.down.K * 2;
  ++p;
  if (i + 1 < L) {
    Layer& nl = e->tl[i + 1];
    chain_phase_gemm(a, m, p, cx, nl.qkv, e->xn);
    ChainPhase& q = a.ph[p];
    q.fin = FIN_QKV_ROPE;
    q.chunks = chain_chunks((e->nh_l + 2 * e->nkv_l + 7) / 8, cx.rows);
    q.q_out = e->q;
    q.k_cache = kv_plane(e->t_kv, i + 1, 0, e->nkv_l, e->cap);
    q.v_cache = kv_plane(e->t_kv, i + 1, 1, e->nkv_l, e->cap);
    q.kv_cap = e->cap;
    q.n_q_heads = e->nh_l;
    q.n_kv_heads = e->nkv_l;
    q.rope_cos = e->t_cos;
    q.rope_sin = e->t_sin;
    q.pos_base = cx.pos_base;
    q.pos_arr = cx.pos_arr;
    q.pos_mstride = cx.pos_mstride;
    q.kv_base = cx.kv_base;
    bytes += static_cast<double>(nl.qkv.N) * nl.qkv.K * 2;
    ++p;
  } else if (head_mode != HEAD_NONE && e->chain_head) {
    chain_head_phase(e, a, m, p, cx, head_mode);
    bytes += static_cast<double>(e->t_head.N) * e->t_head.K * 2;
    ++p;
  }
  a.n_phases = p;
  if (e->chain_trace && e->in_verify && i == std::min(5, L - 2)) a.trace = e->chain_trace;
  if (skip_kernel("chain")) return 0;
  ProfScope ps(e, 0, bytes, "gemm_chain");
  CKL(launch_gemm_chain(e->dtype, cx.mpad, m, a, e->stream));
  e->stats.chain_bytes += bytes;
  return 0;
}

// lm_head over the rows in e->xn (ea_model.py:190): one reduction-free chain launch (whole 128-row vocabulary tiles per CTA,
// per-row arg-max straight from the staged accumulator tile, merged per row) or, for the sampling path, the logits of this rank's shard.
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
  a.ws = e->ws;
  a.sync = e->chain_sync;
  a.timing = e->chain_timing;
  chain_fill_tp(e, a);
  chain_head_phase(e, a, m, 0, cx, head_mode);
  a.n_phases = 1;
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
  if (e->chain_target) {
    // lead-in (embedding -> first block's norm + qkv) as single kernels, then per block: attention + ONE chain launch
    if (e->c.eagle3 && feat_dst && is_tap_layer(e, 0)) {
      TRY(gather(e, e->x, H, nullptr, e->ident, feat_dst, e->F, slot * H, H, cx.rows));
      ++slot;
    }
    TRY(rmsnorm(e, e->x, H, nullptr, nullptr, e->tl[0].ln1, e->xn.p, H, 0, H, eps, cx.rows));
    TRY(gemm_qkv(e, cx, e->tl[0].qkv, e->xn, e->q, kv_plane(e->t_kv, 0, 0, e->nkv_l, e->cap), kv_plane(e->t_kv, 0, 1, e->nkv_l, e->cap), e->cap,
                 e->nh_l, e->nkv_l, e->t_cos, e->t_sin));
    for (int i = 0; i < L; ++i) {
      void* kc = kv_plane(e->t_kv, i, 0, e->nkv_l, e->cap);
      void* vc = kv_plane(e->t_kv, i, 1, e->nkv_l, e->cap);
      TRY(attention(e, cx, e->q, kc, vc, e->attn.p, e->cap, e->nh_l, e->nkv_l, &e->tl[i].o, &e->tl[i].gu));
      TRY(target_segment_chain(e, cx, i, feat_dst, &slot, head_mode));
    }
    if (!e->c.eagle3 && feat_dst) TRY(gather(e, e->xn.p, H, nullptr, e->ident, feat_dst, e->F, 0, H, cx.rows));
    if (!e->chain_head) TRY(target_head(e, cx, head_mode));  // else: already the last phase of the last segment
    return 0;
  }
  bool have_xn = false;   // xn already holds this layer's input_layernorm(x) (written by the previous down_proj's fused TP kernel)
  bool tap_done = false;  // ... and the EAGLE-3 tap of this layer was written there too
  for (int i = 0; i < L; ++i) {
    Layer& l = e->tl[i];
    if (e->c.eagle3 && feat_dst && is_tap_layer(e, i)) {
      if (!tap_done) TRY(gather(e, e->x, H, nullptr, e->ident, feat_dst, e->F, slot * H, H, cx.rows));
      ++slot;
    }
    if (!have_xn) TRY(rmsnorm(e, e->x, H, nullptr, nullptr, l.ln1, e->xn.p, H, 0, H, eps, cx.rows));
    void* kc = kv_plane(e->t_kv, i, 0, e->nkv_l, e->cap);
    void* vc = kv_plane(e->t_kv, i, 1, e->nkv_l, e->cap);
    TRY(gemm_qkv(e, cx, l.qkv, e->xn, e->q, kc, vc, e->cap, e->nh_l, e->nkv_l, e->t_cos, e->t_sin));
    TRY(attention(e, cx, e->q, kc, vc, e->attn.p, e->cap, e->nh_l, e->nkv_l));
    bool did = false;
    TRY(row_parallel_residual(e, cx, l.o, e->attn, e->x, H, l.ln2, nullptr, &did));
    if (!did) TRY(rmsnorm(e, e->x, H, nullptr, nullptr, l.ln2, e->xn.p, H, 0, H, eps, cx.rows));
    TRY(gemm_swiglu(e, cx, l.gu, e->xn, e->act.p, e->I_l));
    const void* next_norm = (i + 1 < L) ? e->tl[i + 1].ln1 : e->t_norm;
    void* tap = nullptr;
    if (e->c.eagle3 && feat_dst && i + 1 < L && is_tap_layer(e, i + 1)) tap = reinterpret_cast<char*>(feat_dst) + static_cast<size_t>(slot) * H * 2;
    TRY(row_parallel_residual(e, cx, l.down, e->act, e->x, H, next_norm, tap, &did));
    have_xn = did;
    tap_done = did && tap != nullptr;
  }
  if (!have_xn) TRY(rmsnorm(e, e->x, H, nullptr, nullptr, e->t_norm, e->xn.p, H, 0, H, eps, cx.rows));
  if (!e->c.eagle3 && feat_dst) TRY(gather(e, e->xn.p, H, nullptr, e->ident, feat_dst, e->F, 0, H, cx.rows));
  TRY(target_head(e, cx, head_mode));  // lm_head on all rows (ea_model.py:190)
  return 0;
}

// Tail of one draft decoder layer as ONE chain launch: o_proj(+residual, post-attention norm) -> gate/up(SwiGLU) ->
// down_proj(+residual [, next norm]) [-> lm_head over all rows when it is the last layer].
static int draft_segment_chain(eb200_engine* e, const RowCtx& cx, int i) {
  const int Hh = e->Hh;
  const bool last = (i == e->hL - 1);
  Layer& l = e->hl[i];
  ChainArgs a;
  ChainMaps m;
  memset(&a, 0, sizeof(a));
  memset(&m, 0, sizeof(m));
  a.m_rows = cx.rows;
  a.m_idx = cx.rows_idx;
  a.st = e->st;
  a.ws = e->ws;
  a.sync = e->chain_sync;
  a.timing = e->chain_timing;
  double bytes = 0;
  int p = 0;
  chain_phase_gemm(a, m, p, cx, l.o, e->d_attn);  // h2 = h + o_proj(attn); xn = post_attention_layernorm(h2)   (cnets.py:432-441)
  a.ph[p].fin = FIN_RESID_NORM;
  a.ph[p].chunks = 1;
  a.ph[p].res = e->d_h.p;
  a.ph[p].ld_res = Hh;
  a.ph[p].x = e->d_h2;
  a.ph[p].ld_x = Hh;
  a.ph[p].norm_w = l.ln2;
  a.ph[p].xn = e->d_xn.p;
  a.ph[p].ld_xn = Hh;
  a.ph[p].eps = e->c.head_rms_norm_eps;
  bytes += static_cast<double>(l.o.N) * l.o.K * 2;
  ++p;
  chain_phase_gemm(a, m, p, cx, l.gu, e->d_xn);
  a.ph[p].fin = FIN_SWIGLU_IL;
  a.ph[p].chunks = chain_chunks((e->Ih + 511) / 512, cx.rows);
  a.ph[p].out = e->d_act.p;
  a.ph[p].ld_out = e->Ih;
  a.ph[p].silu_lut = silu_lut(e->dtype, e->stream);
  if (!a.ph[p].silu_lut) return fail("SiLU table not ready (first use inside stream capture)");
  bytes += static_cast<double>(l.gu.N) * l.gu.K * 2;
  ++p;
  chain_phase_gemm(a, m, p, cx, l.down, e->d_act);  // out = h2 + mlp(xn)
  a.ph[p].fin = FIN_RESID_NORM;
  a.ph[p].chunks = 1;
  a.ph[p].res = e->d_h2;
  a.ph[p].ld_res = Hh;
  a.ph[p].x = last ? e->d_out.p : e->d_h.p;
  a.ph[p].ld_x = Hh;
  if (e->c.eagle3) a.ph[p].norm_w = e->h_norm;  // lm_head(norm(out))  cnets.py:700, :734
  else if (!last) a.ph[p].norm_w = e->hl[i + 1].ln1;
  a.ph[p].xn = e->d_xn.p;
  a.ph[p].ld_xn = Hh;
  a.ph[p].eps = e->c.head_rms_norm_eps;
  bytes += static_cast<double>(l.down.N) * l.down.K * 2;
  ++p;
  if (last) {
    const Linear& head = e->c.eagle3 ? e->h_head : (e->t_head_full.w ? e->t_head_full : e->t_head);
    chain_phase_gemm(a, m, p, cx, head, e->c.eagle3 ? e->d_xn : e->d_out);
    a.ph[p].fin = chain_phase_ok(head.N, head.K, FIN_STORE) ? FIN_STORE : FIN_STORE_DIRECT;
    a.ph[p].chunks = a.ph[p].fin == FIN_STORE ? chain_chunks((head.N + 511) / 512, cx.rows) : 1;
    a.ph[p].out = e->d_logits;
    a.ph[p].ld_out = e->Vd;
    bytes += static_cast<double>(head.N) * head.K * 2;
    ++p;
  }
  a.n_phases = p;
  if (skip_kernel("chain")) return 0;
  ProfScope ps(e, 0, bytes, "gemm_chain_draft");
  CKL(launch_gemm_chain(e->dtype, cx.mpad, m, a, e->stream));
  e->stats.chain_bytes += bytes;
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
    if (first_pass) TRY(gemm_store(e, cx, e->h_fc, e->d_feat, e->d_h.p, Hh, nullptr));  // cnets.py:639-640
    // cat(norm(emb(ids)), norm(hidden))  cnets.py:427-430
    if (e->fused_e3_input) {
      ProfScope ps(e, 2, 0, "e3_input");
      CKL(launch_e3_input(e->dtype, e->h_embed, Hh, ids64, ids32, l.ln1, src_rows ? e->d_out.p : e->d_h.p, Hh, src_rows, e->d_h.p, Hh,
                          e->h_hidden_norm, e->d_cat.p, 2 * Hh, Hh, eps, cx.rows, e->stream));
    } else {
      if (src_rows) TRY(gather(e, e->d_out.p, Hh, nullptr, src_rows, e->d_h.p, Hh, 0, Hh, cx.rows));
      TRY(rmsnorm(e, e->h_embed, Hh, ids64, ids32, l.ln1, e->d_cat.p, 2 * Hh, 0, Hh, eps, cx.rows));
      TRY(rmsnorm(e, e->d_h.p, Hh, nullptr, nullptr, e->h_hidden_norm, e->d_cat.p, 2 * Hh, Hh, Hh, eps, cx.rows));
    }
    void* kc = kv_plane(e->d_kv, 0, 0, e->hnkv, e->dcap);
    void* vc = kv_plane(e->d_kv, 0, 1, e->hnkv, e->dcap);
    TRY(gemm_qkv(e, cx, l.qkv, e->d_cat, e->d_q, kc, vc, e->dcap, e->hnh, e->hnkv, e->h_cos, e->h_sin));
    TRY(attention(e, cx, e->d_q, kc, vc, e->d_attn.p, e->dcap, e->hnh, e->hnkv, e->chain_draft ? &l.o : nullptr, e->chain_draft ? &l.gu : nullptr));
    if (e->chain_draft) return draft_segment_chain(e, cx, 0);
    TRY(gemm_residual(e, cx, l.o, e->d_attn, e->d_h.p, e->d_h2, Hh));
    TRY(rmsnorm(e, e->d_h2, Hh, nullptr, nullptr, l.ln2, e->d_xn.p, Hh, 0, Hh, eps, cx.rows));
    TRY(gemm_swiglu(e, cx, l.gu, e->d_xn, e->d_act.p, e->Ih));
    TRY(gemm_residual(e, cx, l.down, e->d_act, e->d_h2, e->d_out.p, Hh));
    // lm_head(norm(out))  cnets.py:700, :734
    TRY(rmsnorm(e, e->d_out.p, Hh, nullptr, nullptr, e->h_norm, e->d_xn.p, Hh, 0, Hh, eps, cx.rows));
    TRY(gemm_store(e, cx, e->h_head, e->d_xn, e->d_logits, e->Vd, nullptr));
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
      // chain mode: the previous layer's down_proj finish already produced input_layernorm(h) in d_xn
      if (!e->chain_draft) TRY(rmsnorm(e, e->d_h.p, Hh, nullptr, nullptr, l.ln1, e->d_xn.p, Hh, 0, Hh, eps, cx.rows));
      xin = &e->d_xn;
    }
    void* kc = kv_plane(e->d_kv, i, 0, e->hnkv, e->dcap);
    void* vc = kv_plane(e->d_kv, i, 1, e->hnkv, e->dcap);
    TRY(gemm_qkv(e, cx, l.qkv, *xin, e->d_q, kc, vc, e->dcap, e->hnh, e->hnkv, e->h_cos, e->h_sin));
    TRY(attention(e, cx, e->d_q, kc, vc, e->d_attn.p, e->dcap, e->hnh, e->hnkv));
    if (e->chain_draft) {
      TRY(draft_segment_chain(e, cx, i));
      continue;
    }
    TRY(gemm_residual(e, cx, l.o, e->d_attn, e->d_h.p, e->d_h2, Hh));
    TRY(rmsnorm(e, e->d_h2, Hh, nullptr, nullptr, l.ln2, e->d_xn.p, Hh, 0, Hh, eps, cx.rows));
    TRY(gemm_swiglu(e, cx, l.gu, e->d_xn, e->d_act.p, e->Ih));
    void* dst = (i == e->hL - 1) ? e->d_out.p : e->d_h.p;
    TRY(gemm_residual(e, cx, l.down, e->d_act, e->d_h2, dst, Hh));
  }
  if (!e->chain_draft) TRY(gemm_store(e, cx, e->t_head_full.w ? e->t_head_full : e->t_head, e->d_out, e->d_logits, e->Vd, nullptr));
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
  const int chunk = (e->act_rows >= 256 && !e->chain_target) ? 256 : 64;
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

extern "C" int eb200_k_gemm(int32_t dtype, int32_t simt, int32_t epilogue, const void* W, const void* W2, const void* X, void* out,
                            const void* res, const void* bias, int32_t M, int32_t N, int32_t K, int32_t splitk, void* stream) {
  if (M < 1 || M > 64 || epilogue < EPI_STORE || (epilogue > EPI_SWIGLU && epilogue != EPI_SWIGLU_IL)) return fail("eb200_k_gemm: bad arguments");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int mpad = M <= 16 ? 16 : 64;
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
    TRY(make_tmap(&tx, dtype, X, 64, K, mpad));
    CUtensorMap txh;
    TRY(make_tmap(&txh, dtype, X, 64, K, 32));
    const bool cluster = simt == 2 || (simt == 0 && gemm_mode() == 1);
    if (cluster) {
      if (p.splitk > 8) p.splitk = 8;
      CKL(launch_gemm(dtype, mpad, epilogue, &tw, W2 ? &tw2 : nullptr, &tx, p, s, mpad == 64 ? &txh : nullptr));
    } else {
      float* skws = sc.get<float>(streamk_ws_bytes() / 4, false);
      if (!skws) return fail("scratch allocation failed");
      CKL(launch_gemm_streamk(dtype, mpad, epilogue, &tw, W2 ? &tw2 : nullptr, &tx, p, skws, counters, s));
    }
  }
  CK(cudaStreamSynchronize(s));
  return 0;
}

// One decoder-layer segment through the persistent chain kernel (mega.cu), on caller tensors (all DEVICE pointers):
//   x += attn . Wo^T ; xn = ln2 * norm(x) ; act = swiglu(xn . Wgu^T) ; x += act . Wd^T ; xn = ln1n * norm(x) ;
//   q / K-cache / V-cache rows <- rope(xn . Wqkv^T)                         (n_phases = 4; 3 stops before the qkv)
// Wgu is the [2I, H] matrix with gate/up interleaved in 64-row groups.  attn/xn/act are [64][*] buffers (rows >= M ignored).
extern "C" int eb200_k_chain_layer(int32_t dtype, int32_t M, int32_t H, int32_t I, int32_t n_heads, int32_t n_kv_heads, int32_t n_phases,
                                   const void* Wo, const void* Wgu, const void* Wdown, const void* Wqkv, const void* ln2, const void* ln1n,
                                   const void* attn, void* x, void* xn, void* act, void* tap, void* q_out, void* k_cache, void* v_cache,
                                   int64_t kv_cap, const void* cosp, const void* sinp, const int32_t* pos, int32_t kv_base, float eps,
                                   void* stream) {
  if (M < 1 || M > 64 || n_phases < 1 || n_phases > 4) return fail("eb200_k_chain_layer: bad arguments");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int mpad = M <= 16 ? 16 : 64;
  const int A = n_heads * 128;
  if (!chain_phase_ok(H, A, FIN_RESID_NORM) || !chain_phase_ok(2 * I, H, FIN_SWIGLU_IL) || !chain_phase_ok(H, I, FIN_RESID_NORM) ||
      !chain_phase_ok((n_heads + 2 * n_kv_heads) * 128, H, FIN_QKV_ROPE))
    return fail("eb200_k_chain_layer: shape not supported by the chain kernel");
  Scratch sc;
  float* ws = sc.get<float>(chain_ws_bytes(mpad) / 4, false);
  int* sync = sc.get<int>(16);
  if (!ws || !sync) return fail("scratch allocation failed");
  ChainArgs a;
  ChainMaps m;
  memset(&a, 0, sizeof(a));
  memset(&m, 0, sizeof(m));
  a.n_phases = n_phases;
  a.m_rows = M;
  a.m_idx = -1;
  a.ws = ws;
  a.sync = sync;
  const void* lut = silu_lut(dtype, s);
  if (!lut) return fail("SiLU table unavailable");
  auto rows_chunks = [&](int passes) { return std::max(1, std::min(passes, std::max(1, chain_grid()) / M)); };
  // phase 0: o_proj
  a.ph[0].N = H; a.ph[0].K = A; a.ph[0].fin = FIN_RESID_NORM; a.ph[0].chunks = 1;
  a.ph[0].x = x; a.ph[0].ld_x = H; a.ph[0].norm_w = ln2; a.ph[0].xn = xn; a.ph[0].ld_xn = H; a.ph[0].eps = eps;
  TRY(make_tmap(&m.w[0], dtype, Wo, H, A, 128));
  TRY(make_tmap(&m.x[0], dtype, attn, 64, A, mpad));
  if (n_phases > 1) {
    a.ph[1].N = 2 * I; a.ph[1].K = H; a.ph[1].fin = FIN_SWIGLU_IL; a.ph[1].chunks = rows_chunks((I + 511) / 512);
    a.ph[1].out = act; a.ph[1].ld_out = I; a.ph[1].silu_lut = lut;
    TRY(make_tmap(&m.w[1], dtype, Wgu, 2 * I, H, 128));
    TRY(make_tmap(&m.x[1], dtype, xn, 64, H, mpad));
  }
  if (n_phases > 2) {
    a.ph[2].N = H; a.ph[2].K = I; a.ph[2].fin = FIN_RESID_NORM; a.ph[2].chunks = 1;
    a.ph[2].x = x; a.ph[2].ld_x = H; a.ph[2].tap = tap; a.ph[2].ld_tap = H; a.ph[2].norm_w = ln1n; a.ph[2].xn = xn; a.ph[2].ld_xn = H; a.ph[2].eps = eps;
    TRY(make_tmap(&m.w[2], dtype, Wdown, H, I, 128));
    TRY(make_tmap(&m.x[2], dtype, act, 64, I, mpad));
  }
  if (n_phases > 3) {
    const int NH = n_heads + 2 * n_kv_heads;
    ChainPhase& q = a.ph[3];
    q.N = NH * 128; q.K = H; q.fin = FIN_QKV_ROPE; q.chunks = rows_chunks((NH + 7) / 8);
    q.q_out = q_out; q.k_cache = k_cache; q.v_cache = v_cache; q.kv_cap = kv_cap; q.n_q_heads = n_heads; q.n_kv_heads = n_kv_heads;
    q.rope_cos = cosp; q.rope_sin = sinp; q.pos_base = DynInt{-1, 0}; q.pos_arr = pos; q.pos_mstride = 0; q.kv_base = DynInt{-1, kv_base};
    TRY(make_tmap(&m.w[3], dtype, Wqkv, NH * 128, H, 128));
    TRY(make_tmap(&m.x[3], dtype, xn, 64, H, mpad));
  }
  CKL(launch_gemm_chain(dtype, mpad, m, a, s));
  CK(cudaStreamSynchronize(s));
  return 0;
}

// A single GEMM through the chain kernel.  mode 0: stream-K partials + row-wise finish, out = T(X . W^T [+ bias]);
// mode 1: whole tiles, direct store; mode 2: fused arg-max -> out_idx[M] (int32).  `repeat` launches back to back (exercises
// the self-resetting phase counters).
extern "C" int eb200_k_chain_gemm(int32_t dtype, int32_t mode, const void* W, const void* X, void* out, const void* bias, int32_t* out_idx,
                                  int32_t M, int32_t N, int32_t K, int32_t repeat, void* stream) {
  if (M < 1 || M > 64 || mode < 0 || mode > 2 || repeat < 1) return fail("eb200_k_chain_gemm: bad arguments");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int mpad = M <= 16 ? 16 : 64;
  const int fin = mode == 0 ? FIN_STORE : (mode == 1 ? FIN_STORE_DIRECT : FIN_ARGMAX);
  if (!chain_phase_ok(N, K, fin)) return fail("eb200_k_chain_gemm: shape not supported by the chain kernel in this mode");
  Scratch sc;
  float* ws = sc.get<float>(chain_ws_bytes(mpad) / 4, false);
  int* sync = sc.get<int>(16);
  const int tiles = (N + 127) / 128;
  float* tv = sc.get<float>(static_cast<size_t>(tiles) * 64);
  int* ti = sc.get<int>(static_cast<size_t>(tiles) * 64);
  if (!ws || !sync || !tv || !ti) return fail("scratch allocation failed");
  ChainArgs a;
  ChainMaps m;
  memset(&a, 0, sizeof(a));
  memset(&m, 0, sizeof(m));
  a.n_phases = 1;
  a.m_rows = M;
  a.m_idx = -1;
  a.ws = ws;
  a.sync = sync;
  ChainPhase& ph = a.ph[0];
  ph.N = N; ph.K = K; ph.fin = fin;
  ph.chunks = mode == 0 ? std::max(1, std::min((N + 511) / 512, std::max(1, chain_grid()) / M)) : 1;
  ph.out = out; ph.ld_out = N; ph.bias = bias;
  ph.tile_val = tv; ph.tile_idx = ti; ph.out_idx = out_idx;
  TRY(make_tmap(&m.w[0], dtype, W, N, K, 128));
  TRY(make_tmap(&m.x[0], dtype, X, 64, K, mpad));
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
  CUtensorMap tx, txh;
  TRY(make_tmap(&tx, dtype, X, 64, K, mpad));
  TRY(make_tmap(&txh, dtype, X, 64, K, 32));
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
  float* bws = sc.get<float>(streamk_ws_bytes() / 4, false);
  int* bflags = sc.get<int>(8192);
  if (!bws || !bflags) return fail("allocation failed");
  cudaStream_t s;
  CK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
  auto run_all = [&]() -> int {
    for (int i = 0; i < iters; ++i) {
      const int wi = i % n_weights;
      if (gemm_mode() == 1) CKL(launch_gemm(dtype, mpad, epilogue, &tw[wi], epilogue == EPI_SWIGLU ? &tw2[wi] : nullptr, &tx, p, s, mpad == 64 ? &txh : nullptr));
      else CKL(launch_gemm_streamk(dtype, mpad, epilogue, &tw[wi], epilogue == EPI_SWIGLU ? &tw2[wi] : nullptr, &tx, p, bws, bflags, s));
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
  if (M < 1 || M > 64) return fail("eb200_k_qkv_rope: bad M");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int mpad = M <= 16 ? 16 : 64;
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
  p.pos_base = DynInt{-1, 0};
  p.pos_arr = pos;
  p.pos_mstride = 0;
  p.kv_base = DynInt{-1, kv_base};
  if (simt == 1) {
    CKL(launch_gemm_simt(dtype, mpad, EPI_QKV_ROPE, Wqkv, nullptr, X, K, p, s));
  } else {
    CUtensorMap tw, tx;
    TRY(make_tmap(&tw, dtype, Wqkv, N, K, 128));
    TRY(make_tmap(&tx, dtype, X, 64, K, mpad));
    CUtensorMap txh;
    TRY(make_tmap(&txh, dtype, X, 64, K, 32));
    const bool cluster = simt == 2 || (simt == 0 && gemm_mode() == 1);
    if (cluster) {
      if (p.splitk > 8) p.splitk = 8;
      CKL(launch_gemm(dtype, mpad, EPI_QKV_ROPE, &tw, nullptr, &tx, p, s, mpad == 64 ? &txh : nullptr));
    } else {
      float* skws = sc.get<float>(streamk_ws_bytes() / 4, false);
      if (!skws) return fail("scratch allocation failed");
      CKL(launch_gemm_streamk(dtype, mpad, EPI_QKV_ROPE, &tw, nullptr, &tx, p, skws, counters, s));
    }
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
  a.rows_idx = -1;
  a.st = nullptr;
  a.n_ctx = DynInt{-1, n_ctx};
  a.n_tree = n_tree;
  a.mask = mask;
  a.max_kv = n_ctx + n_tree;
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
