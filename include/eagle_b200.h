/* eagle_b200 -- C ABI of the H100-native EAGLE speculative-decoding engine.
 *
 * The reference (SafeAILab/EAGLE) has no FFI layer: its drop-in boundary is the Python surface of
 * `EaModel` (eagle/model/ea_model.py:25-558).  This library is what a thin `EaModel`-compatible class binds
 * (eagle_b200/ea_model.py via ctypes; INTEGRATION.md shows the stub a reference maintainer would add).
 * One engine handle replaces, wholesale, the reference's
 *     initialize_tree / tree_decoding / evaluate_posterior / update_inference_inputs   (eagle/model/utils.py:232-473)
 *     Model.forward / Model.topK_genrate                                                (eagle/model/cnets.py:586-827,
 *                                                                                        eagle/model/cnets1.py:570-822)
 *     LlamaModel.forward with tree mask + preallocated KV                               (eagle/model/modeling_llama_kv.py:
 *                                                                                        1046-1200, kv_cache.py:4-157)
 * Conventions: plain pointers and sizes only, no torch types; every function returns 0 on success and a
 * non-zero code on failure with a message in eb200_last_error(); nothing throws across the boundary; one
 * handle == one CUDA stream == not thread-safe and not re-entrant, exactly like the reference's EaModel
 * (mutable per-model KV / stable_kv / tree_mask state, ea_model.py:223-244).  Pointers marked "host or device"
 * are copied with cudaMemcpyDefault (UVA), so the caller may pass either; device buffers must be complete when the
 * call is made (the engine's stream is non-blocking and is not ordered after the caller's streams).
 */
#ifndef EAGLE_B200_H_
#define EAGLE_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define EB200_ABI_VERSION 5

enum { EB200_BF16 = 0, EB200_FP16 = 1 };
enum { EB200_DT_BF16 = 0, EB200_DT_FP16 = 1, EB200_DT_FP32 = 2, EB200_DT_INT64 = 3, EB200_DT_BOOL = 4, EB200_DT_INT8 = 5, EB200_DT_UINT8 = 6,
       EB200_DT_FP8_E4M3 = 7 };

typedef struct eb200_engine eb200_engine;

/* Shapes of the target (HF LlamaConfig) and of the draft head (EConfig, eagle/model/configs.py:77-124), the
 * tree parameters of EaModel.from_pretrained (ea_model.py:88-98) and the KV capacity (`max_length`,
 * ea_model.py:206, kv_cache.py:69). */
typedef struct eb200_config {
  int32_t abi_version;      /* EB200_ABI_VERSION */
  int32_t dtype;            /* EB200_BF16 | EB200_FP16: the model dtype (`torch_dtype` of from_pretrained) */
  /* target */
  int32_t vocab_size, hidden_size, intermediate_size, num_layers, num_heads, num_kv_heads;
  float rms_norm_eps;
  /* draft head */
  int32_t eagle3;           /* 1: EAGLE-3 head (cnets.py), 0: EAGLE-1/2 head (cnets1.py) */
  int32_t head_hidden_size, head_intermediate_size, head_num_layers, head_num_heads, head_num_kv_heads;
  int32_t draft_vocab_size; /* EAGLE-3 lm_head rows; == vocab_size means no d2t map (ea_model.py:74-75) */
  int32_t head_fc_bias;     /* EAGLE-1 `bias` key of the head's config.json (ea_model.py:49-54) */
  float head_rms_norm_eps;
  /* tree */
  int32_t total_token;      /* API value: total_token - 1 draft nodes + root are verified (cnets.py:522) */
  int32_t depth, top_k;
  /* runtime */
  int32_t max_length;       /* KV rows (ea_model.py:206) */
  int32_t max_rope_positions;
  int32_t tp_rank, tp_size; /* tensor-parallel shard of the TARGET model (draft head is replicated) */
  int32_t device;           /* CUDA ordinal */
  int32_t flags;            /* EB200_FLAG_* */
} eb200_config;

#define EB200_FLAG_SIMT_GEMM 1   /* bring-up only: route GEMMs through the plain-FMA kernel */
#define EB200_FLAG_NO_GRAPH 2    /* launch kernels directly instead of replaying the captured cycle graph */
#define EB200_FLAG_NO_CHAIN 4    /* target lm_head as a GEMM launch + vocab_argmax instead of the fused arg-max launch */
/* The q/k/v/o/gate/up/down projections of every TARGET decoder layer are stored as int8 plus one fp32 scale per row
 * (bitsandbytes' 8-bit weight format) and multiplied by a W8A16 GEMM that computes exactly what the model-dtype GEMM computes on
 * W' = dtype((q * SCB) * 7.874015718698502e-3).  lm_head, embeddings, norms and the draft head stay in the model dtype.
 * Single GPU, default GEMM path only: eb200_finalize refuses tp_size > 1 and EB200_FLAG_SIMT_GEMM. */
#define EB200_FLAG_TARGET_INT8 8
/* The same projections stored as bitsandbytes 4-bit codes (NF4 or FP4 table, blocksize 64: one fp32 absmax per 64 consecutive
 * elements of a row) and multiplied by a W4A16 GEMM that computes exactly what the model-dtype GEMM computes on
 * W' = dtype(code[q] * absmax) (one fp32 product, one round-to-nearest cast).  The two flags exclude each other and
 * EB200_FLAG_TARGET_INT8; the in-features of every projection must be a multiple of 64.  Same restrictions as int8, and
 * eb200_create already refuses them with tp_size > 1 (the loader places whole tensors). */
#define EB200_FLAG_TARGET_NF4 16
#define EB200_FLAG_TARGET_FP4 32
/* The same projections stored the way transformers' FineGrainedFP8Config stores them: float8_e4m3fn weights with one fp32
 * weight_scale_inv per 128 x 128 block, multiplied by a W8A16 GEMM that computes exactly what the model-dtype GEMM computes on
 * W' = dtype(fp32(q) * weight_scale_inv[n / 128][k / 128]) (one fp32 product, one round-to-nearest cast).  Excludes the int8 and
 * 4-bit flags; out- and in-features of every projection must be multiples of 128.  Same restrictions as int8, and eb200_create
 * already refuses it with tp_size > 1 (the loader places whole tensors). */
#define EB200_FLAG_TARGET_FP8 64

typedef struct eb200_gen_params {
  float temperature, top_p;   /* eagenerate(temperature, top_p, top_k, ...) ea_model.py:199-208 */
  int32_t top_k;
  int32_t max_new_tokens;
  int32_t max_length;         /* loop bound of this call (ea_model.py:206, :250); 0 or > capacity -> engine capacity */
  int32_t eos_token_id;       /* tokenizer.eos_token_id; < 0 disables (ea_model.py:294) */
  int32_t stop_token_id;      /* <|eot_id|> when is_llama3; < 0 disables (ea_model.py:290-292) */
  uint64_t seed;              /* sampling path RNG seed */
} eb200_gen_params;

const char* eb200_last_error(void);
int eb200_abi_version(void);

/* ---- lifetime ---- */
int eb200_create(const eb200_config* cfg, eb200_engine** out);
void eb200_destroy(eb200_engine* e);

/* ---- weights: the reference's own state-dict keys.
 *   target : HF names, "model.embed_tokens.weight", "model.layers.{i}.self_attn.{q,k,v,o}_proj.weight",
 *            "model.layers.{i}.mlp.{gate,up,down}_proj.weight", "model.layers.{i}.{input,post_attention}_layernorm.weight",
 *            "model.norm.weight", "lm_head.weight"                  (loaded by ea_model.py:101-118)
 *   head   : prefix "head." + the draft checkpoint keys (SURVEY.md 5 / cnets.py:486-541, cnets1.py:480-528), e.g.
 *            "head.fc.weight", "head.midlayer.self_attn.q_proj.weight", "head.lm_head.weight", "head.d2t",
 *            "head.embed_tokens.weight" (optional: defaults to the target embedding, ea_model.py:55-60 load_emb)
 * `data` is the FULL tensor (host or device, row-major, `dtype` as given); with tp_size > 1 the engine keeps only
 * this rank's shard.  shape has ndim entries.
 * EB200_FLAG_TARGET_INT8 engines take each target projection as "model.layers.{i}.<proj>.weight" in EB200_DT_INT8 [out, in]
 * plus "model.layers.{i}.<proj>.SCB" in EB200_DT_FP32 [out] (its row absmax, the key transformers serializes bnb 8-bit models
 * with); model-dtype data for those names is rejected, and so is int8 data anywhere else or for an engine without the flag.
 * EB200_FLAG_TARGET_NF4 / _FP4 engines take "model.layers.{i}.<proj>.weight" in EB200_DT_UINT8 [out, in / 2] (bitsandbytes' packing:
 * element 2j in the high nibble of byte j) plus "model.layers.{i}.<proj>.weight.absmax" in EB200_DT_FP32 [out, in / 64]; the engine
 * repacks both on the device into its kernel's private layout.
 * EB200_FLAG_TARGET_FP8 engines take "model.layers.{i}.<proj>.weight" in EB200_DT_FP8_E4M3 [out, in] plus
 * "model.layers.{i}.<proj>.weight_scale_inv" in EB200_DT_FP32 [out / 128, in / 128] (transformers' keys) and repack both on the
 * device; model-dtype data for those names is rejected, and so is FP8 data anywhere else or for an engine without the flag. */
int eb200_load_tensor(eb200_engine* e, const char* name, const void* data, const int64_t* shape, int32_t ndim,
                      int32_t dtype);
/* cos/sin tables [n_pos][head_dim/2] in the model dtype, built by the caller exactly like the reference's
 * LlamaRotaryEmbedding (modeling_llama_kv.py:148-186, cnets.py:110-133).  which: 0 = target, 1 = head. */
int eb200_set_rope_table(eb200_engine* e, int32_t which, const void* cos, const void* sin, int32_t n_pos);
/* checks that every tensor arrived, fuses q/k/v, builds TMA descriptors */
int eb200_finalize(eb200_engine* e);
/* tensor parallel: 128-byte ncclUniqueId created by rank 0 and broadcast by the caller's launcher */
int eb200_tp_unique_id(void* out_id128);
/* which block of a [rows, cols] target tensor rank `tp_rank` keeps: out4 = {row0, n_rows, col0, n_cols} (pure host logic) */
int eb200_tp_shard(const char* name, int64_t rows, int64_t cols, int32_t tp_rank, int32_t tp_size, int64_t* out4);
int eb200_tp_init(eb200_engine* e, const void* id128);
/* NVLink peer windows (optional, after eb200_tp_init and before eb200_finalize): each rank exports a 64-byte CUDA IPC handle, the
 * launcher all-gathers them and every rank opens the others'.  With the peers open, the row-parallel projections are reduced
 * over peer memory by one kernel behind each of them, and the lm_head's arg-max is exchanged through the same windows (no NCCL
 * call on the decode path).  eb200_tp_open_peers fails (and the engine keeps the NCCL path) when the GPUs have no peer access. */
int eb200_tp_ipc_handle(eb200_engine* e, void* out64);
int eb200_tp_open_peers(eb200_engine* e, const void* handles, int32_t n);

/* ---- generation: EaModel.eagenerate / naivegenerate (ea_model.py:198-380) ----
 * prompt: P int64 ids (host or device).  out_ids: capacity out_cap int64 (host), receives prompt + committed tokens.
 * out_len = total ids written, out_new_token / out_steps = the `log=True` tuple (new_token, idx). */
int eb200_generate(eb200_engine* e, const int64_t* prompt, int32_t P, const eb200_gen_params* gp, int64_t* out_ids,
                   int32_t out_cap, int32_t* out_len, int32_t* out_new_token, int32_t* out_steps);
int eb200_naive_generate(eb200_engine* e, const int64_t* prompt, int32_t P, const eb200_gen_params* gp, int64_t* out_ids,
                         int32_t out_cap, int32_t* out_len, int32_t* out_new_token, int32_t* out_steps);

/* streaming form of naive_generate (ea_model.py:485-558): begin = prefill + first token, step = feed the pending token and
 * return it together with the next one */
int eb200_naive_begin(eb200_engine* e, const int64_t* prompt, int32_t P, const eb200_gen_params* gp, int64_t* first_token);
int eb200_naive_step(eb200_engine* e, int64_t* fed_token, int64_t* next_token);
/* total_token = -1 (ea_model.py:148-168): device-timed target forward over `rows` rows, `iters` times -> ms_total; then fix the
 * tree size (<= the total_token the engine was created with) */
int eb200_time_target_forward(eb200_engine* e, int32_t rows, int32_t iters, double* ms_total);
int eb200_set_total_token(eb200_engine* e, int32_t total_token);

/* ---- static draft tree (the reference's fixed-tree variant: generate_tree_buffers utils.py:89-207, tree choices.py:1-3,
 * generate_candidates utils.py:284-303, level-by-level draft growth modeling_eagle.py:562-692,863-957) ----
 * A tree is n_choices paths, flattened: choices = concatenation of the paths, choice_len[i] = length of path i; a path
 * [c0, c1, ..] is "the c0-th best child of the root, then its c1-th best child, ..." (values < top_k).
 * eb200_set_static_tree switches the engine from the dynamic (re-ranked) tree to this fixed one for every following
 * prefill / step / generate; the engine must have been created with total_token = n_choices + 1 and
 * depth = longest path - 1.  n_choices = 0 switches back.  Errors (orphan path, duplicate, depth-1 tree, value >= top_k)
 * mirror the inputs the reference's builders raise on. */
int eb200_set_static_tree(eb200_engine* e, const int32_t* choices, const int32_t* choice_len, int32_t n_choices);
/* host-only (no GPU touched): the integer tables of a fixed tree in the reference's formats.  With n = n_choices the
 * caller provides tree_indices / tree_position_ids [n+1], tree_attn_mask [(n+1)^2] (1/0), retrieve_indices [(n+1)^2]
 * (n_leaf x width written, -1 padded, rows sorted with -1 last), level_count [n], level_sel / level_src [n]
 * (concatenated over the n_levels draft levels), level_mask [n*n] (n_inner x n_inner written: ancestor bits among the
 * nodes that have children).  Any output pointer may be NULL. */
int eb200_static_tree_buffers(const int32_t* choices, const int32_t* choice_len, int32_t n_choices, int32_t top_k,
                              int32_t* tree_indices, int32_t* tree_position_ids, float* tree_attn_mask,
                              int32_t* retrieve_indices, int32_t* n_leaf, int32_t* width, int32_t* n_levels,
                              int32_t* level_count, int32_t* level_sel, int32_t* level_src, float* level_mask,
                              int32_t* n_inner);

/* sampling path (temperature > 0) only: inject up to 4096 uniforms in (0,1) (host pointer) that the posterior consumes
 * in order -- one per candidate tried, one per sampled token -- before falling back to the seeded counter RNG; n = 0
 * clears.  Lets a test replay the reference's `random.random()` stream (utils.py:396). */
int eb200_set_uniforms(eb200_engine* e, const float* host_uniforms, int32_t n);

/* ---- step-wise driver (ea_generate yields after every cycle, ea_model.py:382-483) ----
 * eb200_prefill == initialize_tree (utils.py:232-254): target prefill, first token, first draft tree.
 * eb200_step    == one tree_decoding + evaluate_posterior + update_inference_inputs cycle; writes the
 *                  accept_length+1 committed tokens to out_tokens (host, capacity depth+2) and the next root token. */
int eb200_prefill(eb200_engine* e, const int64_t* prompt, int32_t P, const eb200_gen_params* gp, int64_t* first_token);
int eb200_step(eb200_engine* e, int64_t* out_tokens, int32_t* out_n, int64_t* next_token);

/* ---- inspection (tests, INTEGRATION.md): copies of the current tree in the reference's own formats ----
 * draft_tokens[T] int64, tree_mask[T*T] float (1/0), tree_position_ids[T] int64,
 * retrieve_indices[n_leaf*max_depth] int64 (cnets.py:823-827).  Any pointer may be NULL. */
int eb200_get_tree(eb200_engine* e, int64_t* draft_tokens, float* tree_mask, int64_t* tree_position_ids,
                   int64_t* retrieve_indices, int32_t* n_leaf, int32_t* max_depth);
/* arg-max token per tree node of the last verify pass, accepted feature rows, committed length */
int eb200_get_verify(eb200_engine* e, int64_t* node_argmax, int32_t* best, int32_t* accept_length, int32_t* committed_len);
/* copy a named device buffer of the last pass to host as float32 (names: "verify_features", "verify_logits",
 * "draft_stable_out", "draft_logits", "target_k", "target_v", ...); returns rows/cols actually written */
int eb200_debug_read(eb200_engine* e, const char* what, float* out, int64_t cap, int32_t* rows, int32_t* cols);

/* ---- counters / profiling ---- */
typedef struct eb200_stats {
  uint64_t kernel_launches;      /* kernels of this library launched since create */
  uint64_t cycles;               /* draft->verify->accept cycles run */
  uint64_t tokens_committed;
  double gemm_ms;                /* device time in the skinny GEMM, when profiling is on */
  double gemm_bytes;             /* algorithmic weight bytes those launches streamed */
  uint64_t gemm_launches;
  double attn_ms, other_ms;
  double verify_gemm_ms, verify_gemm_bytes;  /* the target verify pass' share */
  /* lm_head launch (mega.cu), measured INSIDE the kernel with %globaltimer (valid under graph replay, no profiler): time from
   * "dependencies resolved" on CTA 0 to the exit of the last CTA, summed over launches; algorithmic weight bytes of those launches */
  double chain_ms, chain_bytes;
  uint64_t chain_launches;
} eb200_stats;
/* the engine's cudaStream_t (so a caller can bracket calls with its own CUDA events) */
void* eb200_get_stream(eb200_engine* e);
int eb200_set_profiling(eb200_engine* e, int32_t on);   /* per-launch CUDA events on the engine's stream */
int eb200_get_stats(eb200_engine* e, eb200_stats* out);
int eb200_reset_stats(eb200_engine* e);

/* ---- per-kernel entry points (parity tests call each kernel in isolation through the same library) ----
 * All pointers are DEVICE pointers unless noted; dtype is EB200_BF16/FP16.
 * simt (eb200_k_gemm, eb200_k_qkv_rope): 1 runs the SIMT bring-up kernel; 0 and 2 both run the engine's cluster split-K kernel.
 * Rows (eb200_k_gemm*, eb200_k_qkv_rope): 1 <= M <= 64 launches 16 or 64 activation rows and X is a [64, K] buffer; 64 < M <= 256
 * launches the prompt prefill's 256 rows and X is a [256, K] buffer.  Above 64 rows only the cluster kernel with the residual (1),
 * interleaved SwiGLU (5) and QKV + RoPE epilogues runs; store, two-matrix SwiGLU and the SIMT kernel are refused. */
int eb200_k_gemm(int32_t dtype, int32_t simt, int32_t epilogue, const void* W, const void* W2, const void* X, void* out,
                 const void* res, const void* bias, int32_t M, int32_t N, int32_t K, int32_t splitk, void* stream);
/* the W8A16 cluster split-K GEMM (EB200_FLAG_TARGET_INT8): Wq int8 [N, K], scb fp32 [N]; epilogue codes and M as
 * eb200_k_gemm (0 store, 1 residual, 5 interleaved SwiGLU with N output columns over a [2N, K] weight); bias: store only */
int eb200_k_gemm_w8(int32_t dtype, int32_t epilogue, const void* Wq, const void* scb, const void* X, void* out, const void* res,
                    const void* bias, int32_t M, int32_t N, int32_t K, int32_t splitk, void* stream);
/* the W4A16 GEMM (EB200_FLAG_TARGET_NF4 / _FP4) on bitsandbytes' layout: Wq uint8 [N, K/2], absmax fp32 [N, K/64], quant_type
 * 0 = nf4, 1 = fp4; the engine's load-time repack is applied first.  Epilogues and M as eb200_k_gemm_w8; K % 64 == 0. */
/* the FP8 GEMM (EB200_FLAG_TARGET_FP8) on transformers' layout: Wq float8_e4m3fn [N, K], scale_inv fp32 [N/128, K/128]; the
 * engine's load-time repack is applied first.  Epilogues and M as eb200_k_gemm_w8; K % 128 == 0 and the weight's rows (2N for the
 * interleaved SwiGLU) a multiple of 128. */
int eb200_k_gemm_fp8(int32_t dtype, int32_t epilogue, const void* Wq, const void* scale_inv, const void* X, void* out, const void* res,
                     const void* bias, int32_t M, int32_t N, int32_t K, int32_t splitk, void* stream);
int eb200_k_gemm_w4(int32_t dtype, int32_t quant_type, int32_t epilogue, const void* Wq, const void* absmax, const void* X, void* out,
                    const void* res, const void* bias, int32_t M, int32_t N, int32_t K, int32_t splitk, void* stream);
/* the lm_head launch (mega.cu, whole 128-row weight tiles per CTA) as a single GEMM: mode 1 stores out = T(X . W^T [+ bias]),
 * mode 2 writes the fused arg-max of every row to out_idx (int32); any other mode is refused.  `repeat` launches back to back. */
int eb200_k_chain_gemm(int32_t dtype, int32_t mode, const void* W, const void* X, void* out, const void* bias, int32_t* out_idx,
                       int32_t M, int32_t N, int32_t K, int32_t repeat, void* stream);
/* micro-benchmark of the skinny GEMM: `iters` back-to-back launches cycling over `n_weights` distinct [N,K] weight
 * matrices (so the stream is HBM-, not L2-resident), timed with CUDA events; optionally replayed from a CUDA graph.
 * epilogue: 0 store, 1 residual, 2 swiglu.  Returns the average microseconds per launch. */
int eb200_k_gemm_bench(int32_t dtype, int32_t epilogue, int32_t M, int32_t N, int32_t K, int32_t splitk, int32_t n_weights,
                       int32_t iters, int32_t use_graph, double* us_per_launch);
int eb200_k_rmsnorm(int32_t dtype, const void* x, const void* w, void* y, int32_t rows, int32_t H, float eps, void* stream);
/* a kernel that also prefetches another GEMM's weight into L2; its outputs must equal the kernel's own.  kernel 0: the cluster
 * GEMM of eb200_k_gemm (epilogue 0 store / 1 residual, W [N, K], X, out, res, M, splitk); kernel 1: eb200_k_rmsnorm (W = the
 * norm weight [N], X = x [M, N], eps).  The prefetched weight is P [PN, PK] (model dtype) under the grid (PN / 128 tiles x
 * p_splitk): k-block rows [j0, j1) of every (tile, split), passed unclipped to the device. */
int eb200_k_prefetch(int32_t dtype, int32_t kernel, int32_t epilogue, const void* W, const void* X, void* out, const void* res, int32_t M,
                     int32_t N, int32_t K, int32_t splitk, float eps, const void* P, int32_t PN, int32_t PK, int32_t p_splitk, int32_t j0,
                     int32_t j1, void* stream);
int eb200_k_attention(int32_t dtype, const void* q, const void* k_cache, const void* v_cache, void* out, int32_t rows,
                      int32_t n_heads, int32_t n_kv_heads, int64_t kv_cap, int32_t n_ctx, int32_t n_tree,
                      const uint64_t* mask, void* stream);
/* host only, no kernel: the tree attention's launch geometry for a score strip of max_kv columns -- query heads per CTA
 * (hpc), KV split over a cluster (kvs), strip columns per CTA row (kv_stride) and dynamic shared memory in bytes.  hpc_cap /
 * kvs_cap: 1, 2 or 4 caps the choice, 0 keeps the engine's policy (EB200_ATTN_HPC / EB200_ATTN_KVS, default 2 / 4).  Fails
 * with a message when max_kv exceeds what shared memory holds (16896 under the default caps). */
int eb200_k_attention_plan(int32_t max_kv, int32_t n_heads, int32_t n_kv_heads, int32_t hpc_cap, int32_t kvs_cap, int32_t* hpc,
                           int32_t* kvs, int32_t* kv_stride, int64_t* smem);
/* eb200_k_attention as the engine launches it: the strip is sized for max_kv columns (kv_len = min(n_ctx + n_tree, max_kv));
 * st (device int32, may be null) supplies the valid row count min(rows, st[rows_idx]) when rows_idx >= 0 and
 * n_ctx = st[n_ctx_idx] + n_ctx_add (n_ctx_add alone when n_ctx_idx < 0); caps as in eb200_k_attention_plan. */
int eb200_k_attention_ex(int32_t dtype, const void* q, const void* k_cache, const void* v_cache, void* out, int32_t rows,
                         int32_t n_heads, int32_t n_kv_heads, int64_t kv_cap, int32_t max_kv, const int32_t* st, int32_t rows_idx,
                         int32_t n_ctx_idx, int32_t n_ctx_add, int32_t n_tree, const uint64_t* mask, int32_t hpc_cap,
                         int32_t kvs_cap, void* stream);
/* X . Wqkv^T with RoPE: q_out [M, n_heads * 128], K / V rows [kv_base, kv_base + M) of the [n_kv_heads, kv_cap, 128] caches;
 * cos / sin [positions, 64].  Row m is rotated to position pos[m] (the cycle's form), or to kv_base + m when pos is null (the
 * prompt prefill's form). */
int eb200_k_qkv_rope(int32_t dtype, int32_t simt, const void* Wqkv, const void* X, void* q_out, void* k_cache,
                     void* v_cache, const void* cos, const void* sin, const int32_t* pos, int32_t M, int32_t n_heads,
                     int32_t n_kv_heads, int32_t K, int64_t kv_cap, int32_t kv_base, int32_t splitk, void* stream);
int eb200_k_argmax(int32_t dtype, const void* logits, int32_t rows, int32_t V, int32_t* out, void* stream);
int eb200_k_logsoftmax_topk(int32_t dtype, const void* logits, int32_t rows, int32_t V, int32_t k, float* topk_p,
                            int32_t* topk_i, void* stream);
/* top-k of the raw logits (value desc, index asc) -- torch.topk(last_headout) of the static tree, modeling_eagle.py:900-903 */
int eb200_k_topk_raw(int32_t dtype, const void* logits, int32_t rows, int32_t V, int32_t k, float* topk_v, int32_t* topk_i,
                     void* stream);
/* generate_candidates (utils.py:284-303) on device; HOST in/out: table [rows*k] draft-vocab ids, optional d2t [d2t_len],
 * tree_indices [T] (eb200_static_tree_buffers), out tree_candidates [T] */
int eb200_k_generate_candidates(const int32_t* table, int32_t rows, int32_t k, const int64_t* d2t, int32_t d2t_len,
                                const int32_t* tree_indices, int32_t T, int32_t sample_token, int64_t* tree_candidates);
/* tree build from a flattened candidate pool (cnets.py:760-827); HOST in/out for convenience.
 * scores[k+depth*k*k] float, tokens same int32, parents[1+depth*k] int32; outputs as eb200_get_tree. */
int eb200_k_tree_finalize(int32_t dtype, const float* scores, const int32_t* tokens, const int32_t* parents, int32_t k,
                          int32_t depth, int32_t total_token, int32_t sample_token, int32_t sort_rows,
                          int64_t* draft_tokens, float* tree_mask, int64_t* tree_position_ids, int64_t* retrieve_indices,
                          int32_t* n_leaf, int32_t* max_depth);
/* draft-tree growth (cnets.py:703-757) on host-supplied top-k tables: the level-0 seed, then one expansion per level.  HOST in/out.
 * topk_p / topk_i [1 + depth*k][k]: row 0 = top-k of the stable pass' last row, rows 1 + l*k .. 1 + (l+1)*k = top-k of the k
 * draft rows of level l (log-probs and draft-vocab ids); optional d2t [d2t_len]; last_row = the stable-pass row that seeds level 0.
 * Outputs (any may be NULL): the candidate pool as eb200_k_tree_finalize takes it -- scores / tokens [k + depth*k*k],
 * parents [1 + depth*k] -- and the frontier after the seed (slot 0) and after each level l (slot l + 1): front_ids / front_src /
 * front_cs / front_scores [depth + 1][k], front_mask [depth + 1][k][2] (ancestor bits over draft tree columns, word 1 = columns
 * 64..127).  k <= 32, depth <= 14, depth*k <= 128. */
int eb200_k_tree_grow(int32_t dtype, const float* topk_p, const int32_t* topk_i, const int64_t* d2t, int32_t d2t_len, int32_t k,
                      int32_t depth, int32_t last_row, float* scores, int32_t* tokens, int32_t* parents, int32_t* front_ids,
                      int32_t* front_src, int32_t* front_cs, float* front_scores, uint64_t* front_mask);
/* greedy posterior on a host-described tree (utils.py:360-373): node_argmax[T], draft_tokens[T],
 * retrieve[n_leaf*max_depth] -> best, accept_length, bonus token */
int eb200_k_greedy_accept(const int32_t* node_argmax, const int32_t* draft_tokens, const int32_t* retrieve, int32_t T,
                          int32_t n_leaf, int32_t max_depth, int32_t* best, int32_t* accept_length, int32_t* bonus);

/* sampling posterior on a host-described tree (utils.py:375-415 + the warpers of utils.py:38-54): logits is a DEVICE
 * [T][V] model-dtype tensor; uniforms (host) are consumed in order: one per candidate tried, then one for the bonus token */
int eb200_k_sample_posterior(int32_t dtype, const void* logits, int32_t V, const int32_t* draft_tokens, const int32_t* retrieve,
                             int32_t T, int32_t n_leaf, int32_t max_depth, float temperature, float top_p, int32_t top_k,
                             const float* uniforms, int32_t n_uniforms, int32_t* best, int32_t* accept_length, int32_t* bonus,
                             int32_t* uniforms_used);
/* softmax statistics of the warped rows (temperature -> top-p -> top-k) as the sampling posterior uses them: logits is a DEVICE
 * [rows][V] model-dtype tensor; stats (HOST) [rows][3] = max, sum, thr, where p(v) = lt_v >= thr ? exp(lt_v - max) / sum : 0 */
int eb200_k_sample_stats(int32_t dtype, const void* logits, int32_t rows, int32_t V, float temperature, float top_p, int32_t top_k,
                         float* stats);
/* one token drawn by inverse CDF from the warped logits row 0 (DEVICE [V], model dtype) with the uniform u: the draw of the
 * first token after prefill and of vanilla sampling; token (HOST) */
int eb200_k_sample_token(int32_t dtype, const void* logits, int32_t V, float temperature, float top_p, int32_t top_k, float u,
                         int32_t* token);

#ifdef __cplusplus
}
#endif
#endif /* EAGLE_B200_H_ */
