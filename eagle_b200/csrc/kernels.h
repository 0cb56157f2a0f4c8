// Host-side launcher declarations shared by the engine (engine.cu) and the kernel translation units.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <string>
#include <vector>
#include <stddef.h>
#include <stdint.h>

namespace eb {

// ----------------------------------------------------------------------------------------------
// Device-resident cycle state (int32 array).  Every kernel reads row counts / KV lengths from here,
// so one draft->verify->accept cycle is a fixed launch sequence with no host round trip inside.
// ----------------------------------------------------------------------------------------------
enum StateIdx : int {
  S_N = 0,        // committed target-KV length (== draft stable-KV length after the stable pass)
  S_NPREV = 1,    // committed length before the last accept
  S_ACC = 2,      // rows committed by the last accept (accept_length + 1)
  S_NLEAF = 3,    // leaves of the current tree
  S_MAXDEPTH = 4, // columns of retrieve_indices (max position id + 1)
  S_BEST = 5,     // best candidate row of the last accept
  S_BONUS = 6,    // bonus (next root) token of the last accept
  S_TMP0 = 7,     // scratch (prefill chunk base etc.)
  S_TMP1 = 8,
  S_LASTROW = 9,  // S_ACC - 1 (row whose draft logits seed level 0)
  S_ROWS = 10,    // generic dynamic row count slot
  S_NEWTOK = 11,  // total tokens committed since prefill
  S_UCOUNT = 12,  // uniforms consumed by the sampling posterior
  S_SNODE = 13,   // sampling: tree node whose distribution yields the bonus token
  S_SNREJ = 14,   // sampling: rejected candidates zeroed in that distribution
  S_COUNT = 16
};

enum Dtype : int { DT_BF16 = 0, DT_FP16 = 1 };

enum GemmEpilogue : int {
  EPI_STORE = 0,     // out = T(acc [+ bias])
  EPI_RESIDUAL = 1,  // out = T(T(acc) + res)
  EPI_SWIGLU = 2,    // out = T(T(silu(T(gate))) * T(up))      (two weight tiles per stage)
  EPI_QKV_ROPE = 3,  // q -> q buffer (rope), k -> K cache (rope), v -> V cache; one 128-row tile == one head
  EPI_PARTIAL_F32 = 4,  // out(float) = acc, unrounded: a tensor-parallel rank's partial sum, all-reduced before the residual add
  // SwiGLU over ONE weight matrix whose 128-row tiles interleave 64 gate rows with the 64 up rows of the same output
  // columns (the engine's layout): a single accumulator per tile, 2x the CTAs of EPI_SWIGLU, no second W stream.
  // N counts the interleaved rows (2 x intermediate); out[m, 64*tile + r] for r < 64.
  EPI_SWIGLU_IL = 5,
};

// value = (idx >= 0 ? st[idx] : 0) + add
struct DynInt {
  int idx;
  int add;
};

struct GemmParams {
  int N, K;          // weight rows (output features), reduction length
  int m_rows;        // static bound on valid activation rows (<= MPAD)
  int m_idx;         // >= 0: additionally clamp to st[m_idx]
  const int* st;     // device state
  int splitk;
  int w4_quant;      // launch_gemm_w4: code table of the 4-bit weights (W4_NF4 / W4_FP4); fills the padding before ws
  float* ws;         // split-K partials  [split][acc][MPAD][n_tiles*128]
  int* counters;     // per-n-tile arrival counters (self-resetting)
  // EPI_STORE / RESIDUAL / SWIGLU
  void* out;
  long ld_out;
  const void* bias;
  const void* res;
  long ld_res;
  // EPI_SWIGLU / EPI_SWIGLU_IL: T(silu(g)) for every 16-bit pattern g of the model dtype (filled in by the launchers)
  const void* silu_lut;
  // EPI_QKV_ROPE
  void* q_out;       // [MPAD][n_q_heads*128]
  void* k_cache;     // [n_kv_heads][kv_cap][128]
  void* v_cache;
  long kv_cap;       // rows per kv head plane
  int n_q_heads, n_kv_heads;
  const void* rope_cos;  // [n_pos][64]
  const void* rope_sin;
  DynInt pos_base;       // rope position of row m = pos_base + pos_arr[m] (if non-null) + pos_mstride*m
  const int* pos_arr;
  int pos_mstride;
  DynInt kv_base;        // K/V rows are appended at kv_base + m
  // launch_gemm_w8: fp32 scale of each int8 weight row [N] (bitsandbytes' SCB, the row absmax)
  const float* w_scale;
};

// L2 prefetch of the weight tiles a later skinny_gemm_wgmma launch reads first.  Weights depend on no kernel, so a kernel that
// leaves HBM idle (attention, RMSNorm, a GEMM's drain) can fetch them before its griddepcontrol.wait.  That GEMM runs the grid
// n_tiles x splitk over num_kb k-blocks; split s reads k-blocks [kb_begin(s), kb_end(s)) in order.  The plan covers k-block
// kb_begin(s) + j of every (n-tile, split) for j in [j0, j1): all CTAs of that GEMM are resident at once, so j-major is the
// order in which it consumes them.  j1 <= j0 prefetches nothing.  Host side: l2_plan in engine.cu.
struct alignas(64) L2Prefetch {
  CUtensorMap tm;  // the weight's map (box 128 rows x 64 K-elements, as the GEMM loads it)
  int n_tiles, splitk, num_kb;
  int j0, j1;
};

// Returns cudaError_t-compatible int (0 = ok).  mpad in {16, 64}.  tm* are HOST pointers to encoded maps.
// pf (optional): after its last weight load, the producer lane of every CTA prefetches its share of that plan (the GEMM that
// follows), so HBM keeps streaming while this launch drains (cluster reduction, epilogue) and the next kernels ramp.
int launch_gemm(int dtype, int mpad, int epi, const CUtensorMap* tmW, const CUtensorMap* tmW2, const CUtensorMap* tmX,
                const GemmParams& p, cudaStream_t s, const L2Prefetch* pf = nullptr);
// W8A16 form of launch_gemm: tmW maps an int8 [N][K] weight (make_tmap_w8 layout: box 128 rows x 64 bytes, no swizzle) and
// p.w_scale its row scales.  The kernel forms W' = T((q * scale) * kInv127) in shared memory and runs the same wgmma sequence and
// epilogue as launch_gemm, so the result is bit-identical to launch_gemm on W'.  mpad 16 / 64: EPI_STORE, EPI_RESIDUAL,
// EPI_QKV_ROPE, EPI_SWIGLU_IL; mpad 256: the last three.
int launch_gemm_w8(int dtype, int mpad, int epi, const CUtensorMap* tmW, const CUtensorMap* tmX, const GemmParams& p, cudaStream_t s,
                   const L2Prefetch* pf = nullptr);
// W4A16 form (bitsandbytes nf4 / fp4 with blocksize 64): tmW maps the nibble tiles written by launch_w4_repack (2-D, rows of 256 B,
// box 256 x 16 = one 4 KB tile), tmA the transposed absmax [K/64][n_pad] (box 128 x 1).  The MMA warpgroups convert each k16 step of
// nibbles into their wgmma A fragments, W' = T(code[q] * absmax) (one fp32 product, one round-to-nearest cast), while the previous
// step's MMA runs, so the result is bit-identical to launch_gemm on W'.  Epilogues and mpad as launch_gemm_w8.
enum W4Quant : int { W4_NF4 = 0, W4_FP4 = 1 };
int launch_gemm_w4(int dtype, int mpad, int epi, const CUtensorMap* tmW, const CUtensorMap* tmA, const CUtensorMap* tmX, const GemmParams& p,
                   cudaStream_t s, const L2Prefetch* pf = nullptr);
// Load-time repack of bitsandbytes' 4-bit layout into the kernel's.  Source row i (of nr) of a [nr][K/2] nibble matrix (element 2j in
// the high nibble of byte j) and of its [nr][K/64] absmax goes to destination row d(i) = row0 + i, or, for half >= 0, to the gate/up
// interleave (i / 64) * 128 + half * 64 + i % 64.  Nibbles land in tiles [n_pad / 128][K / 64][4096 B], each thread's four k16 steps of
// A-fragment bytes contiguous (16 B); absmax lands transposed in [K / 64][n_pad].  K % 64 == 0.
int launch_w4_repack(const uint8_t* src, const float* src_absmax, int nr, int K, int row0, int half, uint8_t* dst, float* dst_absmax,
                     int n_pad, cudaStream_t s);
// W8A16 form on FP8 weights (transformers' FineGrainedFP8Config: e4m3, one fp32 weight_scale_inv per 128 x 128 block): tmW maps the
// e4m3 [N][K] written by launch_fp8_repack exactly like an int8 weight (box 128 rows x 64 bytes, so the L2 prefetch plan applies
// unchanged), tmS the block scales [N / 128][K / 128][4] fp32 (box 4 x 1).  The MMA warpgroups convert each k16 step into their
// wgmma A fragments, W' = T(fp32(q) * scale) (one fp32 product, one round-to-nearest cast), while the previous step's MMA runs, so
// the result is bit-identical to launch_gemm on W'.  N % 128 == 0, K % 128 == 0; epilogues and mpad as launch_gemm_w8.
int launch_gemm_fp8(int dtype, int mpad, int epi, const CUtensorMap* tmW, const CUtensorMap* tmS, const CUtensorMap* tmX, const GemmParams& p,
                    cudaStream_t s, const L2Prefetch* pf = nullptr);
// Load-time repack of transformers' FP8 layout into the kernel's.  Source row i (of nr, a multiple of 128) of an e4m3 [nr][K] matrix
// goes to destination row d(i) = row0 + i (row0 % 64 == 0), or, for half >= 0, to the gate/up interleave (i / 64) * 128 + half * 64 +
// i % 64; within each 128 x 64 tile the bytes are permuted so that thread t of the MMA warpgroups finds its A-fragment bytes of k16
// steps 0, 1 at 16 t and of steps 2, 3 at 4096 + 16 t.  The scales [nr / 128][K / 128] land per 64-row destination group: entry
// (d / 64) % 2 of [n_rows / 128][K / 128][4] (entries 2, 3 stay as they are).  K % 128 == 0, n_rows % 128 == 0.
int launch_fp8_repack(const uint8_t* src, const float* src_scale, int nr, int K, int row0, int half, uint8_t* dst, float* dst_scale,
                      int n_rows, cudaStream_t s);
// bring-up / debugging aid: same epilogues, plain FMA main loop, no TMA/wgmma.  W/W2/X are raw pointers.
int launch_gemm_simt(int dtype, int mpad, int epi, const void* W, const void* W2, const void* X, long ldx,
                     const GemmParams& p, cudaStream_t s);
// Device table lut[bits(g)] = T(g / (1 + exp(-g))) over all 65536 patterns of the model dtype: the SwiGLU epilogues look the
// activation up instead of evaluating exp + divide per element (same values by construction).  Built once per device on `s`.
const void* silu_lut(int dtype, cudaStream_t s);
// How many bytes of dynamic shared memory / pipeline stages the wgmma kernel uses (for reporting)
int gemm_stage_count(int mpad, int epi);

// ----------------------------------------------------------------------------------------------
// lm_head GEMM (mega.cu): ONE launch of one CTA per SM, CTA c owns the whole 128-row weight tiles c, c+G, ...; the epilogue
// finishes each tile straight from the staged accumulators (no split-K, no partials in global memory).
// ----------------------------------------------------------------------------------------------
enum ChainFinish : int {
  FIN_ARGMAX,        // per-tile (max, first index) from the staged tile, merged per row (verify lm_head)
  FIN_STORE_DIRECT,  // out = T(acc [+ bias]) from the staged tile                  (lm_head, sampling path)
};
struct ChainPhase {
  int N, K;      // weight rows, reduction length
  int fin;       // ChainFinish
  // FIN_STORE_DIRECT
  void* out;
  long ld_out;
  const void* bias;
  // FIN_ARGMAX
  float* tile_val;  // [n_tiles][64]
  int* tile_idx;    // [n_tiles][64]
  int* out_idx;     // [rows]
  int idx_offset;   // tensor parallel: first vocabulary row of this rank's lm_head shard
};
// Tensor parallelism over NVLink peer memory: every rank's "window" (one cudaMalloc block, opened on the peers through CUDA
// IPC) holds the replicated activations (x, xn, feature taps), a per-source inbox for fp32 partial rows, the row flags and
// the lm_head's arg-max exchange.  The row-parallel projections (o_proj, down_proj) finish in tp_fused.cu behind the
// per-projection GEMMs; the vocabulary-parallel arg-max of the lm_head exchanges its (value, index) pairs in the chain launch.
constexpr int kMaxTp = 8;
struct ChainTP {
  int size, rank;
  char* win[kMaxTp];        // window base of every rank as mapped in THIS process (win[rank] = the local one)
  long inbox_off;           // float [tp][64][ld_inbox]
  long ld_inbox;
  long flag_off;            // int [tp][64]: epoch of the last row pushed by (src, m)
  long ready_off;           // 1 KB block, ints [64, 128): row flags of the two-shot exchange (tp_fused.cu)
  long am_off;              // arg-max exchange: float2-like {val, idx} [tp][64], then int flags [tp][64]
  int* epoch;               // local: exchanges executed so far (monotonic; identical on every rank)
};
// standalone form of the same exchange behind the per-projection GEMMs (tp_fused.cu): all-reduce + residual + RMSNorm in one launch
struct TpResidParams {
  ChainTP tp;
  const float* partial;  // this rank's unrounded partial sums [rows][ld_partial] (EPI_PARTIAL_F32)
  long ld_partial;
  int N;
  void* x;               // in the window; in place unless res != nullptr
  long ld_x;
  const void* res;
  long ld_res;
  void* tap;             // optional, in the window
  long ld_tap;
  const void* norm_w;    // optional RMSNorm weight -> xn (in the window)
  void* xn;
  long ld_xn;
  float eps;
};
int launch_tp_resid_norm(int dtype, const TpResidParams& p, int rows, cudaStream_t s);
struct ChainArgs {
  ChainTP tp;
  int m_rows, m_idx;  // valid activation rows = min(m_rows, st[m_idx]) (m_idx < 0: m_rows)
  const int* st;
  int* sync;          // >= 2 zeroed ints, owned by this stream (self-resetting)
  // optional in-kernel timing (works inside a replayed CUDA graph, no profiler): [0] += ns from "dependencies resolved" on CTA 0
  // to the exit of the last CTA, [1] += 1 per launch, [2] scratch (start stamp of the running launch)
  unsigned long long* timing;
  ChainPhase ph;
};
struct ChainMaps {
  CUtensorMap w;  // weights [N][K], box 128 x 64
  CUtensorMap x;  // activations [64][K], box mpad x 64
};
int launch_gemm_chain(int dtype, int mpad, const ChainMaps& maps, const ChainArgs& args, cudaStream_t s);
// can an [N, K] weight run through the lm_head launch on the current device?  (TMA row stride, device attributes)
bool chain_phase_ok(int N, int K);

// ----------------------------------------------------------------------------------------------
// elementwise / reduction kernels (misc.cu)
// ----------------------------------------------------------------------------------------------
// y[m, col_off : col_off+H] = w * T(x_row * rsqrt(mean(x_row^2) + eps));  x_row = src[row_ids ? row_ids[m] : m]
// pf (optional, also for launch_e3_input): weight tiles of the GEMM that follows, prefetched into L2 at kernel start
int launch_rmsnorm(int dtype, const void* src, long ld_src, const int64_t* row_ids64, const int* row_ids32,
                   const void* w, void* y, long ld_y, int col_off, int H, float eps, int rows, cudaStream_t s, const L2Prefetch* pf = nullptr);
// EAGLE-3 draft input: cat[m] = (w_emb * norm(table[ids[m]]), w_hid * norm(h_m)) with h_m = hsrc[src_rows ? src_rows[m] : m]
// (src_rows: also copies h_m to hdst[m])
int launch_e3_input(int dtype, const void* table, long ld_table, const int64_t* ids64, const int* ids32, const void* w_emb, const void* hsrc,
                    long ld_hsrc, const int* src_rows, void* hdst, long ld_hdst, const void* w_hid, void* cat, long ld_cat, int H, float eps,
                    int rows, cudaStream_t s, const L2Prefetch* pf = nullptr);
// dst[m, col_off: col_off+H] = table[ids[m]]
int launch_gather_rows(int dtype, const void* table, long ld_table, const int64_t* ids64, const int* ids32, void* dst,
                       long ld_dst, int col_off, int H, int rows, cudaStream_t s);
// out_idx[m] = first argmax over logits[m, :V]
int launch_argmax(int dtype, const void* logits, long ld, int V, int rows, int* out_idx, cudaStream_t s);
// per row: log-softmax in fp32 rounded to T (raw != 0: the logits themselves), then top-k (value desc, index asc).
// row = (row_idx>=0 ? st[row_idx] : 0) + blockIdx
int launch_logsoftmax_topk(int dtype, const void* logits, long ld, int V, int rows, const int* st, int row_idx, int k, int raw,
                           float* topk_p, int* topk_i, cudaStream_t s);
// tensor parallel: x[m, n] = T(T(sum[m, n]) + x[m, n]) after the all-reduce of the row-parallel partial sums
int launch_residual_add_f32(int dtype, const float* sum, void* x, int rows, int H, cudaStream_t s);
// arg-max with value over the first V_valid columns: out_val[m] (model-dtype value as float), out_idx[m] (+ idx_offset)
int launch_argmax_val(int dtype, const void* logits, long ld, int V_valid, int rows, int idx_offset, float* out_val, int* out_idx,
                      cudaStream_t s);
// merge per-rank (value, index) pairs (rank r at vals + r*stride, idxs + r*stride) -> out_idx[rows]; ties -> lowest index
int launch_argmax_merge(const float* vals, const int* idxs, int n_ranks, int rows, int stride, int* out_idx, cudaStream_t s);
int launch_set_state(int* st, int idx, int value, cudaStream_t s);
int launch_state_to(int* dst, const int* st, int idx, cudaStream_t s);
int launch_unshard_rows(const void* in, void* out, int ranks, int rows, int cols, cudaStream_t s);
int launch_copy_state(int* st, int dst_idx, int src_idx, int add, cudaStream_t s);

// ----------------------------------------------------------------------------------------------
// attention (attention.cu): q rows attend to ctx [0, n_ctx) plus tree columns n_ctx + j where bit j of mask[row]
// ----------------------------------------------------------------------------------------------
struct AttnParams {
  const void* q;        // [rows][n_heads*128]
  const void* k_cache;  // [n_kv][kv_cap][128]
  const void* v_cache;
  // TMA descriptors (host pointers) of the two planes viewed as [n_kv * kv_cap][128], box 64 rows x 64 columns, SWIZZLE_128B
  const CUtensorMap* tmK;
  const CUtensorMap* tmV;
  void* out;            // [rows][n_heads*128]
  long kv_cap;
  int n_heads, n_kv_heads;
  int rows;             // static bound on q rows
  int rows_idx;         // >= 0: clamp to st[rows_idx]
  const int* st;
  DynInt n_ctx;         // fully visible prefix length
  int n_tree;           // tree columns appended after the prefix (<= 128)
  const uint64_t* mask; // [rows][2] ancestor bits over the tree columns; nullptr => causal (row r sees columns 0..r)
  int max_kv;           // capacity used to size shared memory (n_ctx + n_tree <= max_kv)
  unsigned long long* trace;  // optional (EB200_ATTN_TRACE): [n_ctas][16] %globaltimer stamps of thread 0 at the phase boundaries
  // optional (host pointer): weight tiles of the GEMM that follows; every CTA prefetches its share into L2 at kernel start, so
  // HBM keeps streaming while this latency-bound kernel runs
  const L2Prefetch* pf;
  // caps on the query heads per CTA and on the KV split, each 1, 2 or 4; 0 = the EB200_ATTN_HPC / EB200_ATTN_KVS policy
  int hpc_cap, kvs_cap;
};
// Launch geometry of the attention kernel for a score strip of max_kv columns: HPC query heads of one kv head per CTA, a KV
// split over a cluster of KVS CTAs (each holds kv_stride strip columns per row) and the dynamic shared memory.  Host only.
struct AttnGeometry {
  int hpc, kvs, kv_stride;
  size_t smem;
};
// 0, or cudaErrorInvalidValue when a cap is not 0/1/2/4 or the strip does not fit in shared memory
int attention_geometry(int max_kv, int n_heads, int n_kv_heads, int hpc_cap, int kvs_cap, AttnGeometry* g);
// largest max_kv the kernel accepts under the default caps (16896 with EB200_ATTN_KVS unset)
int attention_max_kv();
int launch_attention(int dtype, const AttnParams& p, cudaStream_t s);

// ----------------------------------------------------------------------------------------------
// tree / accept / compaction kernels (tree.cu)
// ----------------------------------------------------------------------------------------------
struct TreeBuffers {
  // candidate pool, flattened level-major exactly like the reference (cnets.py:760-761)
  float* scores;     // [k + depth*k*k]
  int* tokens;       // same, target-vocab ids
  int* parents;      // [1 + depth*k]
  // frontier of the current level
  float* front_scores;  // [k]
  int* front_ids;       // [k] tokens fed to the next draft forward
  int* front_src;       // [k] row of the previous level's output feeding each slot
  uint64_t* front_mask; // [k][2] ancestor bits over draft-KV tree columns
  int* front_cs;        // [k] topk_cs_index of the previous level
  // finished tree
  int* draft_tokens;    // [T]
  uint64_t* tree_mask;  // [T][2] (ancestor bits over tree nodes; word 1 always 0 for T <= 64)
  int* tree_pos;        // [T]
  int* retrieve;        // [T][depth+2], -1 padded, rows < n_leaf valid
  int* parent_node;     // [T]
};
// level 0: seed the pool from the stable pass' top-k (cnets.py:703-716)
int launch_tree_seed(const float* topk_p, const int* topk_i, const int64_t* d2t, int k, TreeBuffers tb, int* st,
                     cudaStream_t s);
// level i expansion (cnets.py:728-757)
int launch_tree_expand(int dtype, const float* topk_p, const int* topk_i, const int64_t* d2t, int k, int level,
                       TreeBuffers tb, cudaStream_t s);
// global rerank + mask / positions / retrieve (cnets.py:760-827)
int launch_tree_finalize(int dtype, int k, int depth, int total /* T-1 */, int sort_rows, TreeBuffers tb, int* st,
                         cudaStream_t s);
// greedy posterior (utils.py:360-373) + commit bookkeeping (utils.py:435-441, :458-464)
struct AcceptOut {
  int* accepted_tokens;  // [depth+2]
  int* sel_nodes;        // [depth+2] tree-node index of each committed row
  int64_t* host_visible; // optional pinned mirror: [0]=accept rows, [1]=bonus, [2..] tokens
};
int launch_greedy_accept(const int* node_argmax, TreeBuffers tb, int T, int depth, AcceptOut out, int* st,
                         int64_t* out_ids, int out_cap, cudaStream_t s);
// ---- sampling posterior (utils.py:375-415 with the warpers of utils.py:38-54) ----
struct SampleParams {
  float temperature, top_p;
  int top_k;
  unsigned long long seed;
  const float* uniforms;  // optional injected uniforms (tests); consumed in order, then the counter RNG takes over
  int n_uniforms;
};
struct RowStats {  // softmax statistics of one (warped) logits row: p(v) = lt_v >= thr ? exp(lt_v - max) / sum : 0
  float max, sum, thr, pad;
};
int launch_row_softmax_stats(int dtype, const void* logits, long ld, int V, int rows, SampleParams sp, RowStats* stats, cudaStream_t s);
// sequential multi-candidate speculative sampling over the current tree; leaves (best, accept_length) in the state and the
// bonus-token spec (node, rejected tokens) for launch_sample_commit
int launch_sample_posterior(int dtype, const void* logits, long ld, int V, const RowStats* stats, TreeBuffers tb, int depth, SampleParams sp,
                            int* rej_tokens, int* st, cudaStream_t s);
// inverse-CDF sample of the bonus token from row st[S_SNODE] (minus the rejected tokens), then the commit bookkeeping.
// first_token != 0: prefill mode (row 0 of `logits`, no tree): only writes st[S_BONUS].
int launch_sample_commit(int dtype, const void* logits, long ld, int V, const RowStats* stats, TreeBuffers tb, int depth, SampleParams sp,
                         const int* rej_tokens, AcceptOut out, int* st, int64_t* out_ids, int out_cap, int first_token, cudaStream_t s);
// KV compaction (utils.py:444-452): rows N+sel[j] -> N+j for every plane
int launch_kv_compact(int dtype, void* kv_base, long plane_stride, int n_planes, long kv_cap, const int* sel,
                      const int* st, cudaStream_t s);

// ----------------------------------------------------------------------------------------------
// static draft tree (static_tree.cu): utils.py:89-207,284-303 and modeling_eagle.py:562-692,863-957
// ----------------------------------------------------------------------------------------------
constexpr int kStaticMaxNodes = 128;
struct StaticTreeHost {
  int n_choices = 0, T = 0, topk = 0;
  int width = 0;    // longest root-to-leaf path in nodes (= max choice length + 1)
  int n_leaf = 0;
  // verify side (node 0 = root, node i+1 = i-th choice sorted by (depth, lexicographic))
  std::vector<int> tree_indices, pos, parent;  // [T]
  std::vector<uint64_t> mask;                  // [T][2] ancestor bits (bit 0 and the node's own bit always set)
  std::vector<int> retrieve;                   // [n_leaf][width], -1 padded, rows sorted with -1 last
  // draft side: level l feeds count[l] nodes-with-children to the head; cum = running total (draft-KV tree columns)
  int n_levels = 0;
  std::vector<int> count, cum;
  std::vector<int> sel, src;      // concatenated over levels: index into the previous level's [rows][topk] table, source row
  std::vector<uint64_t> lmask;    // concatenated [inner][2]: ancestor bits over the nodes-with-children
};
// returns 0 or 1 with a message in err
int build_static_tree(const int32_t* choices, const int32_t* choice_len, int n, int topk, StaticTreeHost& t, std::string& err);
struct StaticLevelArgs {
  const int* topk_i;       // [rows_prev][k] draft-vocab indices of the previous pass
  const int64_t* d2t;      // optional draft->target offset table
  int k, rows_prev, ss_row0;
  int* ss_tokens;          // flattened top-k table in target-vocab ids
  int count;               // rows fed to the next draft pass (0 on the final call)
  const int* sel;
  const int* src;
  const uint64_t* lmask;
  int first;               // level 0: every row takes the hidden state of the stable pass' last row
  int final_T;             // > 0: also gather the T candidate tokens and publish n_leaf / width
  const int* tree_indices;
  int n_leaf, width;
};
int launch_static_level(const StaticLevelArgs& a, TreeBuffers tb, int* st, cudaStream_t s);

}  // namespace eb
