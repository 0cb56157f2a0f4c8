// Persistent GEMM chain for sm_90a: up to four dependent skinny-M weight-streaming GEMMs in one launch.
//
// Why: at batch 1 every projection of the verify pass is HBM-bound on its weights, but a chain of ~10 dependent kernels
// per layer pays a launch/drain/fill bubble around each projection's weight stream (DESIGN.md 10: ~316 launches per
// cycle).  Here one CTA per SM stays resident for a whole
// layer segment
//     o_proj(+residual) -> RMSNorm -> gate/up(SwiGLU) -> down_proj(+residual) -> RMSNorm -> next layer's qkv(+RoPE,+KV append)
// (or ... -> final norm -> lm_head(arg-max) for the last layer) and
//   * the WEIGHT producer (one lane) walks the whole task list without ever waiting for a phase boundary: the next
//     projection's tiles fill the shared-memory ring while the current one is reduced, so HBM never idles;
//   * every phase is split stream-K style: CTA c owns units [c*U/G, (c+1)*U/G) of the (n-tile, k-block) grid, so all
//     SMs stream the same number of bytes whatever the tile count (32 / 48 / 224 tiles);
//   * an MMA warpgroup accumulates each (tile, k-range) segment with wgmma in registers and hands it to the epilogue warps
//     through a shared-memory staging tile; they drain it as an fp32 partial tile into an L2-resident workspace while the
//     next segment's MMAs run;
//   * a global arrival counter per phase replaces the kernel boundary (release/acquire at gpu scope);
//   * the FINISH step runs row-wise on the first rows*chunks CTAs: fixed-order split-K reduction (deterministic) + the
//     reference's epilogue arithmetic with its rounding points + the RMSNorm feeding the next phase (the row is complete
//     inside one CTA, so the norm costs no extra pass, launch or barrier);
//   * the ACTIVATION producer (another lane) waits for the finish counter of the previous phase and then TMA-loads the
//     X tiles of its k-blocks behind the already-resident W tiles.
// The lm_head (1002 tiles) runs in "direct" mode: whole tiles per CTA, per-row (max, first index) straight from the staged tile,
// merged per row in the finish step: the 15.4 MB logits round trip and the arg-max launch disappear.
//
// Status (DESIGN.md 6): the single-phase lm_head(+arg-max) form is the default; the multi-phase layer chain is parity-green
// but its row-wise finish reads the split-K partials through one SM's load/store path, where the per-projection kernels
// reduce through distributed shared memory, so it stays opt-in (EB200_CHAIN=1).
//
// Replaces (per layer) modeling_llama_kv.py:801-863 (decoder layer), :118-132 (RMSNorm), :501-535 (MLP) op sites.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "gemm_common.cuh"

namespace eb {

constexpr int kChainThreads = 320;   // warps 0-3 MMA, warps 4-7 epilogue/finish, warp 8 W producer, warp 9 X producer
constexpr int kChainMaxSlots = 4;    // partial tiles one CTA may produce per phase
constexpr int kChainMaxStages = 12;
constexpr int kChainCtrlBytes = 8192;
constexpr int kChainMaxTableTiles = 448;
constexpr int kSyncPartials = 0;     // [4] CTAs that have written all partials of phase p
constexpr int kSyncReady = 4;        // [4] finish items of phase p completed
constexpr int kSyncExit = 8;

// ------------------------------------------------------------------------------------------------------------
// small device helpers
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_gpu_add(int* p, int v) {
  asm volatile("red.release.gpu.global.add.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }
// Bounded spin: a mis-programmed chain traps (CUDA error on the host) instead of hanging the GPU.  No printf in this kernel:
// ptxas serialises every wgmma of a kernel in which a call may run while MMAs are in flight (see mbar_wait_mma).
__device__ __forceinline__ void spin_until_ge(const int* p, int target) {
  uint32_t n = 0;
  while (ld_acquire_gpu(p) < target) {
    __nanosleep(32);
    if (++n > (1u << 23)) __trap();
  }
}
__device__ __forceinline__ void chain_epi_bar() { asm volatile("bar.sync 1, 128;" ::: "memory"); }
// ---- system scope (other GPUs over NVLink peer memory) ----
__device__ __forceinline__ int ld_acquire_sys(const int* p) {
  int v;
  asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(int* p, int v) { asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ void red_release_sys_add(int* p, int v) {
  asm volatile("red.release.sys.global.add.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long chain_gtimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// wait for a peer GPU: the peers run the same launch sequence but are not lock-stepped (host launch skew in eager mode), so the
// bound is wall-clock (20 s), not an iteration count
__device__ __forceinline__ void spin_until_ge_sys(const int* p, int target) {
  unsigned long long t0 = 0;
  uint32_t n = 0;
  while (ld_acquire_sys(p) - target < 0) {
    __nanosleep(64);
    if ((++n & 4095u) == 0) {
      const unsigned long long now = chain_gtimer();
      if (!t0) t0 = now;
      if (now - t0 > 20000000000ull) __trap();
    }
  }
}
template <typename P> __device__ __forceinline__ P* peer_ptr(const ChainTP& tp, P* local, int r) {
  return reinterpret_cast<P*>(tp.win[r] + (reinterpret_cast<char*>(local) - tp.win[tp.rank]));
}

struct Geo {
  int nkb, ntiles;
  uint32_t U;
  bool direct;
};
__device__ __forceinline__ Geo geo_of(const ChainPhase& ph) {
  Geo g;
  g.nkb = (ph.K + kBlockK - 1) / kBlockK;
  g.ntiles = (ph.N + kBlockN - 1) / kBlockN;
  g.U = static_cast<uint32_t>(g.nkb) * static_cast<uint32_t>(g.ntiles);
  g.direct = ph.fin == FIN_ARGMAX || ph.fin == FIN_STORE_DIRECT;
  return g;
}
// first unit of CTA c (U * G < 2^31 is checked on the host)
__device__ __forceinline__ uint32_t unit0(uint32_t U, int c, int G) { return (U * static_cast<uint32_t>(c)) / static_cast<uint32_t>(G); }

// f(tile, kb_begin, kb_end, slot) for every (tile, k-range) segment of CTA `cta`, in execution order
template <typename F> __device__ __forceinline__ void for_each_segment(const Geo& g, int cta, int G, F&& f) {
  if (g.direct) {
    for (int t = cta; t < g.ntiles; t += G) f(t, 0, g.nkb, 0);
  } else {
    uint32_t u = unit0(g.U, cta, G);
    const uint32_t u1 = unit0(g.U, cta + 1, G);
    int j = 0;
    while (u < u1) {
      const int t = static_cast<int>(u / static_cast<uint32_t>(g.nkb));
      const int a = static_cast<int>(u - static_cast<uint32_t>(t) * g.nkb);
      const int b = min(g.nkb, a + static_cast<int>(u1 - u));
      f(t, a, b, j);
      u += static_cast<uint32_t>(b - a);
      ++j;
    }
  }
}

// The weight producer's view of the same schedule: one (phase, tile, k-block) unit at a time, without segment bookkeeping, so
// that a second cursor can run ahead of the loads and prefetch into L2 while the shared-memory ring is full.
struct UnitCursor {
  int p, t, kb, nkb, ntiles;
  uint32_t u, u1;
  bool direct, done;
};
__device__ __forceinline__ void cursor_enter_phase(UnitCursor& c, const ChainArgs& args, int cta, int G) {
  while (c.p < args.n_phases) {
    const Geo g = geo_of(args.ph[c.p]);
    c.nkb = g.nkb;
    c.ntiles = g.ntiles;
    c.direct = g.direct;
    if (g.direct) {
      c.t = cta;
      c.kb = 0;
      if (c.t < g.ntiles) return;
    } else {
      c.u = unit0(g.U, cta, G);
      c.u1 = unit0(g.U, cta + 1, G);
      if (c.u < c.u1) {
        c.t = static_cast<int>(c.u / static_cast<uint32_t>(g.nkb));
        c.kb = static_cast<int>(c.u - static_cast<uint32_t>(c.t) * g.nkb);
        return;
      }
    }
    ++c.p;
  }
  c.done = true;
}
__device__ __forceinline__ void cursor_advance(UnitCursor& c, const ChainArgs& args, int cta, int G) {
  if (++c.kb == c.nkb) {
    c.kb = 0;
    c.t += c.direct ? G : 1;
  }
  bool phase_done;
  if (c.direct) phase_done = (c.kb == 0 && c.t >= c.ntiles);
  else phase_done = (++c.u == c.u1);
  if (phase_done) {
    ++c.p;
    cursor_enter_phase(c, args, cta, G);
  }
}
__device__ __forceinline__ void tma_prefetch_l2_2d(const CUtensorMap* m, int c0, int c1) {
  asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];" ::"l"(reinterpret_cast<uint64_t>(m)), "r"(c0), "r"(c1)
               : "memory");
}

// per-tile contributor table (shared memory): CTAs [c_first, c_last] hold partials of tile t; the first one at slot
// slot_first, every later one at slot 0 (its range starts inside the tile)
struct TileSrc {
  short c_first, c_last, slot_first, pad;
};
__device__ __forceinline__ void build_tile_table(TileSrc* tab, const Geo& g, int G, int etid) {
  for (int t = etid; t < g.ntiles; t += 128) {
    const uint32_t lo = static_cast<uint32_t>(t) * g.nkb, hi = lo + g.nkb;
    int c = static_cast<int>((static_cast<uint64_t>(lo) * G) / g.U);
    while (c + 1 < G && unit0(g.U, c + 1, G) <= lo) ++c;
    while (c > 0 && unit0(g.U, c, G) > lo) --c;
    int cl = c;
    while (cl + 1 < G && unit0(g.U, cl + 1, G) < hi) ++cl;
    TileSrc s;
    s.c_first = static_cast<short>(c);
    s.c_last = static_cast<short>(cl);
    s.slot_first = static_cast<short>(t - static_cast<int>(unit0(g.U, c, G) / g.nkb));
    s.pad = 0;
    tab[t] = s;
  }
}
// sum over all contributors (ascending CTA == ascending k: deterministic) of rows [r, r+4) of tile t, activation row m.
// The loads of one call are independent and issued back to back (up to 8 in flight): the finish is an L2-latency problem, a
// load -> add -> load chain would cost a full L2 round trip per contributor.
template <int MPAD>
__device__ __forceinline__ float4 reduce4(const float* ws, const TileSrc* tab, const Geo& g, int G, int t, int m, int r) {
  const TileSrc s = tab[t];
  const long row_off = static_cast<long>(m) * kBlockN + r;
  const int n = s.c_last - s.c_first + 1;
  const bool sparse = g.U < static_cast<uint32_t>(G);  // tiny problems: some CTAs own no unit at all
  if (n <= 8 && !sparse) {
    float4 v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = s.c_first + j;
      const int slot = (j == 0) ? s.slot_first : 0;
      if (j < n) v[j] = __ldcg(reinterpret_cast<const float4*>(ws + (static_cast<long>(c) * kChainMaxSlots + slot) * MPAD * kBlockN + row_off));
      else v[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    float4 acc = v[0];
#pragma unroll
    for (int j = 1; j < 8; ++j) {
      acc.x += v[j].x;
      acc.y += v[j].y;
      acc.z += v[j].z;
      acc.w += v[j].w;
    }
    return acc;
  }
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int c = s.c_first; c <= s.c_last; ++c) {
    if (sparse && unit0(g.U, c + 1, G) == unit0(g.U, c, G)) continue;
    const int slot = (c == s.c_first) ? s.slot_first : 0;
    const float4 v = __ldcg(reinterpret_cast<const float4*>(ws + (static_cast<long>(c) * kChainMaxSlots + slot) * MPAD * kBlockN + row_off));
    acc.x += v.x;
    acc.y += v.y;
    acc.z += v.z;
    acc.w += v.w;
  }
  return acc;
}

// The row-wise pull-reduce is bound by the L2 latency seen by one SM's load/store path (its in-flight sectors are bounded),
// not by the load flavour (ld.cg or weak): the loads of a batch are therefore all issued before the first add.
__device__ __forceinline__ float4 ld_partial(const float* p) { return __ldcg(reinterpret_cast<const float4*>(p)); }
// Branch-free batch: NB (tile, row-offset) requests x up to MAXC contributors each, ALL loads issued before the first add.
// An L2 round trip between SMs is expensive under load; the finish must pay it once or twice per item, not once per pass.  Callers check chain_fast_path(g, G, MAXC) (phase-uniform) first.
__device__ __forceinline__ bool chain_fast_path(const Geo& g, int G, int maxc) {
  if (g.U < static_cast<uint32_t>(G)) return false;
  const int per = static_cast<int>(g.U / static_cast<uint32_t>(G));
  return (g.nkb + per - 2) / per + 1 <= maxc;
}
template <int MPAD, int NB, int MAXC>
__device__ __forceinline__ void reduce4_batch(const float* ws, const TileSrc* tab, const int (&t)[NB], const int (&r)[NB], const bool (&ok)[NB],
                                              int m, float4 (&out)[NB]) {
  const float* base[NB];
  int cnt[NB];
  long first_off[NB];
#pragma unroll
  for (int u = 0; u < NB; ++u) {
    cnt[u] = 0;
    base[u] = ws;
    first_off[u] = 0;
    if (ok[u]) {
      const TileSrc s = tab[t[u]];
      cnt[u] = s.c_last - s.c_first + 1;
      base[u] = ws + (static_cast<long>(s.c_first) * kChainMaxSlots * MPAD + m) * kBlockN + r[u];
      first_off[u] = static_cast<long>(s.slot_first) * MPAD * kBlockN;
    }
  }
  float4 v[NB][MAXC];
#pragma unroll
  for (int j = 0; j < MAXC; ++j) {
#pragma unroll
    for (int u = 0; u < NB; ++u) {
      const long off = (j == 0) ? first_off[u] : static_cast<long>(j) * kChainMaxSlots * MPAD * kBlockN;
      v[u][j] = (j < cnt[u]) ? ld_partial(base[u] + off) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
#pragma unroll
  for (int u = 0; u < NB; ++u) {
    float4 a = v[u][0];
#pragma unroll
    for (int j = 1; j < MAXC; ++j) {
      a.x += v[u][j].x;
      a.y += v[u][j].y;
      a.z += v[u][j].z;
      a.w += v[u][j].w;
    }
    out[u] = a;
  }
}

template <typename T> __device__ __forceinline__ void ld4(const T* p, float (&f)[4]) {
  const uint2 raw = __ldcg(reinterpret_cast<const uint2*>(p));
  const T* e = reinterpret_cast<const T*>(&raw);
#pragma unroll
  for (int k = 0; k < 4; ++k) f[k] = DT<T>::to_f(e[k]);
}
template <typename T> __device__ __forceinline__ void st4(T* p, const float (&f)[4]) {
  uint2 raw;
  T* e = reinterpret_cast<T*>(&raw);
#pragma unroll
  for (int k = 0; k < 4; ++k) e[k] = DT<T>::from_f(f[k]);
  *reinterpret_cast<uint2*>(p) = raw;
}
__device__ __forceinline__ float epi_block_sum(float v, float* red, int etid) {
  v = warp_sum(v);
  if ((etid & 31) == 0) red[etid >> 5] = v;
  chain_epi_bar();
  const float t = (red[0] + red[1]) + (red[2] + red[3]);
  chain_epi_bar();
  return t;
}
__device__ __forceinline__ bool better(float v, int i, float bv, int bi) { return v > bv || (v == bv && i < bi); }

// ------------------------------------------------------------------------------------------------------------
// finish items (128 epilogue threads; etid = 0..127)
// ------------------------------------------------------------------------------------------------------------
template <typename T, int MPAD>
__device__ __forceinline__ void finish_resid_norm(const ChainPhase& ph, const float* ws, const TileSrc* tab, const Geo& g, int G, int m,
                                                  int etid, float* red, unsigned long long* sub = nullptr) {
  constexpr int kMaxPass = 16;  // N <= 8192
  constexpr int kBatch = 4;     // passes whose loads are issued together
  const bool fast = chain_fast_path(g, G, 6);
  float v[kMaxPass][4];
  float ss = 0.f;
  T* xrow = reinterpret_cast<T*>(ph.x) + static_cast<long>(m) * ph.ld_x;
  const T* resrow = ph.res ? reinterpret_cast<const T*>(ph.res) + static_cast<long>(m) * ph.ld_res : xrow;
  T* taprow = ph.tap ? reinterpret_cast<T*>(ph.tap) + static_cast<long>(m) * ph.ld_tap : nullptr;
  // residual row and norm weights do not depend on the partials: all their loads go out first (8 bytes per pass each), so the
  // arithmetic below never waits for a second or third L2 round trip
  uint2 res_raw[kMaxPass], w_raw[kMaxPass];
  const T* w = reinterpret_cast<const T*>(ph.norm_w);
#pragma unroll
  for (int i = 0; i < kMaxPass; ++i) {
    const int n = (i * 128 + etid) * 4;
    if (n < ph.N) {
      res_raw[i] = __ldcg(reinterpret_cast<const uint2*>(resrow + n));
      if (w) w_raw[i] = __ldg(reinterpret_cast<const uint2*>(w + n));
    }
  }
#pragma unroll
  for (int i0 = 0; i0 < kMaxPass; i0 += kBatch) {
    if (i0 * 512 >= ph.N) break;
    float4 a[kBatch];
    float res[kBatch][4];
    if (fast) {
      int tt[kBatch], rr[kBatch];
      bool ok[kBatch];
#pragma unroll
      for (int u = 0; u < kBatch; ++u) {
        const int n = ((i0 + u) * 128 + etid) * 4;
        ok[u] = n < ph.N;
        tt[u] = n >> 7;
        rr[u] = n & 127;
      }
      reduce4_batch<MPAD, kBatch, 6>(ws, tab, tt, rr, ok, m, a);
    } else {
#pragma unroll
      for (int u = 0; u < kBatch; ++u) {
        const int n = ((i0 + u) * 128 + etid) * 4;
        if (n < ph.N) a[u] = reduce4<MPAD>(ws, tab, g, G, n >> 7, m, n & 127);
      }
    }
#pragma unroll
    for (int u = 0; u < kBatch; ++u) {
      const int i = i0 + u;
      const int n = (i * 128 + etid) * 4;
      if (n < ph.N) {
        const T* re = reinterpret_cast<const T*>(&res_raw[i]);
#pragma unroll
        for (int k = 0; k < 4; ++k) res[u][k] = DT<T>::to_f(re[k]);
        v[i][0] = rnd<T>(rnd<T>(a[u].x) + res[u][0]);  // T(T(acc) + residual): modeling_llama_kv.py:838-845
        v[i][1] = rnd<T>(rnd<T>(a[u].y) + res[u][1]);
        v[i][2] = rnd<T>(rnd<T>(a[u].z) + res[u][2]);
        v[i][3] = rnd<T>(rnd<T>(a[u].w) + res[u][3]);
        st4<T>(xrow + n, v[i]);
        if (taprow) st4<T>(taprow + n, v[i]);
#pragma unroll
        for (int k = 0; k < 4; ++k) ss = fmaf(v[i][k], v[i][k], ss);
      }
    }
    if (sub && i0 == 0) sub[0] = chain_gtimer();  // first batch reduced and stored
  }
  if (sub) sub[1] = chain_gtimer();  // all batches done
  if (!ph.norm_w) return;  // uniform
  ss = epi_block_sum(ss, red, etid);
  if (sub) sub[2] = chain_gtimer();  // row statistics known
  const float inv = rsqrtf(ss / static_cast<float>(ph.N) + ph.eps);  // modeling_llama_kv.py:128-132
  T* orow = reinterpret_cast<T*>(ph.xn) + static_cast<long>(m) * ph.ld_xn;
#pragma unroll
  for (int i = 0; i < kMaxPass; ++i) {
    const int n = (i * 128 + etid) * 4;
    if (n < ph.N) {
      float o[4];
      const T* we = reinterpret_cast<const T*>(&w_raw[i]);
#pragma unroll
      for (int k = 0; k < 4; ++k) o[k] = DT<T>::to_f(we[k]) * rnd<T>(v[i][k] * inv);
      st4<T>(orow + n, o);
    }
  }
}

template <typename T, int MPAD>
__device__ __forceinline__ void finish_swiglu(const ChainPhase& ph, const float* ws, const TileSrc* tab, const Geo& g, int G, int m, int chunk,
                                              int etid) {
  using D = DT<T>;
  constexpr int kBatch = 4;
  const bool fast = chain_fast_path(g, G, 3);
  const int I = ph.N / 2;
  const int np = (I + 511) / 512;
  const int per = (np + ph.chunks - 1) / ph.chunks;
  const int p0 = chunk * per, p1 = min(np, p0 + per);
  const T* lut = reinterpret_cast<const T*>(ph.silu_lut);
  T* orow = reinterpret_cast<T*>(ph.out) + static_cast<long>(m) * ph.ld_out;
  for (int i0 = p0; i0 < p1; i0 += kBatch) {
    float4 ga[kBatch], ua[kBatch];
    if (fast) {
      int tt[2 * kBatch], rr[2 * kBatch];
      bool ok[2 * kBatch];
      float4 o8[2 * kBatch];
#pragma unroll
      for (int u = 0; u < kBatch; ++u) {
        const int j = ((i0 + u) * 128 + etid) * 4;
        ok[2 * u] = ok[2 * u + 1] = (i0 + u < p1 && j < I);
        tt[2 * u] = tt[2 * u + 1] = j >> 6;
        rr[2 * u] = j & 63;
        rr[2 * u + 1] = (j & 63) + 64;
      }
      reduce4_batch<MPAD, 2 * kBatch, 3>(ws, tab, tt, rr, ok, m, o8);
#pragma unroll
      for (int u = 0; u < kBatch; ++u) {
        ga[u] = o8[2 * u];
        ua[u] = o8[2 * u + 1];
      }
    } else {
#pragma unroll
      for (int u = 0; u < kBatch; ++u) {
        const int j = ((i0 + u) * 128 + etid) * 4;
        if (i0 + u < p1 && j < I) {
          ga[u] = reduce4<MPAD>(ws, tab, g, G, j >> 6, m, j & 63);
          ua[u] = reduce4<MPAD>(ws, tab, g, G, j >> 6, m, (j & 63) + 64);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < kBatch; ++u) {
      const int j = ((i0 + u) * 128 + etid) * 4;
      if (i0 + u < p1 && j < I) {
        const float gf[4] = {ga[u].x, ga[u].y, ga[u].z, ga[u].w}, uf[4] = {ua[u].x, ua[u].y, ua[u].z, ua[u].w};
        float o[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const T gt = D::from_f(gf[k]);
          const unsigned short bits = *reinterpret_cast<const unsigned short*>(&gt);
          const float sg = D::to_f(__ldg(lut + bits));  // T(silu(T(gate))), tabulated (gemm.cu: silu_lut)
          o[k] = sg * rnd<T>(uf[k]);
        }
        st4<T>(orow + j, o);
      }
    }
  }
}

template <typename T, int MPAD>
__device__ __forceinline__ void finish_qkv_rope(const ChainPhase& ph, const int* st, const float* ws, const TileSrc* tab, const Geo& g, int G,
                                                int m, int chunk, int etid) {
  constexpr int kBatch = 3;
  const bool fast = chain_fast_path(g, G, 5);
  const int NH = ph.n_q_heads + 2 * ph.n_kv_heads;
  const int np = (NH + 7) / 8;
  const int per = (np + ph.chunks - 1) / ph.chunks;
  const int p0 = chunk * per, p1 = min(np, p0 + per);
  const long kv0 = (ph.kv_base.idx >= 0 ? ld_dep(st + ph.kv_base.idx) : 0) + ph.kv_base.add;
  const int pos = (ph.pos_base.idx >= 0 ? ld_dep(st + ph.pos_base.idx) : 0) + ph.pos_base.add + (ph.pos_arr ? ld_dep(ph.pos_arr + m) : 0) +
                  ph.pos_mstride * m;
  const int d4 = (etid & 15) * 4;
  float c[4], s[4];
  ld4<T>(reinterpret_cast<const T*>(ph.rope_cos) + static_cast<long>(pos) * 64 + d4, c);
  ld4<T>(reinterpret_cast<const T*>(ph.rope_sin) + static_cast<long>(pos) * 64 + d4, s);
  for (int i0 = p0; i0 < p1; i0 += kBatch) {
    float4 lo4[kBatch], hi4[kBatch];
    if (fast) {
      int tt[2 * kBatch], rr[2 * kBatch];
      bool ok[2 * kBatch];
      float4 o6[2 * kBatch];
#pragma unroll
      for (int u = 0; u < kBatch; ++u) {
        const int h = (i0 + u) * 8 + (etid >> 4);
        ok[2 * u] = ok[2 * u + 1] = (i0 + u < p1 && h < NH);
        tt[2 * u] = tt[2 * u + 1] = h;
        rr[2 * u] = d4;
        rr[2 * u + 1] = d4 + 64;
      }
      reduce4_batch<MPAD, 2 * kBatch, 5>(ws, tab, tt, rr, ok, m, o6);
#pragma unroll
      for (int u = 0; u < kBatch; ++u) {
        lo4[u] = o6[2 * u];
        hi4[u] = o6[2 * u + 1];
      }
    } else {
#pragma unroll
      for (int u = 0; u < kBatch; ++u) {
        const int h = (i0 + u) * 8 + (etid >> 4);
        if (i0 + u < p1 && h < NH) {
          lo4[u] = reduce4<MPAD>(ws, tab, g, G, h, m, d4);
          hi4[u] = reduce4<MPAD>(ws, tab, g, G, h, m, d4 + 64);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < kBatch; ++u) {
      const int h = (i0 + u) * 8 + (etid >> 4);
      if (!(i0 + u < p1 && h < NH)) continue;
      float lo[4] = {rnd<T>(lo4[u].x), rnd<T>(lo4[u].y), rnd<T>(lo4[u].z), rnd<T>(lo4[u].w)};
      float hi[4] = {rnd<T>(hi4[u].x), rnd<T>(hi4[u].y), rnd<T>(hi4[u].z), rnd<T>(hi4[u].w)};
      if (h < ph.n_q_heads + ph.n_kv_heads) {  // q or k: rotate_half rope with three roundings (modeling_llama_kv.py:295-330)
        float olo[4], ohi[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          olo[k] = rnd<T>(lo[k] * c[k]) + rnd<T>(-hi[k] * s[k]);
          ohi[k] = rnd<T>(hi[k] * c[k]) + rnd<T>(lo[k] * s[k]);
        }
        T* dst;
        if (h < ph.n_q_heads) dst = reinterpret_cast<T*>(ph.q_out) + (static_cast<long>(m) * ph.n_q_heads + h) * 128;
        else dst = reinterpret_cast<T*>(ph.k_cache) + (static_cast<long>(h - ph.n_q_heads) * ph.kv_cap + kv0 + m) * 128;
        st4<T>(dst + d4, olo);
        st4<T>(dst + d4 + 64, ohi);
      } else {
        T* dst = reinterpret_cast<T*>(ph.v_cache) + (static_cast<long>(h - ph.n_q_heads - ph.n_kv_heads) * ph.kv_cap + kv0 + m) * 128;
        st4<T>(dst + d4, lo);
        st4<T>(dst + d4 + 64, hi);
      }
    }
  }
}

template <typename T, int MPAD>
__device__ __forceinline__ void finish_store(const ChainPhase& ph, const float* ws, const TileSrc* tab, const Geo& g, int G, int m, int chunk,
                                             int etid) {
  constexpr int kBatch = 4;
  const bool fast = chain_fast_path(g, G, 6);
  const int np = (ph.N + 511) / 512;
  const int per = (np + ph.chunks - 1) / ph.chunks;
  const int p0 = chunk * per, p1 = min(np, p0 + per);
  T* orow = reinterpret_cast<T*>(ph.out) + static_cast<long>(m) * ph.ld_out;
  for (int i0 = p0; i0 < p1; i0 += kBatch) {
    float4 a[kBatch];
    if (fast) {
      int tt[kBatch], rr[kBatch];
      bool ok[kBatch];
#pragma unroll
      for (int u = 0; u < kBatch; ++u) {
        const int n = ((i0 + u) * 128 + etid) * 4;
        ok[u] = (i0 + u < p1 && n < ph.N);
        tt[u] = n >> 7;
        rr[u] = n & 127;
      }
      reduce4_batch<MPAD, kBatch, 6>(ws, tab, tt, rr, ok, m, a);
    } else {
#pragma unroll
      for (int u = 0; u < kBatch; ++u) {
        const int n = ((i0 + u) * 128 + etid) * 4;
        if (i0 + u < p1 && n < ph.N) a[u] = reduce4<MPAD>(ws, tab, g, G, n >> 7, m, n & 127);
      }
    }
#pragma unroll
    for (int u = 0; u < kBatch; ++u) {
      const int n = ((i0 + u) * 128 + etid) * 4;
      if (i0 + u < p1 && n < ph.N) {
        float o[4] = {a[u].x, a[u].y, a[u].z, a[u].w};
        if (ph.bias) {
          float bb[4];
          ld4<T>(reinterpret_cast<const T*>(ph.bias) + n, bb);
#pragma unroll
          for (int k = 0; k < 4; ++k) o[k] += bb[k];
        }
        st4<T>(orow + n, o);
      }
    }
  }
}

// Row-parallel projection under tensor parallelism, one row m: (A) every rank reduces its own split-K partials of the row and
// pushes the fp32 row into the inbox of the row's owner (m % tp) over NVLink; (B) the owner adds the tp rows in rank order
// (deterministic, identical on every run), applies residual + RMSNorm exactly like the single-GPU finish and pushes the new x / xn
// (/ tap) rows into every rank's window.  Replaces gemm_partial_f32 -> ncclAllReduce -> residual_add_f32 -> rmsnorm.
template <typename T, int MPAD>
__device__ __forceinline__ void finish_resid_norm_tp(const ChainPhase& ph, const ChainTP& tp, const float* ws, const TileSrc* tab, const Geo& g,
                                                     int G, int m, int etid, float* red, int epoch) {
  constexpr int kMaxPass = 16;
  constexpr int kBatch = 4;
  const bool fast = chain_fast_path(g, G, 6);
  const int owner = m % tp.size;
  float* dst = reinterpret_cast<float*>(tp.win[owner] + tp.inbox_off) + (static_cast<long>(tp.rank) * 64 + m) * tp.ld_inbox;
#pragma unroll
  for (int i0 = 0; i0 < kMaxPass; i0 += kBatch) {
    if (i0 * 512 >= ph.N) break;
    float4 a[kBatch];
    if (fast) {
      int tt[kBatch], rr[kBatch];
      bool ok[kBatch];
#pragma unroll
      for (int u = 0; u < kBatch; ++u) {
        const int n = ((i0 + u) * 128 + etid) * 4;
        ok[u] = n < ph.N;
        tt[u] = n >> 7;
        rr[u] = n & 127;
      }
      reduce4_batch<MPAD, kBatch, 6>(ws, tab, tt, rr, ok, m, a);
    } else {
#pragma unroll
      for (int u = 0; u < kBatch; ++u) {
        const int n = ((i0 + u) * 128 + etid) * 4;
        if (n < ph.N) a[u] = reduce4<MPAD>(ws, tab, g, G, n >> 7, m, n & 127);
      }
    }
#pragma unroll
    for (int u = 0; u < kBatch; ++u) {
      const int n = ((i0 + u) * 128 + etid) * 4;
      if (n < ph.N) *reinterpret_cast<float4*>(dst + n) = a[u];
    }
  }
  __threadfence_system();
  chain_epi_bar();
  if (etid == 0) st_release_sys(reinterpret_cast<int*>(tp.win[owner] + tp.flag_off) + tp.rank * 64 + m, epoch);
  if (owner != tp.rank) return;  // uniform over the CTA
  // ---- owner: wait for every rank's row, then the single-GPU arithmetic on the fp32 total ----
  if (etid < tp.size) spin_until_ge_sys(reinterpret_cast<const int*>(tp.win[tp.rank] + tp.flag_off) + etid * 64 + m, epoch);
  chain_epi_bar();
  __threadfence_system();
  const float* inbox = reinterpret_cast<const float*>(tp.win[tp.rank] + tp.inbox_off) + static_cast<long>(m) * tp.ld_inbox;
  float v[kMaxPass][4];
  float ss = 0.f;
  T* xrow = reinterpret_cast<T*>(ph.x) + static_cast<long>(m) * ph.ld_x;
  const T* resrow = ph.res ? reinterpret_cast<const T*>(ph.res) + static_cast<long>(m) * ph.ld_res : xrow;
  T* taprow = ph.tap ? reinterpret_cast<T*>(ph.tap) + static_cast<long>(m) * ph.ld_tap : nullptr;
#pragma unroll
  for (int i = 0; i < kMaxPass; ++i) {
    const int n = (i * 128 + etid) * 4;
    if (n < ph.N) {
      float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int src = 0; src < tp.size; ++src) {
        const float4 p4 = __ldcg(reinterpret_cast<const float4*>(inbox + static_cast<long>(src) * 64 * tp.ld_inbox + n));
        a.x += p4.x;
        a.y += p4.y;
        a.z += p4.z;
        a.w += p4.w;
      }
      float res[4];
      ld4<T>(resrow + n, res);
      v[i][0] = rnd<T>(rnd<T>(a.x) + res[0]);
      v[i][1] = rnd<T>(rnd<T>(a.y) + res[1]);
      v[i][2] = rnd<T>(rnd<T>(a.z) + res[2]);
      v[i][3] = rnd<T>(rnd<T>(a.w) + res[3]);
      for (int r = 0; r < tp.size; ++r) {
        st4<T>(peer_ptr(tp, xrow, r) + n, v[i]);
        if (taprow) st4<T>(peer_ptr(tp, taprow, r) + n, v[i]);
      }
#pragma unroll
      for (int k = 0; k < 4; ++k) ss = fmaf(v[i][k], v[i][k], ss);
    }
  }
  if (ph.norm_w) {
    ss = epi_block_sum(ss, red, etid);
    const float inv = rsqrtf(ss / static_cast<float>(ph.N) + ph.eps);
    const T* w = reinterpret_cast<const T*>(ph.norm_w);
    T* orow = reinterpret_cast<T*>(ph.xn) + static_cast<long>(m) * ph.ld_xn;
#pragma unroll
    for (int i = 0; i < kMaxPass; ++i) {
      const int n = (i * 128 + etid) * 4;
      if (n < ph.N) {
        float wf[4], o[4];
        ld4<T>(w + n, wf);
#pragma unroll
        for (int k = 0; k < 4; ++k) o[k] = wf[k] * rnd<T>(v[i][k] * inv);
        for (int r = 0; r < tp.size; ++r) st4<T>(peer_ptr(tp, orow, r) + n, o);
      }
    }
  }
  __threadfence_system();
  fence_proxy_async_all();
  chain_epi_bar();
  if (etid < tp.size) red_release_sys_add(reinterpret_cast<int*>(tp.win[etid] + tp.ready_off), 1);
}

// merge the per-tile (max, first index) pairs of row m (torch.argmax: first maximal index; ea_model.py:190 + utils.py:362)
__device__ __forceinline__ void finish_argmax(const ChainPhase& ph, const ChainTP& tp, int epoch, const Geo& g, int m, int etid, float* sval,
                                              int* sidx) {
  float bv = -INFINITY;
  int bi = 0x7fffffff;
  for (int t = etid; t < g.ntiles; t += 128) {
    const float v = __ldcg(ph.tile_val + static_cast<long>(t) * 64 + m);
    const int i = __ldcg(ph.tile_idx + static_cast<long>(t) * 64 + m);
    if (better(v, i, bv, bi)) {
      bv = v;
      bi = i;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (better(ov, oi, bv, bi)) {
      bv = ov;
      bi = oi;
    }
  }
  if ((etid & 31) == 0) {
    sval[etid >> 5] = bv;
    sidx[etid >> 5] = bi;
  }
  chain_epi_bar();
  if (etid == 0) {
    for (int w = 1; w < 4; ++w)
      if (better(sval[w], sidx[w], bv, bi)) {
        bv = sval[w];
        bi = sidx[w];
      }
    if (tp.size > 1) {
      // vocabulary-parallel lm_head: exchange the (value, global index) pairs of the shards; lowest index wins ties, like one GPU
      bi += ph.idx_offset;
      for (int r = 0; r < tp.size; ++r) {
        float* slot = reinterpret_cast<float*>(tp.win[r] + tp.am_off) + (static_cast<long>(tp.rank) * 64 + m) * 2;
        slot[0] = bv;
        reinterpret_cast<int*>(slot)[1] = bi;
        __threadfence_system();
        st_release_sys(reinterpret_cast<int*>(tp.win[r] + tp.am_off + static_cast<long>(kMaxTp) * 64 * 8) + tp.rank * 64 + m, epoch);
      }
      const int* flags = reinterpret_cast<const int*>(tp.win[tp.rank] + tp.am_off + static_cast<long>(kMaxTp) * 64 * 8);
      const float* mine = reinterpret_cast<const float*>(tp.win[tp.rank] + tp.am_off);
      bv = -INFINITY;
      bi = 0x7fffffff;
      for (int src = 0; src < tp.size; ++src) {
        spin_until_ge_sys(flags + src * 64 + m, epoch);
        const float v = __ldcg(mine + (static_cast<long>(src) * 64 + m) * 2);
        const int i = __ldcg(reinterpret_cast<const int*>(mine + (static_cast<long>(src) * 64 + m) * 2) + 1);
        if (better(v, i, bv, bi)) {
          bv = v;
          bi = i;
        }
      }
    }
    ph.out_idx[m] = bi;
  }
  chain_epi_bar();
}

// ------------------------------------------------------------------------------------------------------------
// the kernel
// ------------------------------------------------------------------------------------------------------------
template <typename T, int MPAD>
__global__ void __launch_bounds__(kChainThreads, 1)
gemm_chain_kernel(const __grid_constant__ ChainMaps maps, const __grid_constant__ ChainArgs args, const int stages) {
  constexpr int kXBytes = x_tile_bytes(MPAD);
  constexpr int kStageBytes = kWTileBytes + kXBytes;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* ctrl = smem + stages * kStageBytes;
  uint64_t* fullW = reinterpret_cast<uint64_t*>(ctrl);
  uint64_t* fullX = fullW + kChainMaxStages;
  uint64_t* empty = fullX + kChainMaxStages;
  uint64_t* acc_full = empty + kChainMaxStages;   // the staging tile holds a segment's accumulators (128 arrivals)
  uint64_t* acc_empty = acc_full + 1;             // the epilogue has drained it
  float* accbuf = reinterpret_cast<float*>(ctrl + kChainCtrlBytes);  // [MPAD][128] staged fp32 accumulators
  float* red = reinterpret_cast<float*>(ctrl + 512);                // [4] block-sum scratch, then [4][64] arg-max pairs
  float* sval = reinterpret_cast<float*>(ctrl + 1024);              // [4][64]
  int* sidx = reinterpret_cast<int*>(ctrl + 1024 + 4 * 64 * 4);     // [4][64]
  TileSrc* tab = reinterpret_cast<TileSrc*>(ctrl + 4096);           // [kChainMaxTableTiles]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int cta = blockIdx.x, G = gridDim.x;
  pdl_launch_dependents();

  if (threadIdx.x == 0) {
    for (int p = 0; p < args.n_phases; ++p) {
      tma_prefetch_desc(&maps.w[p]);
      tma_prefetch_desc(&maps.x[p]);
    }
    for (int i = 0; i < stages; ++i) {
      mbar_init(&fullW[i], 1);
      mbar_init(&fullX[i], 1);
      mbar_init(&empty[i], 1);
    }
    mbar_init(acc_full, 128);
    mbar_init(acc_empty, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ===== weight producer: the whole task list, never blocked by a phase boundary (weights depend on nothing).  While the
    // ring is full (the MMA side waits for a finish step) a second cursor keeps HBM busy: it prefetches the next l2_window weight
    // tiles into L2, from where the ring refills faster than from HBM once the MMAs resume. =====
    if (lane == 0) {
      int s = 0;
      uint32_t par = 0;
      UnitCursor ld, pf;
      ld.p = 0;
      ld.done = false;
      cursor_enter_phase(ld, args, cta, G);
      pf = ld;
      int ahead = 0;  // units the prefetch cursor is ahead of the load cursor
      const int window = args.l2_window;
      // Run-ahead throttle: the finish of phase p reads ~5 MB of partials through the same L2 the weight stream saturates;
      // letting the ring refill at full speed during the finish can stretch the (critical-path) finish.  So only w_ahead tiles
      // of phase p+1 are fetched before ready[p] is observed (EB200_CHAIN_W_AHEAD; default -1 = no throttle).
      int cur_phase = ld.done ? 0 : ld.p, into_phase = 0;
      bool prev_ready = true;
      int m_valid_w = -1;
      int tp_ready0_w = 0;
      while (!ld.done) {
        if (ld.p != cur_phase) {
          cur_phase = ld.p;
          into_phase = 0;
          prev_ready = false;
        }
        if (!prev_ready && args.w_ahead >= 0 && into_phase >= args.w_ahead) {
          if (m_valid_w < 0) {
            pdl_wait();
            m_valid_w = args.m_idx >= 0 ? min(args.m_rows, ld_dep(args.st + args.m_idx)) : args.m_rows;
            tp_ready0_w = args.tp.size > 1 ? ld_dep(args.tp.ready_base) : 0;
          }
          // same condition the activation producer waits for (all phases before cur_phase are finished once phase cur_phase-1 is)
          const ChainPhase& prev = args.ph[cur_phase - 1];
          if (args.tp.size > 1 && prev.fin == FIN_RESID_NORM) {
            int seen = 0;
            for (int q = 0; q < cur_phase; ++q) seen += args.ph[q].fin == FIN_RESID_NORM ? 1 : 0;
            spin_until_ge_sys(reinterpret_cast<const int*>(args.tp.win[args.tp.rank] + args.tp.ready_off), tp_ready0_w + seen * m_valid_w);
          } else {
            spin_until_ge(args.sync + kSyncReady + (cur_phase - 1), m_valid_w * prev.chunks);
          }
          prev_ready = true;
        }
        ++into_phase;
        uint32_t spins = 0;
        while (!mbar_try_wait(&empty[s], par ^ 1)) {
          if (!pf.done && ahead < window) {
            tma_prefetch_l2_2d(&maps.w[pf.p], pf.kb * kBlockK, pf.t * kBlockN);
            cursor_advance(pf, args, cta, G);
            ++ahead;
          } else if (++spins > (1u << 26)) {
            __trap();
          }
        }
        mbar_arrive_expect_tx(&fullW[s], kWTileBytes);
        tma_load_2d(smem + s * kStageBytes, &maps.w[ld.p], &fullW[s], ld.kb * kBlockK, ld.t * kBlockN, kEvictFirst);
        cursor_advance(ld, args, cta, G);
        if (ahead > 0) --ahead;
        else pf = ld;
        if (++s == stages) {
          s = 0;
          par ^= 1;
        }
      }
    }
  } else if (warp == 9) {
    // ===== activation producer: X tiles of phase p exist once finish(p-1) has completed (phase 0: the previous kernel) =====
    if (lane == 0) {
      pdl_wait();
      const int m_valid = args.m_idx >= 0 ? min(args.m_rows, ld_dep(args.st + args.m_idx)) : args.m_rows;
      const int tp_ready0 = args.tp.size > 1 ? ld_dep(args.tp.ready_base) : 0;
      int tp_resid_seen = 0;
      int s = 0;
      uint32_t par = 0;
      for (int p = 0; p < args.n_phases; ++p) {
        if (p > 0) {
          const ChainPhase& prev = args.ph[p - 1];
          if (args.tp.size > 1 && prev.fin == FIN_RESID_NORM) {
            // rows of this phase's X operand are pushed by their owners on all ranks (finish_resid_norm_tp)
            tp_resid_seen += 1;
            spin_until_ge_sys(reinterpret_cast<const int*>(args.tp.win[args.tp.rank] + args.tp.ready_off), tp_ready0 + tp_resid_seen * m_valid);
          } else {
            spin_until_ge(args.sync + kSyncReady + (p - 1), m_valid * prev.chunks);
          }
          fence_proxy_async_all();  // generic-proxy writes of other SMs (acquired above) -> this thread's async-proxy (TMA) reads
        }
        const Geo g = geo_of(args.ph[p]);
        for_each_segment(g, cta, G, [&](int, int a, int b, int) {
          for (int kb = a; kb < b; ++kb) {
            mbar_wait_mma(&empty[s], par ^ 1);
            mbar_arrive_expect_tx(&fullX[s], kXBytes);
            tma_load_2d(smem + s * kStageBytes + kWTileBytes, &maps.x[p], &fullX[s], kb * kBlockK, 0, kEvictLast);
            if (++s == stages) {
              s = 0;
              par ^= 1;
            }
          }
        });
      }
    }
  } else if (warp < 4) {
    // ===== MMA warpgroup: both 64-row halves of each tile, fp32 accumulators in registers =====
    const bool lead = threadIdx.x == 0;
    int s = 0;
    uint32_t par = 0, seg = 0;
    unsigned long long* trc = (args.trace && lead) ? args.trace + 32ull * cta : nullptr;
    for (int p = 0; p < args.n_phases; ++p) {
      const Geo g = geo_of(args.ph[p]);
      bool first = true;
      for_each_segment(g, cta, G, [&](int, int a, int b, int) {
        float acc[2][MPAD / 2];
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int i = 0; i < MPAD / 2; ++i) acc[h][i] = 0.f;
        int prev = -1;
        for (int kb = a; kb < b; ++kb) {
          mbar_wait_mma(&fullW[s], par);
          mbar_wait_mma(&fullX[s], par);
          if (trc && first) {
            trc[1 + 6 * p + 4] = chain_gtimer();  // first X tile of the phase has landed
            first = false;
          }
          const uint32_t st = smem_u32(smem + s * kStageBytes);
          const uint64_t b_desc = make_kmajor_sw128_desc(st + kWTileBytes);
          wgmma_fence();
#pragma unroll
          for (int h = 0; h < 2; ++h) wgmma_kblock<T, MPAD>(acc[h], make_kmajor_sw128_desc(st + h * (kWTileBytes / 2)), b_desc);
          wgmma_commit();
          wgmma_wait<1>();  // the previous k-block's MMAs have retired: its slot can be refilled
          if (prev >= 0 && lead) mbar_arrive(&empty[prev]);
          prev = s;
          if (++s == stages) {
            s = 0;
            par ^= 1;
          }
        }
        wgmma_wait<0>();
        if (prev >= 0 && lead) mbar_arrive(&empty[prev]);
#pragma unroll
        for (int h = 0; h < 2; ++h) wgmma_fence_acc(acc[h]);
        mbar_wait_mma(acc_empty, (seg & 1) ^ 1);  // the epilogue has drained the staging tile (first use passes)
#pragma unroll
        for (int h = 0; h < 2; ++h) wgmma_store_acc<MPAD>(acc[h], accbuf, kBlockN, h * 64);
        mbar_arrive(acc_full);
        ++seg;
      });
      if (trc) trc[1 + 6 * p + 5] = chain_gtimer();  // last MMA of the phase issued
    }
  } else if (warp >= 4) {
    // ===== epilogue + finish warps (thread <-> weight row quad * 32 + lane) =====
    const int quad = warp & 3;
    const int etid = threadIdx.x - 128;
    const int row = quad * 32 + lane;  // weight row inside the tile
    pdl_wait();
    const int m_valid = args.m_idx >= 0 ? min(args.m_rows, ld_dep(args.st + args.m_idx)) : args.m_rows;
    if (args.timing && cta == 0 && etid == 0) *reinterpret_cast<volatile unsigned long long*>(args.timing + 2) = chain_gtimer();
    const int tp_epoch0 = args.tp.size > 1 ? ld_dep(args.tp.epoch) : 0;
    unsigned long long* tre = (args.trace && etid == 0) ? args.trace + 32ull * cta : nullptr;
    if (tre) tre[0] = chain_gtimer();
    float* my_ws = args.ws + static_cast<long>(cta) * kChainMaxSlots * MPAD * kBlockN;
    uint32_t seg = 0;
    for (int p = 0; p < args.n_phases; ++p) {
      const ChainPhase& ph = args.ph[p];
      const Geo g = geo_of(ph);
      bool first_seg = true;
      for_each_segment(g, cta, G, [&](int t, int, int, int slot) {
        mbar_wait_mma(acc_full, seg & 1);
        if (tre && first_seg) {
          tre[1 + 6 * p + 0] = chain_gtimer();  // first accumulator of the phase complete
          first_seg = false;
        }
        if (!g.direct) {
          float* part = my_ws + static_cast<long>(slot) * MPAD * kBlockN + row;
#pragma unroll 1
          for (int c = 0; c < MPAD / 16; ++c) {
            if (c * 16 >= m_valid) break;
            float r[16];
            acc_ld16(accbuf, kBlockN, row, c * 16, r);
#pragma unroll
            for (int j = 0; j < 16; ++j)
              if (c * 16 + j < m_valid) __stcg(part + (c * 16 + j) * kBlockN, r[j]);
          }
        } else if (ph.fin == FIN_STORE_DIRECT) {
          GemmParams gp;
          gp.N = ph.N;
          gp.out = ph.out;
          gp.ld_out = ph.ld_out;
          gp.bias = ph.bias;
          float acc[16], acc2[16];
#pragma unroll 1
          for (int c = 0; c < MPAD / 16; ++c) {
            if (c * 16 >= m_valid) break;
            float r[16];
            acc_ld16(accbuf, kBlockN, row, c * 16, r);
#pragma unroll
            for (int j = 0; j < 16; ++j) acc[j] = acc2[j] = r[j];
            final_chunk<T, EPI_STORE>(gp, acc, acc2, c * 16, m_valid, row, t, nullptr);
          }
        } else {  // FIN_ARGMAX: per-row (max, first index) of this tile's 128 vocabulary rows
          const int n = t * kBlockN + row;
#pragma unroll 1
          for (int c = 0; c < MPAD / 16; ++c) {
            if (c * 16 >= m_valid) break;
            float r[16];
            acc_ld16(accbuf, kBlockN, row, c * 16, r);
#pragma unroll
            for (int j = 0; j < 16; ++j) {
              float v = (n < ph.N) ? rnd<T>(r[j]) : -INFINITY;  // the logits tensor is model dtype (ea_model.py:190)
              int idx = n;
#pragma unroll
              for (int o = 16; o > 0; o >>= 1) {
                const float ov = __shfl_xor_sync(0xffffffffu, v, o);
                const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
                if (better(ov, oi, v, idx)) {
                  v = ov;
                  idx = oi;
                }
              }
              if (lane == 0) {
                sval[quad * 64 + c * 16 + j] = v;
                sidx[quad * 64 + c * 16 + j] = idx;
              }
            }
          }
          chain_epi_bar();
          if (etid < m_valid) {
            float bv = sval[etid];
            int bi = sidx[etid];
#pragma unroll
            for (int w = 1; w < 4; ++w)
              if (better(sval[w * 64 + etid], sidx[w * 64 + etid], bv, bi)) {
                bv = sval[w * 64 + etid];
                bi = sidx[w * 64 + etid];
              }
            __stcg(ph.tile_val + static_cast<long>(t) * 64 + etid, bv);
            __stcg(ph.tile_idx + static_cast<long>(t) * 64 + etid, bi);
          }
        }
        chain_epi_bar();  // every epilogue thread is done with the staging tile (and with sval/sidx)
        if (etid == 0) mbar_arrive(acc_empty);
        ++seg;
      });
      // ---- all partials / tile results of this CTA for phase p are written ----
      __threadfence();
      chain_epi_bar();
      if (etid == 0) red_release_gpu_add(args.sync + kSyncPartials + p, 1);
      if (tre) tre[1 + 6 * p + 1] = chain_gtimer();  // this CTA's partials are published
      if (ph.fin == FIN_STORE_DIRECT) {  // no row-wise step: the phase is complete when every CTA has stored its tiles
        if (etid == 0 && cta < m_valid * ph.chunks) {
          int mine = 0;
          for (int it = cta; it < m_valid * ph.chunks; it += G) ++mine;
          spin_until_ge(args.sync + kSyncPartials + p, G);
          red_release_gpu_add(args.sync + kSyncReady + p, mine);
        }
        continue;
      }
      // ---- finish: row-wise split-K reduction + epilogue arithmetic (+ RMSNorm) on the first rows*chunks CTAs ----
      const int n_items = m_valid * ph.chunks;
      if (cta < n_items) {
        if (!g.direct) build_tile_table(tab, g, G, etid);
        if (etid == 0) spin_until_ge(args.sync + kSyncPartials + p, G);
        chain_epi_bar();
        __threadfence();
        if (tre) tre[1 + 6 * p + 2] = chain_gtimer();  // every CTA's partials have arrived: finish starts
        int done = 0;
        for (int item = cta; item < n_items; item += G) {
          const int m = item / ph.chunks, chunk = item - m * ph.chunks;
          switch (ph.fin) {
            case FIN_RESID_NORM:
              if (args.tp.size > 1) finish_resid_norm_tp<T, MPAD>(ph, args.tp, args.ws, tab, g, G, m, etid, red, tp_epoch0 + p + 1);
              else finish_resid_norm<T, MPAD>(ph, args.ws, tab, g, G, m, etid, red, (tre && p == 0) ? tre + 25 : nullptr);
              break;
            case FIN_SWIGLU_IL: finish_swiglu<T, MPAD>(ph, args.ws, tab, g, G, m, chunk, etid); break;
            case FIN_QKV_ROPE: finish_qkv_rope<T, MPAD>(ph, args.st, args.ws, tab, g, G, m, chunk, etid); break;
            case FIN_STORE: finish_store<T, MPAD>(ph, args.ws, tab, g, G, m, chunk, etid); break;
            default: finish_argmax(ph, args.tp, tp_epoch0 + p + 1, g, m, etid, sval, sidx); break;
          }
          ++done;
        }
        if (tre && p == 0) tre[28] = chain_gtimer();  // items done (before the fences)
        __threadfence();
        fence_proxy_async_all();  // these rows are the next phase's TMA-loaded X operand
        if (tre && p == 0) tre[29] = chain_gtimer();  // fences done
        chain_epi_bar();
        if (etid == 0) red_release_gpu_add(args.sync + kSyncReady + p, done);
        if (tre) tre[1 + 6 * p + 3] = chain_gtimer();  // finish items published
      }
    }
    if (tre) tre[31] = chain_gtimer();
  }

  __syncthreads();
  if (threadIdx.x == 0) {
    pdl_wait();  // (returns at once: the epilogue warps already waited) keeps every global access of this thread behind the wait
    // the last CTA to leave resets the counters for the next launch on this stream (nobody polls after its own exit ticket)
    const int old = atomicAdd(args.sync + kSyncExit, 1);
    if (old == G - 1) {
      for (int i = 0; i < 16; ++i) args.sync[i] = 0;
      if (args.tp.size > 1) {
        const int m_valid = args.m_idx >= 0 ? min(args.m_rows, ld_dep(args.st + args.m_idx)) : args.m_rows;
        int n_resid = 0;
        for (int p = 0; p < args.n_phases; ++p) n_resid += args.ph[p].fin == FIN_RESID_NORM ? 1 : 0;
        *args.tp.epoch += args.n_phases;
        *args.tp.ready_base += n_resid * m_valid;
      }
      if (args.timing) {
        volatile unsigned long long* tm = args.timing;
        const unsigned long long t0 = tm[2], t1 = chain_gtimer();
        if (t0 != 0 && t1 > t0) {
          tm[0] += t1 - t0;
          tm[1] += 1;
        }
        tm[2] = 0;
      }
      __threadfence();
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------------------------
static int chain_grid_for(int dev) {
  static int sms[64] = {};
  if (dev < 0 || dev >= 64) return 0;
  if (!sms[dev]) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0;
    const char* e = getenv("EB200_CHAIN_CTAS");  // tuning / debugging only
    if (e && atoi(e) > 0 && atoi(e) < n) n = atoi(e);
    sms[dev] = n;
  }
  return sms[dev];
}
int chain_grid() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  return chain_grid_for(dev);
}
static int current_device() {
  int dev = 0;
  return cudaGetDevice(&dev) == cudaSuccess ? dev : -1;
}
size_t chain_ws_bytes(int mpad) {
  const int G = chain_grid_for(current_device());
  return static_cast<size_t>(G > 0 ? G : 256) * kChainMaxSlots * mpad * kBlockN * sizeof(float);
}
bool chain_phase_ok(int N, int K, int fin) {
  const int G = chain_grid_for(current_device());
  if (G <= 0 || N < 1 || K < 8 || K % 8) return false;
  const long nkb = (K + kBlockK - 1) / kBlockK, ntiles = (N + kBlockN - 1) / kBlockN;
  const long U = nkb * ntiles;
  if (U * (G + 1) >= (1L << 31)) return false;
  if (fin == FIN_ARGMAX || fin == FIN_STORE_DIRECT) return true;
  if (N % 4) return false;
  if (fin == FIN_RESID_NORM && N > 8192) return false;
  if (fin == FIN_SWIGLU_IL && N % 128) return false;
  if (ntiles > kChainMaxTableTiles) return false;
  const long per = (U + G - 1) / G;
  const long max_segs = (per <= 1) ? 1 : 1 + (per - 1 + nkb - 1) / nkb;
  return max_segs <= kChainMaxSlots;
}

template <typename T, int MPAD> static int launch_chain_t(const ChainMaps& maps, const ChainArgs& a, cudaStream_t s) {
  auto kern = gemm_chain_kernel<T, MPAD>;
  const int dev = current_device();
  const int G = chain_grid_for(dev);
  if (G <= 0) return static_cast<int>(cudaErrorInvalidDevice);
  constexpr int kStageBytes = kWTileBytes + x_tile_bytes(MPAD);
  constexpr int kAccBytes = MPAD * kBlockN * 4;
  const int max_smem = 227 * 1024;
  int stages = (max_smem - 1024 - kChainCtrlBytes - kAccBytes) / kStageBytes;
  if (stages > kChainMaxStages) stages = kChainMaxStages;
  {
    const char* e = getenv("EB200_CHAIN_STAGES");
    if (e && atoi(e) >= 2 && atoi(e) < stages) stages = atoi(e);
  }
  const size_t smem = static_cast<size_t>(stages) * kStageBytes + kChainCtrlBytes + kAccBytes + 1024;
  static bool configured[64] = {};  // per device (and per instantiation: this is a template)
  if (!configured[dev]) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem);
    if (e != cudaSuccess) return static_cast<int>(e);
    configured[dev] = true;
  }
  return static_cast<int>(launch_k(kern, dim3(G), dim3(kChainThreads), smem, s, 1, maps, a, stages));
}

int launch_gemm_chain(int dtype, int mpad, const ChainMaps& maps, const ChainArgs& args_in, cudaStream_t s) {
  ChainArgs args = args_in;
  {
    static int window = -1;
    if (window < 0) {
      const char* e = getenv("EB200_CHAIN_L2_WINDOW");
      window = e ? atoi(e) : 0;  // off by default: prefetch traffic competes with the finish reads
      if (window < 0) window = 0;
      if (window > 256) window = 256;
    }
    if (args.l2_window <= 0) args.l2_window = window;
    if (args.l2_window < 0) args.l2_window = 0;
    static int w_ahead = -2;
    if (w_ahead == -2) {
      const char* e = getenv("EB200_CHAIN_W_AHEAD");
      w_ahead = e ? atoi(e) : -1;
    }
    if (args.w_ahead == 0) args.w_ahead = w_ahead;
  }
  if (args.n_phases < 1 || args.n_phases > kChainMaxPhases || args.m_rows < 1 || args.m_rows > mpad || !args.ws || !args.sync)
    return static_cast<int>(cudaErrorInvalidValue);
  for (int p = 0; p < args.n_phases; ++p) {
    const ChainPhase& ph = args.ph[p];
    if (!chain_phase_ok(ph.N, ph.K, ph.fin) || ph.chunks < 1) return static_cast<int>(cudaErrorInvalidValue);
    if (ph.fin == FIN_RESID_NORM && ph.chunks != 1) return static_cast<int>(cudaErrorInvalidValue);
    if (ph.fin == FIN_ARGMAX && ph.chunks != 1) return static_cast<int>(cudaErrorInvalidValue);
  }
  if (dtype == DT_BF16) {
    if (mpad == 16) return launch_chain_t<__nv_bfloat16, 16>(maps, args, s);
    if (mpad == 64) return launch_chain_t<__nv_bfloat16, 64>(maps, args, s);
  } else if (dtype == DT_FP16) {
    if (mpad == 16) return launch_chain_t<__half, 16>(maps, args, s);
    if (mpad == 64) return launch_chain_t<__half, 64>(maps, args, s);
  }
  return static_cast<int>(cudaErrorInvalidValue);
}

}  // namespace eb
