// Tensor-parallel "all-reduce + residual + RMSNorm" in ONE kernel over NVLink peer memory (no NCCL on the decode path).
//
// A row-parallel projection (o_proj, down_proj: modeling_llama_kv.py:768, :838-845) leaves an unrounded fp32 partial
// [rows][H] on every rank (gemm.cu EPI_PARTIAL_F32).  The NCCL path runs ncclAllReduce (983 KB, latency-bound) ->
// residual_add_f32 -> rmsnorm: three launches per projection, 64 projections per verify pass.  Here one CTA per row does a
// ONE-SHOT exchange (one NVLink hop, no reduce-scatter/all-gather round trip):
//   A. pushes its rank's fp32 row into inbox[epoch parity][rank][row] of EVERY rank's peer window (plain 16-byte stores over
//      NVLink), then -- after a CTA barrier -- one thread publishes the row with a release flag carrying the phase epoch;
//   B. waits for the tp flags of its row, adds the tp rows in rank order (deterministic; every rank computes the same bits),
//      applies T(T(sum) + residual) and the row's RMSNorm and writes x / xn (/ EAGLE-3 tap) LOCALLY.
// Kernel completion therefore means the all-reduce is complete on this rank.  The inbox is double-buffered by epoch parity: a
// fast rank can be at most one phase ahead of a slow rank's reads (it needs the slow rank's flags of the phase in between).
// Flags are monotonic epochs kept in device memory (all ranks run the same launch sequence), so nothing is reset between
// launches or CUDA-graph replays.  The windows are opened with CUDA IPC (engine.cu: eb200_tp_open_peers).
#include <stdio.h>

#include "common.cuh"
#include "kernels.h"

namespace eb {

__device__ __forceinline__ int tpf_ld_acquire_sys(const int* p) {
  int v;
  asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void tpf_st_release_sys(int* p, int v) { asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ void tpf_red_release_sys_add(int* p, int v) {
  asm volatile("red.release.sys.global.add.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long tpf_gtimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// peers run the same launch sequence but are not lock-stepped: wall-clock bound (20 s), then trap instead of hanging the box
__device__ __forceinline__ void tpf_spin_ge(const int* p, int target, int what) {
  unsigned long long t0 = 0;
  unsigned n = 0;
  while (tpf_ld_acquire_sys(p) - target < 0) {
    __nanosleep(64);
    if ((++n & 4095u) == 0) {
      const unsigned long long now = tpf_gtimer();
      if (!t0) t0 = now;
      if (now - t0 > 20000000000ull) {
        printf("eagle_b200: tp_resid_norm timed out waiting for a peer (row %d, flag %d, have %d, want %d)\n", blockIdx.x, what, tpf_ld_acquire_sys(p), target);
        __trap();
      }
    }
  }
}
template <typename P> __device__ __forceinline__ P* tpf_peer(const ChainTP& tp, P* local, int r) {
  return reinterpret_cast<P*>(tp.win[r] + (reinterpret_cast<char*>(local) - tp.win[tp.rank]));
}

constexpr int kTpThreads = 256;
constexpr int kTpMaxPass = 8;  // H <= 8192

template <typename T>
__global__ void __launch_bounds__(kTpThreads) tp_resid_norm_kernel(const TpResidParams p) {
  using D = DT<T>;
  __shared__ float red[kTpThreads / 32];
  pdl_launch_dependents();
  pdl_wait();
  const ChainTP& tp = p.tp;
  const int m = blockIdx.x, rows = gridDim.x, tid = threadIdx.x;
  const int epoch = ld_dep(tp.epoch) + 1;
  const long half = static_cast<long>(tp.size) * 64 * tp.ld_inbox;  // floats per inbox buffer
  const long buf_off = (epoch & 1) ? half : 0;
  // ---- A: this rank's fp32 row -> inbox[parity][rank][m] on every rank
  {
    const float* src = p.partial + static_cast<long>(m) * p.ld_partial;
    const long slot = buf_off + (static_cast<long>(tp.rank) * 64 + m) * tp.ld_inbox;
    float4 v[kTpMaxPass];
#pragma unroll
    for (int i = 0; i < kTpMaxPass; ++i) {
      const int n = (i * kTpThreads + tid) * 4;
      if (n < p.N) v[i] = __ldcg(reinterpret_cast<const float4*>(src + n));
    }
    for (int r = 0; r < tp.size; ++r) {
      float* dst = reinterpret_cast<float*>(tp.win[r] + tp.inbox_off) + slot;
#pragma unroll
      for (int i = 0; i < kTpMaxPass; ++i) {
        const int n = (i * kTpThreads + tid) * 4;
        if (n < p.N) *reinterpret_cast<float4*>(dst + n) = v[i];
      }
    }
  }
  __syncthreads();  // CTA barrier + the release below by one thread per destination (the CUTLASS semaphore pattern)
  if (tid < tp.size) tpf_st_release_sys(reinterpret_cast<int*>(tp.win[tid] + tp.flag_off) + tp.rank * 64 + m, epoch);
  // ---- B: reduce the tp rows of row m and finish it locally
  if (tid < tp.size) tpf_spin_ge(reinterpret_cast<const int*>(tp.win[tp.rank] + tp.flag_off) + tid * 64 + m, epoch, tid);
  __syncthreads();
  const float* inbox = reinterpret_cast<const float*>(tp.win[tp.rank] + tp.inbox_off) + buf_off + static_cast<long>(m) * tp.ld_inbox;
  T* xrow = reinterpret_cast<T*>(p.x) + static_cast<long>(m) * p.ld_x;
  const T* resrow = p.res ? reinterpret_cast<const T*>(p.res) + static_cast<long>(m) * p.ld_res : xrow;
  T* taprow = p.tap ? reinterpret_cast<T*>(p.tap) + static_cast<long>(m) * p.ld_tap : nullptr;
  const T* w = reinterpret_cast<const T*>(p.norm_w);
  float xv[kTpMaxPass][4];
  float ss = 0.f;
  // residual row and norm weights do not depend on the exchange: their loads go out first
  uint2 res_raw[kTpMaxPass], w_raw[kTpMaxPass];
#pragma unroll
  for (int i = 0; i < kTpMaxPass; ++i) {
    const int n = (i * kTpThreads + tid) * 4;
    if (n < p.N) {
      res_raw[i] = __ldcg(reinterpret_cast<const uint2*>(resrow + n));
      if (w) w_raw[i] = __ldg(reinterpret_cast<const uint2*>(w + n));
    }
  }
#pragma unroll
  for (int i = 0; i < kTpMaxPass; ++i) {
    const int n = (i * kTpThreads + tid) * 4;
    if (n < p.N) {
      float4 part[kMaxTp];
#pragma unroll
      for (int src = 0; src < kMaxTp; ++src)
        part[src] = (src < tp.size) ? __ldcg(reinterpret_cast<const float4*>(inbox + static_cast<long>(src) * 64 * tp.ld_inbox + n)) : make_float4(0.f, 0.f, 0.f, 0.f);
      float4 a = part[0];
#pragma unroll
      for (int src = 1; src < kMaxTp; ++src) {  // fixed rank order
        a.x += part[src].x;
        a.y += part[src].y;
        a.z += part[src].z;
        a.w += part[src].w;
      }
      const T* re = reinterpret_cast<const T*>(&res_raw[i]);
      xv[i][0] = rnd<T>(rnd<T>(a.x) + D::to_f(re[0]));  // T(T(sum) + residual)
      xv[i][1] = rnd<T>(rnd<T>(a.y) + D::to_f(re[1]));
      xv[i][2] = rnd<T>(rnd<T>(a.z) + D::to_f(re[2]));
      xv[i][3] = rnd<T>(rnd<T>(a.w) + D::to_f(re[3]));
      uint2 raw;
      T* e = reinterpret_cast<T*>(&raw);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        e[k] = D::from_f(xv[i][k]);
        ss = fmaf(xv[i][k], xv[i][k], ss);
      }
      *reinterpret_cast<uint2*>(xrow + n) = raw;
      if (taprow) *reinterpret_cast<uint2*>(taprow + n) = raw;
    }
  }
  if (w) {
    ss = warp_sum(ss);
    if ((tid & 31) == 0) red[tid >> 5] = ss;
    __syncthreads();
    float tot = 0.f;
#pragma unroll
    for (int k = 0; k < kTpThreads / 32; ++k) tot += red[k];
    const float inv = rsqrtf(tot / static_cast<float>(p.N) + p.eps);  // modeling_llama_kv.py:128-132
    T* orow = reinterpret_cast<T*>(p.xn) + static_cast<long>(m) * p.ld_xn;
#pragma unroll
    for (int i = 0; i < kTpMaxPass; ++i) {
      const int n = (i * kTpThreads + tid) * 4;
      if (n < p.N) {
        const T* we = reinterpret_cast<const T*>(&w_raw[i]);
        uint2 raw;
        T* e = reinterpret_cast<T*>(&raw);
#pragma unroll
        for (int k = 0; k < 4; ++k) e[k] = D::from_f(D::to_f(we[k]) * rnd<T>(xv[i][k] * inv));
        *reinterpret_cast<uint2*>(orow + n) = raw;
      }
    }
  }
  __syncthreads();
  if (tid == 0) {
    const int old = atomicAdd(tp.epoch + 1, 1);  // exit ticket: the last row advances the epoch for the next launch
    if (old == rows - 1) {
      tp.epoch[1] = 0;
      tp.epoch[0] = epoch;
      __threadfence();
    }
  }
}

// Two-shot variant for large tp (reduce-scatter + all-gather by rows): the one-shot kernel pushes (tp-1) x 16 KB per row and
// rank -- 6.9 MB per projection at tp = 8, and every CTA waits for 8 flags.  Here row m is reduced only on
// its owner (m % tp): every rank pushes the row to the owner (1.7 MB per projection at tp = 8), the owner finishes it and pushes
// the bf16 x / xn (/ tap) rows to every rank, then raises a per-row flag there; a CTA leaves when its row has arrived locally.
template <typename T>
__global__ void __launch_bounds__(kTpThreads) tp_resid_norm_2shot_kernel(const TpResidParams p) {
  using D = DT<T>;
  __shared__ float red[kTpThreads / 32];
  pdl_launch_dependents();
  pdl_wait();
  const ChainTP& tp = p.tp;
  const int m = blockIdx.x, rows = gridDim.x, tid = threadIdx.x;
  const int epoch = ld_dep(tp.epoch) + 1;
  const long half = static_cast<long>(tp.size) * 64 * tp.ld_inbox;
  const long buf_off = (epoch & 1) ? half : 0;
  const int owner = m % tp.size;
  // ---- A: this rank's fp32 row -> the owner's inbox
  {
    const float* src = p.partial + static_cast<long>(m) * p.ld_partial;
    float* dst = reinterpret_cast<float*>(tp.win[owner] + tp.inbox_off) + buf_off + (static_cast<long>(tp.rank) * 64 + m) * tp.ld_inbox;
    float4 v[kTpMaxPass];
#pragma unroll
    for (int i = 0; i < kTpMaxPass; ++i) {
      const int n = (i * kTpThreads + tid) * 4;
      if (n < p.N) v[i] = __ldcg(reinterpret_cast<const float4*>(src + n));
    }
#pragma unroll
    for (int i = 0; i < kTpMaxPass; ++i) {
      const int n = (i * kTpThreads + tid) * 4;
      if (n < p.N) *reinterpret_cast<float4*>(dst + n) = v[i];
    }
  }
  __syncthreads();
  if (tid == 0) tpf_st_release_sys(reinterpret_cast<int*>(tp.win[owner] + tp.flag_off) + tp.rank * 64 + m, epoch);
  int* rowflag_local = reinterpret_cast<int*>(tp.win[tp.rank] + tp.ready_off) + 64 + m;  // ints [64, 128) of the counter block
  if (owner == tp.rank) {
    // ---- B: reduce, finish, publish the row on every rank
    if (tid < tp.size) tpf_spin_ge(reinterpret_cast<const int*>(tp.win[tp.rank] + tp.flag_off) + tid * 64 + m, epoch, tid);
    __syncthreads();
    const float* inbox = reinterpret_cast<const float*>(tp.win[tp.rank] + tp.inbox_off) + buf_off + static_cast<long>(m) * tp.ld_inbox;
    T* xrow = reinterpret_cast<T*>(p.x) + static_cast<long>(m) * p.ld_x;
    const T* resrow = p.res ? reinterpret_cast<const T*>(p.res) + static_cast<long>(m) * p.ld_res : xrow;
    T* taprow = p.tap ? reinterpret_cast<T*>(p.tap) + static_cast<long>(m) * p.ld_tap : nullptr;
    const T* w = reinterpret_cast<const T*>(p.norm_w);
    float xv[kTpMaxPass][4];
    float ss = 0.f;
    uint2 res_raw[kTpMaxPass], w_raw[kTpMaxPass];
#pragma unroll
    for (int i = 0; i < kTpMaxPass; ++i) {
      const int n = (i * kTpThreads + tid) * 4;
      if (n < p.N) {
        res_raw[i] = __ldcg(reinterpret_cast<const uint2*>(resrow + n));
        if (w) w_raw[i] = __ldg(reinterpret_cast<const uint2*>(w + n));
      }
    }
#pragma unroll
    for (int i = 0; i < kTpMaxPass; ++i) {
      const int n = (i * kTpThreads + tid) * 4;
      if (n < p.N) {
        float4 part[kMaxTp];
#pragma unroll
        for (int src = 0; src < kMaxTp; ++src)
          part[src] = (src < tp.size) ? __ldcg(reinterpret_cast<const float4*>(inbox + static_cast<long>(src) * 64 * tp.ld_inbox + n)) : make_float4(0.f, 0.f, 0.f, 0.f);
        float4 a = part[0];
#pragma unroll
        for (int src = 1; src < kMaxTp; ++src) {
          a.x += part[src].x;
          a.y += part[src].y;
          a.z += part[src].z;
          a.w += part[src].w;
        }
        const T* re = reinterpret_cast<const T*>(&res_raw[i]);
        xv[i][0] = rnd<T>(rnd<T>(a.x) + D::to_f(re[0]));
        xv[i][1] = rnd<T>(rnd<T>(a.y) + D::to_f(re[1]));
        xv[i][2] = rnd<T>(rnd<T>(a.z) + D::to_f(re[2]));
        xv[i][3] = rnd<T>(rnd<T>(a.w) + D::to_f(re[3]));
        uint2 raw;
        T* e = reinterpret_cast<T*>(&raw);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          e[k] = D::from_f(xv[i][k]);
          ss = fmaf(xv[i][k], xv[i][k], ss);
        }
        for (int r = 0; r < tp.size; ++r) {
          *reinterpret_cast<uint2*>(tpf_peer(tp, xrow, r) + n) = raw;
          if (taprow) *reinterpret_cast<uint2*>(tpf_peer(tp, taprow, r) + n) = raw;
        }
      }
    }
    if (w) {
      ss = warp_sum(ss);
      if ((tid & 31) == 0) red[tid >> 5] = ss;
      __syncthreads();
      float tot = 0.f;
#pragma unroll
      for (int k = 0; k < kTpThreads / 32; ++k) tot += red[k];
      const float inv = rsqrtf(tot / static_cast<float>(p.N) + p.eps);
      T* orow = reinterpret_cast<T*>(p.xn) + static_cast<long>(m) * p.ld_xn;
#pragma unroll
      for (int i = 0; i < kTpMaxPass; ++i) {
        const int n = (i * kTpThreads + tid) * 4;
        if (n < p.N) {
          const T* we = reinterpret_cast<const T*>(&w_raw[i]);
          uint2 raw;
          T* e = reinterpret_cast<T*>(&raw);
#pragma unroll
          for (int k = 0; k < 4; ++k) e[k] = D::from_f(D::to_f(we[k]) * rnd<T>(xv[i][k] * inv));
          for (int r = 0; r < tp.size; ++r) *reinterpret_cast<uint2*>(tpf_peer(tp, orow, r) + n) = raw;
        }
      }
    }
    __syncthreads();
    if (tid < tp.size) tpf_st_release_sys(reinterpret_cast<int*>(tp.win[tid] + tp.ready_off) + 64 + m, epoch);
  }
  // ---- C: the row has arrived on this rank (from its owner)
  if (tid == 0) tpf_spin_ge(rowflag_local, epoch, 98);
  __syncthreads();
  if (tid == 0) {
    const int old = atomicAdd(tp.epoch + 1, 1);
    if (old == rows - 1) {
      tp.epoch[1] = 0;
      tp.epoch[0] = epoch;
      __threadfence();
    }
  }
}

int launch_tp_resid_norm(int dtype, const TpResidParams& p, int rows, cudaStream_t s) {
  if (rows < 1 || rows > 64 || p.N % 4 || p.N > kTpMaxPass * kTpThreads * 4 || p.tp.size < 2 || p.tp.size > kMaxTp) return static_cast<int>(cudaErrorInvalidValue);
  static int two_shot_min = -1;  // smallest tp that uses the two-shot exchange (EB200_TP_TWO_SHOT_MIN)
  if (two_shot_min < 0) {
    const char* e = getenv("EB200_TP_TWO_SHOT_MIN");
    two_shot_min = e ? atoi(e) : 8;  // from 8 ranks the one-shot volume ((tp-1) x 16 KB per row and rank) dominates
    if (two_shot_min < 2) two_shot_min = 2;
  }
  if (p.tp.size >= two_shot_min) {
    if (dtype == DT_BF16) return static_cast<int>(launch_k(tp_resid_norm_2shot_kernel<__nv_bfloat16>, dim3(rows), dim3(kTpThreads), 0, s, 1, p));
    return static_cast<int>(launch_k(tp_resid_norm_2shot_kernel<__half>, dim3(rows), dim3(kTpThreads), 0, s, 1, p));
  }
  if (dtype == DT_BF16) return static_cast<int>(launch_k(tp_resid_norm_kernel<__nv_bfloat16>, dim3(rows), dim3(kTpThreads), 0, s, 1, p));
  return static_cast<int>(launch_k(tp_resid_norm_kernel<__half>, dim3(rows), dim3(kTpThreads), 0, s, 1, p));
}

}  // namespace eb
