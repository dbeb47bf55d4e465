// Internal helpers shared by the kernels of libcup2d_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>

#define CUP2D_BS 8
#define CUP2D_BS2 64

namespace cup2d {

// ---- error plumbing ------------------------------------------------------------------------
void set_error(const std::string &msg);
#define CUP2D_CUDA(call)                                                                         \
  do {                                                                                           \
    cudaError_t _e = (call);                                                                     \
    if (_e != cudaSuccess) {                                                                     \
      cup2d::set_error(std::string(#call) + ": " + cudaGetErrorString(_e) + " (" + __FILE__ +    \
                       ":" + std::to_string(__LINE__) + ")");                                    \
      return CUP2D_ECUDA;                                                                        \
    }                                                                                            \
  } while (0)

// ---- mbarrier + 1-D TMA bulk copy (cp.async.bulk: SASS UBLKCP) -----------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
  asm volatile("{\n"
               ".reg .pred p;\n"
               "WAIT_%=:\n"
               "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
               "@p bra DONE_%=;\n"
               "bra WAIT_%=;\n"
               "DONE_%=:\n"
               "}" ::"r"(smem_u32(bar)),
               "r"(parity)
               : "memory");
}
// global -> shared bulk copy; bytes % 16 == 0, both addresses 16-byte aligned
__device__ __forceinline__ void tma_load_1d(void *smem_dst, const void *gmem_src, uint32_t bytes,
                                            uint64_t *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
                   "r"(smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// ---- numerics ------------------------------------------------------------------------------
// U > 0 for finite doubles without touching the FP64 pipe (NaN is treated as > 0)
__device__ __forceinline__ bool is_pos(double x) {
  int hi = __double2hiint(x), lo = __double2loint(x);
  return hi >= 0 && (hi | lo) != 0;
}
// reciprocal of a positive normal double: MUFU.RCP64H seed + 2 Newton steps (~1 ulp)
__device__ __forceinline__ double fast_rcp_pos(double x) {
  double r;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
  double e = fma(-x, r, 1.0);
  r = fma(r, e, r);
  e = fma(-x, r, 1.0);
  r = fma(r, e, r);
  return r;
}

// ---- cross-GPU plumbing over NVLink peer memory ---------------------------------------------------
// One process per GPU; every rank maps every peer's mailbox (CUDA IPC).  Mailbox layout (u64 words):
//   [0..8)     halo-pull READY epochs, one per source rank     [8..16) halo-pull DONE epochs
//   [16 + (src*2 + parity)*16 ...]  reduction slot: up to 7 doubles, each as two words (32 data bits | epoch << 32)   (16 .. 272)
//   [288..296) PUSHED epochs, one per source rank (halo rows pushed by the producing Krylov kernel)
//   [496] reduction epoch   [497] halo-pull epoch   [498] push epoch   (this rank's counters; device-side, so that a
//         step captured in a CUDA graph carries no host-supplied epoch)
//   [499] error word: first failed wait of this rank (0 = none); the host reads it at its synchronisation points
constexpr int MB_READY = 0, MB_DONE = 8, MB_RED = 16, MB_RED_STRIDE = 16, MB_PUSHED = 288, MB_EPOCH = 496,
              MB_HEPOCH = 497, MB_PEPOCH = 498, MB_ERR = 499, MB_WORDS = 512;
constexpr int COMM_MAX_RANKS = 8;
constexpr unsigned long long COMM_ERR_TIMEOUT = 1; // codes in the error word: (code << 32) | (what << 8) | peer
enum CommWait { CW_REDUCE = 1, CW_HALO_READY = 2, CW_HALO_DONE = 3, CW_PUSHED = 4 };
struct Comm {
  int rank, nranks;
  unsigned long long *mb[COMM_MAX_RANKS]; // mb[r] = rank r's mailbox (mb[rank] is local memory)
  unsigned long long timeout_ns;          // bound of every cross-GPU wait (0 = wait for ever)
};
__device__ __forceinline__ void st_release_sys(unsigned long long *p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long *p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_sys(unsigned long long *p, unsigned long long v) {
  asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_relaxed_sys(const unsigned long long *p) {
  unsigned long long v;
  asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned long long global_timer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)::"memory");
  return t;
}
// coherent (never the non-coherent/texture path, never a stale L1 line) loads of data another GPU wrote into this
// GPU's memory during the running kernel; used after an acquire of the flag that announces the data
__device__ __forceinline__ double ld_coherent(const double *p) {
  double v;
  asm volatile("ld.relaxed.sys.global.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ double2 ld_coherent2(const double2 *p) {
  double2 v;
  asm volatile("ld.relaxed.sys.global.v2.f64 {%0, %1}, [%2];" : "=d"(v.x), "=d"(v.y) : "l"(p) : "memory");
  return v;
}
// Bounded wait for *flag >= target (a peer's release store).  Returns false when the wait was given up: either this
// one ran into the time limit (the error word is set: code, what, peer) or an earlier one did (then nothing waits any
// more, so a step with a dead peer drains in milliseconds and the host finds the error word at its next
// synchronisation point — CUP2D_ECOMM — instead of eight GPUs spinning for ever; the reference aborts through MPI).
__device__ __forceinline__ bool wait_flag(const unsigned long long *flag, unsigned long long target, const Comm &c,
                                          int what, int peer) {
  if (ld_acquire_sys(flag) >= target) return true;
  unsigned long long *err = c.mb[c.rank] + MB_ERR;
  if (ld_relaxed_sys(err) != 0) return false;
  const unsigned long long t0 = global_timer_ns();
  for (unsigned n = 1;; n++) {
    if (ld_acquire_sys(flag) >= target) return true;
    if ((n & 255u) == 0) {
      if (ld_relaxed_sys(err) != 0) return false;
      if (c.timeout_ns && global_timer_ns() - t0 > c.timeout_ns) {
        st_relaxed_sys(err, (COMM_ERR_TIMEOUT << 32) | ((unsigned long long)what << 8) | (unsigned long long)peer);
        return false;
      }
    }
  }
}
// Same bound for a "low-latency" word: 32 data bits in the low half, the epoch in the high half (the flag travels WITH
// the data in one 8-byte store, which is single-copy atomic, so neither fences nor a separate flag round trip are needed)
__device__ __forceinline__ unsigned long long wait_ll_word(const unsigned long long *w, unsigned ep32, const Comm &c, int peer) {
  unsigned long long v = ld_relaxed_sys(w);
  if ((unsigned)(v >> 32) == ep32) return v;
  unsigned long long *err = c.mb[c.rank] + MB_ERR;
  if (ld_relaxed_sys(err) != 0) return v;
  const unsigned long long t0 = global_timer_ns();
  for (unsigned n = 1;; n++) {
    v = ld_relaxed_sys(w);
    if ((unsigned)(v >> 32) == ep32) return v;
    if ((n & 255u) == 0) {
      if (ld_relaxed_sys(err) != 0) return v;
      if (c.timeout_ns && global_timer_ns() - t0 > c.timeout_ns) {
        st_relaxed_sys(err, (COMM_ERR_TIMEOUT << 32) | ((unsigned long long)CW_REDUCE << 8) | (unsigned long long)peer);
        return v;
      }
    }
  }
}
// All-reduce of NS sums + 1 max across ranks, executed by ONE WARP per rank (warp 0 of the last CTA of a
// grid reduction; every lane enters with the same local totals).  Lane r < nranks writes this rank's
// values into rank r's mailbox over NVLink (one peer per lane: one NVLink round trip in total, not one
// per peer), then waits for rank r's contribution in the local mailbox; the contributions are combined
// in rank order with shuffles, so the result is bitwise identical on every lane and on every rank.
template <int NS>
__device__ __forceinline__ void peer_allreduce(const Comm &c, double (&tot)[NS], double &mx, int lane) {
  static_assert(2 * (NS + 1) <= MB_RED_STRIDE, "reduction slot too small");
  if (c.nranks <= 1) return;
  unsigned long long *mine = c.mb[c.rank];
  unsigned long long ep = 0;
  if (lane == 0) {
    ep = ld_relaxed_sys(mine + MB_EPOCH) + 1;
    st_relaxed_sys(mine + MB_EPOCH, ep);
  }
  ep = __shfl_sync(0xffffffffu, ep, 0);
  const int par = (int)(ep & 1);
  const unsigned ep32 = (unsigned)ep; // never 0 within 2^32 - 1 reductions of a context (the mailbox starts zeroed)
  // Every value goes out as two 8-byte words, each carrying 32 bits of the double and the epoch: a word is valid the
  // moment its epoch matches, whatever order the stores arrive in.  A slot of parity p is rewritten two reductions
  // later, which the writer can only reach after the reader contributed to the reduction in between, i.e. after it
  // finished reading.
  if (lane < c.nranks) {
    unsigned long long *dst = c.mb[lane] + MB_RED + (c.rank * 2 + par) * MB_RED_STRIDE;
#pragma unroll
    for (int k = 0; k <= NS; k++) {
      const unsigned long long b = (unsigned long long)__double_as_longlong(k < NS ? tot[k] : mx);
      st_relaxed_sys(dst + 2 * k, (b & 0xffffffffull) | ((unsigned long long)ep32 << 32));
      st_relaxed_sys(dst + 2 * k + 1, (b >> 32) | ((unsigned long long)ep32 << 32));
    }
  }
  double v[NS + 1];
#pragma unroll
  for (int k = 0; k <= NS; k++) v[k] = 0.0;
  if (lane < c.nranks) {
    const unsigned long long *src = mine + MB_RED + (lane * 2 + par) * MB_RED_STRIDE;
#pragma unroll
    for (int k = 0; k <= NS; k++) {
      const unsigned long long lo = wait_ll_word(src + 2 * k, ep32, c, lane), hi = wait_ll_word(src + 2 * k + 1, ep32, c, lane);
      v[k] = __longlong_as_double((long long)((lo & 0xffffffffull) | (hi << 32)));
    }
  }
  double acc[NS];
#pragma unroll
  for (int k = 0; k < NS; k++) acc[k] = 0;
  double am = 0;
  for (int r = 0; r < c.nranks; r++) {
#pragma unroll
    for (int k = 0; k < NS; k++) acc[k] += __shfl_sync(0xffffffffu, v[k], r);
    am = fmax(am, __shfl_sync(0xffffffffu, v[NS], r));
  }
#pragma unroll
  for (int k = 0; k < NS; k++) tot[k] = acc[k];
  mx = am;
}

// ---- block reductions -----------------------------------------------------------------------
template <int N> __device__ __forceinline__ void warp_sum(double (&v)[N]) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
#pragma unroll
    for (int k = 0; k < N; k++) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Deterministic grid reduction: every CTA writes its partial (NS sums + 1 max) to
// partials[blockIdx.x]; the CTA that finishes last re-reduces all partials in a fixed order and
// calls fin(sums, max).  Result is independent of CTA scheduling.  `counter` must be 0 on entry and
// is reset to 0 by the last CTA.  With more than one rank the finalizer first all-reduces the local
// totals over NVLink peer memory (peer_allreduce), so fin sees global values on every rank.
template <int NS, int NT, class Fin>
__device__ __forceinline__ void grid_reduce(double (&sums)[NS], double mx, double *partials,
                                            unsigned int *counter, const Comm &comm, Fin fin) {
  __shared__ double s_red[(NS + 1) * (NT / 32)];
  __shared__ bool s_last;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  warp_sum<NS>(sums);
  mx = warp_max(mx);
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < NS; k++) s_red[k * (NT / 32) + warp] = sums[k];
    s_red[NS * (NT / 32) + warp] = mx;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double *out = partials + (size_t)blockIdx.x * (NS + 1);
#pragma unroll
    for (int k = 0; k < NS; k++) {
      double a = 0;
      for (int w = 0; w < NT / 32; w++) a += s_red[k * (NT / 32) + w];
      out[k] = a;
    }
    double m = 0;
    for (int w = 0; w < NT / 32; w++) m = fmax(m, s_red[NS * (NT / 32) + w]);
    out[NS] = m;
    __threadfence();
    unsigned int done = atomicAdd(counter, 1u);
    s_last = (done == gridDim.x - 1);
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  // last CTA: fixed-order re-reduction over all CTA partials
  double acc[NS];
#pragma unroll
  for (int k = 0; k < NS; k++) acc[k] = 0;
  double am = 0;
  for (unsigned int b = threadIdx.x; b < gridDim.x; b += NT) {
    const volatile double *in = partials + (size_t)b * (NS + 1);
#pragma unroll
    for (int k = 0; k < NS; k++) acc[k] += in[k];
    am = fmax(am, in[NS]);
  }
  __syncthreads(); // s_red reuse
  warp_sum<NS>(acc);
  am = warp_max(am);
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < NS; k++) s_red[k * (NT / 32) + warp] = acc[k];
    s_red[NS * (NT / 32) + warp] = am;
  }
  __syncthreads();
  if (warp == 0) { // warp 0 finishes: lane 0 sums the warps in order, the warp all-reduces across GPUs
    double tot[NS];
    double m = 0;
#pragma unroll
    for (int k = 0; k < NS; k++) {
      double a = 0;
      for (int w = 0; w < NT / 32; w++) a += s_red[k * (NT / 32) + w];
      tot[k] = a;
    }
    for (int w = 0; w < NT / 32; w++) m = fmax(m, s_red[NS * (NT / 32) + w]);
    peer_allreduce<NS>(comm, tot, m, lane);
    if (lane == 0) {
      *counter = 0;
      fin(tot, m);
      __threadfence();
    }
  }
}

} // namespace cup2d
