// Shared device/host helpers for libb200rl (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/b200rl.h"

namespace b200rl {

// ---- error plumbing ---------------------------------------------------------------------
void set_error(const char* fmt, ...);
void count_launch(int n = 1);

#define B200RL_CHECK_ARG(cond, ...)          \
  do {                                       \
    if (!(cond)) {                           \
      ::b200rl::set_error(__VA_ARGS__);      \
      return B200RL_ERR_INVALID;             \
    }                                        \
  } while (0)

#define B200RL_CHECK_LAUNCH(name)                                                   \
  do {                                                                              \
    cudaError_t e__ = cudaGetLastError();                                           \
    if (e__ != cudaSuccess) {                                                       \
      ::b200rl::set_error("%s: CUDA launch failed: %s", name, cudaGetErrorString(e__)); \
      return B200RL_ERR_CUDA;                                                       \
    }                                                                               \
    ::b200rl::count_launch();                                                       \
  } while (0)

constexpr int kNumSMs = 132;  // H100 SXM

// ---- programmatic dependent launch (PDL) ---------------------------------------------------
// Every kernel of the library starts with pdl_prologue(): `griddepcontrol.wait` blocks until the
// grids this launch depends on have completed and flushed their memory (a no-op for launches
// without the attribute), then `griddepcontrol.launch_dependents` lets the NEXT kernel of the
// stream be scheduled while this one runs.  With the wait first, ordering is exactly stream
// order; what is gained is that the next grid's launch latency and block scheduling overlap this
// grid's execution instead of following it (2-3 us per node in a captured step).
// Kernels with a global-memory-free prologue (tc_gemm: shared-memory set-up) call
// pdl_launch_dependents() first and pdl_wait() after the prologue instead.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
__device__ __forceinline__ void pdl_prologue() {
  pdl_wait();
  pdl_launch_dependents();
}

// Every launch carries cudaLaunchAttributeProgrammaticStreamSerialization.
template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
                            cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<Args&&>(args)...);
}
// Launch errors are picked up by the B200RL_CHECK_LAUNCH that follows every launch.
#define B200RL_LAUNCH(kernel, grid, block, smem, st, ...) \
  (void)::b200rl::launch_k(kernel, dim3(grid), dim3(block), (size_t)(smem), st, __VA_ARGS__)

// 256-thread blocks for n elements, one element per thread.
static inline unsigned blocks_of_256(int64_t n) { return (unsigned)((n + 255) / 256); }

// Width of a one-block reduction over n elements: n rounded up to whole warps, at most 1024.
static inline unsigned reduce_threads(int64_t n) {
  return n >= 1024 ? 1024u : (unsigned)((n + 31) / 32 * 32);
}

// ---- Philox4x32-10 (Salmon et al. 2011), the counter-based generator of this library -----
// counter = (elem_lo, elem_hi, call_lo, call_hi), key = (seed_lo, seed_hi).
// oracle/philox.py restates exactly this; tests/test_philox.py pins both against the
// Random123 known-answer vectors.
struct Philox4 {
  uint32_t x, y, z, w;
};

__host__ __device__ __forceinline__ uint32_t mulhi32(uint32_t a, uint32_t b) {
#ifdef __CUDA_ARCH__
  return __umulhi(a, b);
#else
  return (uint32_t)(((uint64_t)a * (uint64_t)b) >> 32);
#endif
}

__host__ __device__ __forceinline__ Philox4 philox4x32_10(uint64_t elem, uint64_t call,
                                                           uint64_t seed) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
  uint32_t c0 = (uint32_t)elem, c1 = (uint32_t)(elem >> 32);
  uint32_t c2 = (uint32_t)call, c3 = (uint32_t)(call >> 32);
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0 = mulhi32(M0, c0), lo0 = M0 * c0;
    uint32_t hi1 = mulhi32(M1, c2), lo1 = M1 * c2;
    uint32_t n0 = hi1 ^ c1 ^ k0;
    uint32_t n2 = hi0 ^ c3 ^ k1;
    c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
    k0 += W0; k1 += W1;
  }
  return Philox4{c0, c1, c2, c3};
}

// uniform int64 in [lo, hi): lo + u64 % (hi-lo)  (TF's int64 uniform also reduces by modulo).
__host__ __device__ __forceinline__ int64_t uniform_i64(uint32_t a, uint32_t b, int64_t lo,
                                                         int64_t hi) {
  uint64_t u = ((uint64_t)b << 32) | (uint64_t)a;
  uint64_t range = (uint64_t)(hi - lo);
  return lo + (int64_t)(u % range);
}
// uniform f32 in [0,1) with 24 random bits.
__host__ __device__ __forceinline__ float uniform_f32(uint32_t a) {
  return (float)(a >> 8) * (1.0f / 16777216.0f);
}

// N(0, 1) by Box-Muller on one Philox draw (u1 in (0, 1] from x, the angle from y).
__device__ __forceinline__ float philox_normal(uint64_t elem, uint64_t call, uint64_t seed) {
  const Philox4 r = philox4x32_10(elem, call, seed);
  const float u1 = ((float)(r.x >> 8) + 1.0f) * (1.0f / 16777216.0f);
  return sqrtf(-2.f * logf(u1)) * cospif(2.f * uniform_f32(r.y));
}

// ---- last-block-done ticket -----------------------------------------------------------------
// The device-resident counters (Philox call index, replay last_id, optimiser step, Periodically
// counter) are advanced once per launch by the last block of the grid to finish, so a captured
// graph sees the new value on every replay.  One thread per block calls this after a
// __syncthreads() that follows the block's last read of the counters.  It returns true in exactly
// one block, with the ticket already back at 0; that block then stores the counters and calls
// __threadfence().  The ticket counts every block of the grid, whatever its shape.
__device__ __forceinline__ bool last_block_ticket(uint32_t* ticket) {
  __threadfence();
  const unsigned int tk = atomicAdd(ticket, 1u);
  if (tk != gridDim.x * gridDim.y * gridDim.z - 1) return false;
  *ticket = 0u;
  return true;
}

// Advances the Philox call counter rng_call = uint64[2] {call, ticket} once per launch, so a
// captured graph draws fresh values on every replay.  Every thread of the grid must reach it, and
// every block must have read rng_call[0] before.
__device__ __forceinline__ void next_rng_call(uint64_t* rng_call) {
  __syncthreads();
  if (threadIdx.x == 0 && last_block_ticket((uint32_t*)(rng_call + 1))) {
    rng_call[0] = rng_call[0] + 1;
    __threadfence();
  }
}

// ---- TD element loss (td3.cu, ddpg.cu, qtopt.cu) ------------------------------------------------
// l = l(e) + l0 and g = dl/dq for the TD error e = y - q.  Huber (delta 1): l(e) = 0.5 e^2 for
// |e| <= 1 else |e| - 0.5, dl/dq = -clip(e, -1, 1); squared: l(e) = e^2, dl/dq = -2e.
// l0 takes a second critic's loss, so the twin-critic squared sum is fma(e1, e1, e2^2).  The
// default l0 = -0 is the exact additive identity (x + -0 = x and fma(e, e, -0) = e * e for
// every x and e).
__device__ __forceinline__ void td_elem_loss(float e, int kind, float& l, float& g,
                                             float l0 = -0.f) {
  if (kind == B200RL_LOSS_HUBER) {
    const float a = fabsf(e);
    l = (a <= 1.f ? 0.5f * e * e : a - 0.5f) + l0;
    g = -fminf(fmaxf(e, -1.f), 1.f);
  } else {
    l = fmaf(e, e, l0);
    g = -2.f * e;
  }
}

// ---- 16-byte streaming copies -------------------------------------------------------------
__device__ __forceinline__ int4 ld_stream16(const void* p) {
  int4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ void st_stream16(void* p, const int4& v) {
  asm volatile("st.global.L1::no_allocate.v4.s32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x),
               "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---- tanh-Normal helpers (sac.cu, cql.cu) --------------------------------------------------
constexpr float kLog2PiS = 1.8378770664093453f;
constexpr float kLog2 = 0.6931471805599453f;

__device__ __forceinline__ float softplus_f(float x) {
  return x > 20.f ? x : log1pf(expf(x));
}

// ---- row groups: a row of a [N, W] array handled by G lanes (lane l takes columns l, l+G, ...) --
// Every warp runs the same number of row iterations (groups past N repeat their warp's first row
// and discard the result), so the full-mask shuffles never diverge.
template <int G>
__device__ __forceinline__ float grp_max(float v) {
#pragma unroll
  for (int o = G / 2; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o, G));
  return v;
}
template <int G>
__device__ __forceinline__ float grp_sum(float v) {
#pragma unroll
  for (int o = G / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o, G);
  return v;
}

// Lanes per row of width W: one thread for narrow rows, 8 or 32 lanes once a row spans more than
// 8 / 64 columns (coalesced row reads, shuffle reductions).
static inline int lane_group(int64_t width) { return width <= 8 ? 1 : (width <= 64 ? 8 : 32); }

// 256-thread blocks for N rows of G lanes each, at most `cap` (the partials one final block
// reduces); the group kernels stride over the rest.
static inline unsigned group_blocks(int64_t N, int G, int64_t cap) {
  const int64_t nb = (N * G + 255) / 256;
  return (unsigned)(nb > cap ? cap : nb);
}

// Row iteration shared by the group kernels: n is this group's row, n0 the row of the warp's first
// group (warp-uniform loop bound).
#define B200RL_GROUP_ROWS(G, N)                                                              \
  const int lane = (int)(threadIdx.x % (G));                                                 \
  const int64_t stride_ = (int64_t)gridDim.x * blockDim.x / (G);                             \
  for (int64_t n = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / (G),                   \
               n0 = ((int64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u)) / (G);         \
       n0 < (N); n += stride_, n0 += stride_)

// ---- Categorical rows (ppo.cu, reinforce.cu) ---------------------------------------------------
// Max-subtracted log-softmax statistics of one row: m = max z, s = sum exp(z - m),
// t = sum exp(z - m) * (z - m).  log p_j = (z_j - m) - log s, entropy = log s - t / s.
template <int G>
__device__ __forceinline__ void row_softmax_stats(const float* __restrict__ z, int64_t A, int lane,
                                                  float& m, float& s, float& t) {
  m = -INFINITY;
  for (int64_t j = lane; j < A; j += G) m = fmaxf(m, z[j]);
  m = grp_max<G>(m);
  s = 0.f; t = 0.f;
  for (int64_t j = lane; j < A; j += G) {
    const float d = z[j] - m;
    const float e = expf(d);
    s += e;
    t += e > 0.f ? e * d : 0.f;
  }
  s = grp_sum<G>(s);
  t = grp_sum<G>(t);
}

__device__ __forceinline__ int clamp_action(int32_t a, int64_t A, int32_t* nan_flag) {
  if (a < 0 || a >= A) {          // out-of-range action: read a valid column, report it
    if (nan_flag) *nan_flag = 1;
    a = a < 0 ? 0 : (int32_t)(A - 1);
  }
  return a;
}

// Block-wide sum (blockDim.x multiple of 32, <= 1024). Deterministic order.
__device__ __forceinline__ float block_sum(float v, float* smem32) {
  int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) smem32[wid] = v;
  __syncthreads();
  int nw = (blockDim.x + 31) >> 5;
  float r = (threadIdx.x < nw) ? smem32[threadIdx.x] : 0.f;
  if (wid == 0) r = warp_sum(r);
  if (threadIdx.x == 0) smem32[0] = r;
  __syncthreads();
  r = smem32[0];
  return r;
}

// ---- multi-CTA sequence-loss totals (ddpg.cu, sac.cu) -------------------------------------------
// Every block stores its block_sum of `partial` in partials[blockIdx.x]; the block that takes the
// last ticket adds the partials in index order and returns the total there (threads of other
// blocks return 0 and must not use it).  No float atomics: the sum has a fixed order per grid.
__device__ __forceinline__ float seq_loss_total(float partial, float* partials, uint32_t* ticket,
                                                float* red, bool* last) {
  const float total = block_sum(partial, red);
  if (threadIdx.x == 0) {
    partials[blockIdx.x] = total;
    *last = last_block_ticket(ticket);
  }
  __syncthreads();
  if (!*last) return 0.f;
  float s = 0.f;
  for (unsigned i = threadIdx.x; i < gridDim.x; i += blockDim.x) s += __ldcg(partials + i);
  return block_sum(s, red);
}

}  // namespace b200rl
