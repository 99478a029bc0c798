// Fused multi-tensor optimisers and target-network updates on flat fp32 buffers
// (kernel family iii-e/f).  Every network in this repo keeps its parameters in ONE contiguous
// buffer, so each of these is a single HBM-bound launch:
//   Adam   28 B/param (read g,m,v,p; write m,v,p)     Polyak 12 B/param
// The reference issues one assign op per variable (utils/common.py:328-331) and leaves the
// optimiser to TensorFlow (agents/dqn/dqn_agent.py:444).  Counters live on the device as
// int64[2] {value, ticket} and are advanced by the last block to finish, so the launches are
// CUDA-graph replayable.  last_block_ticket uses the low 32-bit word of the ticket; the word is
// back at 0 after every launch, so the high word stays 0.
#include <math.h>

#include "common.cuh"

namespace b200rl {

// kGated: every block returns before touching anything unless *gate % gate_period == 0, so a
// skipped update leaves p, m, v and the step counter as they were.
template <bool kGated>
__global__ void __launch_bounds__(256) adam_tf_kernel(float* __restrict__ p,
                                                      const float* __restrict__ g,
                                                      float* __restrict__ m,
                                                      float* __restrict__ v, int64_t n, float lr,
                                                      float b1, float b2, float eps,
                                                      int64_t* step, const float* grad_scale,
                                                      const int64_t* gate, int64_t gate_period) {
  pdl_prologue();
  if (kGated && gate[0] % gate_period != 0) return;
  __shared__ float s_lr_t;
  const int64_t t = step[0] + 1;
  if (threadIdx.x == 0) {
    // lr_t = lr * sqrt(1 - b2^t) / (1 - b1^t), evaluated in fp32 like the TF kernel inputs
    const float b1p = powf(b1, (float)t), b2p = powf(b2, (float)t);
    s_lr_t = lr * sqrtf(1.f - b2p) / (1.f - b1p);
  }
  __syncthreads();
  const float lr_t = s_lr_t;
  const float gs = grad_scale ? *grad_scale : 1.f;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const float gi = g[i] * gs;
    const float mi = m[i] + (gi - m[i]) * (1.f - b1);          // m += (g - m) * (1 - b1)
    const float vi = v[i] + (gi * gi - v[i]) * (1.f - b2);     // v += (g*g - v) * (1 - b2)
    m[i] = mi;
    v[i] = vi;
    p[i] = p[i] - (mi * lr_t) / (sqrtf(vi) + eps);
  }
  __syncthreads();
  if (threadIdx.x == 0 && last_block_ticket((uint32_t*)(step + 1))) {
    step[0] = t;
    __threadfence();
  }
}

__device__ __forceinline__ void rmsprop_one(float& p, float g, float& ms, float* mg, float& mom,
                                            float lr, float decay, float momentum, float eps,
                                            int centered) {
  const float msi = ms + (g * g - ms) * (1.f - decay);
  ms = msi;
  float denom = msi + eps;
  if (centered) {
    const float mgi = *mg + (g - *mg) * (1.f - decay);
    *mg = mgi;
    denom = msi - mgi * mgi + eps;
  }
  const float mo = mom * momentum + lr * g * rsqrtf(denom);
  mom = mo;
  p = p - mo;
}

// 16-byte accesses when the buffers allow it (flat parameter buffers are 16 B aligned and padded
// to 4 floats per variable): 44 B/param of traffic for the centered form, HBM-bound.
__global__ void __launch_bounds__(256) rmsprop_tf_kernel(float* __restrict__ p,
                                                         const float* __restrict__ g,
                                                         float* __restrict__ ms,
                                                         float* __restrict__ mg,
                                                         float* __restrict__ mom, int64_t n,
                                                         float lr, float decay, float momentum,
                                                         float eps, int centered,
                                                         const float* grad_scale, int vec) {
  pdl_prologue();
  const float gs = grad_scale ? *grad_scale : 1.f;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (vec) {
    const int64_t n4 = n >> 2;
    for (int64_t i = tid; i < n4; i += stride) {
      float4 pv = reinterpret_cast<float4*>(p)[i];
      const float4 gv = reinterpret_cast<const float4*>(g)[i];
      float4 msv = reinterpret_cast<float4*>(ms)[i];
      float4 mgv = centered ? reinterpret_cast<float4*>(mg)[i] : make_float4(0.f, 0.f, 0.f, 0.f);
      float4 mov = reinterpret_cast<float4*>(mom)[i];
      rmsprop_one(pv.x, gv.x * gs, msv.x, &mgv.x, mov.x, lr, decay, momentum, eps, centered);
      rmsprop_one(pv.y, gv.y * gs, msv.y, &mgv.y, mov.y, lr, decay, momentum, eps, centered);
      rmsprop_one(pv.z, gv.z * gs, msv.z, &mgv.z, mov.z, lr, decay, momentum, eps, centered);
      rmsprop_one(pv.w, gv.w * gs, msv.w, &mgv.w, mov.w, lr, decay, momentum, eps, centered);
      reinterpret_cast<float4*>(p)[i] = pv;
      reinterpret_cast<float4*>(ms)[i] = msv;
      if (centered) reinterpret_cast<float4*>(mg)[i] = mgv;
      reinterpret_cast<float4*>(mom)[i] = mov;
    }
    return;
  }
  for (int64_t i = tid; i < n; i += stride)
    rmsprop_one(p[i], g[i] * gs, ms[i], centered ? mg + i : nullptr, mom[i], lr, decay, momentum, eps,
                centered);
}

__global__ void __launch_bounds__(256) soft_update_kernel(float* __restrict__ target,
                                                          const float* __restrict__ source,
                                                          int64_t n, float tau, int64_t period,
                                                          int64_t* counter) {
  pdl_prologue();
  bool fire = true;
  int64_t c = 0;
  if (period > 1) {
    c = counter[0] + 1;  // Periodically: assign_add(1) then mod (utils/common.py:494-497)
    fire = (c % period) == 0;
  }
  if (fire) {
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
      if (tau == 1.f) target[i] = source[i];
      else target[i] = (1.f - tau) * target[i] + tau * source[i];  // utils/common.py:328-331
    }
  }
  if (period > 1) {
    __syncthreads();
    if (threadIdx.x == 0 && last_block_ticket((uint32_t*)(counter + 1))) {
      counter[0] = c;
      __threadfence();
    }
  }
}

__global__ void __launch_bounds__(1024) clip_by_norm_segments_kernel(float* __restrict__ g,
                                                                     const int64_t* __restrict__ offs,
                                                                     float max_norm) {
  pdl_prologue();
  __shared__ float red[32];
  const int64_t b = offs[blockIdx.x], e = offs[blockIdx.x + 1];
  float s = 0.f;
  for (int64_t i = b + threadIdx.x; i < e; i += blockDim.x) s += g[i] * g[i];
  s = block_sum(s, red);
  const float l2 = sqrtf(s);
  // tf.clip_by_norm: t * clip / max(l2, clip)
  const float scale = max_norm / fmaxf(l2, max_norm);
  for (int64_t i = b + threadIdx.x; i < e; i += blockDim.x) g[i] = g[i] * scale;
}

constexpr int kNormBlocks = 296;
__global__ void __launch_bounds__(256) sumsq_partial_kernel(const float* __restrict__ g, int64_t n,
                                                            float* __restrict__ part) {
  pdl_prologue();
  __shared__ float red[32];
  float s = 0.f;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    s += g[i] * g[i];
  s = block_sum(s, red);
  if (threadIdx.x == 0) part[blockIdx.x] = s;
}
__global__ void __launch_bounds__(512) global_norm_final_kernel(const float* __restrict__ part,
                                                                int nparts, float clip,
                                                                float* scale, float* norm) {
  pdl_prologue();
  __shared__ float red[32];
  float s = (threadIdx.x < nparts) ? part[threadIdx.x] : 0.f;
  s = block_sum(s, red);
  if (threadIdx.x == 0) {
    const float l2 = sqrtf(s);
    if (norm) *norm = l2;
    // tf.clip_by_global_norm: scale = clip * min(1/norm, 1/clip) = clip / max(norm, clip)
    if (scale) *scale = clip > 0.f ? clip / fmaxf(l2, clip) : 1.f;
  }
}

__global__ void add_scaled_kernel(float* __restrict__ dst, const float* __restrict__ src,
                                  int64_t n, float alpha) {
  pdl_prologue();
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    dst[i] = dst[i] + alpha * src[i];
}

__global__ void __launch_bounds__(1024) l2_sum_kernel(const float* __restrict__ x, int64_t n,
                                                      float coef, float* out) {
  pdl_prologue();
  __shared__ float red[32];
  float s = 0.f;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) s += x[i] * x[i];
  s = block_sum(s, red);
  if (threadIdx.x == 0) *out = *out + coef * s;
}

__global__ void counter_add_kernel(int64_t* c, int64_t inc) {
  pdl_prologue(); *c = *c + inc; }

static unsigned flat_grid(int64_t n) {
  int64_t blocks = (n + 255) / 256;
  const int64_t cap = (int64_t)kNumSMs * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (unsigned)blocks;
}

}  // namespace b200rl

using namespace b200rl;

extern "C" {

int b200rl_adam_tf(float* p, const float* g, float* m, float* v, int64_t n, float lr,
                   float b1, float b2, float eps, int64_t* step_dev,
                   const float* grad_scale_dev, void* stream) {
  B200RL_CHECK_ARG(p && g && m && v && step_dev && n >= 0, "adam_tf: bad argument");
  if (n == 0) return B200RL_OK;
  B200RL_LAUNCH(adam_tf_kernel<false>, flat_grid(n), 256, 0, (cudaStream_t)stream, p, g, m, v, n, lr, b1, b2, eps, step_dev, grad_scale_dev, (const int64_t*)nullptr, (int64_t)1);
  B200RL_CHECK_LAUNCH("adam_tf");
  return B200RL_OK;
}

int b200rl_adam_tf_gated(float* p, const float* g, float* m, float* v, int64_t n, float lr,
                         float b1, float b2, float eps, int64_t* step_dev,
                         const float* grad_scale_dev, const int64_t* gate_counter_dev,
                         int64_t gate_period, void* stream) {
  B200RL_CHECK_ARG(p && g && m && v && step_dev && n >= 0, "adam_tf_gated: bad argument");
  B200RL_CHECK_ARG(gate_counter_dev && gate_period >= 1, "adam_tf_gated: bad gate");
  if (n == 0) return B200RL_OK;
  B200RL_LAUNCH(adam_tf_kernel<true>, flat_grid(n), 256, 0, (cudaStream_t)stream, p, g, m, v, n, lr, b1, b2, eps, step_dev, grad_scale_dev, gate_counter_dev, gate_period);
  B200RL_CHECK_LAUNCH("adam_tf_gated");
  return B200RL_OK;
}

int b200rl_rmsprop_tf(float* p, const float* g, float* ms, float* mg, float* mom, int64_t n,
                      float lr, float decay, float momentum, float eps, int centered,
                      const float* grad_scale_dev, void* stream) {
  B200RL_CHECK_ARG(p && g && ms && mom && n >= 0, "rmsprop_tf: bad argument");
  B200RL_CHECK_ARG(!centered || mg, "rmsprop_tf: centered needs mg");
  if (n == 0) return B200RL_OK;
  const int vec = (n & 3) == 0 && ((((uintptr_t)p | (uintptr_t)g | (uintptr_t)ms | (uintptr_t)mom |
                                     (uintptr_t)(centered ? mg : p)) & 15) == 0);
  B200RL_LAUNCH(rmsprop_tf_kernel, flat_grid(vec ? n / 4 : n), 256, 0, (cudaStream_t)stream, p, g, ms, mg, mom, n, lr, decay, momentum, eps, centered, grad_scale_dev, vec);
  B200RL_CHECK_LAUNCH("rmsprop_tf");
  return B200RL_OK;
}

int b200rl_soft_update(float* target, const float* source, int64_t n, float tau, int64_t period,
                       int64_t* counter_dev, void* stream) {
  B200RL_CHECK_ARG(target && source && n >= 0, "soft_update: bad argument");
  B200RL_CHECK_ARG(tau >= 0.f && tau <= 1.f, "Input `tau` should be in [0, 1].");
  B200RL_CHECK_ARG(period <= 1 || counter_dev, "soft_update: period>1 needs a counter");
  // tau == 0 or no variables: the blend is a no-op (utils/common.py:301-302), but a Periodically
  // counter still advances on every call (assign_add before tf.cond, utils/common.py:494-497)
  if (n == 0 || tau == 0.f) {
    if (period <= 1) return B200RL_OK;
    n = 0;
  }
  B200RL_LAUNCH(soft_update_kernel, flat_grid(n), 256, 0, (cudaStream_t)stream, target, source, n, tau, period, counter_dev);
  B200RL_CHECK_LAUNCH("soft_update");
  return B200RL_OK;
}

int b200rl_clip_by_norm_segments(float* g, const int64_t* offsets_dev, int64_t nseg,
                                 float max_norm, void* stream) {
  B200RL_CHECK_ARG(g && offsets_dev && nseg >= 0, "clip_by_norm_segments: bad argument");
  if (nseg == 0) return B200RL_OK;
  B200RL_LAUNCH(clip_by_norm_segments_kernel, (unsigned)nseg, 1024, 0, (cudaStream_t)stream, g, offsets_dev, max_norm);
  B200RL_CHECK_LAUNCH("clip_by_norm_segments");
  return B200RL_OK;
}

int b200rl_global_norm_scale(const float* g, int64_t n, float clip, float* scale_dev,
                             float* norm_dev, void* workspace, int64_t ws_bytes, void* stream) {
  B200RL_CHECK_ARG(g && n >= 0, "global_norm_scale: bad argument");
  B200RL_CHECK_ARG(workspace && ws_bytes >= (int64_t)(kNormBlocks * sizeof(float)),
                   "global_norm_scale: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  B200RL_LAUNCH(sumsq_partial_kernel, kNormBlocks, 256, 0, st, g, n, (float*)workspace);
  B200RL_CHECK_LAUNCH("sumsq_partial");
  B200RL_LAUNCH(global_norm_final_kernel, 1, 512, 0, st, (const float*)workspace, kNormBlocks, clip, scale_dev, norm_dev);
  B200RL_CHECK_LAUNCH("global_norm_final");
  return B200RL_OK;
}

int b200rl_add_scaled(float* dst, const float* src, int64_t n, float alpha, void* stream) {
  B200RL_CHECK_ARG(dst && src && n >= 0, "add_scaled: bad argument");
  if (n == 0) return B200RL_OK;
  B200RL_LAUNCH(add_scaled_kernel, flat_grid(n), 256, 0, (cudaStream_t)stream, dst, src, n, alpha);
  B200RL_CHECK_LAUNCH("add_scaled");
  return B200RL_OK;
}

int b200rl_l2_sum(const float* x, int64_t n, float coef, float* out_accum, void* stream) {
  B200RL_CHECK_ARG(x && out_accum && n >= 0, "l2_sum: bad argument");
  B200RL_LAUNCH(l2_sum_kernel, 1, 1024, 0, (cudaStream_t)stream, x, n, coef, out_accum);
  B200RL_CHECK_LAUNCH("l2_sum");
  return B200RL_OK;
}

int b200rl_counter_add(int64_t* counter_dev, int64_t inc, void* stream) {
  B200RL_CHECK_ARG(counter_dev, "counter_add: NULL");
  B200RL_LAUNCH(counter_add_kernel, 1, 1, 0, (cudaStream_t)stream, counter_dev, inc);
  B200RL_CHECK_LAUNCH("counter_add");
  return B200RL_OK;
}

}  // extern "C"
