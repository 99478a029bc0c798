// REINFORCE update math (kernel family iii-d): episode masks, return / advantage normalisation,
// policy-gradient / entropy / value losses and their gradients, including the path through which
// the policy-gradient loss also trains the value network.
//
// Restates, per (b,t) element of a batch-major [B,T] batch (agents/reinforce/reinforce_agent.py):
//   num_episodes, valid mask, weights   :327-350 (is_last = next_step_type == LAST)
//   advantages, _standard_normalize     :48-61, :352-379 (moments over all B*T entries,
//                                        (adv - mean) / (sqrt(var) + float32 eps))
//   policy_gradient_loss                :442-506 (masked by step_type != LAST, / num_episodes)
//   _entropy_loss / entropy term        :64-80, :508-534 (mean over B*T)
//   value_estimation_loss               :536-567 (/ num_episodes)
// value_preds are not stop-gradient inside the advantages (:284-292, :355-364), so with a baseline
// d(pg)/dV = -d(pg)/d(adv), through the normalisation when it is on.
//
// Stages (every reduction has a fixed order, so a graph replay equals the eager call bit for bit):
//   1. rf_stats_kernel       a warp per trajectory row: last[b] = largest t with is_last (-1 if
//                            none), the row's is_last count, Welford moments of adv; Chan-merged
//                            per block.
//   2. rf_stats_final_kernel one warp merges the block partials in index order: mean, sigma,
//                            D = sigma + eps, num_episodes.
//   3. rf_loss_{normal,cat}  per row: losses, d(distribution params), the value-loss part of dV and
//                            g = d(pg)/d(adv_n) with block partials of sum g, sum g (adv - mean).
//   4. rf_loss_final_kernel  losses[6], the dV coefficients, the flag bits.
//   5. rf_dv_kernel          (baseline + normalisation only) the policy-gradient part of dV.
#include <math.h>

#include "common.cuh"

namespace b200rl {

namespace {

constexpr int kStepLastR = 2;
constexpr float kEpsF32 = 1.1920928955078125e-07f;   // np.finfo(np.float32).eps
constexpr int kRfStatBlocks = 2 * kNumSMs;            // stage-1 partials (<= 32 * 9 per lane)
constexpr int kRfLossBlocks = 512;                    // stage-3 partials, one per final thread
// workspace layout (floats)
constexpr int kWsStat = 0;                            // [kRfStatBlocks, 4] {n, mean, m2, episodes}
constexpr int kWsScalars = 1088;                      // [8] see rf_stats_final_kernel
constexpr int kWsLoss = 1152;                         // [kRfLossBlocks, 5]
constexpr int kWsLast = 4096;                         // int32 [round4(B)], then g [N]

struct Mom {
  float n, mean, m2;
};

// Chan et al. pairwise merge of (count, mean, M2); with b = {1, x, 0} it is Welford's update.
__device__ __forceinline__ Mom mom_merge(Mom a, const Mom& b) {
  const float n = a.n + b.n;
  if (b.n == 0.f) return a;
  const float d = b.mean - a.mean;
  const float f = b.n / n;
  return Mom{n, a.mean + d * f, a.m2 + b.m2 + d * d * a.n * f};
}

__device__ __forceinline__ Mom mom_shfl_down(const Mom& m, int o) {
  return Mom{__shfl_down_sync(0xffffffffu, m.n, o), __shfl_down_sync(0xffffffffu, m.mean, o),
             __shfl_down_sync(0xffffffffu, m.m2, o)};
}

// lane 0 ends with the merge of the warp's 32 values (fixed tree order)
__device__ __forceinline__ Mom warp_mom(Mom m) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = mom_merge(m, mom_shfl_down(m, o));
  return m;
}

struct RfArgs {
  const float* p0; const float* p1; int64_t ld;   // Normal (loc, scale) or Categorical logits
  const void* action;                             // float [N, A] or int32 [N]
  const float* ret; const float* v;               // [B, T]; v may be NULL
  const int32_t* step_type; const int32_t* next_step_type;
  const float* w;                                 // user weights [B, T] or NULL
  int64_t B, T, N, A;
  int use_adv, normalize;
  float ent_coef, value_coef;
  float* d0; float* d1; int64_t ld_g;             // gradients, same layout as the params
  float* dv;                                      // [N] or NULL
  int32_t* flag;
  float* ws;
};

__device__ __forceinline__ float rf_adv(const RfArgs& a, int64_t n) {
  return a.use_adv ? a.ret[n] - a.v[n] : a.ret[n];
}

// ---- stage 1 ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) rf_stats_kernel(const RfArgs a) {
  pdl_prologue();
  __shared__ Mom sm[8];
  __shared__ float se[8];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int32_t* last = reinterpret_cast<int32_t*>(a.ws + kWsLast);
  Mom acc{0.f, 0.f, 0.f};
  float eps_cnt = 0.f;
  const int64_t warps = (int64_t)gridDim.x * 8;
  for (int64_t b = (int64_t)blockIdx.x * 8 + wid; b < a.B; b += warps) {
    int lt = -1;
    float cnt = 0.f;
    Mom m{0.f, 0.f, 0.f};
    for (int64_t t = lane; t < a.T; t += 32) {
      const int64_t n = b * a.T + t;
      if (a.next_step_type[n] == kStepLastR) { lt = (int)t; cnt += 1.f; }
      m = mom_merge(m, Mom{1.f, rf_adv(a, n), 0.f});
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      lt = max(lt, __shfl_down_sync(0xffffffffu, lt, o));
      cnt += __shfl_down_sync(0xffffffffu, cnt, o);
    }
    m = warp_mom(m);
    if (lane == 0) {
      last[b] = lt;
      acc = mom_merge(acc, m);
      eps_cnt += cnt;
    }
  }
  if (lane == 0) { sm[wid] = acc; se[wid] = eps_cnt; }
  __syncthreads();
  if (threadIdx.x == 0) {
    Mom r = sm[0];
    float e = se[0];
    for (int i = 1; i < 8; ++i) { r = mom_merge(r, sm[i]); e += se[i]; }
    float* p = a.ws + kWsStat + (int64_t)blockIdx.x * 4;
    p[0] = r.n; p[1] = r.mean; p[2] = r.m2; p[3] = e;
  }
}

// ---- stage 2 ---------------------------------------------------------------------------------
// scalars[0..7] = {mean, sigma, D = sigma + eps, num_episodes, 1/num_episodes (0 when there is
// none), g_bar, S / (N sigma D^2) (0 when sigma = 0), unused}
__global__ void rf_stats_final_kernel(float* __restrict__ ws, int nblocks,
                                      float* __restrict__ num_episodes_out) {
  pdl_prologue();
  const int lane = threadIdx.x;
  Mom m{0.f, 0.f, 0.f};
  float e = 0.f;
  for (int i = lane; i < nblocks; i += 32) {
    const float* p = ws + kWsStat + i * 4;
    m = mom_merge(m, Mom{p[0], p[1], p[2]});
    e += p[3];
  }
  m = warp_mom(m);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) e += __shfl_down_sync(0xffffffffu, e, o);
  if (lane == 0) {
    float* s = ws + kWsScalars;
    const float sigma = sqrtf(m.m2 / m.n);
    s[0] = m.mean;
    s[1] = sigma;
    s[2] = sigma + kEpsF32;
    s[3] = e;
    s[4] = e > 0.f ? 1.f / e : 0.f;
    if (num_episodes_out) *num_episodes_out = e;
  }
}

// ---- stage 3 ---------------------------------------------------------------------------------
// Per-row terms shared by both heads.  Returns the row's weight w_eff = user weight * valid and
// c = w_eff * (step_type != LAST); writes the value-loss part of dV (and all of dV when the
// stage-5 pass is not needed).
struct RowTerms {
  float w_eff, c, adv_n, adv_c, g_lp_scale;
};

__device__ __forceinline__ RowTerms rf_row(const RfArgs& a, int64_t n, const float* sc) {
  const int64_t b = n / a.T, t = n - b * a.T;
  const int32_t* last = reinterpret_cast<const int32_t*>(a.ws + kWsLast);
  RowTerms r;
  const float valid = t <= (int64_t)last[b] ? 1.f : 0.f;
  r.w_eff = a.w ? a.w[n] * valid : valid;
  r.c = a.step_type[n] == kStepLastR ? 0.f : r.w_eff;
  const float adv = rf_adv(a, n);
  r.adv_c = adv - sc[0];
  r.adv_n = a.normalize ? r.adv_c / sc[2] : adv;
  return r;
}

__device__ __forceinline__ void rf_row_value(const RfArgs& a, int64_t n, const RowTerms& r,
                                             float logp, const float* sc, float& s_v, float& s_g,
                                             float& s_gd) {
  if (!a.v) return;
  const float R = a.ret[n], v = a.v[n];
  s_v += (R - v) * (R - v) * r.w_eff;
  float dv = a.value_coef * 2.f * (v - R) * r.w_eff * sc[4];
  if (a.use_adv) {
    const float g = -logp * r.c * sc[4];        // d(pg) / d(adv_n)
    if (a.normalize) {
      a.ws[kWsLast + ((a.B + 3) & ~3LL) + n] = g;
      s_g += g;
      s_gd += g * r.adv_c;
    } else {
      dv -= g;                                   // adv = R - V
    }
  }
  a.dv[n] = dv;
}

__device__ __forceinline__ void rf_block_partials(const RfArgs& a, float s_pg, float s_ent,
                                                  float s_v, float s_g, float s_gd, float* red) {
  const float t_pg = block_sum(s_pg, red);
  const float t_ent = block_sum(s_ent, red);
  const float t_v = block_sum(s_v, red);
  const float t_g = block_sum(s_g, red);
  const float t_gd = block_sum(s_gd, red);
  if (threadIdx.x == 0) {
    float* p = a.ws + kWsLoss + (int64_t)blockIdx.x * 5;
    p[0] = t_pg; p[1] = t_ent; p[2] = t_v; p[3] = t_g; p[4] = t_gd;
  }
}

// Normal(loc, scale), one thread per row: log pi and entropy summed over the A action dims.
__global__ void __launch_bounds__(256) rf_loss_normal_kernel(const RfArgs a) {
  pdl_prologue();
  __shared__ float red[32];
  const float* sc = a.ws + kWsScalars;
  const float inv_n = 1.f / (float)a.N;
  const float* action = static_cast<const float*>(a.action);
  float s_pg = 0.f, s_ent = 0.f, s_v = 0.f, s_g = 0.f, s_gd = 0.f;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; n < a.N; n += stride) {
    const RowTerms r = rf_row(a, n, sc);
    float logp = 0.f, ent = 0.f;
    for (int64_t k = 0; k < a.A; ++k) {
      const float mu = a.p0[n * a.ld + k], sg = a.p1[n * a.ld + k];
      const float z = (action[n * a.A + k] - mu) / sg;
      const float lsg = logf(sg);
      logp += -0.5f * z * z - lsg - 0.5f * kLog2PiS;
      ent += 0.5f + 0.5f * kLog2PiS + lsg;
    }
    s_pg -= logp * r.c * r.adv_n;
    s_ent -= ent * r.w_eff;
    const float g_lp = -r.c * r.adv_n * sc[4];            // d(pg) / d(log pi)
    const float g_ent = -a.ent_coef * r.w_eff * inv_n;    // d(entropy loss) / d(H)
    for (int64_t k = 0; k < a.A; ++k) {
      const float mu = a.p0[n * a.ld + k], sg = a.p1[n * a.ld + k];
      const float d = action[n * a.A + k] - mu;
      const float inv = 1.f / sg;
      a.d0[n * a.ld_g + k] = g_lp * d * inv * inv;
      a.d1[n * a.ld_g + k] = g_lp * (d * d * inv * inv * inv - inv) + g_ent * inv;
    }
    rf_row_value(a, n, r, logp, sc, s_v, s_g, s_gd);
  }
  rf_block_partials(a, s_pg, s_ent, s_v, s_g, s_gd, red);
}

// Categorical(logits), G lanes per row (as ppo_loss_cat_kernel).
template <int G>
__global__ void __launch_bounds__(256) rf_loss_cat_kernel(const RfArgs a) {
  pdl_prologue();
  __shared__ float red[32];
  const float* sc = a.ws + kWsScalars;
  const float inv_n = 1.f / (float)a.N;
  const int32_t* action = static_cast<const int32_t*>(a.action);
  float s_pg = 0.f, s_ent = 0.f, s_v = 0.f, s_g = 0.f, s_gd = 0.f;
  B200RL_GROUP_ROWS(G, a.N) {
    const bool valid = n < a.N;
    const int64_t r_ = valid ? n : n0;
    const float* z = a.p0 + r_ * a.ld;
    const int32_t raw = action[r_];
    if (valid && lane == 0 && (raw < 0 || raw >= a.A)) atomicOr(a.flag, 1);
    const int act = clamp_action(raw, a.A, nullptr);
    float m, s, t;
    row_softmax_stats<G>(z, a.A, lane, m, s, t);
    const float log_s = logf(s);
    const float ent = log_s - t / s;
    const float logp = (z[act] - m) - log_s;
    const RowTerms r = rf_row(a, r_, sc);
    const float g_lp = -r.c * r.adv_n * sc[4];
    const float g_ent = -a.ent_coef * r.w_eff * inv_n;
    if (valid && lane == 0) {
      s_pg -= logp * r.c * r.adv_n;
      s_ent -= ent * r.w_eff;
      rf_row_value(a, r_, r, logp, sc, s_v, s_g, s_gd);
    }
    if (valid) {
      for (int64_t j = lane; j < a.A; j += G) {
        const float lpj = (z[j] - m) - log_s;
        const float p = expf(lpj);
        a.d0[r_ * a.ld_g + j] = g_lp * ((j == act ? 1.f : 0.f) - p) + g_ent * (-p * (lpj + ent));
      }
    }
  }
  rf_block_partials(a, s_pg, s_ent, s_v, s_g, s_gd, red);
}

// ---- stage 4 ---------------------------------------------------------------------------------
// losses[6] = {policy_gradient, policy_network_regularization (0 here), entropy_regularization,
//              value_estimation, value_network_regularization (0 here), total}
__global__ void __launch_bounds__(512) rf_loss_final_kernel(float* __restrict__ ws, int nblocks,
                                                            float n_total, float ent_coef,
                                                            float value_coef, int has_value,
                                                            float* __restrict__ losses,
                                                            int32_t* flag) {
  pdl_prologue();
  __shared__ float red[32];
  float v[5];
#pragma unroll
  for (int j = 0; j < 5; ++j) {
    const float s = (threadIdx.x < nblocks) ? ws[kWsLoss + threadIdx.x * 5 + j] : 0.f;
    v[j] = block_sum(s, red);
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    float* sc = ws + kWsScalars;
    const float inv_ep = sc[4];
    const float pg = v[0] * inv_ep;
    const float en = ent_coef != 0.f ? ent_coef * (v[1] / n_total) : 0.f;
    const float ve = has_value ? v[2] * value_coef * inv_ep : 0.f;
    losses[0] = pg;
    losses[1] = 0.f;
    losses[2] = en;
    losses[3] = ve;
    losses[4] = 0.f;
    losses[5] = pg + en + ve;
    const float sigma = sc[1], D = sc[2];
    sc[5] = v[3] / n_total;
    sc[6] = sigma > 0.f ? v[4] / (n_total * sigma * D * D) : 0.f;   // sigma = 0: defined as 0
    int32_t bits = 0;
    if (!isfinite(losses[5])) bits |= 1;
    if (sc[3] == 0.f) bits |= 2;
    if (bits) atomicOr(flag, bits);
  }
}

// ---- stage 5 ---------------------------------------------------------------------------------
// dV_j -= d(pg)/d(adv_j) = (g_j - g_bar) / D - (adv_j - mean) * S / (N sigma D^2)
__global__ void rf_dv_kernel(const RfArgs a) {
  pdl_prologue();
  const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= a.N) return;
  const float* sc = a.ws + kWsScalars;
  const float g = a.ws[kWsLast + ((a.B + 3) & ~3LL) + n];
  const float adv_c = rf_adv(a, n) - sc[0];
  a.dv[n] -= (g - sc[5]) / sc[2] - adv_c * sc[6];
}

}  // namespace

}  // namespace b200rl

using namespace b200rl;

static int64_t rf_workspace_bytes(int64_t B, int64_t T) {
  return 4 * (kWsLast + ((B + 3) & ~3LL) + B * T);
}

extern "C" {

int b200rl_reinforce_loss(const float* p0, const float* p1, int64_t ld, const void* action,
                          int64_t A, const float* returns, const float* value,
                          const int32_t* step_type, const int32_t* next_step_type,
                          const float* weights, int64_t B, int64_t T, int use_advantage,
                          int normalize, float entropy_coef, float value_coef, float* losses,
                          float* d0, float* d1, int64_t ld_g, float* dvalue, float* num_episodes,
                          int32_t* flag, void* workspace, int64_t ws_bytes, void* stream) {
  B200RL_CHECK_ARG(p0 && action && returns && step_type && next_step_type && losses && d0 && flag,
                   "reinforce_loss: NULL argument");
  B200RL_CHECK_ARG((p1 == nullptr) == (d1 == nullptr),
                   "reinforce_loss: scale and dscale must be given together (Normal head)");
  B200RL_CHECK_ARG(B >= 1 && T >= 1 && A >= 1 && ld >= A && ld_g >= A,
                   "reinforce_loss: bad sizes");
  B200RL_CHECK_ARG(B * T < (1LL << 24), "reinforce_loss: B*T must stay below 2^24");
  B200RL_CHECK_ARG((value == nullptr) == (dvalue == nullptr),
                   "reinforce_loss: value and dvalue must be given together");
  B200RL_CHECK_ARG(!use_advantage || value, "reinforce_loss: use_advantage needs value predictions");
  B200RL_CHECK_ARG(workspace && ws_bytes >= rf_workspace_bytes(B, T),
                   "reinforce_loss: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t N = B * T;
  RfArgs a{p0, p1, ld, action, returns, value, step_type, next_step_type, weights, B, T, N, A,
           use_advantage ? 1 : 0, normalize ? 1 : 0, entropy_coef, value_coef, d0, d1, ld_g,
           dvalue, flag, (float*)workspace};
  int nb1 = (int)((B + 7) / 8);
  if (nb1 > kRfStatBlocks) nb1 = kRfStatBlocks;
  B200RL_LAUNCH(rf_stats_kernel, nb1, 256, 0, st, a);
  B200RL_CHECK_LAUNCH("reinforce_stats");
  B200RL_LAUNCH(rf_stats_final_kernel, 1, 32, 0, st, (float*)workspace, nb1, num_episodes);
  B200RL_CHECK_LAUNCH("reinforce_stats_final");
  unsigned nb3;
  if (p1 != nullptr) {
    const int64_t want = (N + 255) / 256;
    nb3 = (unsigned)(want > kRfLossBlocks ? kRfLossBlocks : want);
    B200RL_LAUNCH(rf_loss_normal_kernel, nb3, 256, 0, st, a);
  } else {
    const int G = lane_group(A);
    nb3 = group_blocks(N, G, kRfLossBlocks);
    if (G == 1) B200RL_LAUNCH(rf_loss_cat_kernel<1>, nb3, 256, 0, st, a);
    else if (G == 8) B200RL_LAUNCH(rf_loss_cat_kernel<8>, nb3, 256, 0, st, a);
    else B200RL_LAUNCH(rf_loss_cat_kernel<32>, nb3, 256, 0, st, a);
  }
  B200RL_CHECK_LAUNCH("reinforce_loss");
  B200RL_LAUNCH(rf_loss_final_kernel, 1, 512, 0, st, (float*)workspace, (int)nb3, (float)N, entropy_coef, value_coef, value ? 1 : 0, losses, flag);
  B200RL_CHECK_LAUNCH("reinforce_loss_final");
  if (value && use_advantage && normalize) {
    B200RL_LAUNCH(rf_dv_kernel, (unsigned)((N + 255) / 256), 256, 0, st, a);
    B200RL_CHECK_LAUNCH("reinforce_dv");
  }
  return B200RL_OK;
}

}  // extern "C"
