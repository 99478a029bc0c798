// LSTM sequence kernels: the recurrence of a Keras LSTMCell (implementation=2) over a whole
// [B, T] sequence in one launch, forward and backward-through-time.
//
// Restates keras LSTMCell (gates i, f, g, o in column order; sigmoid gates, tanh cell input and
// output; c_t = f c_{t-1} + i g, h_t = o tanh(c_t)) under tf_agents' DynamicUnroll
// (keras_layers/dynamic_unroll_layer.py): a step whose step_type is FIRST starts from the zero
// state.  The input projection x W + b over all B*T rows is one GEMM on the dense routes, so these
// kernels take xw = x W + b and only run the h_{t-1} U term, which is strictly sequential.
//
// Layout.  A cluster of `cs` CTAs (1, 2, 4 or 8) runs one tile of BT batch rows for all T steps.
// CTA r owns hidden units [r*Hc, r*Hc + Hc): the four gate columns of those units, so the cell
// update never leaves the CTA.  Its slice of U stays in shared memory for the whole sequence
// (forward: U[:, gates of own units]; backward: U[own units, :]).  Every step each CTA writes its
// slice of h_t (forward) or dG_t (backward) into the double-buffered shared array of every CTA
// of the cluster (distributed shared memory), then the cluster meets at one barrier.  The
// per-step inputs (xw; the stored gates, c and dh in the backward) are copied into a ring of
// `depth` steps with cp.async, so the step's critical path is the recurrent product, the gate
// math and the barrier.  Thread (rg, jl) owns unit jl for kRows rows of the tile; c and the
// backward's cell-gradient carry stay in its registers.
#include <cooperative_groups.h>

#include "common.cuh"

namespace cg = cooperative_groups;

namespace b200rl {

constexpr int kLstmRows = 4;          // rows of the tile per thread
constexpr int kLstmMaxH = 256;
// Hc * BT / kLstmRows threads: at most 89 units x 4 row groups on one CTA (U slice 128 KB).
constexpr int kLstmMaxThreads = 384;
constexpr int64_t kLstmUBytes = 128 * 1024;     // resident U slice per CTA
constexpr int64_t kLstmSmemMax = 227 * 1024;    // opt-in shared memory per block on sm_90
constexpr int64_t kLstmMaxTiles = 65535;        // gridDim.y limit: tiles of BT rows per launch
constexpr int kStepFirst = 0;

__device__ __forceinline__ void cp_async4(float* dst, const float* src, bool valid) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(d), "l"(src),
               "r"(valid ? 4 : 0)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

__device__ __forceinline__ float sigmoid_f(float z) { return 1.f / (1.f + expf(-z)); }

struct LstmTile {
  int cs, Hc, BT, H, Hp;
};

// Forward ring slot of one step: [BT][4][Hc] floats of xw.
__device__ __forceinline__ void lstm_fwd_prefetch(float* slot, const float* __restrict__ xw,
                                                  int64_t B, int64_t T, int64_t t, int64_t b0,
                                                  int j0, int nj, const LstmTile& g) {
  const int n = g.BT * 4 * g.Hc;
  const int64_t H4 = 4 * (int64_t)g.H;
  for (int e = threadIdx.x; e < n; e += blockDim.x) {
    const int bl = e / (4 * g.Hc), q = (e / g.Hc) & 3, jl = e % g.Hc;
    const int64_t b = b0 + bl;
    const bool valid = t < T && b < B && jl < nj;
    const float* src = valid ? xw + (b * T + t) * H4 + q * g.H + j0 + jl : xw;
    cp_async4(slot + e, src, valid);
  }
  cp_async_commit();
}

template <int D>
__global__ void __launch_bounds__(kLstmMaxThreads) lstm_seq_fwd_kernel(
    const float* __restrict__ xw, const float* __restrict__ U, const int32_t* __restrict__ step_type,
    const float* __restrict__ h0, const float* __restrict__ c0, int64_t B, int64_t T, LstmTile g,
    float* __restrict__ h_out, float* __restrict__ gates, float* __restrict__ c_out,
    float* __restrict__ h_used, float* __restrict__ hT, float* __restrict__ cT) {
  extern __shared__ __align__(16) float smem[];
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int H = g.H, Hp = g.Hp, Hc = g.Hc, BT = g.BT;
  float4* Us = reinterpret_cast<float4*>(smem);             // [Hp][Hc]: gates of unit jl, row k
  float* hs = smem + (size_t)4 * Hp * Hc;                   // [2][BT][Hp]
  float* ring = hs + (size_t)2 * BT * Hp;                   // [D][BT][4][Hc]
  const int j0 = rank * Hc, nj = min(Hc, H - j0);
  const int64_t b0 = (int64_t)blockIdx.y * BT;
  const int jl = threadIdx.x % Hc, rg = threadIdx.x / Hc;
  const bool active = rg < BT / kLstmRows && jl < nj;
  const int j = j0 + jl;
  const int64_t H4 = 4 * (int64_t)H;

  pdl_prologue();
  for (int e = threadIdx.x; e < Hp * Hc; e += blockDim.x) {
    const int k = e / Hc, u = e % Hc;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (k < H && u < nj) {
      const float* row = U + (int64_t)k * H4 + j0 + u;
      v = make_float4(row[0], row[H], row[2 * H], row[3 * H]);
    }
    Us[e] = v;
  }
  for (int e = threadIdx.x; e < 2 * BT * Hp; e += blockDim.x) {
    const int k = e % Hp, bl = (e / Hp) % BT;
    const int64_t b = b0 + bl;
    hs[e] = (e < BT * Hp && h0 && k < H && b < B) ? h0[b * H + k] : 0.f;
  }
  for (int s = 0; s < D; ++s)
    lstm_fwd_prefetch(ring + (size_t)s * BT * 4 * Hc, xw, B, T, s, b0, j0, nj, g);

  float c[kLstmRows], hprev[kLstmRows];
#pragma unroll
  for (int r = 0; r < kLstmRows; ++r) {
    const int64_t b = b0 + rg * kLstmRows + r;
    const bool ok = active && b < B;
    c[r] = (ok && c0) ? c0[b * H + j] : 0.f;
    hprev[r] = (ok && h0) ? h0[b * H + j] : 0.f;
  }
  cp_async_wait<D - 1>();
  cluster.sync();

  for (int64_t t = 0; t < T; ++t) {
    const int cur = (int)(t & 1);
    const float* slot = ring + (size_t)(t % D) * BT * 4 * Hc;
    if (active) {
      float acc[4][kLstmRows];
#pragma unroll
      for (int r = 0; r < kLstmRows; ++r) acc[0][r] = acc[1][r] = acc[2][r] = acc[3][r] = 0.f;
      const float4* hrow = reinterpret_cast<const float4*>(hs + (size_t)(cur * BT + rg * kLstmRows) * Hp);
      const int Hp4 = Hp / 4;
      for (int k4 = 0; k4 < Hp4; ++k4) {
        const float4 u0 = Us[(4 * k4 + 0) * Hc + jl], u1 = Us[(4 * k4 + 1) * Hc + jl];
        const float4 u2 = Us[(4 * k4 + 2) * Hc + jl], u3 = Us[(4 * k4 + 3) * Hc + jl];
#pragma unroll
        for (int r = 0; r < kLstmRows; ++r) {
          const float4 h = hrow[r * Hp4 + k4];
          acc[0][r] += h.x * u0.x + h.y * u1.x + h.z * u2.x + h.w * u3.x;
          acc[1][r] += h.x * u0.y + h.y * u1.y + h.z * u2.y + h.w * u3.y;
          acc[2][r] += h.x * u0.z + h.y * u1.z + h.z * u2.z + h.w * u3.z;
          acc[3][r] += h.x * u0.w + h.y * u1.w + h.z * u2.w + h.w * u3.w;
        }
      }
#pragma unroll
      for (int r = 0; r < kLstmRows; ++r) {
        const int bl = rg * kLstmRows + r;
        const int64_t b = b0 + bl;
        if (b >= B) continue;
        const bool reset = step_type[b * T + t] == kStepFirst;
        const float* x = slot + (size_t)bl * 4 * Hc + jl;
        const float zi = x[0] + (reset ? 0.f : acc[0][r]);
        const float zf = x[Hc] + (reset ? 0.f : acc[1][r]);
        const float zg = x[2 * Hc] + (reset ? 0.f : acc[2][r]);
        const float zo = x[3 * Hc] + (reset ? 0.f : acc[3][r]);
        const float gi = sigmoid_f(zi), gf = sigmoid_f(zf), gg = tanhf(zg), go = sigmoid_f(zo);
        const float cp = reset ? 0.f : c[r];
        const float cn = gf * cp + gi * gg;
        const float hn = go * tanhf(cn);
        const int64_t row = b * T + t;
        h_out[row * H + j] = hn;
        c_out[row * H + j] = cn;
        h_used[row * H + j] = reset ? 0.f : hprev[r];
        float* gr = gates + row * H4 + j;
        gr[0] = gi; gr[H] = gf; gr[2 * H] = gg; gr[3 * H] = go;
        c[r] = cn;
        hprev[r] = hn;
        float* dst = hs + (size_t)((cur ^ 1) * BT + bl) * Hp + j;
        for (int p = 0; p < g.cs; ++p) *cluster.map_shared_rank(dst, p) = hn;
      }
    }
    cp_async_wait<D - 2>();
    cluster.sync();
    lstm_fwd_prefetch(ring + (size_t)(t % D) * BT * 4 * Hc, xw, B, T, t + D, b0, j0, nj, g);
  }
  cp_async_wait<0>();
  if (active) {
#pragma unroll
    for (int r = 0; r < kLstmRows; ++r) {
      const int64_t b = b0 + rg * kLstmRows + r;
      if (b >= B) continue;
      if (hT) hT[b * H + j] = hprev[r];
      if (cT) cT[b * H + j] = c[r];
    }
  }
}

// Backward ring slot of one step: [BT][7][Hc] floats: i, f, g, o, c_t, c_{t-1}, dh_t.
__device__ __forceinline__ void lstm_bwd_prefetch(float* slot, const float* __restrict__ gates,
                                                  const float* __restrict__ c,
                                                  const float* __restrict__ c0,
                                                  const float* __restrict__ dh, int64_t B,
                                                  int64_t T, int64_t t, int64_t b0, int j0, int nj,
                                                  const LstmTile& g) {
  const int n = g.BT * 7 * g.Hc;
  const int64_t H = g.H;
  for (int e = threadIdx.x; e < n; e += blockDim.x) {
    const int bl = e / (7 * g.Hc), f = (e / g.Hc) % 7, jl = e % g.Hc;
    const int64_t b = b0 + bl;
    bool valid = t >= 0 && b < B && jl < nj;
    const float* src = dh;
    if (valid) {
      const int64_t row = b * T + t, j = j0 + jl;
      if (f < 4) {
        src = gates + row * 4 * H + f * H + j;
      } else if (f == 4) {
        src = c + row * H + j;
      } else if (f == 5) {
        valid = t > 0 || c0 != nullptr;
        src = t > 0 ? c + (row - 1) * H + j : (c0 ? c0 + b * H + j : dh);
      } else {
        src = dh + row * H + j;
      }
    }
    cp_async4(slot + e, src, valid);
  }
  cp_async_commit();
}

template <int D>
__global__ void __launch_bounds__(kLstmMaxThreads) lstm_seq_bwd_kernel(
    const float* __restrict__ dh, const float* __restrict__ gates, const float* __restrict__ c,
    const float* __restrict__ c0, const float* __restrict__ U,
    const int32_t* __restrict__ step_type, int64_t B, int64_t T, LstmTile g,
    float* __restrict__ dG) {
  extern __shared__ __align__(16) float smem[];
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int H = g.H, Hc = g.Hc, BT = g.BT;
  float4* Ut = reinterpret_cast<float4*>(smem);            // [H][Hc]: U[unit kl, 4c4 .. 4c4+3]
  float* dgs = smem + (size_t)4 * H * Hc;                   // [2][BT][4H]
  float* ring = dgs + (size_t)2 * BT * 4 * H;               // [D][BT][7][Hc]
  const int j0 = rank * Hc, nj = min(Hc, H - j0);
  const int64_t b0 = (int64_t)blockIdx.y * BT;
  const int jl = threadIdx.x % Hc, rg = threadIdx.x / Hc;
  const bool active = rg < BT / kLstmRows && jl < nj;
  const int j = j0 + jl;
  const int64_t H4 = 4 * (int64_t)H;

  pdl_prologue();
  for (int e = threadIdx.x; e < H * Hc; e += blockDim.x) {
    const int c4 = e / Hc, u = e % Hc;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (u < nj) v = *reinterpret_cast<const float4*>(U + (int64_t)(j0 + u) * H4 + 4 * c4);
    Ut[e] = v;
  }
  for (int e = threadIdx.x; e < 2 * BT * 4 * H; e += blockDim.x) dgs[e] = 0.f;
  for (int s = 0; s < D; ++s)
    lstm_bwd_prefetch(ring + (size_t)s * BT * 7 * Hc, gates, c, c0, dh, B, T, T - 1 - s, b0, j0,
                      nj, g);
  float dc[kLstmRows];
#pragma unroll
  for (int r = 0; r < kLstmRows; ++r) dc[r] = 0.f;
  cp_async_wait<D - 1>();
  cluster.sync();

  for (int64_t s = 0; s < T; ++s) {
    const int64_t t = T - 1 - s;
    const int cur = (int)(s & 1);
    const float* slot = ring + (size_t)(s % D) * BT * 7 * Hc;
    if (active) {
      float acc[kLstmRows];
#pragma unroll
      for (int r = 0; r < kLstmRows; ++r) acc[r] = 0.f;
      const float4* grow = reinterpret_cast<const float4*>(dgs + (size_t)((cur ^ 1) * BT + rg * kLstmRows) * 4 * H);
      for (int c4 = 0; c4 < H; ++c4) {
        const float4 u = Ut[c4 * Hc + jl];
#pragma unroll
        for (int r = 0; r < kLstmRows; ++r) {
          const float4 d = grow[r * H + c4];
          acc[r] += d.x * u.x + d.y * u.y + d.z * u.z + d.w * u.w;
        }
      }
#pragma unroll
      for (int r = 0; r < kLstmRows; ++r) {
        const int bl = rg * kLstmRows + r;
        const int64_t b = b0 + bl;
        if (b >= B) continue;
        // no gradient crosses into step t from t+1 when t+1 starts an episode (or t is last)
        const bool carry = t + 1 < T && step_type[b * T + t + 1] != kStepFirst;
        const bool reset = step_type[b * T + t] == kStepFirst;
        const float* v = slot + (size_t)bl * 7 * Hc + jl;
        const float gi = v[0], gf = v[Hc], gg = v[2 * Hc], go = v[3 * Hc];
        const float ct = v[4 * Hc], cp = reset ? 0.f : v[5 * Hc];
        const float dht = v[6 * Hc] + (carry ? acc[r] : 0.f);
        const float tc = tanhf(ct);
        const float dct = (carry ? dc[r] : 0.f) + dht * go * (1.f - tc * tc);
        const float dzi = dct * gg * gi * (1.f - gi);
        const float dzf = dct * cp * gf * (1.f - gf);
        const float dzg = dct * gi * (1.f - gg * gg);
        const float dzo = dht * tc * go * (1.f - go);
        dc[r] = dct * gf;
        float* out = dG + (b * T + t) * H4 + j;
        out[0] = dzi; out[H] = dzf; out[2 * H] = dzg; out[3 * H] = dzo;
        float* dst = dgs + (size_t)(cur * BT + bl) * 4 * H + j;
        for (int p = 0; p < g.cs; ++p) {
          float* q = cluster.map_shared_rank(dst, p);
          q[0] = dzi; q[H] = dzf; q[2 * H] = dzg; q[3 * H] = dzo;
        }
      }
    }
    cp_async_wait<D - 2>();
    cluster.sync();
    lstm_bwd_prefetch(ring + (size_t)(s % D) * BT * 7 * Hc, gates, c, c0, dh, B, T, t - D, b0, j0,
                      nj, g);
  }
  cp_async_wait<0>();
}

// Shared memory of one CTA (bytes).
static int64_t lstm_fwd_smem(const LstmTile& g, int D) {
  return 4 * ((int64_t)4 * g.Hp * g.Hc + 2LL * g.BT * g.Hp + (int64_t)D * g.BT * 4 * g.Hc);
}
static int64_t lstm_bwd_smem(const LstmTile& g, int D) {
  return 4 * ((int64_t)4 * g.H * g.Hc + 2LL * g.BT * 4 * g.H + (int64_t)D * g.BT * 7 * g.Hc);
}

// Cluster size: the fewest CTAs whose U slices fit kLstmUBytes.  Tile: the most rows (<= 16, no
// more than B needs) and then the deepest ring (4, else 2) that fit the shared memory.
static bool lstm_plan(int64_t B, int H, bool bwd, LstmTile* g, int* depth) {
  g->H = H;
  g->Hp = (H + 3) / 4 * 4;
  g->cs = 8;
  for (int cs = 1; cs <= 8; cs *= 2) {
    if ((int64_t)16 * g->Hp * ((H + cs - 1) / cs) <= kLstmUBytes) { g->cs = cs; break; }
  }
  g->Hc = (H + g->cs - 1) / g->cs;
  const int bt_max = B >= 16 ? 16 : (int)((B + kLstmRows - 1) / kLstmRows * kLstmRows);
  const int bts[3] = {bt_max, 8, 4};
  for (int bt : bts) {
    if (bt > bt_max || g->Hc * (bt / kLstmRows) > kLstmMaxThreads) continue;
    g->BT = bt;
    for (int d = 4; d >= 2; d -= 2) {
      const int64_t sm = bwd ? lstm_bwd_smem(*g, d) : lstm_fwd_smem(*g, d);
      if (sm <= kLstmSmemMax) { *depth = d; return true; }
    }
  }
  return false;
}

template <typename... KArgs, typename... Args>
static cudaError_t lstm_launch(void (*kernel)(KArgs...), const LstmTile& g, int64_t B, size_t smem,
                               cudaStream_t st, Args&&... args) {
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)g.cs, (unsigned)((B + g.BT - 1) / g.BT));
  cfg.blockDim = dim3((unsigned)(g.Hc * (g.BT / kLstmRows)));
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  attr[1].id = cudaLaunchAttributeClusterDimension;
  attr[1].val.clusterDim.x = (unsigned)g.cs;
  attr[1].val.clusterDim.y = 1;
  attr[1].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 2;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<Args&&>(args)...);
}

}  // namespace b200rl

using namespace b200rl;

extern "C" {

int b200rl_lstm_plan(int64_t B, int64_t H, int* cluster, int* rows_fwd, int* rows_bwd,
                     int* depth_fwd, int* depth_bwd, int64_t* smem_fwd, int64_t* smem_bwd) {
  B200RL_CHECK_ARG(B >= 1, "lstm_plan: B must be >= 1");
  B200RL_CHECK_ARG(H >= 1 && H <= kLstmMaxH, "lstm: units must be in [1, %d], got %lld",
                   kLstmMaxH, (long long)H);
  LstmTile gf, gb;
  int df = 0, db = 0;
  B200RL_CHECK_ARG(lstm_plan(B, (int)H, false, &gf, &df) && lstm_plan(B, (int)H, true, &gb, &db),
                   "lstm_plan: no tile fits shared memory");
  const int bt = gf.BT < gb.BT ? gf.BT : gb.BT;
  B200RL_CHECK_ARG((B + bt - 1) / bt <= kLstmMaxTiles,
                   "lstm_plan: B = %lld needs more than %lld tiles of %d rows; B must be <= %lld "
                   "for %lld units", (long long)B, (long long)kLstmMaxTiles, bt,
                   (long long)(kLstmMaxTiles * bt), (long long)H);
  if (cluster) *cluster = gf.cs;
  if (rows_fwd) *rows_fwd = gf.BT;
  if (rows_bwd) *rows_bwd = gb.BT;
  if (depth_fwd) *depth_fwd = df;
  if (depth_bwd) *depth_bwd = db;
  if (smem_fwd) *smem_fwd = lstm_fwd_smem(gf, df);
  if (smem_bwd) *smem_bwd = lstm_bwd_smem(gb, db);
  return B200RL_OK;
}

int b200rl_lstm_seq_fwd(const float* xw, const float* U, const int32_t* step_type,
                        const float* h0, const float* c0, int64_t B, int64_t T, int64_t H,
                        float* h, float* gates, float* c, float* h_used, float* hT, float* cT,
                        void* stream) {
  B200RL_CHECK_ARG(xw && U && step_type && h && gates && c && h_used && B >= 1 && T >= 1,
                   "lstm_seq_fwd: bad argument");
  B200RL_CHECK_ARG(H >= 1 && H <= kLstmMaxH, "lstm: units must be in [1, %d], got %lld",
                   kLstmMaxH, (long long)H);
  LstmTile g;
  int d = 0;
  B200RL_CHECK_ARG(lstm_plan(B, (int)H, false, &g, &d), "lstm_seq_fwd: no tile fits");
  B200RL_CHECK_ARG((B + g.BT - 1) / g.BT <= kLstmMaxTiles,
                   "lstm_seq_fwd: B = %lld needs more than %lld tiles of %d rows; B must be <= %lld "
                   "for %lld units", (long long)B, (long long)kLstmMaxTiles, g.BT,
                   (long long)(kLstmMaxTiles * g.BT), (long long)H);
  const size_t smem = (size_t)lstm_fwd_smem(g, d);
  const cudaStream_t st = (cudaStream_t)stream;
  if (d == 4)
    (void)lstm_launch(lstm_seq_fwd_kernel<4>, g, B, smem, st, xw, U, step_type, h0, c0, B, T, g, h, gates, c, h_used, hT, cT);
  else
    (void)lstm_launch(lstm_seq_fwd_kernel<2>, g, B, smem, st, xw, U, step_type, h0, c0, B, T, g, h, gates, c, h_used, hT, cT);
  B200RL_CHECK_LAUNCH("lstm_seq_fwd");
  return B200RL_OK;
}

int b200rl_lstm_seq_bwd(const float* dh, const float* gates, const float* c, const float* c0,
                        const float* U, const int32_t* step_type, int64_t B, int64_t T,
                        int64_t H, float* dG, void* stream) {
  B200RL_CHECK_ARG(dh && gates && c && U && step_type && dG && B >= 1 && T >= 1,
                   "lstm_seq_bwd: bad argument");
  B200RL_CHECK_ARG(H >= 1 && H <= kLstmMaxH, "lstm: units must be in [1, %d], got %lld",
                   kLstmMaxH, (long long)H);
  B200RL_CHECK_ARG(((uintptr_t)U & 15) == 0, "lstm_seq_bwd: U must be 16-byte aligned");
  LstmTile g;
  int d = 0;
  B200RL_CHECK_ARG(lstm_plan(B, (int)H, true, &g, &d), "lstm_seq_bwd: no tile fits");
  B200RL_CHECK_ARG((B + g.BT - 1) / g.BT <= kLstmMaxTiles,
                   "lstm_seq_bwd: B = %lld needs more than %lld tiles of %d rows; B must be <= %lld "
                   "for %lld units", (long long)B, (long long)kLstmMaxTiles, g.BT,
                   (long long)(kLstmMaxTiles * g.BT), (long long)H);
  const size_t smem = (size_t)lstm_bwd_smem(g, d);
  const cudaStream_t st = (cudaStream_t)stream;
  if (d == 4)
    (void)lstm_launch(lstm_seq_bwd_kernel<4>, g, B, smem, st, dh, gates, c, c0, U, step_type, B, T, g, dG);
  else
    (void)lstm_launch(lstm_seq_bwd_kernel<2>, g, B, smem, st, dh, gates, c, c0, U, step_type, B, T, g, dG);
  B200RL_CHECK_LAUNCH("lstm_seq_bwd");
  return B200RL_OK;
}

}  // extern "C"
