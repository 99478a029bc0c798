// Dense / Conv2D forward + backward in true fp32 (kernel family iii, network part).
//
// The reference runs these through Keras -> TensorFlow CPU kernels (Eigen fp32):
//   networks/encoding_network.py:224-312 (conv + dense stack), q_network.py:126-135 (Q head),
//   examples/dqn/mnih15/dqn_train_eval_atari.py:104-110 (the Atari net incl. cast+/255).
// North-star parity is 1e-5 relative on the loss, which BF16/TF32 MMA cannot hold over a
// 3136-wide reduction (SURVEY.md §7 "hard parts"), so this file is a register-tiled fp32 FFMA
// GEMM with pluggable operand views:
//   ARow  A(m,k)=X[m*ld+k]              dense forward, dX = dZ @ W^T
//   ACol  A(m,k)=X[k*ld+m]              dW = X^T @ dZ
//   AConv A(m,k)=im2col(X)(m,k)         implicit-GEMM conv forward (u8 or f32 input, fused
//                                       cast * scale of the reference's preprocessing layer)
//   AConvT A(m,k)=im2col(X)(k,m)        conv filter gradient
//   BRow  B(k,n)=W[k*ld+n]   BCol  B(k,n)=W[n*ld+k]
// Small output grids (fc layers, filter gradients) use deterministic split-K: partial tiles
// go to the caller's workspace and a second kernel reduces them in fixed order and applies
// bias + activation, so results are run-to-run bit-stable.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

namespace b200rl {

struct FastDiv {
  uint32_t d, mul, shr;
  __host__ FastDiv() : d(1), mul(0), shr(0) {}
  __host__ explicit FastDiv(uint32_t div) : d(div) {
    // round-up magic number method, valid for n < 2^31
    if (div == 1) { mul = 0; shr = 0; return; }
    uint32_t l = 0;
    while ((1u << l) < div) ++l;
    uint64_t m = ((1ull << 32) * ((1ull << l) - div)) / div + 1;
    mul = (uint32_t)m;
    shr = l;
  }
  __device__ __forceinline__ uint32_t div(uint32_t n) const {
    if (d == 1) return n;
    uint32_t t = __umulhi(mul, n);
    return (t + ((n - t) >> 1)) >> (shr - 1);
  }
  __device__ __forceinline__ void divmod(uint32_t n, uint32_t& q, uint32_t& r) const {
    q = div(n);
    r = n - q * d;
  }
};

// Operand views.  Every view is separable: element (row, k) lives at row_off(row) + k_off(k),
// where "row" is m for A views and n for B views.  kKContig says which index is contiguous in
// memory (4 consecutive elements along it can then be copied as one 16-byte / 4-byte chunk when
// vec4_ok()).  `at` is the scalar accessor used by the fp32 FFMA kernel; the tensor-core kernel
// copies raw Elem values from addr() and converts them to fp32 with cvt().
struct ARow {
  using Elem = float;
  const float* p;
  int64_t ld;
  static constexpr bool kKContig = true;
  static constexpr bool kExact = false;
  __device__ __forceinline__ float at(int64_t m, int64_t k) const { return p[m * ld + k]; }
  __device__ __forceinline__ int64_t row_off(int64_t m) const { return m * ld; }
  __device__ __forceinline__ int64_t k_off(int64_t k) const { return k; }
  __device__ __forceinline__ bool vec4_ok() const { return (ld & 3) == 0 && ((uintptr_t)p & 15) == 0; }
  __device__ __forceinline__ float cvt(Elem x) const { return x; }
  __device__ __forceinline__ const void* addr(int64_t off) const { return p + off; }
};
struct ACol {
  using Elem = float;
  const float* p;
  int64_t ld;
  static constexpr bool kKContig = false;
  static constexpr bool kExact = false;
  __device__ __forceinline__ float at(int64_t m, int64_t k) const { return p[k * ld + m]; }
  __device__ __forceinline__ int64_t row_off(int64_t m) const { return m; }
  __device__ __forceinline__ int64_t k_off(int64_t k) const { return k * ld; }
  __device__ __forceinline__ bool vec4_ok() const { return (ld & 3) == 0 && ((uintptr_t)p & 15) == 0; }
  __device__ __forceinline__ float cvt(Elem x) const { return x; }
  __device__ __forceinline__ const void* addr(int64_t off) const { return p + off; }
};
struct BRow {  // B(k, n) = p[k*ld + n]  (n contiguous)
  using Elem = float;
  const float* p;
  int64_t ld;
  static constexpr bool kNContig = true;
  static constexpr bool kKContig = false;
  static constexpr bool kExact = false;
  __device__ __forceinline__ float at(int64_t k, int64_t n) const { return p[k * ld + n]; }
  __device__ __forceinline__ int64_t row_off(int64_t n) const { return n; }
  __device__ __forceinline__ int64_t k_off(int64_t k) const { return k * ld; }
  __device__ __forceinline__ bool vec4_ok() const { return (ld & 3) == 0 && ((uintptr_t)p & 15) == 0; }
  __device__ __forceinline__ float cvt(Elem x) const { return x; }
  __device__ __forceinline__ const void* addr(int64_t off) const { return p + off; }
};
struct BCol {  // B(k, n) = p[n*ld + k]  (k contiguous)
  using Elem = float;
  const float* p;
  int64_t ld;
  static constexpr bool kNContig = false;
  static constexpr bool kKContig = true;
  static constexpr bool kExact = false;
  __device__ __forceinline__ float at(int64_t k, int64_t n) const { return p[n * ld + k]; }
  __device__ __forceinline__ int64_t row_off(int64_t n) const { return n * ld; }
  __device__ __forceinline__ int64_t k_off(int64_t k) const { return k; }
  __device__ __forceinline__ bool vec4_ok() const { return (ld & 3) == 0 && ((uintptr_t)p & 15) == 0; }
  __device__ __forceinline__ float cvt(Elem x) const { return x; }
  __device__ __forceinline__ const void* addr(int64_t off) const { return p + off; }
};

struct ConvGeom {
  int H, W, C, KH, KW, F, stride, OH, OW;
  FastDiv d_ohow, d_ow, d_kwc;
  int64_t in_row;   // W*C
  int64_t in_img;   // elements between consecutive images
};

template <typename T>
__device__ __forceinline__ float cvt_in(T v, float scale);
template <>
__device__ __forceinline__ float cvt_in<float>(float v, float) { return v; }
template <>
__device__ __forceinline__ float cvt_in<uint8_t>(uint8_t v, float scale) {
  // tf.cast(obs, f32) / 255 is restated as a division to stay bit-identical to the oracle.
  return __fdiv_rn((float)v, scale);
}

// im2col view: pos = (n, oy, ox), patch = (ky, kx, c) with c fastest (Keras HWIO order).
template <typename T>
struct ConvView {
  const T* x;
  ConvGeom g;
  float scale;
  __device__ __forceinline__ int64_t pos_offset(uint32_t pos) const {
    uint32_t n, r, oy, ox;
    g.d_ohow.divmod(pos, n, r);
    g.d_ow.divmod(r, oy, ox);
    return (int64_t)n * g.in_img + (int64_t)(oy * g.stride) * g.in_row +
           (int64_t)(ox * g.stride) * g.C;
  }
  __device__ __forceinline__ int64_t patch_offset(uint32_t kidx) const {
    uint32_t ky, r;
    g.d_kwc.divmod(kidx, ky, r);
    return (int64_t)ky * g.in_row + r;
  }
  __device__ __forceinline__ float load(int64_t off) const { return cvt_in<T>(x[off], scale); }
  __device__ __forceinline__ bool vec4_ok() const {
    return (g.C & 3) == 0 && (g.in_img & 3) == 0 && ((uintptr_t)x & (4 * sizeof(T) - 1)) == 0;
  }
  // tensor-core path: x * (1/scale) instead of the IEEE division (differs by <= 1 ulp; the
  // parity bar is 1e-5, and the division costs ~25 instructions per element in the split)
  __device__ __forceinline__ float cvt_fast(T v) const;
};
template <>
__device__ __forceinline__ float ConvView<float>::cvt_fast(float v) const { return v; }
template <>
__device__ __forceinline__ float ConvView<uint8_t>::cvt_fast(uint8_t v) const {
  return (float)v * __frcp_rn(scale);
}
template <typename T>
struct AConv {
  using Elem = T;
  ConvView<T> v;
  static constexpr bool kKContig = true;
  static constexpr bool kExact = false;
  __device__ __forceinline__ float at(int64_t m, int64_t k) const {
    return v.load(v.pos_offset((uint32_t)m) + v.patch_offset((uint32_t)k));
  }
  __device__ __forceinline__ int64_t row_off(int64_t m) const { return v.pos_offset((uint32_t)m); }
  __device__ __forceinline__ int64_t k_off(int64_t k) const { return v.patch_offset((uint32_t)k); }
  __device__ __forceinline__ bool vec4_ok() const { return v.vec4_ok(); }
  __device__ __forceinline__ float cvt(Elem x) const { return v.cvt_fast(x); }
  __device__ __forceinline__ const void* addr(int64_t off) const { return v.x + off; }
};
template <typename T>
struct AConvT {
  using Elem = T;
  ConvView<T> v;
  static constexpr bool kKContig = false;
  static constexpr bool kExact = false;
  __device__ __forceinline__ float at(int64_t m, int64_t k) const {
    return v.load(v.pos_offset((uint32_t)k) + v.patch_offset((uint32_t)m));
  }
  __device__ __forceinline__ int64_t row_off(int64_t m) const { return v.patch_offset((uint32_t)m); }
  __device__ __forceinline__ int64_t k_off(int64_t k) const { return v.pos_offset((uint32_t)k); }
  __device__ __forceinline__ bool vec4_ok() const { return v.vec4_ok(); }
  __device__ __forceinline__ float cvt(Elem x) const { return v.cvt_fast(x); }
  __device__ __forceinline__ const void* addr(int64_t off) const { return v.x + off; }
};

// Raw uint8 pixel views for the tensor-core path: values 0..255 are exact in TF32, the 1/scale of
// the reference's cast+/255 layer is applied to the accumulator in the epilogue instead.
struct AConvU8Raw {
  using Elem = uint8_t;
  ConvView<uint8_t> v;
  static constexpr bool kKContig = true;
  static constexpr bool kExact = true;
  __device__ __forceinline__ float at(int64_t m, int64_t k) const { return 0.f; }
  __device__ __forceinline__ int64_t row_off(int64_t m) const { return v.pos_offset((uint32_t)m); }
  __device__ __forceinline__ int64_t k_off(int64_t k) const { return v.patch_offset((uint32_t)k); }
  __device__ __forceinline__ bool vec4_ok() const { return v.vec4_ok(); }
  __device__ __forceinline__ float cvt(Elem x) const { return (float)x; }
  __device__ __forceinline__ const void* addr(int64_t off) const { return v.x + off; }
};
struct AConvTU8Raw {
  using Elem = uint8_t;
  ConvView<uint8_t> v;
  static constexpr bool kKContig = false;
  static constexpr bool kExact = true;
  __device__ __forceinline__ float at(int64_t m, int64_t k) const { return 0.f; }
  __device__ __forceinline__ int64_t row_off(int64_t m) const { return v.patch_offset((uint32_t)m); }
  __device__ __forceinline__ int64_t k_off(int64_t k) const { return v.pos_offset((uint32_t)k); }
  __device__ __forceinline__ bool vec4_ok() const { return v.vec4_ok(); }
  __device__ __forceinline__ float cvt(Elem x) const { return (float)x; }
  __device__ __forceinline__ const void* addr(int64_t off) const { return v.x + off; }
};

__device__ __forceinline__ float apply_act(float v, int act) {
  if (act == B200RL_ACT_RELU) return fmaxf(v, 0.f);
  if (act == B200RL_ACT_TANH) return tanhf(v);
  return v;
}

// Input-gradient mask: when the GEMM input X is the OUTPUT of an activation (the previous layer
// of the stack), dLoss/dX is multiplied by act'(X) on its way out, so the caller receives the
// gradient w.r.t. that layer's pre-activation and the separate act_bwd pass disappears.
struct ActMask {
  const float* y = nullptr;   // X as produced by the previous layer (nullptr: no mask)
  int64_t ld = 0;             // dense: row stride of y; conv: elements between images
  int act = 0;
};
__device__ __forceinline__ float dact(float y, float g, int act) {
  if (act == B200RL_ACT_RELU) return y > 0.f ? g : 0.f;
  if (act == B200RL_ACT_TANH) return g * (1.f - y * y);
  return g;
}

}  // namespace b200rl
#include "tc_gemm.cuh"
namespace b200rl {

constexpr int BK = 16;

// C[M,N] (+)= act(A @ B + bias)   or   ws[split] = partial(A @ B) when splits > 1.
template <int BM, int BN, int TM, int TN, class AL, class BL>
__global__ void __launch_bounds__(256) sgemm_kernel(const AL a, const BL b, float* __restrict__ C,
                                                    const float* __restrict__ bias, int64_t M,
                                                    int64_t N, int64_t K, int act, int beta,
                                                    int splits, int64_t k_per_split,
                                                    float* __restrict__ ws, const ActMask mask) {
  pdl_prologue();
  static_assert((BM / TM) * (BN / TN) == 256, "thread grid must be 256");
  constexpr int TX = BN / TN;
  constexpr int GM = TM >= 4 ? 4 : TM, GN = TN >= 4 ? 4 : TN;  // contiguous group widths
  constexpr int NGM = TM / GM, NGN = TN / GN;
  constexpr int APT = BM * BK / 256, BPT = BN * BK / 256;  // elements per thread per tile
  __shared__ __align__(16) float As[2][BK][BM + 4];
  __shared__ __align__(16) float Bs[2][BK][BN + 4];

  const int tid = threadIdx.x;
  const int tx = tid % TX, ty = tid / TX;
  const int64_t m0 = (int64_t)blockIdx.y * BM, n0 = (int64_t)blockIdx.x * BN;
  const int split = blockIdx.z;
  const int64_t kb = (int64_t)split * k_per_split;
  const int64_t ke = (kb + k_per_split < K) ? kb + k_per_split : K;

  // tile-load coordinates
  int a_m[APT], a_k[APT], b_n[BPT], b_k[BPT];
#pragma unroll
  for (int i = 0; i < APT; ++i) {
    if (AL::kKContig) { a_k[i] = tid % BK; a_m[i] = tid / BK + i * (256 / BK); }
    else { a_m[i] = tid % BM; a_k[i] = tid / BM + i * (256 / BM); }
  }
#pragma unroll
  for (int i = 0; i < BPT; ++i) {
    if (BL::kNContig) { b_n[i] = tid % BN; b_k[i] = tid / BN + i * (256 / BN); }
    else { b_k[i] = tid % BK; b_n[i] = tid / BK + i * (256 / BK); }
  }

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  float ra[APT], rb[BPT];
  auto load_tile = [&](int64_t k0) {
#pragma unroll
    for (int i = 0; i < APT; ++i) {
      const int64_t m = m0 + a_m[i], k = k0 + a_k[i];
      ra[i] = (m < M && k < ke) ? a.at(m, k) : 0.f;
    }
#pragma unroll
    for (int i = 0; i < BPT; ++i) {
      const int64_t n = n0 + b_n[i], k = k0 + b_k[i];
      rb[i] = (n < N && k < ke) ? b.at(k, n) : 0.f;
    }
  };
  auto store_tile = [&](int buf) {
#pragma unroll
    for (int i = 0; i < APT; ++i) As[buf][a_k[i]][a_m[i]] = ra[i];
#pragma unroll
    for (int i = 0; i < BPT; ++i) Bs[buf][b_k[i]][b_n[i]] = rb[i];
  };

  int buf = 0;
  if (kb < ke) {
    load_tile(kb);
    store_tile(0);
  }
  __syncthreads();
  for (int64_t k0 = kb; k0 < ke; k0 += BK) {
    const bool has_next = k0 + BK < ke;
    if (has_next) load_tile(k0 + BK);
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float fa[TM], fb[TN];
#pragma unroll
      for (int g = 0; g < NGM; ++g)
#pragma unroll
        for (int i = 0; i < GM; ++i) fa[g * GM + i] = As[buf][kk][g * (BM / NGM) + ty * GM + i];
#pragma unroll
      for (int g = 0; g < NGN; ++g)
#pragma unroll
        for (int j = 0; j < GN; ++j) fb[g * GN + j] = Bs[buf][kk][g * (BN / NGN) + tx * GN + j];
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(fa[i], fb[j], acc[i][j]);
    }
    if (has_next) {
      store_tile(buf ^ 1);
      __syncthreads();
      buf ^= 1;
    }
  }

  float* out = (splits > 1) ? ws + (int64_t)split * M * N : C;
#pragma unroll
  for (int gi = 0; gi < NGM; ++gi)
#pragma unroll
    for (int i = 0; i < GM; ++i) {
      const int64_t m = m0 + gi * (BM / NGM) + ty * GM + i;
      if (m >= M) continue;
#pragma unroll
      for (int gj = 0; gj < NGN; ++gj)
#pragma unroll
        for (int j = 0; j < GN; ++j) {
          const int64_t n = n0 + gj * (BN / NGN) + tx * GN + j;
          if (n >= N) continue;
          float v = acc[gi * GM + i][gj * GN + j];
          if (splits == 1) {
            if (bias) v += bias[n];
            v = apply_act(v, act);
            if (mask.y) v = dact(mask.y[m * mask.ld + n], v, mask.act);
            if (beta) v += out[m * N + n];
          }
          out[m * N + n] = v;
        }
    }
}

__global__ void splitk_reduce_kernel(const float* __restrict__ ws, float* __restrict__ C,
                                     const float* __restrict__ bias, int64_t MN, int64_t N,
                                     int splits, int act, int beta, const ActMask mask) {
  pdl_prologue();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= MN) return;
  float v = 0.f;
  for (int s = 0; s < splits; ++s) v += ws[(int64_t)s * MN + i];
  if (bias) v += bias[i % N];
  v = apply_act(v, act);
  if (mask.y) v = dact(mask.y[(i / N) * mask.ld + i % N], v, mask.act);
  if (beta) v += C[i];
  C[i] = v;
}

// dZ = dY * act'(Y); 16-byte accesses when n and the pointers allow (HBM-bound: 12 B / element)
__global__ void act_bwd_kernel(const float* __restrict__ Y, const float* __restrict__ dY,
                               float* __restrict__ dZ, int64_t n, int act, int vec) {
  pdl_prologue();
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (vec) {
    const int64_t n4 = n >> 2;
    for (int64_t i = tid; i < n4; i += stride) {
      const float4 y = reinterpret_cast<const float4*>(Y)[i];
      const float4 g = reinterpret_cast<const float4*>(dY)[i];
      reinterpret_cast<float4*>(dZ)[i] = make_float4(dact(y.x, g.x, act), dact(y.y, g.y, act),
                                                     dact(y.z, g.z, act), dact(y.w, g.w, act));
    }
    return;
  }
  for (int64_t i = tid; i < n; i += stride) dZ[i] = dact(Y[i], dY[i], act);
}

// Column sums of dZ[M,N] in two deterministic stages.
constexpr int kColRows = 512;  // rows per partial block
// Block = 32 columns x 8 row-lanes: a warp reads 128 contiguous bytes of one row, the 8 warps
// walk kColRows rows in an interleaved fashion and are combined through shared memory in a
// fixed order (deterministic).
__global__ void __launch_bounds__(256) colsum_partial_kernel(const float* __restrict__ dZ,
                                                             float* __restrict__ part, int64_t M,
                                                             int64_t N) {
  pdl_prologue();
  __shared__ float red[8][33];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t n = (int64_t)blockIdx.x * 32 + lane;
  const int64_t mb = (int64_t)blockIdx.y * kColRows;
  const int64_t me = mb + kColRows < M ? mb + kColRows : M;
  float s = 0.f;
  if (n < N) {
#pragma unroll 4
    for (int64_t m = mb + w; m < me; m += 8) s += dZ[m * N + n];
  }
  red[w][lane] = s;
  __syncthreads();
  if (w == 0 && n < N) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += red[i][lane];
    part[(int64_t)blockIdx.y * N + n] = t;
  }
}
__global__ void __launch_bounds__(256) colsum_final_kernel(const float* __restrict__ part,
                                                           float* __restrict__ db, int64_t nparts,
                                                           int64_t N, int beta) {
  pdl_prologue();
  // one warp per column: lanes stride over the partials, fixed-order shuffle reduction
  const int lane = threadIdx.x & 31;
  const int64_t n = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (n >= N) return;
  float s = 0.f;
  for (int64_t p = lane; p < nparts; p += 32) s += part[p * N + n];
  s = warp_sum(s);
  if (lane == 0) db[n] = beta ? db[n] + s : s;
}


// ---------------------------------------------------------------------------------------
// Skinny heads: Dense layers with N <= 16 outputs (Q head, value head, action means).
// A tensor-core tile would be >= 87 % padding and the FFMA tiles need a split-K + reduce pair
// for 256 rows; these three kernels are plain bandwidth-bound sweeps with W staged in shared
// memory.  Used when the GEMM mode is not 0 (their weight gradient accumulates with atomics).
// ---------------------------------------------------------------------------------------
constexpr int kSkinnyMaxN = 16;
constexpr int kSkinnySmem = 48 * 1024;

// Y[m, :] = act(X[m, :] @ W + b): one warp per row, lanes stride over k, N shuffle reductions.
template <int NMAX>
__global__ void __launch_bounds__(256) skinny_fwd_kernel(const float* __restrict__ X, int64_t ldx,
                                                         const float* __restrict__ W,
                                                         const float* __restrict__ bias,
                                                         float* __restrict__ Y, int64_t M, int K,
                                                         int N, int act) {
  pdl_prologue();
  extern __shared__ float sw[];                       // [K, N]
  for (int i = threadIdx.x; i < K * N; i += blockDim.x) sw[i] = W[i];
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int64_t m = (int64_t)blockIdx.x * nw + warp; m < M; m += (int64_t)gridDim.x * nw) {
    float acc[NMAX];
#pragma unroll
    for (int n = 0; n < NMAX; ++n) acc[n] = 0.f;
    const float* x = X + m * ldx;
#pragma unroll 4
    for (int k = lane; k < K; k += 32) {
      const float xv = x[k];
      const float* w = sw + k * N;
#pragma unroll
      for (int n = 0; n < NMAX; ++n)
        if (n < N) acc[n] = fmaf(xv, w[n], acc[n]);
    }
#pragma unroll
    for (int n = 0; n < NMAX; ++n)
      if (n < N) acc[n] = warp_sum(acc[n]);
    if (lane == 0) {
#pragma unroll
      for (int n = 0; n < NMAX; ++n)
        if (n < N) Y[m * N + n] = apply_act(acc[n] + (bias ? bias[n] : 0.f), act);
    }
  }
}

// dX[m, k] = sum_n dY[m, n] W[k, n]  (* act'(X[m, k]) of the producing layer): 4 k per thread.
template <int NMAX>
__global__ void __launch_bounds__(256) skinny_dx_kernel(const float* __restrict__ dY,
                                                        const float* __restrict__ W,
                                                        float* __restrict__ dX, int64_t M, int K,
                                                        int N, const ActMask mask) {
  pdl_prologue();
  extern __shared__ float sw[];                       // [K, N]
  for (int i = threadIdx.x; i < K * N; i += blockDim.x) sw[i] = W[i];
  __syncthreads();
  const int kq = (K + 3) >> 2;                        // k quads per row
  const int64_t total = M * kq;
  const bool vec = (K & 3) == 0 && ((uintptr_t)dX & 15) == 0;   // dX is a caller pointer
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t m = i / kq;
    const int k0 = (int)(i - m * kq) * 4;
    float dy[NMAX];
#pragma unroll
    for (int n = 0; n < NMAX; ++n) dy[n] = n < N ? dY[m * N + n] : 0.f;
    float o[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      if (k0 + q < K) {
        const float* w = sw + (k0 + q) * N;
#pragma unroll
        for (int n = 0; n < NMAX; ++n)
          if (n < N) o[q] = fmaf(dy[n], w[n], o[q]);
        if (mask.y) o[q] = dact(mask.y[m * mask.ld + k0 + q], o[q], mask.act);
      }
    }
    float* dst = dX + m * K + k0;
    if (vec) *reinterpret_cast<float4*>(dst) = make_float4(o[0], o[1], o[2], o[3]);
    else
      for (int q = 0; q < 4; ++q)
        if (k0 + q < K) dst[q] = o[q];
  }
}

// dW[k, n] += sum_m X[m, k] dY[m, n], db[n] += sum_m dY[m, n] over the CTA's slab of rows; thread
// t owns input features k = t, t + blockDim, ...; the slab's dY rows are staged in shared memory.
template <int NMAX, int KPT>
__global__ void __launch_bounds__(256) skinny_dw_kernel(const float* __restrict__ X, int64_t ldx,
                                                        const float* __restrict__ dY,
                                                        float* __restrict__ dW,
                                                        float* __restrict__ db, int64_t M, int K,
                                                        int N, int64_t rows_per_cta) {
  pdl_prologue();
  constexpr int kChunk = 64;                          // rows of dY staged per step
  __shared__ float sdy[kChunk * NMAX];
  const int64_t mb = (int64_t)blockIdx.x * rows_per_cta;
  const int64_t me = (mb + rows_per_cta < M) ? mb + rows_per_cta : M;
  float acc[KPT][NMAX];
#pragma unroll
  for (int j = 0; j < KPT; ++j)
#pragma unroll
    for (int n = 0; n < NMAX; ++n) acc[j][n] = 0.f;
  float bsum = 0.f;
  // K < blockDim: the threads form G = blockDim / K' row groups (K' = K rounded up to a warp), group
  // g takes rows g, g + G, ... of every staged chunk (run 12: 100 of 256 threads worked on the PPO
  // heads); the groups meet in the atomics below.
  const int kpad = (K + 31) & ~31;
  const int G = (KPT == 1 && kpad < (int)blockDim.x) ? (int)blockDim.x / kpad : 1;
  const int rg = G > 1 ? (int)threadIdx.x / kpad : 0;
  const int kt = G > 1 ? (int)threadIdx.x - rg * kpad : (int)threadIdx.x;
  const bool live = rg < G;
  for (int64_t m0 = mb; m0 < me; m0 += kChunk) {
    const int rows = (int)((me - m0 < kChunk) ? me - m0 : kChunk);
    __syncthreads();
    for (int i = threadIdx.x; i < rows * N; i += blockDim.x) sdy[(i / N) * NMAX + i % N] = dY[m0 * N + i];
    __syncthreads();
    if ((int)threadIdx.x < N)
      for (int r = 0; r < rows; ++r) bsum += sdy[r * NMAX + threadIdx.x];
#pragma unroll
    for (int j = 0; j < KPT; ++j) {
      const int k = kt + j * blockDim.x;
      if (k < K && live) {
        const float* xp = X + m0 * ldx + k;
        int r = rg;
        for (; r + 3 * G < rows; r += 4 * G) {        // 4 independent loads in flight per thread
          float xv[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) xv[u] = xp[(int64_t)(r + u * G) * ldx];
#pragma unroll
          for (int u = 0; u < 4; ++u)
#pragma unroll
            for (int n = 0; n < NMAX; ++n)
              if (n < N) acc[j][n] = fmaf(xv[u], sdy[(r + u * G) * NMAX + n], acc[j][n]);
        }
        for (; r < rows; r += G) {
          const float xv = xp[(int64_t)r * ldx];
#pragma unroll
          for (int n = 0; n < NMAX; ++n)
            if (n < N) acc[j][n] = fmaf(xv, sdy[r * NMAX + n], acc[j][n]);
        }
      }
    }
  }
  if (G > 1) {
    // the row groups add their sums in a fixed order (a single-CTA launch stays bit-reproducible)
    extern __shared__ float skinny_red[];             // [K, N]
    for (int i = threadIdx.x; i < K * N; i += blockDim.x) skinny_red[i] = 0.f;
    for (int g = 0; g < G; ++g) {
      __syncthreads();
      if (live && rg == g && kt < K) {
#pragma unroll
        for (int n = 0; n < NMAX; ++n)
          if (n < N) skinny_red[kt * N + n] += acc[0][n];
      }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < K * N; i += blockDim.x) atomicAdd(dW + i, skinny_red[i]);
  } else {
#pragma unroll
    for (int j = 0; j < KPT; ++j) {
      const int k = kt + j * blockDim.x;
      if (k < K && live) {
#pragma unroll
        for (int n = 0; n < NMAX; ++n)
          if (n < N) atomicAdd(dW + (int64_t)k * N + n, acc[j][n]);
      }
    }
  }
  if (db != nullptr && (int)threadIdx.x < N) atomicAdd(db + threadIdx.x, bsum);
}

// ---- thin-input layers (K <= 32: observation -> first hidden layer) ----------------------------
// Run 12 (PPO, 524 288 rows): x[M,17] @ W[17,200] fell through to the first-generation tensor-core
// kernel (K % 4 != 0) at ~900 us and its weight gradient to the FFMA GEMM at ~600 us, against an
// HBM floor of 65 us (the [M,200] activation is written / read once).  Both are one outer product
// per row: thread (cq, rg) owns output columns 4cq..4cq+3 for rows rg*8..rg*8+7 of every 32-row
// chunk; the chunk of X sits in shared memory (broadcast reads), W / dW columns in registers or
// shared memory, the wide operand moves as coalesced float4.
constexpr int kThinMaxK = 32, kThinMaxN = 256, kThinRows = 32;

__global__ void __launch_bounds__(256) thin_fwd_kernel(const float* __restrict__ X, int64_t ldx,
                                                       const float* __restrict__ W,
                                                       const float* __restrict__ bias,
                                                       float* __restrict__ Y, int64_t M, int K,
                                                       int N, int act, int64_t chunks) {
  pdl_prologue();
  extern __shared__ float4 thin_smem[];
  const int KP = (K + 3) & ~3, nq = N >> 2;
  float4* sw = thin_smem;                              // [KP][nq] (rows >= K are zero)
  float* sx = reinterpret_cast<float*>(thin_smem + KP * nq);   // [kThinRows][KP]
  for (int i = threadIdx.x; i < KP * nq; i += blockDim.x)
    sw[i] = (i / nq) < K ? reinterpret_cast<const float4*>(W)[i] : make_float4(0.f, 0.f, 0.f, 0.f);
  const int cq = threadIdx.x & 63, rg = threadIdx.x >> 6;
  const bool active = cq < nq;
  float4 b4 = make_float4(0.f, 0.f, 0.f, 0.f);
  if (bias && active) b4 = reinterpret_cast<const float4*>(bias)[cq];
  for (int64_t chunk = blockIdx.x; chunk < chunks; chunk += gridDim.x) {
    const int64_t m0 = chunk * kThinRows;
    __syncthreads();
    for (int i = threadIdx.x; i < kThinRows * KP; i += blockDim.x) {
      const int r = i / KP, k = i - r * KP;
      sx[i] = (m0 + r < M && k < K) ? X[(m0 + r) * ldx + k] : 0.f;
    }
    __syncthreads();
    if (!active) continue;
    float4 acc[8];
#pragma unroll
    for (int r = 0; r < 8; ++r) acc[r] = b4;
    for (int k = 0; k < KP; k += 4) {
      const float4 w0 = sw[(k + 0) * nq + cq], w1 = sw[(k + 1) * nq + cq];
      const float4 w2 = sw[(k + 2) * nq + cq], w3 = sw[(k + 3) * nq + cq];
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const float4 x = *reinterpret_cast<const float4*>(sx + (rg * 8 + r) * KP + k);
        acc[r].x = fmaf(x.x, w0.x, acc[r].x); acc[r].y = fmaf(x.x, w0.y, acc[r].y);
        acc[r].z = fmaf(x.x, w0.z, acc[r].z); acc[r].w = fmaf(x.x, w0.w, acc[r].w);
        acc[r].x = fmaf(x.y, w1.x, acc[r].x); acc[r].y = fmaf(x.y, w1.y, acc[r].y);
        acc[r].z = fmaf(x.y, w1.z, acc[r].z); acc[r].w = fmaf(x.y, w1.w, acc[r].w);
        acc[r].x = fmaf(x.z, w2.x, acc[r].x); acc[r].y = fmaf(x.z, w2.y, acc[r].y);
        acc[r].z = fmaf(x.z, w2.z, acc[r].z); acc[r].w = fmaf(x.z, w2.w, acc[r].w);
        acc[r].x = fmaf(x.w, w3.x, acc[r].x); acc[r].y = fmaf(x.w, w3.y, acc[r].y);
        acc[r].z = fmaf(x.w, w3.z, acc[r].z); acc[r].w = fmaf(x.w, w3.w, acc[r].w);
      }
    }
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const int64_t m = m0 + rg * 8 + r;
      if (m < M) {
        float4 v = acc[r];
        v.x = apply_act(v.x, act); v.y = apply_act(v.y, act);
        v.z = apply_act(v.z, act); v.w = apply_act(v.w, act);
        reinterpret_cast<float4*>(Y + m * N)[cq] = v;
      }
    }
  }
}

// dW[K,N] += X^T dZ, db[N] += column sums of dZ over the CTA's row range.
template <int KMAX>
__global__ void __launch_bounds__(256, KMAX <= 20 ? 2 : 1) thin_dw_kernel(const float* __restrict__ X, int64_t ldx,
                                                      const float* __restrict__ dZ,
                                                      float* __restrict__ dW,
                                                      float* __restrict__ db, int64_t M, int K,
                                                      int N, int64_t rows_per_cta) {
  pdl_prologue();
  extern __shared__ float4 thin_smem[];
  const int nq = N >> 2;
  float* sx = reinterpret_cast<float*>(thin_smem);     // [kThinRows][KMAX]
  float* sred = sx + kThinRows * KMAX;                 // [(K + 1)][N] cross-row-group sums
  for (int i = threadIdx.x; i < (K + 1) * N; i += blockDim.x) sred[i] = 0.f;
  const int cq = threadIdx.x & 63, rg = threadIdx.x >> 6;
  const bool active = cq < nq;
  float4 acc[KMAX], bsum = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int k = 0; k < KMAX; ++k) acc[k] = make_float4(0.f, 0.f, 0.f, 0.f);
  const int64_t mb = (int64_t)blockIdx.x * rows_per_cta;
  const int64_t me = (mb + rows_per_cta < M) ? mb + rows_per_cta : M;
  for (int64_t m0 = mb; m0 < me; m0 += kThinRows) {
    __syncthreads();
    for (int i = threadIdx.x; i < kThinRows * KMAX; i += blockDim.x) {
      const int r = i / KMAX, k = i - r * KMAX;
      sx[i] = (m0 + r < me && k < K) ? X[(m0 + r) * ldx + k] : 0.f;
    }
    __syncthreads();
    if (!active) continue;
#pragma unroll 1
    for (int h = 0; h < 8; h += 4) {                   // two halves of 4 rows: 128 registers, 2 CTAs / SM
    float4 dz[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int64_t m = m0 + rg * 8 + h + r;
      dz[r] = m < me ? reinterpret_cast<const float4*>(dZ + m * N)[cq] : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      bsum.x += dz[r].x; bsum.y += dz[r].y; bsum.z += dz[r].z; bsum.w += dz[r].w;
      const float* xr = sx + (rg * 8 + h + r) * KMAX;
#pragma unroll
      for (int k = 0; k < KMAX; k += 4) {
        const float4 x = *reinterpret_cast<const float4*>(xr + k);
        acc[k + 0].x = fmaf(x.x, dz[r].x, acc[k + 0].x); acc[k + 0].y = fmaf(x.x, dz[r].y, acc[k + 0].y);
        acc[k + 0].z = fmaf(x.x, dz[r].z, acc[k + 0].z); acc[k + 0].w = fmaf(x.x, dz[r].w, acc[k + 0].w);
        acc[k + 1].x = fmaf(x.y, dz[r].x, acc[k + 1].x); acc[k + 1].y = fmaf(x.y, dz[r].y, acc[k + 1].y);
        acc[k + 1].z = fmaf(x.y, dz[r].z, acc[k + 1].z); acc[k + 1].w = fmaf(x.y, dz[r].w, acc[k + 1].w);
        acc[k + 2].x = fmaf(x.z, dz[r].x, acc[k + 2].x); acc[k + 2].y = fmaf(x.z, dz[r].y, acc[k + 2].y);
        acc[k + 2].z = fmaf(x.z, dz[r].z, acc[k + 2].z); acc[k + 2].w = fmaf(x.z, dz[r].w, acc[k + 2].w);
        acc[k + 3].x = fmaf(x.w, dz[r].x, acc[k + 3].x); acc[k + 3].y = fmaf(x.w, dz[r].y, acc[k + 3].y);
        acc[k + 3].z = fmaf(x.w, dz[r].z, acc[k + 3].z); acc[k + 3].w = fmaf(x.w, dz[r].w, acc[k + 3].w);
      }
    }
    }
  }
  // the four row groups add their partial sums in a fixed order (a single-CTA launch, i.e. a small
  // batch, is bit-reproducible; larger ones meet in the global atomics below)
  for (int g = 0; g < 4; ++g) {
    __syncthreads();
    if (active && rg == g) {
#pragma unroll
      for (int k = 0; k < KMAX; ++k) {
        if (k < K) {
          float4* d = reinterpret_cast<float4*>(sred + k * N) + cq;
          float4 v = *d;
          v.x += acc[k].x; v.y += acc[k].y; v.z += acc[k].z; v.w += acc[k].w;
          *d = v;
        }
      }
      float4* d = reinterpret_cast<float4*>(sred + K * N) + cq;
      float4 v = *d;
      v.x += bsum.x; v.y += bsum.y; v.z += bsum.z; v.w += bsum.w;
      *d = v;
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < K * N; i += blockDim.x) atomicAdd(dW + i, sred[i]);
  if (db != nullptr)
    for (int i = threadIdx.x; i < N; i += blockDim.x) atomicAdd(db + i, sred[K * N + i]);
}

// col2im in gather form (deterministic): dX[n,y,x,c] = sum over kernel taps hitting (y,x).
__global__ void col2im_kernel(const float* __restrict__ dcol, float* __restrict__ dX, ConvGeom g,
                              int64_t total, int Kc, const ActMask mask) {
  pdl_prologue();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = (int)(i % g.C);
  int64_t r = i / g.C;
  const int x = (int)(r % g.W);
  r /= g.W;
  const int y = (int)(r % g.H);
  const int64_t n = r / g.H;
  float s = 0.f;
  for (int ky = y % g.stride; ky < g.KH && ky <= y; ky += g.stride) {
    const int oy = (y - ky) / g.stride;
    if (oy >= g.OH) continue;
    for (int kx = x % g.stride; kx < g.KW && kx <= x; kx += g.stride) {
      const int ox = (x - kx) / g.stride;
      if (ox >= g.OW) continue;
      const int64_t pos = (n * g.OH + oy) * g.OW + ox;
      s += dcol[pos * Kc + (ky * g.KW + kx) * g.C + c];
    }
  }
  if (mask.y) s = dact(mask.y[n * mask.ld + ((int64_t)y * g.W + x) * g.C + c], s, mask.act);
  dX[i] = s;
}

// ---------------------------------------------------------------------------------------
// host-side dispatch
// ---------------------------------------------------------------------------------------
// GEMM mode, read from B200RL_GEMM_MODE once, on first use; b200rl_set_gemm_mode overrides it.
//   0 = fp32 FFMA (sgemm_kernel), 1 = wgmma 3xTF32 (default),
//   2 = wgmma single-pass TF32 (not 1e-5 safe)
static int& gemm_mode() {
  static int mode = [] {
    const char* e = getenv("B200RL_GEMM_MODE");
    return e ? atoi(e) : 1;
  }();
  return mode;
}

static bool al16(const void* p) { return ((uintptr_t)p & 15) == 0; }

// Zeroes bytes at p on st; p == NULL (an optional gradient that is not wanted) is a no-op.
static int zero_async(void* p, size_t bytes, cudaStream_t st, const char* what) {
  if (p == nullptr) return B200RL_OK;
  cudaError_t e = cudaMemsetAsync(p, 0, bytes, st);
  if (e != cudaSuccess) {
    set_error("%s: memset failed: %s", what, cudaGetErrorString(e));
    return B200RL_ERR_CUDA;
  }
  return B200RL_OK;
}

struct GemmArgs {
  float* C;
  const float* bias;
  int64_t M, N, K;
  int act, beta;
  void* ws;
  int64_t ws_bytes;
  cudaStream_t st;
  float out_scale = 1.f;  // tensor-core path only: multiplies the accumulator (raw-u8 operands)
  ActMask mask{};         // input-gradient GEMMs: multiply the result by act'(mask.y)
  // split-K partial slices of C that fit in the workspace (0 without one)
  int64_t ws_slices() const { return ws ? ws_bytes / (M * N * (int64_t)sizeof(float)) : 0; }
};

// The smallest GEMM (in GEMM coordinates) the tensor-core kernels take.
static bool tc_fits(int64_t M, int64_t N, int64_t K) { return N >= 16 && M >= 32 && K >= 8; }

struct SplitK {
  int splits;
  int64_t kps;  // K range per split, a multiple of bk
};
// Split-K over grid.z when the tile grid leaves the chip short of `target` CTAs and K spans at
// least 8 blocks of bk: ceil (round_up) or floor of target / tiles splits, each keeping at least
// 4 blocks, at most max_splits and 65535.  The K range is then rounded up to whole blocks and the
// splits recounted.
static SplitK plan_split_k(int64_t tiles, int64_t K, int64_t bk, int64_t target, bool round_up,
                           int64_t max_splits) {
  int64_t s = 1;
  if (tiles < target && K >= 8 * bk) {
    s = round_up ? (target + tiles - 1) / tiles : target / tiles;
    if (s > K / (4 * bk)) s = K / (4 * bk);
    if (s > max_splits) s = max_splits;
    if (s > 65535) s = 65535;
    if (s < 2) s = 1;
  }
  int64_t kps = (K + s - 1) / s;
  kps = (kps + bk - 1) / bk * bk;
  return {(int)((K + kps - 1) / kps), kps};
}

static int splitk_reduce(const GemmArgs& g, int splits) {
  const int64_t MN = g.M * g.N;
  B200RL_LAUNCH(splitk_reduce_kernel, (unsigned)((MN + 255) / 256), 256, 0, g.st, (const float*)g.ws, g.C, g.bias, MN, g.N, splits, g.act, g.beta, g.mask);
  B200RL_CHECK_LAUNCH("splitk_reduce");
  return B200RL_OK;
}

template <int BM, int BN, int TM, int TN, class AL, class BL>
static int launch_gemm_cfg(const AL& a, const BL& b, const GemmArgs& g) {
  const int64_t tm = (g.M + BM - 1) / BM, tn = (g.N + BN - 1) / BN;
  // two CTAs per SM; the partials always go through the workspace
  const SplitK sk = plan_split_k(tm * tn, g.K, BK, 2 * kNumSMs, true, g.ws_slices());
  B200RL_CHECK_ARG(tm <= 65535, "gemm: M too large for grid.y (%lld tiles)", (long long)tm);
  dim3 grid((unsigned)tn, (unsigned)tm, (unsigned)sk.splits);
  B200RL_LAUNCH((sgemm_kernel<BM, BN, TM, TN, AL, BL>), grid, 256, 0, g.st, a, b, g.C, g.bias, g.M, g.N, g.K, g.act, g.beta, sk.splits, sk.kps, (float*)g.ws, g.mask);
  B200RL_CHECK_LAUNCH("sgemm");
  return sk.splits > 1 ? splitk_reduce(g, sk.splits) : B200RL_OK;
}

template <int BN, int PASSES, int EPI, class AL, class BL>
static int launch_tc_cfg(const AL& a, const BL& b, const GemmArgs& g, const tc::EpiArgs& epi) {
  using L = tc::SmemLayout<BN, PASSES, AL::kExact>;
  auto short_k = tc::tc_gemm_kernel<BN, PASSES, EPI, AL, BL, false>;
  auto long_k = tc::tc_gemm_kernel<BN, PASSES, EPI, AL, BL, PASSES == 3>;
  static bool configured = false;
  if (!configured) {
    for (auto kernel : {short_k, long_k}) {
      cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           L::kBytes);
      if (e != cudaSuccess) {
        set_error("tc_gemm: cannot set dynamic smem to %d: %s", L::kBytes, cudaGetErrorString(e));
        return B200RL_ERR_CUDA;
      }
    }
    configured = true;
  }
  const int64_t tm = (g.M + tc::kBM - 1) / tc::kBM, tn = (g.N + BN - 1) / BN;
  // kCtasPerSM resident CTAs per SM: only split when a whole extra set of CTAs fits on the chip.
  // The atomic and col2im epilogues add their partials in place; only EPI_STORE needs the workspace.
  const SplitK sk = plan_split_k(tm * tn, g.K, tc::kBK, kNumSMs * L::kCtasPerSM, false,
                                 EPI == tc::EPI_STORE ? g.ws_slices() : 65535);
  B200RL_CHECK_ARG(tm <= 65535, "tc_gemm: M too large for grid.y (%lld tiles)", (long long)tm);
  dim3 grid((unsigned)tn, (unsigned)tm, (unsigned)sk.splits);
  // a K range longer than one accumulation chain needs the chained variant to stay fp32-accurate
  auto kernel = sk.kps > tc::kChainBlocks * tc::kBK ? long_k : short_k;
  B200RL_LAUNCH(kernel, grid, tc::kThreads, L::kBytes, g.st, a, b, epi, g.C, g.bias, g.M, g.N, g.K, g.act, g.beta, sk.splits, sk.kps, (float*)g.ws, g.out_scale);
  B200RL_CHECK_LAUNCH("tc_gemm");
  return sk.splits > 1 && EPI == tc::EPI_STORE ? splitk_reduce(g, sk.splits) : B200RL_OK;
}

// Tensor-core GEMM with a fixed pass count: BN by output width (32 / 64 / 128; col2im always 128).
template <int PASSES, int EPI, class AL, class BL>
static int launch_tc_passes(const AL& a, const BL& b, const GemmArgs& g, const tc::EpiArgs& epi) {
  B200RL_CHECK_ARG(!(g.mask.y && g.beta), "gemm: an input-gradient mask cannot be combined with accumulation");
  if constexpr (EPI == tc::EPI_COL2IM) {
    return launch_tc_cfg<128, PASSES, EPI>(a, b, g, epi);
  } else {
    if (g.N <= 32) return launch_tc_cfg<32, PASSES, EPI>(a, b, g, epi);
    if (g.N <= 64) return launch_tc_cfg<64, PASSES, EPI>(a, b, g, epi);
    return launch_tc_cfg<128, PASSES, EPI>(a, b, g, epi);
  }
}

// Tensor-core GEMM in the current mode: 2 = single-pass TF32, otherwise 3xTF32.
template <int EPI, class AL, class BL>
static int launch_tc(const AL& a, const BL& b, const GemmArgs& g, const tc::EpiArgs& epi) {
  if (gemm_mode() == 2) return launch_tc_passes<1, EPI>(a, b, g, epi);
  return launch_tc_passes<3, EPI>(a, b, g, epi);
}

template <class AL, class BL>
static int launch_gemm(const AL& a, const BL& b, const GemmArgs& g) {
  if (g.M <= 0 || g.N <= 0) return B200RL_OK;
  B200RL_CHECK_ARG(g.K > 0, "gemm: K must be > 0");
  B200RL_CHECK_ARG(g.M < (1ll << 31) && g.N < (1ll << 31) && g.K < (1ll << 31), "gemm: dims");
  if (gemm_mode() != 0 && tc_fits(g.M, g.N, g.K)) {
    tc::EpiArgs epi{};
    epi.mask = g.mask;
    return launch_tc<tc::EPI_STORE>(a, b, g, epi);
  }
  if (g.N <= 32) return launch_gemm_cfg<128, 32, 4, 4>(a, b, g);
  if (g.N <= 64) {
    if (g.M >= 4096) return launch_gemm_cfg<128, 64, 8, 4>(a, b, g);
    return launch_gemm_cfg<64, 64, 4, 4>(a, b, g);
  }
  const int64_t t128 = ((g.M + 127) / 128) * ((g.N + 127) / 128);
  if (t128 >= kNumSMs) return launch_gemm_cfg<128, 128, 8, 8>(a, b, g);
  return launch_gemm_cfg<64, 64, 4, 4>(a, b, g);
}

// Weight-gradient GEMMs (no bias / activation): in tensor-core mode the split-K partials are
// accumulated with red.global.add straight into the (zeroed) gradient instead of going through
// a workspace + reduce kernel.  Summation order across splits is not fixed.
// `db` (optional): bias gradient = column sums of B; when the tensor-core path takes the GEMM and
// B is an MN-major view the sums are accumulated by the producers of the same kernel and
// *db_fused is set, otherwise the caller runs the separate column-sum kernels.
template <class AL, class BL>
static int launch_grad_gemm(const AL& a, const BL& b, const GemmArgs& g, float* db, bool* db_fused) {
  *db_fused = false;
  if (gemm_mode() == 0 || !tc_fits(g.M, g.N, g.K)) return launch_gemm(a, b, g);
  tc::EpiArgs epi{};
  if (db != nullptr && !BL::kKContig) epi.colsum = db;
  if (!g.beta) {
    int rc = zero_async(g.C, (size_t)(g.M * g.N) * sizeof(float), g.st, "grad gemm");
    if (rc == B200RL_OK) rc = zero_async(epi.colsum, (size_t)g.N * sizeof(float), g.st, "grad gemm");
    if (rc) return rc;
  }
  *db_fused = epi.colsum != nullptr;
  return launch_tc<tc::EPI_ATOMIC>(a, b, g, epi);
}


// ---- skinny-head dispatch (N <= 16) ----------------------------------------------------------
static bool skinny_ok(int64_t M, int64_t K, int64_t N) {
  return gemm_mode() != 0 && N >= 1 && N <= kSkinnyMaxN && K >= 1 && K <= 1024 &&
         K * N * (int64_t)sizeof(float) <= kSkinnySmem && M >= 1;
}
template <int NMAX>
static int skinny_fwd_launch(const float* X, int64_t ldx, const float* W, const float* bias,
                             float* Y, int64_t M, int64_t K, int64_t N, int act, cudaStream_t st) {
  int64_t blocks = (M + 7) / 8;
  if (blocks > kNumSMs * 8) blocks = kNumSMs * 8;
  B200RL_LAUNCH(skinny_fwd_kernel<NMAX>, (unsigned)blocks, 256, (size_t)(K * N * sizeof(float)), st, X, ldx, W, bias, Y, M, (int)K, (int)N, act);
  B200RL_CHECK_LAUNCH("skinny_fwd");
  return B200RL_OK;
}
template <int NMAX>
static int skinny_dx_launch(const float* dY, const float* W, float* dX, int64_t M, int64_t K,
                            int64_t N, const ActMask& mask, cudaStream_t st) {
  int64_t blocks = (M * ((K + 3) / 4) + 255) / 256;
  if (blocks > kNumSMs * 8) blocks = kNumSMs * 8;
  B200RL_LAUNCH(skinny_dx_kernel<NMAX>, (unsigned)blocks, 256, (size_t)(K * N * sizeof(float)), st, dY, W, dX, M, (int)K, (int)N, mask);
  B200RL_CHECK_LAUNCH("skinny_dx");
  return B200RL_OK;
}
template <int NMAX>
static int skinny_dw_launch(const float* X, int64_t ldx, const float* dY, float* dW, float* db,
                            int64_t M, int64_t K, int64_t N, int accumulate, cudaStream_t st) {
  if (!accumulate) {
    int rc = zero_async(dW, (size_t)(K * N) * sizeof(float), st, "skinny dW");
    if (rc == B200RL_OK) rc = zero_async(db, (size_t)N * sizeof(float), st, "skinny dW");
    if (rc) return rc;
  }
  int64_t rows = (M + 2 * kNumSMs - 1) / (2 * kNumSMs);   // ~2 CTAs per SM; small M: 8-row slabs
  rows = (rows + 7) / 8 * 8;
  const int64_t blocks = (M + rows - 1) / rows;
  if (K <= 256) B200RL_LAUNCH((skinny_dw_kernel<NMAX, 1>), (unsigned)blocks, 256, (size_t)(K * N * sizeof(float)), st, X, ldx, dY, dW, db, M, (int)K, (int)N, rows);
  else if (K <= 512) B200RL_LAUNCH((skinny_dw_kernel<NMAX, 2>), (unsigned)blocks, 256, 0, st, X, ldx, dY, dW, db, M, (int)K, (int)N, rows);
  else B200RL_LAUNCH((skinny_dw_kernel<NMAX, 4>), (unsigned)blocks, 256, 0, st, X, ldx, dY, dW, db, M, (int)K, (int)N, rows);
  B200RL_CHECK_LAUNCH("skinny_dw");
  return B200RL_OK;
}
#define SKINNY_BY_N(fn, N, ...)                                  \
  ((N) <= 4 ? fn<4>(__VA_ARGS__) : (N) <= 8 ? fn<8>(__VA_ARGS__) : fn<16>(__VA_ARGS__))

static int colsum(const float* dZ, float* db, int64_t M, int64_t N, int beta, void* ws,
                  int64_t ws_bytes, cudaStream_t st) {
  const int64_t nparts = (M + kColRows - 1) / kColRows;
  B200RL_CHECK_ARG(ws != nullptr && ws_bytes >= (int64_t)(nparts * N * sizeof(float)),
                   "bias gradient needs %lld bytes of workspace",
                   (long long)(nparts * N * sizeof(float)));
  B200RL_CHECK_ARG(nparts <= 65535, "bias gradient: too many rows");
  dim3 grid((unsigned)((N + 31) / 32), (unsigned)nparts);
  B200RL_LAUNCH(colsum_partial_kernel, grid, 256, 0, st, dZ, (float*)ws, M, N);
  B200RL_CHECK_LAUNCH("colsum_partial");
  B200RL_LAUNCH(colsum_final_kernel, (unsigned)((N + 7) / 8), 256, 0, st, (const float*)ws, db, nparts, N, beta);
  B200RL_CHECK_LAUNCH("colsum_final");
  return B200RL_OK;
}

static int make_geom(const b200rl_conv_t* c, ConvGeom& g) {
  B200RL_CHECK_ARG(c != nullptr, "conv geometry is NULL");
  B200RL_CHECK_ARG(c->N > 0 && c->H > 0 && c->W > 0 && c->C > 0 && c->KH > 0 && c->KW > 0 &&
                       c->F > 0 && c->stride > 0,
                   "conv: non-positive dimension");
  B200RL_CHECK_ARG(c->H >= c->KH && c->W >= c->KW, "conv: kernel larger than input");
  g.H = c->H; g.W = c->W; g.C = c->C; g.KH = c->KH; g.KW = c->KW; g.F = c->F;
  g.stride = c->stride;
  g.OH = (c->H - c->KH) / c->stride + 1;
  g.OW = (c->W - c->KW) / c->stride + 1;
  g.d_ohow = FastDiv((uint32_t)(g.OH * g.OW));
  g.d_ow = FastDiv((uint32_t)g.OW);
  g.d_kwc = FastDiv((uint32_t)(g.KW * g.C));
  g.in_row = (int64_t)c->W * c->C;
  g.in_img = c->x_batch_stride > 0 ? c->x_batch_stride : (int64_t)c->H * c->W * c->C;
  const int64_t M = (int64_t)c->N * g.OH * g.OW;
  B200RL_CHECK_ARG(M < (1ll << 31), "conv: too many output positions");
  return B200RL_OK;
}

}  // namespace b200rl

using namespace b200rl;

extern "C" {

int b200rl_tc_debug_buffer(long long* dev_buf) {
  cudaError_t e = cudaMemcpyToSymbol(tc::g_tc_dbg, &dev_buf, sizeof(dev_buf));
  if (e != cudaSuccess) {
    set_error("tc_debug_buffer: %s", cudaGetErrorString(e));
    return B200RL_ERR_CUDA;
  }
  return B200RL_OK;
}

// ---- thin-input dispatch (K <= 32, 16 < N <= 256, N % 4 == 0) -----------------------------------
static bool thin_ok(const float* W, int64_t M, int64_t K, int64_t N) {
  return gemm_mode() != 0 && K >= 1 && K <= kThinMaxK && N > kSkinnyMaxN && N <= kThinMaxN &&
         (N & 3) == 0 && M >= 1 && al16(W);
}
static int thin_fwd_launch(const float* X, int64_t ldx, const float* W, const float* bias, float* Y,
                           int64_t M, int64_t K, int64_t N, int act, cudaStream_t st) {
  const int64_t chunks = (M + kThinRows - 1) / kThinRows;
  const int KP = ((int)K + 3) & ~3;
  const size_t smem = (size_t)KP * N * sizeof(float) + (size_t)kThinRows * KP * sizeof(float);
  const int64_t blocks = chunks < 4 * kNumSMs ? chunks : 4 * kNumSMs;
  B200RL_LAUNCH(thin_fwd_kernel, (unsigned)blocks, 256, smem, st, X, ldx, W, bias, Y, M, (int)K, (int)N, act, chunks);
  B200RL_CHECK_LAUNCH("thin_fwd");
  return B200RL_OK;
}
static int thin_dw_launch(const float* X, int64_t ldx, const float* dZ, float* dW, float* db,
                          int64_t M, int64_t K, int64_t N, int accumulate, cudaStream_t st) {
  if (!accumulate) {
    int rc = zero_async(dW, (size_t)(K * N) * sizeof(float), st, "thin dW");
    if (rc == B200RL_OK) rc = zero_async(db, (size_t)N * sizeof(float), st, "thin dW");
    if (rc) return rc;
  }
  int64_t rows = (M + 4 * kNumSMs - 1) / (4 * kNumSMs);
  rows = (rows + kThinRows - 1) / kThinRows * kThinRows;
  const int64_t blocks = (M + rows - 1) / rows;
  const int KMAX = K <= 8 ? 8 : K <= 20 ? 20 : 32;
  const size_t smem = ((size_t)kThinRows * KMAX + (size_t)(K + 1) * N) * sizeof(float);
  if (KMAX == 8) B200RL_LAUNCH(thin_dw_kernel<8>, (unsigned)blocks, 256, smem, st, X, ldx, dZ, dW, db, M, (int)K, (int)N, rows);
  else if (KMAX == 20) B200RL_LAUNCH(thin_dw_kernel<20>, (unsigned)blocks, 256, smem, st, X, ldx, dZ, dW, db, M, (int)K, (int)N, rows);
  else B200RL_LAUNCH(thin_dw_kernel<32>, (unsigned)blocks, 256, smem, st, X, ldx, dZ, dW, db, M, (int)K, (int)N, rows);
  B200RL_CHECK_LAUNCH("thin_dw");
  return B200RL_OK;
}

int b200rl_set_gemm_mode(int mode) {
  B200RL_CHECK_ARG(mode >= 0 && mode <= 2, "gemm mode must be 0 (fp32 FFMA), 1 (wgmma 3xTF32) "
                                           "or 2 (wgmma 1xTF32)");
  gemm_mode() = mode;
  return B200RL_OK;
}

int b200rl_dense_fwd(const float* X, int64_t ldx, const float* W, const float* bias, float* Y,
                     int64_t M, int64_t K, int64_t N, int act, void* workspace,
                     int64_t ws_bytes, void* stream) {
  B200RL_CHECK_ARG(X && W && Y, "dense_fwd: NULL argument");
  B200RL_CHECK_ARG(ldx == 0 || ldx >= K, "dense_fwd: ldx < K");
  if (ldx == 0) ldx = K;
  cudaStream_t st = (cudaStream_t)stream;
  if (skinny_ok(M, K, N)) return SKINNY_BY_N(skinny_fwd_launch, N, X, ldx, W, bias, Y, M, K, N, act, st);
  if (thin_ok(W, M, K, N) && al16(Y) && (bias == nullptr || al16(bias)))
    return thin_fwd_launch(X, ldx, W, bias, Y, M, K, N, act, st);
  GemmArgs g{Y, bias, M, N, K, act, 0, workspace, ws_bytes, st};
  return launch_gemm(ARow{X, ldx}, BRow{W, N}, g);
}

int b200rl_dense_bwd(const float* X, int64_t ldx, const float* W, const float* dY, float* dX,
                     float* dW, float* db, int64_t M, int64_t K, int64_t N, int accumulate,
                     int x_act, void* workspace, int64_t ws_bytes, void* stream) {
  B200RL_CHECK_ARG(X && W && dY, "dense_bwd: NULL argument");
  B200RL_CHECK_ARG(ldx == 0 || ldx >= K, "dense_bwd: ldx < K");
  B200RL_CHECK_ARG(x_act >= B200RL_ACT_NONE && x_act <= B200RL_ACT_TANH, "dense_bwd: x_act");
  if (ldx == 0) ldx = K;
  cudaStream_t st = (cudaStream_t)stream;
  ActMask mask{};
  if (x_act != B200RL_ACT_NONE) mask = ActMask{X, ldx, x_act};
  int rc;
  if (skinny_ok(M, K, N)) {
    if (dX) {
      rc = SKINNY_BY_N(skinny_dx_launch, N, dY, W, dX, M, K, N, mask, st);
      if (rc) return rc;
    }
    if (dW) return SKINNY_BY_N(skinny_dw_launch, N, X, ldx, dY, dW, db, M, K, N, accumulate, st);
    if (db) return colsum(dY, db, M, N, accumulate, workspace, ws_bytes, st);
    return B200RL_OK;
  }
  if (dX) {  // dX[M,K] = dY @ W^T
    GemmArgs g{dX, nullptr, M, K, N, B200RL_ACT_NONE, 0, workspace, ws_bytes, st};
    g.mask = mask;
    rc = launch_gemm(ARow{dY, N}, BCol{W, N}, g);
    if (rc) return rc;
  }
  bool db_fused = false;
  if (dW && thin_ok(W, M, K, N) && al16(dY)) {
    rc = thin_dw_launch(X, ldx, dY, dW, db, M, K, N, accumulate, st);
    if (rc) return rc;
    db_fused = true;
  } else if (dW) {  // dW[K,N] = X^T @ dY
    GemmArgs g{dW, nullptr, K, N, M, B200RL_ACT_NONE, accumulate, workspace, ws_bytes, st};
    rc = launch_grad_gemm(ACol{X, ldx}, BRow{dY, N}, g, db, &db_fused);
    if (rc) return rc;
  }
  if (db && !db_fused) return colsum(dY, db, M, N, accumulate, workspace, ws_bytes, st);
  return B200RL_OK;
}

int b200rl_act_bwd(const float* Y, const float* dY, float* dZ, int64_t n, int act,
                   void* stream) {
  B200RL_CHECK_ARG(Y && dY && dZ && n >= 0, "act_bwd: bad argument");
  if (n == 0) return B200RL_OK;
  const int vec = (n & 3) == 0 && ((((uintptr_t)Y | (uintptr_t)dY | (uintptr_t)dZ) & 15) == 0);
  int64_t blocks = ((vec ? n / 4 : n) + 255) / 256;
  if (blocks > kNumSMs * 16) blocks = kNumSMs * 16;
  B200RL_LAUNCH(act_bwd_kernel, (unsigned)blocks, 256, 0, (cudaStream_t)stream, Y, dY, dZ, n, act, vec);
  B200RL_CHECK_LAUNCH("act_bwd");
  return B200RL_OK;
}

int b200rl_conv2d_fwd(const void* X, int x_is_u8, float x_scale, const float* Wt,
                      const float* bias, float* Y, const b200rl_conv_t* c, int act,
                      void* workspace, int64_t ws_bytes, void* stream) {
  B200RL_CHECK_ARG(X && Wt && Y, "conv2d_fwd: NULL argument");
  ConvGeom cg;
  int rc = make_geom(c, cg);
  if (rc) return rc;
  const int64_t M = (int64_t)c->N * cg.OH * cg.OW, K = (int64_t)c->KH * c->KW * c->C;
  GemmArgs g{Y, bias, M, c->F, K, act, 0, workspace, ws_bytes, (cudaStream_t)stream};
  const BRow w{Wt, c->F};
  if (x_is_u8 && gemm_mode() == 1 && tc_fits(M, c->F, K)) {
    // raw pixels, 2-pass 3xTF32, scaled in the epilogue (mode 1 only: no 1-pass kernels are built)
    g.out_scale = 1.f / x_scale;
    AConvU8Raw a{ConvView<uint8_t>{(const uint8_t*)X, cg, x_scale}};
    return launch_tc_passes<3, tc::EPI_STORE>(a, w, g, tc::EpiArgs{});
  }
  if (x_is_u8) return launch_gemm(AConv<uint8_t>{ConvView<uint8_t>{(const uint8_t*)X, cg, x_scale}}, w, g);
  return launch_gemm(AConv<float>{ConvView<float>{(const float*)X, cg, 1.f}}, w, g);
}

int b200rl_conv2d_bwd(const void* X, int x_is_u8, float x_scale, const float* Wt,
                      const float* dY, float* dX, float* dW, float* db,
                      const b200rl_conv_t* c, int accumulate, int x_act, void* workspace,
                      int64_t ws_bytes, void* stream) {
  B200RL_CHECK_ARG(X && Wt && dY, "conv2d_bwd: NULL argument");
  B200RL_CHECK_ARG(!(dX && x_is_u8), "conv2d_bwd: no input gradient for u8 input");
  B200RL_CHECK_ARG(x_act >= B200RL_ACT_NONE && x_act <= B200RL_ACT_TANH, "conv2d_bwd: x_act");
  ConvGeom cg;
  int rc = make_geom(c, cg);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t M = (int64_t)c->N * cg.OH * cg.OW, K = (int64_t)c->KH * c->KW * c->C;
  const int64_t F = c->F;
  const int mode = gemm_mode();
  ActMask mask{};
  if (x_act != B200RL_ACT_NONE && !x_is_u8) mask = ActMask{(const float*)X, cg.in_img, x_act};
  bool db_fused = false;
  if (dW) {  // dW[K,F] = im2col(X)^T @ dY
    GemmArgs g{dW, nullptr, K, F, M, B200RL_ACT_NONE, accumulate, workspace, ws_bytes, st};
    const BRow dy{dY, F};
    if (!x_is_u8) {
      AConvT<float> a{ConvView<float>{(const float*)X, cg, 1.f}};
      rc = launch_grad_gemm(a, dy, g, db, &db_fused);
    } else if (mode == 1 && tc_fits(K, F, M)) {   // raw pixels, scaled in the epilogue
      g.out_scale = 1.f / x_scale;
      AConvTU8Raw a{ConvView<uint8_t>{(const uint8_t*)X, cg, x_scale}};
      rc = launch_grad_gemm(a, dy, g, db, &db_fused);
    } else {  // mode 0 / 2: the STORE epilogue, bias gradient by the column-sum kernels
      AConvT<uint8_t> a{ConvView<uint8_t>{(const uint8_t*)X, cg, x_scale}};
      rc = launch_gemm(a, dy, g);
    }
    if (rc) return rc;
  }
  if (db && !db_fused) {
    rc = colsum(dY, db, M, F, accumulate, workspace, ws_bytes, st);
    if (rc) return rc;
  }
  if (!dX) return B200RL_OK;
  const int64_t total = (int64_t)c->N * c->H * c->W * c->C;
  if (mode != 0 && (c->C & 3) == 0 && tc_fits(M, K, F)) {
    // tensor-core path: dY @ W^T with the col2im scatter-add fused into the epilogue
    rc = zero_async(dX, (size_t)total * sizeof(float), st, "conv2d_bwd");
    if (rc) return rc;
    GemmArgs g{nullptr, nullptr, M, K, F, B200RL_ACT_NONE, 0, nullptr, 0, st};
    tc::EpiArgs epi{cg, dX};
    epi.mask = mask;
    return launch_tc<tc::EPI_COL2IM>(ARow{dY, F}, BCol{Wt, F}, g, epi);
  }
  // dcol[M,K] = dY @ W^T, then gather-form col2im
  const int64_t need = M * K * (int64_t)sizeof(float);
  B200RL_CHECK_ARG(workspace && ws_bytes >= need,
                   "conv2d_bwd: input gradient needs %lld bytes of workspace", (long long)need);
  GemmArgs g{(float*)workspace, nullptr, M, K, F, B200RL_ACT_NONE, 0, nullptr, 0, st};
  rc = launch_gemm(ARow{dY, F}, BCol{Wt, F}, g);
  if (rc) return rc;
  B200RL_LAUNCH(col2im_kernel, (unsigned)((total + 255) / 256), 256, 0, st, (const float*)workspace, dX, cg, total, (int)K, mask);
  B200RL_CHECK_LAUNCH("col2im");
  return B200RL_OK;
}

}  // extern "C"
