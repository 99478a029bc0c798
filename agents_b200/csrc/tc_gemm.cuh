// Tensor-core GEMM for the Q / actor / critic networks: Hopper warpgroup MMA (wgmma, tf32 inputs,
// fp32 register accumulators), fp32-grade accuracy through the 3xTF32 split.
//
//   C[M,N] (+)= act(A[M,K] @ B[K,N] + bias)      A, B given as operand views (see nn.cu)
//
// Why 3xTF32: north_star parity is 1e-5 relative on the loss; one TF32 pass keeps ~11 mantissa
// bits (1e-3).  Each fp32 operand x is split into hi = x with the low 13 mantissa bits cleared
// and lo = x - hi (exact); the tensor core accumulates lo_a*hi_b + hi_a*lo_b + hi_a*hi_b into the
// same fp32 accumulator (the dropped lo*lo term is 2^-22 relative).
//
// Structure (one CTA = one 128 x BN output tile, 256 threads = two warpgroups):
//   operand ring: every thread copies its share of the raw (128 x 32) A tile and (BN x 32) B^T
//   tile of a K block global -> shared with cp.async (16-byte chunks, 4-byte ones for uint8 and
//   misaligned views; zero-fill through src-size past every tail), kRing - 1 K blocks ahead of the
//   block being multiplied, so several blocks of loads are in flight at once;
//   per K block: wait for the block's copies, barrier, issue the copies of block i + kRing - 1,
//   then split: read the raw tile from shared memory (u8 -> f32 conversion here), write TF32 hi /
//   lo K-major into 128B-swizzled planes, the layout wgmma reads (tf32 operands must be K-major,
//   so MN-contiguous views are transposed in this pass); a second barrier, then warpgroup w
//   issues wgmma.m64nBNk8 for rows 64w..64w+63 (4 K steps x up to 3 passes per 32-wide K block)
//   and keeps one group in flight while the next block is split.  Two plane stages: the first
//   barrier of block i comes after every warpgroup retired the MMAs of block i-2.
//   Exact A views (raw uint8 pixels) have no A plane: each thread loads its wgmma fragments of A
//   from the raw ring slot into one of two register sets and only B is split.
//   The epilogue parks the accumulators in the idle planes / ring and drains them row-per-thread:
//   bias / activation / act' mask / split-K partials, the fused col2im scatter-add, or red.add.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200rl {
namespace tc {

constexpr int kBM = 128;
constexpr int kBK = 32;                    // fp32 elements = 128 bytes = one swizzle row
constexpr int kThreads = 256;
constexpr int kPlaneStages = 2;           // TF32 hi / lo planes the MMAs read
constexpr int kMaxRing = 8;               // raw operand stages (K blocks) in the cp.async ring
constexpr int kSmemOptIn = 227 * 1024;    // sm_90: dynamic shared memory one CTA may opt into
constexpr int kSmemPerSM = 228 * 1024;
constexpr int kSmemPerCta = 1024;         // reserved by the system for every resident CTA
constexpr int kChainBlocks = 8;           // K blocks per tensor-core accumulation chain (CHAINS)

// optional phase stamps (b200rl_tc_debug_buffer): [block][8] nanosecond timers
__device__ long long* g_tc_dbg = nullptr;
__device__ __forceinline__ long long gtimer() {
  long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void stamp(int slot) {
  if (g_tc_dbg) {
    const int64_t blk = blockIdx.x + (int64_t)gridDim.x * (blockIdx.y + (int64_t)gridDim.y * blockIdx.z);
    if (blk < 64) g_tc_dbg[blk * 8 + slot] = gtimer();
  }
}

__device__ __forceinline__ uint32_t smem_addr(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}

// Shared-memory matrix descriptor (sm_90 GMMA): K-major, SWIZZLE_128B, 8-row groups 1024 B apart.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);          // start address
  d |= (uint64_t)1 << 16;                          // leading byte offset (unused for SW128 K-major)
  d |= (uint64_t)(1024 >> 4) << 32;                // stride byte offset
  d |= (uint64_t)1 << 62;                          // layout type 1 = SWIZZLE_128B
  return d;
}

// D[64 x N] = A[64 x 8] * B[8 x N] + (scale_d ? D : 0), both operands from shared memory
// (descriptors above).
template <int N>
__device__ __forceinline__ void wgmma_tf32(float (&d)[N / 2], uint64_t a, uint64_t b, int scale_d);
template <>
__device__ __forceinline__ void wgmma_tf32<32>(float (&d)[16], uint64_t a, uint64_t b, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(a), "l"(b), "r"(scale_d));
}
template <>
__device__ __forceinline__ void wgmma_tf32<64>(float (&d)[32], uint64_t a, uint64_t b, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a), "l"(b), "r"(scale_d));
}
template <>
__device__ __forceinline__ void wgmma_tf32<128>(float (&d)[64], uint64_t a, uint64_t b, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b), "r"(scale_d));
}
// The same MMA with A from registers: a[] is this thread's m64k8 fragment (fp32 bit patterns, see
// load_frag_*).
// The registers must not change until a wait_group retires the MMA.
template <int N>
__device__ __forceinline__ void wgmma_tf32_rs(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t b,
                                              int scale_d);
template <>
__device__ __forceinline__ void wgmma_tf32_rs<32>(float (&d)[16], const uint32_t (&a)[4], uint64_t b,
                                                  int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, {%16,%17,%18,%19}, %20, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(scale_d));
}
template <>
__device__ __forceinline__ void wgmma_tf32_rs<64>(float (&d)[32], const uint32_t (&a)[4], uint64_t b,
                                                  int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32,%33,%34,%35}, %36, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(scale_d));
}
template <>
__device__ __forceinline__ void wgmma_tf32_rs<128>(float (&d)[64], const uint32_t (&a)[4], uint64_t b,
                                                   int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, {%64,%65,%66,%67}, %68, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

// byte offset of the 16-byte chunk j (0..7) of row r inside a K-major [rows x 128 B] SWIZZLE_128B tile
__device__ __forceinline__ uint32_t sw128(uint32_t r, uint32_t j) {
  return (r >> 3) * 1024u + (r & 7u) * 128u + ((j ^ (r & 7u)) << 4);
}

__device__ __forceinline__ float tf32_hi(float x) {
  return __uint_as_float(__float_as_uint(x) & 0xFFFFE000u);
}

template <bool WITH_LO>
__device__ __forceinline__ void split_store(unsigned char* hi_tile, unsigned char* lo_tile,
                                            uint32_t off, float4 v) {
  float4 h;
  h.x = tf32_hi(v.x);
  h.y = tf32_hi(v.y);
  h.z = tf32_hi(v.z);
  h.w = tf32_hi(v.w);
  // explicit st.shared: the tile pointers come from integer alignment arithmetic, which makes
  // the compiler fall back to generic ST.E otherwise
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(smem_addr(hi_tile) + off),
               "f"(h.x), "f"(h.y), "f"(h.z), "f"(h.w)
               : "memory");
  if (WITH_LO) {
    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(smem_addr(lo_tile) + off),
                 "f"(v.x - h.x), "f"(v.y - h.y), "f"(v.z - h.z), "f"(v.w - h.w)
                 : "memory");
  }
}
template <bool WITH_LO>
__device__ __forceinline__ void split_store1(unsigned char* hi_tile, unsigned char* lo_tile,
                                             uint32_t off, float v) {
  const float h = tf32_hi(v);
  asm volatile("st.shared.f32 [%0], %1;" ::"r"(smem_addr(hi_tile) + off), "f"(h) : "memory");
  if (WITH_LO)
    asm volatile("st.shared.f32 [%0], %1;" ::"r"(smem_addr(lo_tile) + off), "f"(v - h) : "memory");
}

// K blocks of raw operand tiles that fit next to `fixed` bytes when `ctas` CTAs share an SM
constexpr int ring_depth(int fixed, int raw_stage, int ctas) {
  return (kSmemPerSM / ctas - kSmemPerCta - fixed) / raw_stage;
}
// `ctas` CTAs per SM fit when each keeps a ring >= 4 deep and the registers a thread holds across
// the K loop (accumulators, chain sums, A fragment sets: loop_regs) take at most half of its share
// of the 64 K register file; the other half goes to addresses, offsets and loop state (tighter
// bounds spill, see -Xptxas -v).
constexpr bool ctas_fit(int ctas, int fixed, int raw_stage, int loop_regs) {
  return ring_depth(fixed, raw_stage, ctas) >= 4 && 2 * loop_regs <= 65536 / (kThreads * ctas);
}

// A_EXACT: the A view yields values that are exactly representable in TF32 (raw uint8 pixels), so
// A needs no "lo" part and the product needs only 2 passes (a*b_lo + a*b_hi).  Such A operands go
// to the MMAs from registers, loaded straight from the raw ring slot, so they have no plane.
// Shared memory: [kPlaneStages x split planes][kRing x raw operand tiles][bias slice].  The ring is
// as deep as the opt-in limit allows (at most kMaxRing) when one CTA runs per SM; a layout that
// fits 3 or 2 CTAs per SM (ctas_fit) runs that many (kCtasPerSM, the kernel's launch bound), each
// with the ring of its share.
template <int BN, int PASSES, bool A_EXACT = false>
struct SmemLayout {
  static constexpr int kATile = kBM * 128;
  static constexpr int kBTile = BN * 128;
  static constexpr int kNumA = A_EXACT ? 0 : PASSES == 3 ? 2 : 1;   // A planes
  static constexpr int kNumB = PASSES == 3 ? 2 : 1;                 // B planes
  static constexpr int kStage = kNumA * kATile + kNumB * kBTile;
  static constexpr int kPlanes = kPlaneStages * kStage;
  // raw tiles sized for the larger (MN-contiguous, padded) layout; A_EXACT views are uint8
  static constexpr int kRawA = kBK * (kBM * (A_EXACT ? 1 : 4) + 16);
  static constexpr int kRawB = kBK * (BN * 4 + 16);
  static constexpr int kRawStage = kRawA + kRawB;
  static constexpr int kFixed = kPlanes + 1024 /*alignment slack*/ + BN * 4 /*bias*/;
  // accumulators + chain sums (BN / 2 each) + two A fragment sets of kBK / 8 K steps x 4
  static constexpr int kLoopRegs = BN + (A_EXACT ? 2 * (kBK / 8) * 4 : 0);
  static constexpr int kCtasPerSM = ctas_fit(3, kFixed, kRawStage, kLoopRegs)   ? 3
                                    : ctas_fit(2, kFixed, kRawStage, kLoopRegs) ? 2
                                                                                : 1;
  static constexpr int kRingFit = kCtasPerSM > 1 ? ring_depth(kFixed, kRawStage, kCtasPerSM)
                                                 : (kSmemOptIn - kFixed) / kRawStage;
  static constexpr int kRing = kRingFit < kMaxRing ? kRingFit : kMaxRing;
  static_assert(kRing >= 2, "the operand ring needs two stages");
  static constexpr int kPitch = BN + 4;                             // epilogue staging row (floats)
  static_assert(kBM * kPitch * 4 <= kPlanes + kRing * kRawStage, "epilogue staging tile must fit");
  static constexpr int kBytes = kFixed + kRing * kRawStage;
};

// ---- operand ring: global -> shared with cp.async, then split from shared memory -------------
// One chunk = 4 consecutive elements along the contiguous index of a view (k for K-contiguous
// views, m / n for MN-contiguous ones): 16 bytes of fp32 or 4 bytes of uint8.  When the view is
// vec4_ok() a chunk is one cp.async whose src-size covers only the in-range elements; the rest of
// the 16 / 4 bytes is zero-filled by the copy, so nothing past a K tail, a row end or an image is
// ever read.  Otherwise every element moves on its own (4-byte cp.async for fp32, a plain byte
// load and store for uint8, which cp.async cannot copy).
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
template <int BYTES>
__device__ __forceinline__ void cp_async(uint32_t dst, const void* src, uint32_t src_bytes) {
  if constexpr (BYTES == 16)
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes)
                 : "memory");
  else
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst), "l"(src), "r"(src_bytes)
                 : "memory");
}
// n of the chunk's 4 elements (0..4) are in range and contiguous from `off`
template <class V>
__device__ __forceinline__ void copy_chunk(const V& v, uint32_t dst, int64_t off, int n) {
  constexpr int E = sizeof(typename V::Elem);
  cp_async<4 * E>(dst, v.addr(n > 0 ? off : 0), (uint32_t)(n * E));
}
template <class V>
__device__ __forceinline__ void copy_elem(const V& v, uint32_t dst, int64_t off, bool ok) {
  if constexpr (sizeof(typename V::Elem) == 4) {
    cp_async<4>(dst, v.addr(ok ? off : 0), ok ? 4u : 0u);
  } else {
    const uint32_t x = ok ? *static_cast<const uint8_t*>(v.addr(off)) : 0u;
    asm volatile("st.shared.u8 [%0], %1;" ::"r"(dst), "r"(x) : "memory");
  }
}
// 4 raw elements of a chunk in shared memory -> fp32 (uint8 views convert here)
template <class V>
__device__ __forceinline__ float4 ld_raw4(const V& v, uint32_t saddr) {
  if constexpr (sizeof(typename V::Elem) == 4) {
    float4 x;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(x.x), "=f"(x.y), "=f"(x.z), "=f"(x.w) : "r"(saddr) : "memory");
    return x;
  } else {
    uint32_t w;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(w) : "r"(saddr) : "memory");
    return make_float4(v.cvt((uint8_t)w), v.cvt((uint8_t)(w >> 8)), v.cvt((uint8_t)(w >> 16)),
                       v.cvt((uint8_t)(w >> 24)));
  }
}

// Raw tile of a (ROWS x 32) operand block.  K-contiguous views: chunk j of row r sits where the
// split planes keep it (sw128 for fp32, 32-byte rows for uint8), so the split pass reads and writes
// the same conflict-free pattern.  MN-contiguous views: 32 k-rows of ROWS elements, 16 bytes of
// padding per k-row so that the 8 k-rows a quarter-warp reads in the transposing split fall into
// different banks.
template <class V, int ROWS>
struct RawTile {
  static constexpr int E = sizeof(typename V::Elem);
  static constexpr int kPitch = ROWS * E + 16;   // MN-contiguous k-row
  __device__ static __forceinline__ uint32_t k_chunk(uint32_t r, uint32_t j) {
    return E == 4 ? sw128(r, j) : r * 32u + j * 4u;
  }
};

// K-contiguous views: thread = (row group tid>>3, chunk tid&7), 8 lanes copy one row's 32 k;
// row_offs[i] belongs to row (tid>>3) + 32 i (hoisted once per CTA).
template <int ROWS, class V>
__device__ __forceinline__ void copy_tile_k(const V& v, uint32_t dst, const int64_t* row_offs,
                                            uint32_t row_ok_mask, int64_t k0, int64_t ke,
                                            bool vec, int tid) {
  using R = RawTile<V, ROWS>;
  constexpr int NV = ROWS * 8 / kThreads;
  const int j = tid & 7;
  const int64_t k = k0 + j * 4;
  const int nk = k < ke ? (ke - k < 4 ? (int)(ke - k) : 4) : 0;
  if (vec) {
    const int64_t ko = nk > 0 ? v.k_off(k) : 0;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const uint32_t r = (uint32_t)((tid >> 3) + 32 * i);
      copy_chunk(v, dst + R::k_chunk(r, j), row_offs[i] + ko, ((row_ok_mask >> i) & 1u) ? nk : 0);
    }
  } else {
    int64_t ko[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) ko[e] = e < nk ? v.k_off(k + e) : 0;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const uint32_t r = (uint32_t)((tid >> 3) + 32 * i);
      const bool ok = (row_ok_mask >> i) & 1u;
#pragma unroll
      for (int e = 0; e < 4; ++e)
        copy_elem(v, dst + R::k_chunk(r, j) + e * R::E, row_offs[i] + ko[e], ok && e < nk);
    }
  }
}

// MN-contiguous views: chunk c = tid + 256 i is rows 4 (c % CPR) .. +3 at k = c / CPR, so a warp
// copies whole 4*CPR-element runs of a k-row and a thread keeps one row group (roff = the view's
// row offset of that group's first row, nrow = how many of its 4 rows are in range).
template <int ROWS, class V>
__device__ __forceinline__ void copy_tile_mn(const V& v, uint32_t dst, int64_t r, int64_t roff,
                                             int nrow, int64_t k0, int64_t ke, bool vec, int tid) {
  using R = RawTile<V, ROWS>;
  constexpr int CPR = ROWS / 4, NV = ROWS * 8 / kThreads;
  static_assert(kThreads % CPR == 0, "a thread's row group must not change between its chunks");
  const uint32_t cm = (uint32_t)(tid % CPR);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int kk = (tid + kThreads * i) / CPR;
    const int64_t k = k0 + kk;
    const bool kok = k < ke;
    const uint32_t d = dst + (uint32_t)kk * R::kPitch + cm * 4u * R::E;
    if (vec) {
      copy_chunk(v, d, roff + (kok ? v.k_off(k) : 0), kok ? nrow : 0);
    } else {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const bool ok = kok && e < nrow;
        copy_elem(v, d + e * R::E, ok ? v.row_off(r + e) + v.k_off(k) : 0, ok);
      }
    }
  }
}

// Split pass of K-contiguous tiles: raw chunk (r, j) -> TF32 hi / lo at sw128(r, j).
template <int ROWS, bool WITH_LO, class V>
__device__ __forceinline__ void split_tile_k(const V& v, uint32_t raw, unsigned char* hi,
                                             unsigned char* lo, int tid) {
  using R = RawTile<V, ROWS>;
  constexpr int NV = ROWS * 8 / kThreads;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const uint32_t r = (uint32_t)((tid >> 3) + 32 * i), j = (uint32_t)(tid & 7);
    split_store<WITH_LO>(hi, lo, sw128(r, j), ld_raw4(v, raw + R::k_chunk(r, j)));
  }
}

// Split pass of MN-contiguous tiles, transposed to K-major on the way: chunk c = tid + 256 i holds
// rows 4 cm .. 4 cm + 3 at reduction index k, with k & 7 = c & 7, cm = (c >> 3) % CPR and
// k >> 3 = (c >> 3) / CPR.  The transposing scalar stores of a warp then spread over 16 banks
// (2-way conflicts instead of 16-way for a row-per-lane map).  cm does not depend on i, so every
// chunk of a thread covers the same 4 columns: `colsum` accumulates their sums (fused bias
// gradient).
template <int ROWS>
struct MnMap {
  static constexpr int CPR = ROWS / 4;
  __device__ static __forceinline__ int cm(int c) { return (c >> 3) % CPR; }
  __device__ static __forceinline__ int kk(int c) { return (c & 7) | (((c >> 3) / CPR) << 3); }
};
// Register A fragments of raw uint8 tiles.  Fragment of K step ks (wgmma m64k8, tf32): a[0] / a[1]
// = rows R / R + 8 at column t, a[2] / a[3] = the same rows at column t + 4, with R = 64 wg +
// 16 (warp % 4) + lane / 4 and t = lane % 4.  Values 0..255 are exact in fp32 and TF32:
// byte | 0x4B000000 is the float 2^23 + byte.
__device__ __forceinline__ uint32_t u8_to_f32(uint32_t w, int byte) {
  return __float_as_uint(__uint_as_float(__byte_perm(w, 0x4B000000u, 0x7540u + (uint32_t)byte)) - 8388608.f);
}
// K-contiguous tiles (32-byte rows): four 4-byte loads per block.  That needs the reduction index
// inside a K block reordered: raw byte p of a row is column kperm(p) of the block's MMAs, so that
// byte b of word t + 4 h of a row (h < 2) is K step 2 h + b / 2, column t + 4 (b % 2), and every
// byte of the two words a thread loads per row is one of its fragment values.  The split of B
// (split_tile_mn<..., true>) stores B in the same order; the permutation keeps its stores at
// 2-way bank conflicts, and the words a warp loads are 2-way as well.
__device__ __forceinline__ uint32_t kperm(uint32_t p) {
  return ((p >> 4) << 4) | (((p >> 1) & 1u) << 3) | ((p & 1u) << 2) | ((p >> 2) & 3u);
}
__device__ __forceinline__ void load_frag_k(uint32_t raw, uint32_t (&a)[kBK / 8][4], int wg, int warp,
                                            int lane) {
  const uint32_t r = (uint32_t)(wg * 64 + (warp & 3) * 16 + (lane >> 2)), t = (uint32_t)(lane & 3);
  uint32_t w[2][2];   // [word t / t + 4][row R / R + 8]
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int rr = 0; rr < 2; ++rr)
      asm volatile("ld.shared.u32 %0, [%1];"
                   : "=r"(w[h][rr]) : "r"(raw + (r + 8u * rr) * 32u + (t + 4u * h) * 4u) : "memory");
#pragma unroll
  for (int ks = 0; ks < kBK / 8; ++ks) {
    const int h = ks >> 1, b = 2 * (ks & 1);
    a[ks][0] = u8_to_f32(w[h][0], b);
    a[ks][1] = u8_to_f32(w[h][1], b);
    a[ks][2] = u8_to_f32(w[h][0], b + 1);
    a[ks][3] = u8_to_f32(w[h][1], b + 1);
  }
}
// MN-contiguous tiles ([32 k][ROWS + 16] bytes): one byte load per element, natural K order (the
// 4 t lanes of a load hit k-rows 144 bytes = 4 banks apart, so a load is conflict-free).
template <int ROWS>
__device__ __forceinline__ void load_frag_mn(uint32_t raw, uint32_t (&a)[kBK / 8][4], int wg, int warp,
                                             int lane) {
  constexpr uint32_t kPitch = ROWS + 16;
  const uint32_t r = (uint32_t)(wg * 64 + (warp & 3) * 16 + (lane >> 2)), t = (uint32_t)(lane & 3);
#pragma unroll
  for (int ks = 0; ks < kBK / 8; ++ks) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const uint32_t k = 8u * ks + t + 4u * (i >> 1), m = r + 8u * (i & 1);
      uint32_t x;
      asm volatile("ld.shared.u8 %0, [%1];" : "=r"(x) : "r"(raw + k * kPitch + m) : "memory");
      a[ks][i] = __float_as_uint(__uint_as_float(x | 0x4B000000u) - 8388608.f);
    }
  }
}

// KPERM: store column k at kperm(k) (B of a K-contiguous register A operand, see load_frag_k).
template <int ROWS, bool WITH_LO, class V, bool KPERM = false>
__device__ __forceinline__ void split_tile_mn(const V& v, uint32_t raw, unsigned char* hi,
                                              unsigned char* lo, int tid, bool do_colsum,
                                              float4& colsum) {
  using R = RawTile<V, ROWS>;
  constexpr int NV = ROWS * 8 / kThreads;
  const uint32_t r = 4u * (uint32_t)MnMap<ROWS>::cm(tid);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const uint32_t k = (uint32_t)MnMap<ROWS>::kk(tid + kThreads * i);
    const float4 x = ld_raw4(v, raw + k * R::kPitch + r * R::E);
    if (do_colsum) {
      colsum.x += x.x; colsum.y += x.y; colsum.z += x.z; colsum.w += x.w;
    }
    const uint32_t kc = KPERM ? kperm(k) : k;
    const uint32_t j = kc >> 2, e = (kc & 3u) * 4u;
    split_store1<WITH_LO>(hi, lo, sw128(r + 0, j) + e, x.x);
    split_store1<WITH_LO>(hi, lo, sw128(r + 1, j) + e, x.y);
    split_store1<WITH_LO>(hi, lo, sw128(r + 2, j) + e, x.z);
    split_store1<WITH_LO>(hi, lo, sw128(r + 3, j) + e, x.w);
  }
}

// Epilogue variants.  EPI_STORE: C (+)= act(acc + bias) or split-K partial.  EPI_COL2IM: the
// GEMM is dcol[pos, (ky,kx,c)] = dY @ W^T of a convolution input gradient and every 4-channel
// group is scatter-added straight into dX[n, oy*s+ky, ox*s+kx, c..c+3] with one
// red.global.add.v4.f32 (four scalar atomics when dX is not 16-byte aligned) — the
// [M, KH*KW*C] dcol matrix is never materialised and split-K partials need no reduction pass
// (dX must be zeroed by the caller; summation order of the <= KH*KW/s^2 contributions per
// element is not fixed).
constexpr int EPI_STORE = 0;
constexpr int EPI_COL2IM = 1;
constexpr int EPI_ATOMIC = 2;  // C += acc with red.global.add (split-K without a reduce pass; C pre-zeroed)
struct EpiArgs {
  ConvGeom g;
  float* dx;
  ActMask mask;     // EPI_STORE / EPI_COL2IM: multiply the input gradient by act'(mask.y)
  float* colsum;    // EPI_ATOMIC with an MN-major B view: column sums of B (bias gradient) += here
};

// AL / BL are the fp32 operand views of nn.cu (row index = m for A, n for B).
// CHAINS: the K range of a CTA is long (> kChainBlocks blocks), see `sum` below.
template <int BN, int PASSES, int EPI, class AL, class BL, bool CHAINS>
__global__ void __launch_bounds__(kThreads, SmemLayout<BN, PASSES, AL::kExact>::kCtasPerSM)
tc_gemm_kernel(const AL a, const BL b, const EpiArgs epi, float* __restrict__ C,
               const float* __restrict__ bias, int64_t M, int64_t N, int64_t K, int act, int beta,
               int splits, int64_t k_per_split, float* __restrict__ ws, float out_scale) {
  using L = SmemLayout<BN, PASSES, AL::kExact>;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = reinterpret_cast<unsigned char*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  float* sbias = reinterpret_cast<float*>(smem + L::kPlanes + L::kRing * L::kRawStage);   // bias / column sums

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = tid >> 7;                                  // warpgroup: tile rows 64 wg ..
  const int64_t m0 = (int64_t)blockIdx.y * kBM, n0 = (int64_t)blockIdx.x * BN;
  const int split = blockIdx.z;
  const int64_t kb = (int64_t)split * k_per_split;
  const int64_t ke = (kb + k_per_split < K) ? kb + k_per_split : K;
  const int nkb = (int)((ke - kb + kBK - 1) / kBK);

  pdl_launch_dependents();   // the next kernel of the stream may be scheduled from here on
  if (tid == 0) stamp(0);
  if (EPI == EPI_ATOMIC && tid < BN) sbias[tid] = 0.f;
  // everything above touched no global memory; from here on the producing kernels must be done
  pdl_wait();
  if (tid == 0) stamp(1);

  constexpr bool kLo = PASSES == 3;
  constexpr bool kLoA = PASSES == 3 && !AL::kExact;
  constexpr int NRA = AL::kKContig ? kBM * 8 / kThreads : 1;
  constexpr int NRB = BL::kKContig ? BN * 8 / kThreads : 1;
  static_assert(BN * 8 >= kThreads, "BN must be >= 32");
  // hoisted row offsets (the implicit-im2col index math runs once per CTA).  K-contiguous views:
  // row (tid>>3) + 32 i; MN-contiguous views: the 4-row group of copy_tile_mn.
  int64_t a_off[NRA], b_off[NRB];
  uint32_t a_ok = 0, b_ok = 0;
  int64_t a_r = 0, b_r = 0;
  int a_nrow = 0, b_nrow = 0;
  if constexpr (AL::kKContig) {
#pragma unroll
    for (int i = 0; i < NRA; ++i) {
      const int r = (tid >> 3) + 32 * i;
      const bool ok = m0 + r < M;
      a_off[i] = ok ? a.row_off(m0 + r) : 0;
      a_ok |= (ok ? 1u : 0u) << i;
    }
  } else {
    a_r = m0 + 4 * (tid % (kBM / 4));
    a_nrow = M - a_r < 0 ? 0 : (M - a_r < 4 ? (int)(M - a_r) : 4);
    a_off[0] = a_nrow > 0 ? a.row_off(a_r) : 0;
  }
  if constexpr (BL::kKContig) {
#pragma unroll
    for (int i = 0; i < NRB; ++i) {
      const int r = (tid >> 3) + 32 * i;
      const bool ok = n0 + r < N;
      b_off[i] = ok ? b.row_off(n0 + r) : 0;
      b_ok |= (ok ? 1u : 0u) << i;
    }
  } else {
    b_r = n0 + 4 * (tid % (BN / 4));
    b_nrow = N - b_r < 0 ? 0 : (N - b_r < 4 ? (int)(N - b_r) : 4);
    b_off[0] = b_nrow > 0 ? b.row_off(b_r) : 0;
  }
  const bool a_vec = a.vec4_ok(), b_vec = b.vec4_ok();
  const uint32_t smem_base = smem_addr(smem);
  const uint32_t ring_base = smem_base + L::kPlanes;
  // Copies K block `blk` into its ring slot; commits a (possibly empty) group either way, so that
  // the group count stays in step with the block index.
  auto issue = [&](int blk) {
    if (blk < nkb) {
      const uint32_t slot = ring_base + (uint32_t)(blk % L::kRing) * L::kRawStage;
      const int64_t k0 = kb + (int64_t)blk * kBK;
      if constexpr (AL::kKContig) copy_tile_k<kBM>(a, slot, a_off, a_ok, k0, ke, a_vec, tid);
      else copy_tile_mn<kBM>(a, slot, a_r, a_off[0], a_nrow, k0, ke, a_vec, tid);
      if constexpr (BL::kKContig) copy_tile_k<BN>(b, slot + L::kRawA, b_off, b_ok, k0, ke, b_vec, tid);
      else copy_tile_mn<BN>(b, slot + L::kRawA, b_r, b_off[0], b_nrow, k0, ke, b_vec, tid);
    }
    cp_async_commit();
  };
  // bias gradient fused into the weight-gradient GEMM: B = dY[k, n] passes through these threads
  // in the split; in the MN-major map every chunk of a thread covers the same 4 columns, so one
  // float4 per thread accumulates the column sums of the CTA's K range.
  const bool do_colsum = EPI == EPI_ATOMIC && !BL::kKContig && epi.colsum != nullptr &&
                         blockIdx.y == 0;
  float4 bsum = make_float4(0.f, 0.f, 0.f, 0.f);
  // The wgmma accumulator does not round to nearest: every accumulate loses ~2^-24 of the running
  // sum, always toward zero, so on same-sign data one chain over K = 3136 drifts by ~7e-5 (512:
  // 1.2e-5, 256: 6.6e-6).  With CHAINS, each chain covers kChainBlocks K blocks only and is then
  // added into `sum` with an ordinary (round-to-nearest) fp32 add; the next chain restarts the
  // accumulator (scale-d = 0).  `sum` costs BN/2 registers, which slows the BN=128 kernels by ~12 %
  // even when no chain ends, so the host selects CHAINS only for K ranges longer than one chain.
  float acc[BN / 2], sum[CHAINS ? BN / 2 : 1];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
#pragma unroll
  for (int i = 0; i < (CHAINS ? BN / 2 : 1); ++i) sum[i] = 0.f;
  // the ring's first kRing - 1 blocks are in flight before the loop starts
#pragma unroll 1
  for (int blk = 0; blk < L::kRing - 1; ++blk) issue(blk);
  if constexpr (AL::kExact) {
    // A from registers: each thread loads its fragments of block kbi from the raw ring slot into
    // set kbi % 2 while block kbi - 1's MMAs (set (kbi - 1) % 2) may still run; the wait_group 1
    // of block kbi - 1 retired block kbi - 2, the last reader of set kbi % 2.  Blocks go in pairs
    // so that the set (and the plane stage) is a compile-time index.
    static_assert(!BL::kKContig, "register A operands pair with an MN-contiguous B view");
    constexpr bool kPerm = AL::kKContig;
    uint32_t af[2][kBK / 8][4];
#pragma unroll 1
    for (int kb2 = 0; kb2 < nkb; kb2 += 2) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int kbi = kb2 + h;
        if (kbi >= nkb) break;
        cp_async_wait<L::kRing - 2>();
        __syncthreads();
        issue(kbi + L::kRing - 1);
        const uint32_t raw = ring_base + (uint32_t)(kbi % L::kRing) * L::kRawStage;
        if constexpr (AL::kKContig) load_frag_k(raw, af[h], wg, warp, lane);
        else load_frag_mn<kBM>(raw, af[h], wg, warp, lane);
        unsigned char* b_hi = smem + h * L::kStage;
        split_tile_mn<BN, kLo, BL, kPerm>(b, raw + L::kRawA, b_hi, b_hi + L::kBTile, tid, do_colsum,
                                          bsum);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();
        const uint32_t sb = smem_base + (uint32_t)h * L::kStage;
        const bool fresh = CHAINS && kbi % kChainBlocks == 0;
        if constexpr (CHAINS) {
          if (fresh && kbi > 0) {
            wgmma_wait<0>();
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) sum[i] += acc[i];
          }
        }
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < kBK / 8; ++ks) {
          const uint32_t ko = (uint32_t)ks * 32u;
          const int keep = (fresh && ks == 0) ? 0 : 1;
          if (PASSES == 3) {
            wgmma_tf32_rs<BN>(acc, af[h][ks], make_desc(sb + L::kBTile + ko), keep);
            wgmma_tf32_rs<BN>(acc, af[h][ks], make_desc(sb + ko), 1);
          } else {
            wgmma_tf32_rs<BN>(acc, af[h][ks], make_desc(sb + ko), keep);
          }
        }
        wgmma_commit();
        wgmma_wait<1>();
      }
    }
  } else {
#pragma unroll 1
    for (int kbi = 0; kbi < nkb; ++kbi) {
      // this thread's copies of block kbi have landed; the barrier makes everyone's visible, and it
      // frees the ring slot of block kbi - 1 (split before the last barrier) and plane stage
      // kbi % 2 (its MMAs, block kbi - 2, retired in every warpgroup's wait_group 1 below)
      cp_async_wait<L::kRing - 2>();
      __syncthreads();
      issue(kbi + L::kRing - 1);
      const int s = kbi % kPlaneStages;
      const uint32_t raw = ring_base + (uint32_t)(kbi % L::kRing) * L::kRawStage;
      unsigned char* st = smem + s * L::kStage;
      unsigned char* a_hi = st;
      unsigned char* a_lo = st + L::kATile;
      unsigned char* b_hi = st + L::kNumA * L::kATile;
      unsigned char* b_lo = b_hi + L::kBTile;
      if constexpr (AL::kKContig) split_tile_k<kBM, kLoA>(a, raw, a_hi, a_lo, tid);
      else split_tile_mn<kBM, kLoA>(a, raw, a_hi, a_lo, tid, false, bsum);
      if constexpr (BL::kKContig) split_tile_k<BN, kLo>(b, raw + L::kRawA, b_hi, b_lo, tid);
      else split_tile_mn<BN, kLo>(b, raw + L::kRawA, b_hi, b_lo, tid, do_colsum, bsum);
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic stores -> async proxy
      __syncthreads();
      const uint32_t sa = smem_base + (uint32_t)s * L::kStage + (uint32_t)wg * (64u * 128u);
      const uint32_t sb = smem_base + (uint32_t)s * L::kStage + L::kNumA * L::kATile;
      const uint32_t a_lo_off = L::kATile, b_lo_off = L::kBTile;
      const bool fresh = CHAINS && kbi % kChainBlocks == 0;   // first block of a chain
      if constexpr (CHAINS) {
        if (fresh && kbi > 0) {
          // the previous block's MMAs ran during this block's split; usually retired
          wgmma_wait<0>();
#pragma unroll
          for (int i = 0; i < BN / 2; ++i) sum[i] += acc[i];
        }
      }
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < kBK / 8; ++ks) {
        const uint32_t ko = (uint32_t)ks * 32u;   // 8 tf32 = 32 bytes further inside the 128 B row
        const int keep = (fresh && ks == 0) ? 0 : 1;   // scale-d of the block's first MMA
        if (PASSES == 3) {
          wgmma_tf32<BN>(acc, make_desc(sa + a_lo_off + ko), make_desc(sb + ko), keep);
          wgmma_tf32<BN>(acc, make_desc(sa + ko), make_desc(sb + b_lo_off + ko), 1);
          wgmma_tf32<BN>(acc, make_desc(sa + ko), make_desc(sb + ko), 1);
        } else {
          wgmma_tf32<BN>(acc, make_desc(sa + ko), make_desc(sb + ko), keep);
        }
      }
      wgmma_commit();
      wgmma_wait<1>();
    }
  }
  wgmma_wait<0>();
  if constexpr (CHAINS) {
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] += sum[i];   // the last chain (all zero when nkb == 0)
  }
  if (tid == 0) stamp(2);
  __syncthreads();   // every MMA of the CTA has retired: the stage buffers hold the staging tile now

  // ===================== epilogue =====================
  constexpr int P = L::kPitch;
  float* stg = reinterpret_cast<float*>(smem);
  {
    // wgmma m64nNk8 accumulator: register 4i + 2h + e of lane l in warp w (of the warpgroup) is
    // row 16 w + l / 4 + 8 h, column 8 i + 2 (l % 4) + e
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
      *reinterpret_cast<float2*>(stg + r0 * P + 8 * i + c0) = make_float2(acc[4 * i], acc[4 * i + 1]);
      *reinterpret_cast<float2*>(stg + (r0 + 8) * P + 8 * i + c0) =
          make_float2(acc[4 * i + 2], acc[4 * i + 3]);
    }
  }
  if (do_colsum) {
    // thread tid holds columns 4 cm .. 4 cm + 3 (MnMap); the k-lanes of a column are combined
    // with shared-memory atomics, one red per column goes to global memory
    const int c4 = MnMap<BN>::cm(tid) * 4;
    atomicAdd(&sbias[c4 + 0], bsum.x);
    atomicAdd(&sbias[c4 + 1], bsum.y);
    atomicAdd(&sbias[c4 + 2], bsum.z);
    atomicAdd(&sbias[c4 + 3], bsum.w);
  }
  // bias slice of this tile -> shared memory
  if (EPI == EPI_STORE && tid < BN) sbias[tid] = (bias != nullptr && n0 + tid < N) ? bias[n0 + tid] : 0.f;
  __syncthreads();
  if (do_colsum && tid < BN && n0 + tid < N) atomicAdd(epi.colsum + n0 + tid, sbias[tid]);
  if (tid == 0) stamp(4);
  const int q = warp & 3, half = warp >> 2;   // row quadrant / column half of this warp
  const int row = q * 32 + lane;
  const int64_t m = m0 + row;
  float* out = (splits > 1) ? ws + (int64_t)split * M * N : C;
  const bool vec_out = (N & 3) == 0 && ((uintptr_t)out & 15) == 0;
  constexpr int G = 16;  // columns handled per step
#pragma unroll
  for (int cc = 0; cc < BN / 2; cc += G) {
    const int c = half * (BN / 2) + cc;
    float r[G];
#pragma unroll
    for (int j = 0; j < G; j += 4) {
      const float4 t = *reinterpret_cast<const float4*>(stg + row * P + c + j);
      r[j] = t.x; r[j + 1] = t.y; r[j + 2] = t.z; r[j + 3] = t.w;
    }
    if (m >= M && !(EPI == EPI_STORE && vec_out)) continue;
    const int64_t nb = n0 + c;
    if (EPI == EPI_COL2IM) {
      if (nkb == 0) continue;
      // pos -> (n, oy, ox); patch index -> (ky, kx*C + c)
      uint32_t img, rem, oy, ox;
      epi.g.d_ohow.divmod((uint32_t)m, img, rem);
      epi.g.d_ow.divmod(rem, oy, ox);
      const int64_t wc = (int64_t)epi.g.W * epi.g.C;
      const int64_t in_off = (int64_t)oy * epi.g.stride * wc + (int64_t)ox * epi.g.stride * epi.g.C;
      float* base = epi.dx + (int64_t)img * epi.g.H * wc + in_off;
      // act'(X) of the layer that produced the conv input: the scatter-add is linear, so every
      // contribution is masked on its way out (X is read at the destination index)
      const float* ybase = epi.mask.y ? epi.mask.y + (int64_t)img * epi.mask.ld + in_off : nullptr;
      // C % 4 == 0 keeps every 4-channel group 16-byte aligned relative to dX / X; the base
      // pointers (and the X image stride) are the caller's and need not be
      const bool dx_vec = ((uintptr_t)epi.dx & 15) == 0;
      const bool y_vec = ((uintptr_t)epi.mask.y & 15) == 0 && (epi.mask.ld & 3) == 0;
#pragma unroll
      for (int j = 0; j < G; j += 4) {
        const int64_t kidx = nb + j;
        if (kidx >= N) break;
        uint32_t ky, rr;
        epi.g.d_kwc.divmod((uint32_t)kidx, ky, rr);
        float* dst = base + (int64_t)ky * wc + rr;
        float4 v = make_float4(r[j], r[j + 1], r[j + 2], r[j + 3]);
        if (ybase) {
          const float* yp = ybase + (int64_t)ky * wc + rr;
          const float4 y = y_vec ? *reinterpret_cast<const float4*>(yp)
                                 : make_float4(yp[0], yp[1], yp[2], yp[3]);
          v.x = dact(y.x, v.x, epi.mask.act); v.y = dact(y.y, v.y, epi.mask.act);
          v.z = dact(y.z, v.z, epi.mask.act); v.w = dact(y.w, v.w, epi.mask.act);
        }
        if (dx_vec) {
          asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "f"(v.x),
                       "f"(v.y), "f"(v.z), "f"(v.w)
                       : "memory");
        } else {
          atomicAdd(dst + 0, v.x); atomicAdd(dst + 1, v.y);
          atomicAdd(dst + 2, v.z); atomicAdd(dst + 3, v.w);
        }
      }
      continue;
    }
    if (EPI == EPI_ATOMIC) {
      if (nkb == 0) continue;
      float* dst = C + m * N + nb;
      if ((N & 3) == 0 && ((uintptr_t)C & 15) == 0 && nb + G - 1 < N) {
#pragma unroll
        for (int j = 0; j < G; j += 4)
          asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst + j),
                       "f"(r[j] * out_scale), "f"(r[j + 1] * out_scale),
                       "f"(r[j + 2] * out_scale), "f"(r[j + 3] * out_scale)
                       : "memory");
      } else {
#pragma unroll
        for (int j = 0; j < G; ++j)
          if (nb + j < N) atomicAdd(dst + j, r[j] * out_scale);
      }
      continue;
    }
    float v[G];
#pragma unroll
    for (int j = 0; j < G; ++j) {
      float x = nkb > 0 ? r[j] * out_scale : 0.f;
      if (splits == 1 && nb + j < N && m < M) {
        x += sbias[c + j];
        x = apply_act(x, act);
        if (!vec_out && epi.mask.y) x = dact(epi.mask.y[m * epi.mask.ld + nb + j], x, epi.mask.act);
        if (beta) x += out[m * N + nb + j];
      }
      v[j] = x;
    }
    if (vec_out) {
      // back into the staging row (this thread's own cells) so that global rows are written by
      // adjacent lanes below; row pitch BN+4 floats keeps the 16-byte accesses conflict-free
      float* srow = stg + row * P + c;
#pragma unroll
      for (int j = 0; j < G; j += 4)
        *reinterpret_cast<float4*>(srow + j) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
    } else {
#pragma unroll
      for (int j = 0; j < G; ++j)
        if (nb + j < N) out[m * N + nb + j] = v[j];
    }
  }
  if (EPI == EPI_STORE && vec_out) {
    __syncthreads();
    constexpr int LPR = BN / 4;                        // lanes per tile row
    constexpr int RPI = 32 / LPR;                      // rows per store instruction
    const int col = (lane % LPR) * 4;
#pragma unroll 4
    for (int rr = 0; rr < 16; rr += RPI) {
      const int srow = warp * 16 + rr + lane / LPR;
      const int64_t gm = m0 + srow;
      if (gm < M && n0 + col < N) {
        float4 t = *reinterpret_cast<const float4*>(stg + srow * P + col);
        if (splits == 1 && epi.mask.y) {   // coalesced read of the producing layer's output
          const float* yp = epi.mask.y + gm * epi.mask.ld + n0 + col;
          const bool yv = (epi.mask.ld & 3) == 0 && ((uintptr_t)epi.mask.y & 15) == 0;
          const float4 y = yv ? *reinterpret_cast<const float4*>(yp)
                              : make_float4(yp[0], yp[1], yp[2], yp[3]);
          t.x = dact(y.x, t.x, epi.mask.act); t.y = dact(y.y, t.y, epi.mask.act);
          t.z = dact(y.z, t.z, epi.mask.act); t.w = dact(y.w, t.w, epi.mask.act);
        }
        *reinterpret_cast<float4*>(out + gm * N + n0 + col) = t;
      }
    }
  }
  if (tid == 0) stamp(5);
}

}  // namespace tc
}  // namespace b200rl
