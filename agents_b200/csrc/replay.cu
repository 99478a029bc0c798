// Ring-buffer trajectory write, Philox uniform index draw and segment gather (kernel family ii).
//
// Replaces the TF ops issued by replay_buffers/tf_uniform_replay_buffer.py:182-310,533-579 and
// replay_buffers/table.py:86-137 of the reference: one scatter_update / sparse_read op per
// leaf plus two RandomUniformInt ops become ONE launch that (a) computes the row ids on the
// fly (Philox4x32-10 or externally supplied draws), (b) copies every leaf of every selected
// row with 16-byte streaming loads/stores, (c) maintains the device-resident counters
// (last_id / RNG call index) with a last-block-done ticket so the launch is CUDA-graph safe.
//
// HBM-bound byte movement: algorithmic bytes = 2 * rows * row_bytes (read ring + write batch).
#include <stdlib.h>

#include "common.cuh"

namespace b200rl {

constexpr int kThreads = 256;
constexpr int kUnroll = 4;                 // independent 16 B requests in flight per thread
constexpr int kSmallMax = 512;             // leaves up to this many bytes/row ride along piece 0
constexpr int64_t kPieceTarget = kThreads * kUnroll * 16;  // 16 KiB per CTA

enum Mode : int {
  MODE_SAMPLE = 0,      // ring -> batch, rows from (ids, offs) draws      (_get_next)
  MODE_ROWS = 1,        // ring -> batch, explicit rows                      (Table.read)
  MODE_GATHER_ALL = 2,  // ring -> [B_env, n_valid], age order               (_gather_all)
  MODE_ADD = 3,         // items -> ring at id = last_id+1                   (_add_batch)
  MODE_WRITE_ROWS = 4   // items -> ring, explicit rows                      (Table.write)
};

struct PlanLeaf {
  const char* src;
  char* dst;
  int64_t row_bytes;
  int32_t n_pieces;     // big leaves only
  int32_t piece_bytes;  // multiple of 16 (big) ; unused (small)
  int32_t vec;          // 16 / 8 / 4 / 2 / 1: widest aligned access that divides row_bytes
  int32_t _pad;
};

struct Plan {
  int32_t n_big, n_small, pieces_per_row, rows_per_cta;
  int64_t n_rows;  // number of (dst) rows in this launch
  // ring geometry / counters
  int64_t B_env, L, B, T, n_valid;
  int64_t* id_table;
  int64_t* last_id;
  uint32_t* ticket;
  // sample
  const int64_t* ids;
  const int64_t* offs;
  const int64_t* rows;
  uint64_t seed;
  uint64_t* rng_call;
  int64_t* out_ids;
  int64_t* out_rows;
  int64_t* out_draw_ids;   // b200rl_rb_draw only
  int64_t* out_draw_offs;  // b200rl_rb_draw only
  float* out_prob;
  int32_t* status;
  PlanLeaf big[B200RL_MAX_LEAVES];
  PlanLeaf small[B200RL_MAX_LEAVES];
};

__device__ __forceinline__ void valid_range(int64_t last, int64_t L, int64_t T, int64_t& lo,
                                            int64_t& hi) {
  // _valid_range_ids, tf_uniform_replay_buffer.py:610-635
  if (last < L) {
    lo = 0;
    int64_t m = last + 1 - T + 1;
    hi = m > 0 ? m : 0;
  } else {
    lo = last + 1 - L;
    hi = last + 1 - T + 1;
  }
}

// Copy `len` bytes (len % vec == 0, src/dst aligned to vec) cooperatively by `nthr` threads.
__device__ __forceinline__ void copy_span(const char* __restrict__ src, char* __restrict__ dst,
                                          int64_t len, int vec, int tid, int nthr) {
  if (vec == 16) {
    const int64_t n = len >> 4;
    for (int64_t i = tid; i < n; i += (int64_t)nthr * kUnroll) {
      int4 v[kUnroll];
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        int64_t j = i + (int64_t)u * nthr;
        if (j < n) v[u] = ld_stream16(src + (j << 4));
      }
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        int64_t j = i + (int64_t)u * nthr;
        if (j < n) st_stream16(dst + (j << 4), v[u]);
      }
    }
  } else if (vec == 8) {
    const int64_t n = len >> 3;
    for (int64_t i = tid; i < n; i += nthr)
      reinterpret_cast<int2*>(dst)[i] = __ldg(reinterpret_cast<const int2*>(src) + i);
  } else if (vec == 4) {
    const int64_t n = len >> 2;
    for (int64_t i = tid; i < n; i += nthr)
      reinterpret_cast<int*>(dst)[i] = __ldg(reinterpret_cast<const int*>(src) + i);
  } else if (vec == 2) {
    const int64_t n = len >> 1;
    for (int64_t i = tid; i < n; i += nthr)
      reinterpret_cast<short*>(dst)[i] = __ldg(reinterpret_cast<const short*>(src) + i);
  } else {
    for (int64_t i = tid; i < len; i += nthr) dst[i] = __ldg(src + i);
  }
}

template <int MODE>
__device__ __forceinline__ bool resolve_rows(const Plan& p, int64_t s, int64_t last,
                                             int64_t& src_row, int64_t& dst_row,
                                             int64_t& ring_row, int64_t& new_id) {
  new_id = 0;
  if (MODE == MODE_SAMPLE) {
    int64_t lo, hi;
    valid_range(last, p.L, p.T, lo, hi);
    if (hi <= lo) return false;
    const int64_t b = s / p.T, t = s - b * p.T;
    int64_t id, off;
    if (p.ids != nullptr) {
      id = p.ids[b];
      off = p.offs[b];
    } else {
      Philox4 r = philox4x32_10((uint64_t)b, *p.rng_call, p.seed);
      id = uniform_i64(r.x, r.y, lo, hi);
      off = uniform_i64(r.z, r.w, 0, p.B_env);
    }
    ring_row = (id + t) % p.L + off * p.L;  // tf_uniform_replay_buffer.py:289-292
    src_row = ring_row;
    dst_row = s;
  } else if (MODE == MODE_ROWS) {
    ring_row = p.rows[s];
    src_row = ring_row;
    dst_row = s;
  } else if (MODE == MODE_GATHER_ALL) {
    int64_t lo, hi;
    valid_range(last, p.L, 1, lo, hi);
    const int64_t b = s / p.n_valid, j = s - b * p.n_valid;
    ring_row = b * p.L + (lo + j) % p.L;  // :541-552
    src_row = ring_row;
    dst_row = s;
  } else if (MODE == MODE_ADD) {
    new_id = last + 1;                    // _increment_last_id :582-595
    ring_row = s * p.L + new_id % p.L;    // _get_rows_for_id :603-607
    src_row = s;
    dst_row = ring_row;
  } else {  // MODE_WRITE_ROWS
    ring_row = p.rows[s];
    src_row = s;
    dst_row = ring_row;
  }
  return true;
}

template <int MODE>
__device__ __forceinline__ void small_and_meta(const Plan& p, int64_t s, int64_t src_row,
                                               int64_t dst_row, int64_t ring_row,
                                               int64_t new_id, int64_t last, int tid,
                                               int nthr) {
  for (int i = 0; i < p.n_small; ++i) {
    const PlanLeaf& lf = p.small[i];
    copy_span(lf.src + src_row * lf.row_bytes, lf.dst + dst_row * lf.row_bytes, lf.row_bytes,
              lf.vec, tid, nthr);
  }
  if (tid == 0) {
    if (MODE == MODE_SAMPLE || MODE == MODE_ROWS) {
      if (p.out_ids) p.out_ids[s] = p.id_table[ring_row];
      if (p.out_rows) p.out_rows[s] = ring_row;
    }
    if (MODE == MODE_SAMPLE) {
      const int64_t b = s / p.T;
      if (s == b * p.T && p.out_prob) {
        int64_t lo, hi;
        valid_range(last, p.L, p.T, lo, hi);
        // probability, tf_uniform_replay_buffer.py:255-264
        p.out_prob[b] = 1.0f / (float)((hi - lo) * p.B_env);
      }
    }
    if (MODE == MODE_ADD) p.id_table[ring_row] = new_id;
  }
}

template <int MODE>
__device__ __forceinline__ void finish(const Plan& p, int64_t last, bool ok) {
  // last-block-done: advance the device-resident counters exactly once per launch.
  __syncthreads();
  if (threadIdx.x == 0 && p.ticket != nullptr && last_block_ticket(p.ticket)) {
    if (MODE == MODE_SAMPLE) {
      if (p.rng_call && p.ids == nullptr) *p.rng_call = *p.rng_call + 1;
      if (p.status) *p.status = ok ? 0 : 1;
    }
    if (MODE == MODE_ADD) *p.last_id = last + 1;
    __threadfence();
  }
}

// One CTA per (row, piece): a piece is <= 16 KiB of one big leaf; piece 0 also carries the
// small leaves and the id / row / probability outputs.
template <int MODE>
__global__ void __launch_bounds__(kThreads) row_copy_big(const __grid_constant__ Plan p) {
  pdl_prologue();
  const int64_t blk = blockIdx.x;
  const int64_t s = blk / p.pieces_per_row;
  int piece = (int)(blk - s * p.pieces_per_row);
  const int64_t last = p.last_id ? *p.last_id : 0;
  int64_t src_row, dst_row, ring_row, new_id;
  const bool ok = resolve_rows<MODE>(p, s, last, src_row, dst_row, ring_row, new_id);
  if (ok) {
    int li = 0, pc = piece;
    while (pc >= p.big[li].n_pieces) {
      pc -= p.big[li].n_pieces;
      ++li;
    }
    const PlanLeaf& lf = p.big[li];
    const int64_t begin = (int64_t)pc * lf.piece_bytes;
    int64_t len = lf.row_bytes - begin;
    if (len > lf.piece_bytes) len = lf.piece_bytes;
    copy_span(lf.src + src_row * lf.row_bytes + begin, lf.dst + dst_row * lf.row_bytes + begin,
              len, lf.vec, threadIdx.x, kThreads);
    if (piece == 0)
      small_and_meta<MODE>(p, s, src_row, dst_row, ring_row, new_id, last, threadIdx.x,
                           kThreads);
  }
  finish<MODE>(p, last, ok);
}

// TMA variant of row_copy_big: one warp per (row, piece).  Lane 0 stages the piece through
// shared memory with two bulk-async copies (global -> smem on an mbarrier, smem -> global as a
// bulk group), so the whole transfer is issued by the copy engine in two instructions and
// 16 CTAs x 14 KiB stay in flight per SM.  Lanes 1..31 carry the small leaves / ids.
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}

template <int MODE>
__global__ void __launch_bounds__(32) row_copy_tma(const __grid_constant__ Plan p) {
  pdl_prologue();
  extern __shared__ __align__(128) unsigned char stage[];
  __shared__ __align__(8) unsigned long long bar;
  const int64_t blk = blockIdx.x;
  const int64_t s = blk / p.pieces_per_row;
  int piece = (int)(blk - s * p.pieces_per_row);
  const int64_t last = p.last_id ? *p.last_id : 0;
  int64_t src_row, dst_row, ring_row, new_id;
  const bool ok = resolve_rows<MODE>(p, s, last, src_row, dst_row, ring_row, new_id);
  if (ok) {
    if (threadIdx.x == 0) {
      int li = 0, pc = piece;
      while (pc >= p.big[li].n_pieces) {
        pc -= p.big[li].n_pieces;
        ++li;
      }
      const PlanLeaf& lf = p.big[li];
      const int64_t begin = (int64_t)pc * lf.piece_bytes;
      int64_t len = lf.row_bytes - begin;
      if (len > lf.piece_bytes) len = lf.piece_bytes;
      const char* src = lf.src + src_row * lf.row_bytes + begin;
      char* dst = lf.dst + dst_row * lf.row_bytes + begin;
      const uint32_t bar_a = smem_u32(&bar), st_a = smem_u32(stage), n = (uint32_t)len;
      asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar_a));
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_a), "r"(n)
                   : "memory");
      asm volatile(
          "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
          ::"r"(st_a), "l"(src), "r"(n), "r"(bar_a)
          : "memory");
      // non-blocking poll (mbarrier.try_wait may suspend the thread for a system time limit)
      uint32_t landed;
      do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], 0;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(landed)
            : "r"(bar_a)
            : "memory");
      } while (!landed);
      asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst),
                   "r"(st_a), "r"(n)
                   : "memory");
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
    } else if (piece == 0) {
      small_and_meta<MODE>(p, s, src_row, dst_row, ring_row, new_id, last, threadIdx.x - 1, 31);
    }
  }
  finish<MODE>(p, last, ok);
}

// All-small rows (MuJoCo-shape: 108-160 B): one warp per row, 8 rows per CTA.
template <int MODE>
__global__ void __launch_bounds__(kThreads) row_copy_small(const __grid_constant__ Plan p) {
  pdl_prologue();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t s = (int64_t)blockIdx.x * (kThreads / 32) + warp;
  const int64_t last = p.last_id ? *p.last_id : 0;
  bool ok = true;
  if (s < p.n_rows) {
    int64_t src_row, dst_row, ring_row, new_id;
    ok = resolve_rows<MODE>(p, s, last, src_row, dst_row, ring_row, new_id);
    if (ok) small_and_meta<MODE>(p, s, src_row, dst_row, ring_row, new_id, last, lane, 32);
  } else if (MODE == MODE_SAMPLE) {
    int64_t lo, hi;
    valid_range(last, p.L, p.T, lo, hi);
    ok = hi > lo;
  }
  finish<MODE>(p, last, ok);
}

__global__ void draw_kernel(const __grid_constant__ Plan p) {
  pdl_prologue();
  const int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t last = *p.last_id;
  int64_t lo, hi;
  valid_range(last, p.L, p.T, lo, hi);
  const bool ok = hi > lo;
  if (b < p.B && ok) {
    Philox4 r = philox4x32_10((uint64_t)b, *p.rng_call, p.seed);
    p.out_draw_ids[b] = uniform_i64(r.x, r.y, lo, hi);
    p.out_draw_offs[b] = uniform_i64(r.z, r.w, 0, p.B_env);
  }
  __syncthreads();
  if (threadIdx.x == 0 && last_block_ticket(p.ticket)) {
    *p.rng_call = *p.rng_call + 1;
    __threadfence();
  }
}

__global__ void clear_kernel(int64_t* last_id) {
  pdl_prologue(); *last_id = -1; }

static int widest_vec(int64_t row_bytes, const void* a, const void* b) {
  uintptr_t bits = (uintptr_t)row_bytes | (uintptr_t)a | (uintptr_t)b;
  if ((bits & 15) == 0) return 16;
  if ((bits & 7) == 0) return 8;
  if ((bits & 3) == 0) return 4;
  if ((bits & 1) == 0) return 2;
  return 1;
}

// Build the copy plan. ring_is_src: ring storage is the source (reads) else destination.
static int build_plan(const b200rl_ring_t* ring, const void* const* other, bool ring_is_src,
                      Plan& p) {
  B200RL_CHECK_ARG(ring != nullptr, "ring is NULL");
  B200RL_CHECK_ARG(ring->num_leaves > 0 && ring->num_leaves <= B200RL_MAX_LEAVES,
                   "num_leaves=%d out of range (1..%d)", ring->num_leaves, B200RL_MAX_LEAVES);
  B200RL_CHECK_ARG(ring->batch_size > 0 && ring->max_length > 0, "bad ring geometry");
  B200RL_CHECK_ARG(other != nullptr, "leaf pointer array is NULL");
  p = Plan{};
  p.B_env = ring->batch_size;
  p.L = ring->max_length;
  p.id_table = ring->id_table;
  p.last_id = ring->last_id;
  p.ticket = ring->ticket;
  int pieces = 0;
  for (int i = 0; i < ring->num_leaves; ++i) {
    const b200rl_leaf_t& lf = ring->leaves[i];
    B200RL_CHECK_ARG(lf.storage != nullptr && other[i] != nullptr, "leaf %d has NULL pointer", i);
    B200RL_CHECK_ARG(lf.row_bytes > 0, "leaf %d has row_bytes=%lld", i, (long long)lf.row_bytes);
    PlanLeaf pl{};
    pl.src = (const char*)(ring_is_src ? lf.storage : other[i]);
    pl.dst = (char*)(ring_is_src ? other[i] : lf.storage);
    pl.row_bytes = lf.row_bytes;
    pl.vec = widest_vec(lf.row_bytes, pl.src, pl.dst);
    if (lf.row_bytes <= kSmallMax) {
      p.small[p.n_small++] = pl;
    } else {
      int64_t np = (lf.row_bytes + kPieceTarget - 1) / kPieceTarget;
      int64_t pb = (lf.row_bytes + np - 1) / np;
      pb = (pb + 15) / 16 * 16;  // keep piece starts 16 B aligned
      np = (lf.row_bytes + pb - 1) / pb;
      pl.n_pieces = (int32_t)np;
      pl.piece_bytes = (int32_t)pb;
      pieces += (int)np;
      p.big[p.n_big++] = pl;
    }
  }
  p.pieces_per_row = pieces;
  p.rows_per_cta = kThreads / 32;
  return B200RL_OK;
}

template <int MODE>
static int launch_plan(Plan& p, cudaStream_t st, const char* name) {
  if (p.n_rows <= 0) return B200RL_OK;
  if (p.n_big > 0) {
    int64_t grid = p.n_rows * p.pieces_per_row;
    B200RL_CHECK_ARG(grid < (1ll << 31), "%s: grid too large", name);
    // the TMA bulk copy (row_copy_tma) needs every big leaf 16-byte aligned, else row_copy_big
    bool tma_ok = true;
    int max_piece = 0;
    for (int i = 0; i < p.n_big; ++i) {
      if (p.big[i].vec != 16) tma_ok = false;
      if (p.big[i].piece_bytes > max_piece) max_piece = p.big[i].piece_bytes;
    }
    if (tma_ok) {
      B200RL_LAUNCH(row_copy_tma<MODE>, (unsigned)grid, 32, max_piece, st, p);
    } else {
      B200RL_LAUNCH(row_copy_big<MODE>, (unsigned)grid, kThreads, 0, st, p);
    }
  } else {
    int64_t grid = (p.n_rows + p.rows_per_cta - 1) / p.rows_per_cta;
    B200RL_CHECK_ARG(grid < (1ll << 31), "%s: grid too large", name);
    B200RL_LAUNCH(row_copy_small<MODE>, (unsigned)grid, kThreads, 0, st, p);
  }
  B200RL_CHECK_LAUNCH(name);
  return B200RL_OK;
}

}  // namespace b200rl

using namespace b200rl;

extern "C" {

int b200rl_rb_add_batch(const b200rl_ring_t* ring, const void* const* items, void* stream) {
  Plan p;
  int rc = build_plan(ring, items, /*ring_is_src=*/false, p);
  if (rc) return rc;
  B200RL_CHECK_ARG(ring->last_id && ring->id_table && ring->ticket, "ring counters are NULL");
  p.n_rows = ring->batch_size;
  return launch_plan<MODE_ADD>(p, (cudaStream_t)stream, "rb_add_batch");
}

int b200rl_rb_sample(const b200rl_ring_t* ring, int64_t B, int64_t T, const int64_t* ids_dev,
                     const int64_t* offs_dev, uint64_t seed, uint64_t* rng_call_dev,
                     void* const* out, int64_t* out_ids, int64_t* out_rows, float* out_prob,
                     int32_t* status_dev, void* stream) {
  Plan p;
  int rc = build_plan(ring, (const void* const*)out, /*ring_is_src=*/true, p);
  if (rc) return rc;
  B200RL_CHECK_ARG(B >= 1 && T >= 1, "rb_sample: B=%lld T=%lld", (long long)B, (long long)T);
  B200RL_CHECK_ARG(T <= ring->max_length, "rb_sample: num_steps %lld > max_length %lld",
                   (long long)T, (long long)ring->max_length);
  B200RL_CHECK_ARG((ids_dev == nullptr) == (offs_dev == nullptr),
                   "rb_sample: ids and offs must both be given or both NULL");
  B200RL_CHECK_ARG(ids_dev != nullptr || rng_call_dev != nullptr,
                   "rb_sample: need rng_call_dev when drawing on device");
  B200RL_CHECK_ARG(ring->last_id && ring->id_table && ring->ticket, "ring counters are NULL");
  p.B = B;
  p.T = T;
  p.n_rows = B * T;
  p.ids = ids_dev;
  p.offs = offs_dev;
  p.seed = seed;
  p.rng_call = rng_call_dev;
  p.out_ids = out_ids;
  p.out_rows = out_rows;
  p.out_prob = out_prob;
  p.status = status_dev;
  return launch_plan<MODE_SAMPLE>(p, (cudaStream_t)stream, "rb_sample");
}

int b200rl_rb_read_rows(const b200rl_ring_t* ring, const int64_t* rows_dev, int64_t n,
                        void* const* out, int64_t* out_ids, void* stream) {
  Plan p;
  int rc = build_plan(ring, (const void* const*)out, true, p);
  if (rc) return rc;
  B200RL_CHECK_ARG(rows_dev != nullptr && n >= 0, "rb_read_rows: bad rows");
  p.n_rows = n;
  p.rows = rows_dev;
  p.out_ids = out_ids;
  p.ticket = nullptr;  // no counters to advance
  return launch_plan<MODE_ROWS>(p, (cudaStream_t)stream, "rb_read_rows");
}

int b200rl_rb_write_rows(const b200rl_ring_t* ring, const int64_t* rows_dev, int64_t n,
                         const void* const* items, void* stream) {
  Plan p;
  int rc = build_plan(ring, items, false, p);
  if (rc) return rc;
  B200RL_CHECK_ARG(rows_dev != nullptr && n >= 0, "rb_write_rows: bad rows");
  p.n_rows = n;
  p.rows = rows_dev;
  p.ticket = nullptr;
  return launch_plan<MODE_WRITE_ROWS>(p, (cudaStream_t)stream, "rb_write_rows");
}

int b200rl_rb_gather_all(const b200rl_ring_t* ring, int64_t n_valid, void* const* out,
                         void* stream) {
  Plan p;
  int rc = build_plan(ring, (const void* const*)out, true, p);
  if (rc) return rc;
  B200RL_CHECK_ARG(n_valid >= 0 && n_valid <= ring->max_length, "rb_gather_all: n_valid=%lld",
                   (long long)n_valid);
  p.n_valid = n_valid;
  p.n_rows = ring->batch_size * n_valid;
  p.ticket = nullptr;
  return launch_plan<MODE_GATHER_ALL>(p, (cudaStream_t)stream, "rb_gather_all");
}

int b200rl_rb_clear(const b200rl_ring_t* ring, int clear_all, void* stream) {
  B200RL_CHECK_ARG(ring != nullptr && ring->last_id != nullptr, "rb_clear: ring is NULL");
  cudaStream_t st = (cudaStream_t)stream;
  B200RL_LAUNCH(clear_kernel, 1, 1, 0, st, ring->last_id);
  B200RL_CHECK_LAUNCH("rb_clear");
  if (clear_all) {
    const int64_t cap = ring->batch_size * ring->max_length;
    for (int i = 0; i < ring->num_leaves; ++i) {
      cudaError_t e = cudaMemsetAsync(ring->leaves[i].storage, 0,
                                      (size_t)(cap * ring->leaves[i].row_bytes), st);
      if (e != cudaSuccess) {
        set_error("rb_clear: memset failed: %s", cudaGetErrorString(e));
        return B200RL_ERR_CUDA;
      }
    }
    cudaMemsetAsync(ring->id_table, 0, (size_t)cap * sizeof(int64_t), st);
  }
  return B200RL_OK;
}

int b200rl_rb_draw(const b200rl_ring_t* ring, int64_t B, int64_t T, uint64_t seed,
                   uint64_t* rng_call_dev, int64_t* out_ids, int64_t* out_offs, void* stream) {
  B200RL_CHECK_ARG(ring && ring->last_id && ring->ticket && rng_call_dev && out_ids && out_offs,
                   "rb_draw: NULL argument");
  B200RL_CHECK_ARG(B >= 1 && T >= 1, "rb_draw: B=%lld T=%lld", (long long)B, (long long)T);
  Plan p{};
  p.B_env = ring->batch_size;
  p.L = ring->max_length;
  p.last_id = ring->last_id;
  p.ticket = ring->ticket;
  p.B = B;
  p.T = T;
  p.seed = seed;
  p.rng_call = rng_call_dev;
  p.out_draw_ids = out_ids;
  p.out_draw_offs = out_offs;
  unsigned grid = (unsigned)((B + 255) / 256);
  B200RL_LAUNCH(draw_kernel, grid, 256, 0, (cudaStream_t)stream, p);
  B200RL_CHECK_LAUNCH("rb_draw");
  return B200RL_OK;
}

}  // extern "C"
