// Exact k-nearest-neighbour search by inner product (the retrieval step of scripts/knn2img.py: the reference's ScaNN
// `score_brute_force` searcher over L2-normalised CLIP embeddings), and the pooling of CLIP's text embedding.
//
// sdb_knn_topk streams the fp16 database once, so it is bound by HBM bandwidth. Each CTA takes a contiguous slice of
// 64-row tiles. One producer warp loads the tiles by TMA in 64-column chunks (8 KiB, SWIZZLE_128B) into a ring of
// KNN_STAGES stages; one consumer warpgroup scores each tile against all queries with wgmma m64n64k16: database rows as
// M, the queries (<= 64, zero-padded by TMA, resident in shared memory for the whole pass) as N, fp32 accumulators.
// The 64 x 64 score tile goes through shared memory, and one warp per query admits the rows that beat that query's
// running k-th score into a sorted list of k (score descending, row ascending). Rows arrive in ascending order within a
// CTA, so a row that only ties the k-th score ranks after it and is rejected. A second launch merges the per-CTA lists
// of each query. No atomics: the result is the same on every run.
#include <cuda_fp16.h>
#include <float.h>
#include <limits.h>

#include "../../include/sdb200.h"
#include "host.h"
#include "ptx.cuh"

namespace sdb {

constexpr int KNN_ROWS = 64;        // database rows per tile (wgmma M)
constexpr int KNN_Q = 64;           // query columns (wgmma N); B <= 64
constexpr int KNN_CHUNK = 64;       // columns per TMA box: one 128-byte swizzle atom row
constexpr int KNN_STAGES = 8;
constexpr int KNN_MAX_DIM = 768;
constexpr int KNN_MAX_K = 64;
constexpr int KNN_BOX_BYTES = KNN_ROWS * KNN_CHUNK * 2;   // 8 KiB
constexpr int KNN_S_LD = KNN_Q + 1;                        // score tile row stride (floats)
constexpr int KNN_THREADS = 160;                           // consumer warpgroup + producer warp

struct KnnSmem {
  // 1024-byte aligned operand tiles first
  static constexpr int Q_OFF = 0;
  static constexpr int DB_OFF = Q_OFF + (KNN_MAX_DIM / KNN_CHUNK) * KNN_BOX_BYTES;
  static constexpr int S_OFF = DB_OFF + KNN_STAGES * KNN_BOX_BYTES;
  static constexpr int LS_OFF = S_OFF + KNN_ROWS * KNN_S_LD * 4;
  static constexpr int LI_OFF = LS_OFF + KNN_Q * KNN_MAX_K * 4;
  static constexpr int BAR_OFF = LI_OFF + KNN_Q * KNN_MAX_K * 4;
  static constexpr int BYTES = BAR_OFF + (2 * KNN_STAGES + 1) * 8;
};
constexpr int KNN_SMEM = KnnSmem::BYTES + 1024;   // + alignment slack

__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, 128;" ::: "memory"); }

// a ranks ahead of b: higher score, then lower row
__device__ __forceinline__ bool knn_ahead(float as, int ai, float bs, int bi) { return as > bs || (as == bs && ai < bi); }

__global__ void __launch_bounds__(KNN_THREADS, 1)
    knn_score_kernel(const __grid_constant__ CUtensorMap tm_db, const __grid_constant__ CUtensorMap tm_q, int n_rows,
                     int dim, int nq, int k, float* __restrict__ ws_score, int* __restrict__ ws_idx) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* q_s = smem + KnnSmem::Q_OFF;
  uint8_t* db_s = smem + KnnSmem::DB_OFF;
  float* s_tile = reinterpret_cast<float*>(smem + KnnSmem::S_OFF);
  float* l_score = reinterpret_cast<float*>(smem + KnnSmem::LS_OFF);
  int* l_idx = reinterpret_cast<int*>(smem + KnnSmem::LI_OFF);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + KnnSmem::BAR_OFF);
  uint64_t* empty = full + KNN_STAGES;
  uint64_t* q_bar = empty + KNN_STAGES;

  const int tid = threadIdx.x;
  const int n_chunks = dim / KNN_CHUNK;
  const int n_tiles = (n_rows + KNN_ROWS - 1) / KNN_ROWS;
  const int t0 = static_cast<int>(static_cast<long long>(n_tiles) * blockIdx.x / gridDim.x);
  const int t1 = static_cast<int>(static_cast<long long>(n_tiles) * (blockIdx.x + 1) / gridDim.x);

  if (tid == 0) {
    for (int s = 0; s < KNN_STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 4);   // one arrive per consumer warp
    }
    mbar_init(q_bar, 1);
    fence_barrier_init();
  }
  for (int i = tid; i < KNN_Q * KNN_MAX_K; i += KNN_THREADS) {
    l_score[i] = -INFINITY;
    l_idx[i] = INT_MAX;
  }
  __syncthreads();

  if (tid >= 128) {
    // ------------------------------------------------------------ producer warp
    if (tid == 128) {
      tma_prefetch_desc(&tm_db);
      mbar_arrive_expect_tx(q_bar, n_chunks * KNN_BOX_BYTES);
      for (int c = 0; c < n_chunks; ++c) tma_load_2d(q_s + c * KNN_BOX_BYTES, &tm_q, q_bar, c * KNN_CHUNK, 0);
      int it = 0;
      for (int t = t0; t < t1; ++t) {
        for (int c = 0; c < n_chunks; ++c, ++it) {
          const int s = it % KNN_STAGES;
          if (it >= KNN_STAGES) mbar_wait_mma(&empty[s], ((it / KNN_STAGES) - 1) & 1);
          mbar_arrive_expect_tx(&full[s], KNN_BOX_BYTES);
          tma_load_2d(db_s + s * KNN_BOX_BYTES, &tm_db, &full[s], c * KNN_CHUNK, t * KNN_ROWS);
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------- consumer warpgroup
  const int warp = tid >> 5, lane = tid & 31;
  mbar_wait_mma(q_bar, 0);
  int it = 0;
  for (int t = t0; t < t1; ++t) {
    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
    for (int c = 0; c < n_chunks; ++c, ++it) {
      const int s = it % KNN_STAGES;
      mbar_wait_mma(&full[s], (it / KNN_STAGES) & 1);
      const uint32_t a0 = smem_u32(db_s + s * KNN_BOX_BYTES);
      const uint32_t b0 = smem_u32(q_s + c * KNN_BOX_BYTES);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < KNN_CHUNK / 16; ++kk)
        WgmmaSS<KNN_Q>::mma(acc, wg_desc(a0 + kk * 32), wg_desc(b0 + kk * 32), (c | kk) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_hold(acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);
    }
    // accumulator fragment -> score tile [row][query]
    const int r0 = 16 * warp + (lane >> 2);
#pragma unroll
    for (int j = 0; j < KNN_Q / 8; ++j) {
      const int col = 8 * j + 2 * (lane & 3);
      s_tile[r0 * KNN_S_LD + col] = acc[4 * j];
      s_tile[r0 * KNN_S_LD + col + 1] = acc[4 * j + 1];
      s_tile[(r0 + 8) * KNN_S_LD + col] = acc[4 * j + 2];
      s_tile[(r0 + 8) * KNN_S_LD + col + 1] = acc[4 * j + 3];
    }
    consumer_sync();
    const int row_base = t * KNN_ROWS;
    const bool v0 = row_base + lane < n_rows, v1 = row_base + lane + 32 < n_rows;
    for (int q = warp; q < nq; q += 4) {
      float* ls = l_score + q * KNN_MAX_K;
      int* li = l_idx + q * KNN_MAX_K;
      float thr = ls[k - 1];   // -inf while the list is not full
      const float s0 = s_tile[lane * KNN_S_LD + q], s1 = s_tile[(lane + 32) * KNN_S_LD + q];
      uint32_t m0 = __ballot_sync(0xffffffffu, v0 && s0 > thr);
      uint32_t m1 = __ballot_sync(0xffffffffu, v1 && s1 > thr);
      if (!(m0 | m1)) continue;
      // the list in registers: lane holds entries lane and lane + 32
      float e0 = ls[lane], e1 = ls[lane + 32];
      int i0 = li[lane], i1 = li[lane + 32];
      for (int half = 0; half < 2; ++half) {
        uint32_t m = half ? m1 : m0;
        const float sv = half ? s1 : s0;
        while (m) {
          const int src = __ffs(m) - 1;
          m &= m - 1;
          const float cs = __shfl_sync(0xffffffffu, sv, src);
          const int ci = row_base + 32 * half + src;
          if (!(cs > thr)) continue;   // the threshold rose since the ballot
          // insert at pos = #entries ranking ahead (all of them came from lower rows: score >= cs)
          const int pos = __popc(__ballot_sync(0xffffffffu, e0 >= cs)) + __popc(__ballot_sync(0xffffffffu, e1 >= cs));
          const float up0 = __shfl_up_sync(0xffffffffu, e0, 1), up1 = __shfl_up_sync(0xffffffffu, e1, 1);
          const int iu0 = __shfl_up_sync(0xffffffffu, i0, 1), iu1 = __shfl_up_sync(0xffffffffu, i1, 1);
          const float w31 = __shfl_sync(0xffffffffu, e0, 31);
          const int iw31 = __shfl_sync(0xffffffffu, i0, 31);
          const float p1 = lane == 0 ? w31 : up1;
          const int ip1 = lane == 0 ? iw31 : iu1;
          const int j0 = lane, j1 = lane + 32;
          if (j0 == pos) { e0 = cs; i0 = ci; } else if (j0 > pos) { e0 = up0; i0 = iu0; }
          if (j1 == pos) { e1 = cs; i1 = ci; } else if (j1 > pos) { e1 = p1; i1 = ip1; }
          if (j0 >= k) { e0 = -INFINITY; i0 = INT_MAX; }
          if (j1 >= k) { e1 = -INFINITY; i1 = INT_MAX; }
          const float kth = __shfl_sync(0xffffffffu, (k - 1) < 32 ? e0 : e1, (k - 1) & 31);
          thr = kth;
        }
      }
      ls[lane] = e0;
      ls[lane + 32] = e1;
      li[lane] = i0;
      li[lane + 32] = i1;
      __syncwarp();
    }
    consumer_sync();   // the score tile is rewritten by the next tile
  }
  // this CTA's lists -> workspace [cta][query][k]
  for (int q = warp; q < nq; q += 4) {
    const size_t base = (static_cast<size_t>(blockIdx.x) * nq + q) * k;
    for (int i = lane; i < k; i += 32) {
      ws_score[base + i] = l_score[q * KNN_MAX_K + i];
      ws_idx[base + i] = l_idx[q * KNN_MAX_K + i];
    }
  }
}

// One CTA per query: k rounds of a block-wide pick among the heads of the n_lists sorted lists (one per thread).
__global__ void __launch_bounds__(1024) knn_merge_kernel(const float* __restrict__ ws_score, const int* __restrict__ ws_idx,
                                                         int n_lists, int nq, int k, float* __restrict__ out_score,
                                                         int64_t* __restrict__ out_idx) {
  __shared__ float red_s[32];
  __shared__ int red_i[32], red_l[32];
  const int q = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, n_warps = blockDim.x >> 5;
  const size_t base = (static_cast<size_t>(tid) * nq + q) * k;
  int p = 0;
  for (int r = 0; r < k; ++r) {
    float hs = -INFINITY;
    int hi = INT_MAX, hl = tid;
    if (tid < n_lists && p < k) {
      hs = ws_score[base + p];
      hi = ws_idx[base + p];
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      const float os = __shfl_xor_sync(0xffffffffu, hs, o);
      const int oi = __shfl_xor_sync(0xffffffffu, hi, o), ol = __shfl_xor_sync(0xffffffffu, hl, o);
      if (knn_ahead(os, oi, hs, hi)) { hs = os; hi = oi; hl = ol; }
    }
    if (lane == 0) { red_s[warp] = hs; red_i[warp] = hi; red_l[warp] = hl; }
    __syncthreads();
    if (warp == 0) {
      hs = lane < n_warps ? red_s[lane] : -INFINITY;
      hi = lane < n_warps ? red_i[lane] : INT_MAX;
      hl = lane < n_warps ? red_l[lane] : 0;
#pragma unroll
      for (int o = 16; o; o >>= 1) {
        const float os = __shfl_xor_sync(0xffffffffu, hs, o);
        const int oi = __shfl_xor_sync(0xffffffffu, hi, o), ol = __shfl_xor_sync(0xffffffffu, hl, o);
        if (knn_ahead(os, oi, hs, hi)) { hs = os; hi = oi; hl = ol; }
      }
      if (lane == 0) {
        out_score[static_cast<size_t>(q) * k + r] = hs;
        out_idx[static_cast<size_t>(q) * k + r] = hi;
        red_l[0] = hl;
      }
    }
    __syncthreads();
    if (tid == red_l[0]) ++p;
    __syncthreads();
  }
}

// ids != NULL: out[b] = x[b * n_ctx + argmax_i ids[b, i]] (the EOT row; the first maximum, as torch.argmax);
// else out[b] = x[b]. normalize != 0 divides the row by its L2 norm (fp32, z / torch.linalg.norm(z, dim=1)).
__global__ void rows_pool_kernel(const float* __restrict__ x, const int64_t* __restrict__ ids, int n_ctx, int dim,
                                 int normalize, float* __restrict__ out) {
  __shared__ float red[32];
  __shared__ int src_row;
  const int b = blockIdx.x, tid = threadIdx.x;
  if (tid == 0) {
    int best = 0;
    if (ids) {
      const int64_t* r = ids + static_cast<size_t>(b) * n_ctx;
      for (int i = 1; i < n_ctx; ++i)
        if (r[i] > r[best]) best = i;
      src_row = b * n_ctx + best;
    } else {
      src_row = b;
    }
  }
  __syncthreads();
  const float* src = x + static_cast<size_t>(src_row) * dim;
  float norm = 1.f;
  if (normalize) {
    float ss = 0.f;
    for (int c = tid; c < dim; c += blockDim.x) ss = fmaf(src[c], src[c], ss);
#pragma unroll
    for (int o = 16; o; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    if ((tid & 31) == 0) red[tid >> 5] = ss;
    __syncthreads();
    if (tid < 32) {
      ss = tid < (blockDim.x >> 5) ? red[tid] : 0.f;
#pragma unroll
      for (int o = 16; o; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
      if (tid == 0) red[0] = ss;
    }
    __syncthreads();
    norm = sqrtf(red[0]);
  }
  for (int c = tid; c < dim; c += blockDim.x) out[static_cast<size_t>(b) * dim + c] = normalize ? __fdiv_rn(src[c], norm) : src[c];
}

}  // namespace sdb

using namespace sdb;

extern "C" int64_t sdb_knn_workspace(int64_t n, int32_t b, int32_t k) {
  if (n <= 0 || b <= 0 || k <= 0) return 0;
  const int64_t tiles = (n + KNN_ROWS - 1) / KNN_ROWS;
  const int64_t ctas = tiles < sm_count() ? tiles : sm_count();
  return ctas * b * k;
}

extern "C" int sdb_knn_topk(const void* db, int64_t n, int32_t dim, const void* queries, int32_t b, int32_t k,
                            float* ws_score, int32_t* ws_idx, int64_t ws_entries, float* out_score, int64_t* out_idx,
                            sdb_stream_t stream) {
  SDB_REC(sdb_knn_topk(db, n, dim, queries, b, k, ws_score, ws_idx, ws_entries, out_score, out_idx, s_));
  SDB_CHECK(db && queries && ws_score && ws_idx && out_score && out_idx, "sdb_knn_topk: null pointer");
  SDB_CHECK(dim > 0 && dim % KNN_CHUNK == 0 && dim <= KNN_MAX_DIM, "sdb_knn_topk: dim %d (multiple of 64, <= %d)", dim,
            KNN_MAX_DIM);
  SDB_CHECK(b >= 1 && b <= KNN_Q, "sdb_knn_topk: %d queries (1 .. %d per launch)", b, KNN_Q);
  SDB_CHECK(k >= 1 && k <= KNN_MAX_K && k <= n, "sdb_knn_topk: k %d (1 .. %d, <= rows %lld)", k, KNN_MAX_K, (long long)n);
  SDB_CHECK(n < INT_MAX - KNN_ROWS, "sdb_knn_topk: %lld rows (< 2^31)", (long long)n);
  const int64_t need = sdb_knn_workspace(n, b, k);
  SDB_CHECK(ws_entries >= need, "sdb_knn_topk: workspace of %lld entries, %lld needed", (long long)ws_entries,
            (long long)need);
  const int ctas = static_cast<int>(need / (static_cast<int64_t>(b) * k));
  CUtensorMap tm_db, tm_q;
  {
    const uint64_t dims[2] = {static_cast<uint64_t>(dim), static_cast<uint64_t>(n)};
    const uint64_t str[1] = {static_cast<uint64_t>(dim) * 2};
    const uint32_t box[2] = {KNN_CHUNK, KNN_ROWS};
    if (make_tmap_f16(&tm_db, db, 2, dims, str, box)) return 1;
  }
  {
    const uint64_t dims[2] = {static_cast<uint64_t>(dim), static_cast<uint64_t>(b)};
    const uint64_t str[1] = {static_cast<uint64_t>(dim) * 2};
    const uint32_t box[2] = {KNN_CHUNK, KNN_Q};   // rows past b are zero-filled
    if (make_tmap_f16(&tm_q, queries, 2, dims, str, box)) return 1;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  static bool attr = false;
  if (!attr) {
    SDB_CUDA(cudaFuncSetAttribute(knn_score_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, KNN_SMEM));
    attr = true;
  }
  knn_score_kernel<<<ctas, KNN_THREADS, KNN_SMEM, st>>>(tm_db, tm_q, static_cast<int>(n), dim, b, k, ws_score, ws_idx);
  SDB_LAUNCH_CHECK();
  const int threads = (ctas + 31) / 32 * 32;
  knn_merge_kernel<<<b, threads, 0, st>>>(ws_score, ws_idx, ctas, b, k, out_score, out_idx);
  SDB_LAUNCH_CHECK();
  return 0;
}

extern "C" int sdb_rows_pool(const float* x, const int64_t* ids, int32_t b, int32_t n_ctx, int32_t dim,
                             int32_t normalize, float* out, sdb_stream_t stream) {
  SDB_REC(sdb_rows_pool(x, ids, b, n_ctx, dim, normalize, out, s_));
  SDB_CHECK(x && out && b > 0 && dim > 0 && (!ids || n_ctx > 0), "sdb_rows_pool: bad arguments");
  rows_pool_kernel<<<b, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, ids, n_ctx, dim, normalize, out);
  SDB_LAUNCH_CHECK();
  return 0;
}
