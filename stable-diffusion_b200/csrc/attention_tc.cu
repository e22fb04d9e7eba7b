// Flash-style fused attention on wgmma (sm_90a): S = Q K^T and O += P V on the tensor cores with S, O in registers,
// online softmax on the accumulator fragments, P kept in registers as the A operand of the second MMA.
//
//   warp 8      : TMA producer (Q once; K in 64-column panels and V^T tiles, each through an mbarrier ring)
//   warps 0..7  : two consumer warpgroups of 64 query rows each: wgmma S (M = 64, N = 64 keys), masking, online
//                 softmax (a row lives in the four threads of a quad), wgmma PV (M = 64, N = DV), epilogue O / l
//
//   attention_tc_kernel<DPAD, DPAD>: multi-head attention with the head dim padded to DPAD = 64 / 128 / 192.
//   attention_tc_kernel<512, 128>  : single-head d = 512 (the AutoencoderKL mid-block AttnBlock,
//     ldm/modules/diffusionmodules/model.py:178-202): one CTA = 128 query rows x ONE 128-column slice of the output
//     (grid.y = 4 slices; S is recomputed per slice: a wider O does not fit the registers next to S), Q resident as
//     eight 64-column panels, K streamed panel by panel.
//     The N x N logits never leave the SM.
//
// Replaces the materialised einsum('b i d, b j d -> b i j') * scale -> softmax -> einsum('b i j, b j d -> b i d')
// of ldm/modules/attention.py:178-192 (and CLIP self-attention with a causal mask).
#include "../../include/sdb200.h"
#include "host.h"
#include "ptx.cuh"

#include <stdlib.h>

namespace sdb {

constexpr int AQ = 128;   // query rows per CTA
constexpr int AKV = 64;   // kv rows per iteration
constexpr int ATT_THREADS = 288;
constexpr int ATT_PRODUCER_WARP = 8;

template <int DPAD, int DV>
struct AttnCfg {
  static constexpr int PANELS = DPAD / 64;
  static constexpr int Q_BYTES = AQ * DPAD * 2;
  static constexpr int KP_BYTES = AKV * 64 * 2;   // one 64-column K panel
  static constexpr int V_BYTES = DV * AKV * 2;     // one V^T tile [DV x 64 keys]
  static constexpr int KST = DPAD == 512 ? 4 : (2 * PANELS < 4 ? 4 : 2 * PANELS);   // K panel ring depth
  static constexpr int VST = 2;                                                      // V^T ring depth
  static constexpr int SMEM = Q_BYTES + KST * KP_BYTES + VST * V_BYTES + 1024;
};

struct AttnArgs {
  int nq, nkv, d, heads;
  int ldo;
  long long o_batch_stride;
  __half* out;
  float scale_log2;
  int causal;
};

__device__ __forceinline__ float fast_exp2(float x) {  // one MUFU.EX2, flush-to-zero (exp2(-inf) = 0)
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
  const __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}

template <int DPAD, int DV>
__global__ void __launch_bounds__(ATT_THREADS, 1)
    attention_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                        const __grid_constant__ CUtensorMap tmV, const AttnArgs p) {
  using Cfg = AttnCfg<DPAD, DV>;
  constexpr bool WIDE = DV < DPAD;
  constexpr int PANELS = Cfg::PANELS;
  constexpr int KST = Cfg::KST;
  constexpr int VST = Cfg::VST;

  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment by offset (keeps the shared address space visible to the compiler: STS, not generic ST)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* q_s = smem;
  uint8_t* k_s = q_s + Cfg::Q_BYTES;
  uint8_t* v_s = k_s + KST * Cfg::KP_BYTES;

  __shared__ uint64_t q_full, k_full[KST], k_empty[KST], v_full[VST], v_empty[VST];

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  pdl_launch_dependents();
  const int q0 = blockIdx.x * AQ;
  const int head = WIDE ? 0 : blockIdx.y;
  const int dv0 = WIDE ? blockIdx.y * DV : 0;
  const int b = blockIdx.z;
  int nkv_eff = p.nkv;
  if (p.causal) nkv_eff = min(p.nkv, q0 + AQ);  // kv blocks entirely above the diagonal are skipped
  const int n_iter = (nkv_eff + AKV - 1) / AKV;

  if (warp == ATT_PRODUCER_WARP && lane == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    mbar_init(&q_full, 1);
    for (int i = 0; i < KST; ++i) {
      mbar_init(&k_full[i], 1);
      mbar_init(&k_empty[i], 8);   // one arrive per consumer warp
    }
    for (int i = 0; i < VST; ++i) {
      mbar_init(&v_full[i], 1);
      mbar_init(&v_empty[i], 8);
    }
    fence_barrier_init();
  }
  __syncthreads();

  pdl_wait();   // q / k / v come from the previous kernels; everything above overlapped their tail
  if (warp == ATT_PRODUCER_WARP) {
    if (elect_one()) {
      mbar_arrive_expect_tx(&q_full, Cfg::Q_BYTES);
      for (int pn = 0; pn < PANELS; ++pn) tma_load_3d(q_s + pn * (AQ * 128), &tmQ, &q_full, head * DPAD + pn * 64, q0, b);
      int ks = 0;
      uint32_t kph = 0;
      for (int j = 0; j < n_iter; ++j) {
        for (int pn = 0; pn < PANELS; ++pn) {
          mbar_wait_mma(&k_empty[ks], kph ^ 1);
          mbar_arrive_expect_tx(&k_full[ks], Cfg::KP_BYTES);
          tma_load_3d(k_s + ks * Cfg::KP_BYTES, &tmK, &k_full[ks], head * DPAD + pn * 64, j * AKV, b);
          if (++ks == KST) {
            ks = 0;
            kph ^= 1;
          }
        }
        const int vs = j % VST;
        mbar_wait_mma(&v_empty[vs], ((j / VST) & 1) ^ 1);
        mbar_arrive_expect_tx(&v_full[vs], Cfg::V_BYTES);
        tma_load_3d(v_s + vs * Cfg::V_BYTES, &tmV, &v_full[vs], j * AKV, head * DPAD + dv0, b);
      }
    }
    __syncwarp();
  } else {
    const int wg = warp >> 2;
    const int t4 = lane & 3;
    const int qi0 = q0 + 64 * wg + 16 * (warp & 3) + (lane >> 2);   // fragment rows of this thread: qi0, qi0 + 8
    const int qi1 = qi0 + 8;
    // head dimension d < DPAD: columns d .. DPAD-1 of Q / K are zero padding; only the 16-wide K steps that hold real
    // columns are issued for S
    const int ksteps = (p.d + 15) >> 4;
    const uint32_t q_addr = smem_u32(q_s) + static_cast<uint32_t>(wg * 64 * 128);
    float o[DV / 2];
#pragma unroll
    for (int i = 0; i < DV / 2; ++i) o[i] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY;   // running maxima (log2 domain) of rows qi0 / qi1
    float l0 = 0.f, l1 = 0.f;               // this thread's share of the row sums
    int ks = 0;
    uint32_t kph = 0;
    mbar_wait_mma(&q_full, 0);
    for (int j = 0; j < n_iter; ++j) {
      // ---- S = Q K^T over the K panels of this tile; each panel is handed back once its MMAs have completed
      float s[AKV / 2];
#pragma unroll
      for (int i = 0; i < AKV / 2; ++i) s[i] = 0.f;
      wgmma_hold(s);
      int prev = -1;
#pragma unroll 1
      for (int pn = 0; pn < PANELS; ++pn) {
        mbar_wait_mma(&k_full[ks], kph);
        const uint32_t k_addr = smem_u32(k_s + ks * Cfg::KP_BYTES);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
          if (pn * 4 + kk < ksteps)
            WgmmaSS<AKV>::mma(s, wg_desc(q_addr + pn * (AQ * 128) + kk * 32), wg_desc(k_addr + kk * 32), 1u);
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0 && lane == 0) mbar_arrive(&k_empty[prev]);
        prev = ks;
        if (++ks == KST) {
          ks = 0;
          kph ^= 1;
        }
      }
      wgmma_wait<0>();
      wgmma_hold(s);
      if (lane == 0) mbar_arrive(&k_empty[prev]);

      // ---- mask, online softmax. s[4c + e]: row qi0 (e < 2) or qi1, key kv0 + 8c + 2 t4 + (e & 1)
      const int kv0 = j * AKV;
      if ((kv0 + AKV > p.nkv) || (p.causal && kv0 + AKV - 1 > q0)) {
#pragma unroll
        for (int i = 0; i < AKV / 2; ++i) {
          const int kv = kv0 + 8 * (i >> 2) + 2 * t4 + (i & 1);
          const int qi = (i & 2) ? qi1 : qi0;
          if ((kv >= p.nkv) || (p.causal && kv > qi)) s[i] = -INFINITY;
        }
      }
      float mx0 = s[0], mx1 = s[2];
#pragma unroll
      for (int c = 0; c < AKV / 8; ++c) {
        mx0 = fmaxf(mx0, fmaxf(s[4 * c], s[4 * c + 1]));
        mx1 = fmaxf(mx1, fmaxf(s[4 * c + 2], s[4 * c + 3]));
      }
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
      const float mn0 = fmaxf(m0, mx0 * p.scale_log2);   // scale > 0
      const float mn1 = fmaxf(m1, mx1 * p.scale_log2);
      const float al0 = (m0 == -INFINITY) ? 0.f : exp2f(m0 - mn0);   // nothing accumulated yet: O = 0, l = 0
      const float al1 = (m1 == -INFINITY) ? 0.f : exp2f(m1 - mn1);
      m0 = mn0;
      m1 = mn1;
      l0 *= al0;
      l1 *= al1;
#pragma unroll
      for (int c = 0; c < DV / 8; ++c) {
        o[4 * c] *= al0;
        o[4 * c + 1] *= al0;
        o[4 * c + 2] *= al1;
        o[4 * c + 3] *= al1;
      }
      const float nm0 = (mn0 == -INFINITY) ? 0.f : -mn0;   // a fully masked row so far: exp2(-inf) = 0
      const float nm1 = (mn1 == -INFINITY) ? 0.f : -mn1;
      // P (fp16) in the A-operand layout of wgmma: for key step kk, {row qi0 keys 2 t4 .. +1, row qi1 same, row qi0
      // keys 8 + 2 t4 .. +1, row qi1 same} = the S fragments of n8 blocks 2 kk and 2 kk + 1
      uint32_t pa[AKV / 16][4];
#pragma unroll
      for (int c = 0; c < AKV / 8; ++c) {
        const float e0 = fast_exp2(fmaf(s[4 * c], p.scale_log2, nm0));
        const float e1 = fast_exp2(fmaf(s[4 * c + 1], p.scale_log2, nm0));
        const float e2 = fast_exp2(fmaf(s[4 * c + 2], p.scale_log2, nm1));
        const float e3 = fast_exp2(fmaf(s[4 * c + 3], p.scale_log2, nm1));
        l0 += e0 + e1;
        l1 += e2 + e3;
        pa[c >> 1][(c & 1) * 2] = pack_half2(e0, e1);
        pa[c >> 1][(c & 1) * 2 + 1] = pack_half2(e2, e3);
      }

      // ---- O += P V^T-tile
      const int vs = j % VST;
      mbar_wait_mma(&v_full[vs], (j / VST) & 1);
      const uint32_t v_addr = smem_u32(v_s + vs * Cfg::V_BYTES);
      wgmma_hold(o);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < AKV / 16; ++kk) WgmmaRS<DV>::mma(o, pa[kk], wg_desc(v_addr + kk * 32), 1u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_hold(o);
      if (lane == 0) mbar_arrive(&v_empty[vs]);
    }

    // ---- epilogue: O / l
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
    l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float inv0 = l0 > 0.f ? 1.0f / l0 : 0.f;
    const float inv1 = l1 > 0.f ? 1.0f / l1 : 0.f;
    const int ncols = WIDE ? DV : p.d;
    __half* base = p.out + static_cast<size_t>(b) * p.o_batch_stride + static_cast<size_t>(head) * p.d + dv0;
    __half* row0 = base + static_cast<size_t>(qi0) * p.ldo;
    __half* row1 = base + static_cast<size_t>(qi1) * p.ldo;
#pragma unroll
    for (int c = 0; c < DV / 8; ++c) {
      const int col = 8 * c + 2 * t4;
      if (col < ncols) {
        if (qi0 < p.nq) *reinterpret_cast<uint32_t*>(row0 + col) = pack_half2(o[4 * c] * inv0, o[4 * c + 1] * inv0);
        if (qi1 < p.nq) *reinterpret_cast<uint32_t*>(row1 + col) = pack_half2(o[4 * c + 2] * inv1, o[4 * c + 3] * inv1);
      }
    }
  }
}

template <int DPAD, int DV>
static int launch_attn(const CUtensorMap& q, const CUtensorMap& k, const CUtensorMap& v, const AttnArgs& p, dim3 grid,
                       cudaStream_t st) {
  constexpr int SMEM = AttnCfg<DPAD, DV>::SMEM;
  auto kern = attention_tc_kernel<DPAD, DV>;
  static bool configured = false;
  if (!configured) {
    SDB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    configured = true;
  }
  SDB_CUDA(launch_pdl(kern, grid, dim3(ATT_THREADS), SMEM, st, q, k, v, p));
  SDB_LAUNCH_CHECK();
  return 0;
}

constexpr int WIDE_D = 512;
constexpr int WIDE_DV = 128;

}  // namespace sdb

using namespace sdb;

extern "C" int sdb_attention(const sdb_attn_desc* d, sdb_stream_t stream) {
  if (d && ::sdb::plan_recording()) {
    const sdb_attn_desc c = *d;
    ::sdb::plan_record([c](cudaStream_t s_) { return sdb_attention(&c, s_); });
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  SDB_CHECK(d && d->q && d->k && d->vt && d->out, "sdb_attention: null pointer");
  if (d->dpad == WIDE_D) {
    // single-head d = 512 (AutoencoderKL AttnBlock): q, k [B, n, 512], vt [B, 512, ldvt]
    SDB_CHECK(d->d == WIDE_D && d->heads == 1 && !d->causal, "sdb_attention: dpad 512 is the single-head d = 512 kernel");
    SDB_CHECK(d->batch > 0 && d->nq > 0 && d->nkv > 0, "sdb_attention: bad sizes");
    SDB_CHECK(d->ldq % 8 == 0 && d->ldk % 8 == 0 && d->ldvt % 8 == 0 && d->ldo % 8 == 0 && d->o_batch_stride % 8 == 0,
              "sdb_attention: leading dims must be multiples of 8");
    CUtensorMap tq, tk, tv;
    {
      uint64_t dims[3] = {WIDE_D, static_cast<uint64_t>(d->nq), static_cast<uint64_t>(d->batch)};
      uint64_t str[2] = {static_cast<uint64_t>(d->ldq) * 2, static_cast<uint64_t>(d->q_batch_stride) * 2};
      uint32_t box[3] = {64, AQ, 1};
      if (make_tmap_f16(&tq, d->q, 3, dims, str, box)) return 1;
    }
    {
      uint64_t dims[3] = {WIDE_D, static_cast<uint64_t>(d->nkv), static_cast<uint64_t>(d->batch)};
      uint64_t str[2] = {static_cast<uint64_t>(d->ldk) * 2, static_cast<uint64_t>(d->k_batch_stride) * 2};
      uint32_t box[3] = {64, AKV, 1};
      if (make_tmap_f16(&tk, d->k, 3, dims, str, box)) return 1;
    }
    {
      uint64_t dims[3] = {static_cast<uint64_t>(d->nkv), WIDE_D, static_cast<uint64_t>(d->batch)};
      uint64_t str[2] = {static_cast<uint64_t>(d->ldvt) * 2, static_cast<uint64_t>(d->vt_batch_stride) * 2};
      uint32_t box[3] = {AKV, WIDE_DV, 1};
      if (make_tmap_f16(&tv, d->vt, 3, dims, str, box)) return 1;
    }
    AttnArgs p{};
    p.nq = d->nq;
    p.nkv = d->nkv;
    p.d = d->d;
    p.heads = 1;
    p.ldo = d->ldo;
    p.o_batch_stride = d->o_batch_stride;
    p.out = static_cast<__half*>(d->out);
    p.scale_log2 = d->scale * 1.4426950408889634f;
    p.causal = 0;
    dim3 grid((d->nq + AQ - 1) / AQ, WIDE_D / WIDE_DV, d->batch);
    return launch_attn<WIDE_D, WIDE_DV>(tq, tk, tv, p, grid, st);
  }
  SDB_CHECK(d->dpad == 64 || d->dpad == 128 || d->dpad == 192, "sdb_attention: dpad must be 64/128/192/512 (got %d)",
            d->dpad);
  SDB_CHECK(d->d > 0 && d->d <= d->dpad && d->d % 2 == 0, "sdb_attention: bad head dim %d", d->d);
  SDB_CHECK(d->batch > 0 && d->heads > 0 && d->nq > 0 && d->nkv > 0, "sdb_attention: bad sizes");
  SDB_CHECK(d->ldq % 8 == 0 && d->ldk % 8 == 0 && d->ldvt % 8 == 0, "sdb_attention: leading dims must be multiples of 8");
  SDB_CHECK(d->ldo % 2 == 0 && d->o_batch_stride % 2 == 0, "sdb_attention: output stride must be even");

  CUtensorMap tq, tk, tv;
  const uint64_t hd = static_cast<uint64_t>(d->heads) * d->dpad;
  {
    uint64_t dims[3] = {hd, static_cast<uint64_t>(d->nq), static_cast<uint64_t>(d->batch)};
    uint64_t str[2] = {static_cast<uint64_t>(d->ldq) * 2, static_cast<uint64_t>(d->q_batch_stride) * 2};
    uint32_t box[3] = {64, AQ, 1};
    if (make_tmap_f16(&tq, d->q, 3, dims, str, box)) return 1;
  }
  {
    uint64_t dims[3] = {hd, static_cast<uint64_t>(d->nkv), static_cast<uint64_t>(d->batch)};
    uint64_t str[2] = {static_cast<uint64_t>(d->ldk) * 2, static_cast<uint64_t>(d->k_batch_stride) * 2};
    uint32_t box[3] = {64, AKV, 1};
    if (make_tmap_f16(&tk, d->k, 3, dims, str, box)) return 1;
  }
  {
    uint64_t dims[3] = {static_cast<uint64_t>(d->nkv), hd, static_cast<uint64_t>(d->batch)};
    uint64_t str[2] = {static_cast<uint64_t>(d->ldvt) * 2, static_cast<uint64_t>(d->vt_batch_stride) * 2};
    uint32_t box[3] = {AKV, static_cast<uint32_t>(d->dpad), 1};
    if (make_tmap_f16(&tv, d->vt, 3, dims, str, box)) return 1;
  }
  AttnArgs p{};
  p.nq = d->nq;
  p.nkv = d->nkv;
  p.d = d->d;
  p.heads = d->heads;
  p.ldo = d->ldo;
  p.o_batch_stride = d->o_batch_stride;
  p.out = static_cast<__half*>(d->out);
  p.scale_log2 = d->scale * 1.4426950408889634f;
  p.causal = d->causal;
  dim3 grid((d->nq + AQ - 1) / AQ, d->heads, d->batch);
  switch (d->dpad) {
    case 64: return launch_attn<64, 64>(tq, tk, tv, p, grid, st);
    case 128: return launch_attn<128, 128>(tq, tk, tv, p, grid, st);
    default: return launch_attn<192, 192>(tq, tk, tv, p, grid, st);
  }
}
