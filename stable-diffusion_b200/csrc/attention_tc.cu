// Flash-style fused attention on wgmma (sm_90a): S = Q K^T and O += P V on the tensor cores with S, O in registers,
// online softmax on the accumulator fragments, P kept in registers as the A operand of the second MMA.
//
//   warp 8      : TMA producer (Q once, or with each K panel at d = 960; K in 64-column panels and V^T tiles, each
//                 through an mbarrier ring)
//   warps 0..7  : two consumer warpgroups of 64 query rows each: wgmma S (M = 64, N = 64 keys), masking, online
//                 softmax (a row lives in the four threads of a quad), wgmma PV (M = 64, N = DV), epilogue O / l
//
//   attention_tc_kernel<DPAD, DV>: multi-head attention, head dim d <= DPAD (64 / 128 / 192 = the K panels of S),
//     DV = the PV width, ceil8(d) for the head dims the engine runs, else the slot width (d <= 160 at DPAD 192). Heads are read through 4-D
//     tensor maps whose innermost extent is d, so the panel columns d .. DPAD-1 and the V^T rows d .. DV-1 arrive as
//     TMA zero fill whatever the head stride in memory is. The consumer loop is software-pipelined (FA3-style):
//       window j (tensor-core issue, ping-ponged between the warpgroups by two named barriers): S_j = Q K_j^T, then
//         O += P_{j-1} V_{j-1}
//       after the window: wait for S_j only, softmax of tile j into the S registers while PV_{j-1} runs, wait for
//         PV_{j-1}, rescale O, pack P_j
//     so one warpgroup's exp work overlaps its own PV and the other warpgroup's MMAs. A quarter of the exponentials
//     run as a polynomial on the FMA pipe (poly_exp2) next to the MUFU ones.
//     The 288 threads x 224 registers of one CTA per SM fit the register file, so there is no setmaxnreg rebalancing.
//   attention_tc_kernel<D, DV>, D in {384, 512, 576, 960}: single-head attention at d = D, not causal (the
//     AutoencoderKL mid-block AttnBlock at 512, ldm/modules/diffusionmodules/model.py:178-202; the SpatialTransformers of
//     the class-conditional ImageNet LDM at 384 / 576 / 960, num_heads 1 with legacy dim_head = ch). One CTA = 128 query
//     rows x ONE DV-column slice of the output (grid.y = D / DV slices; S is recomputed per slice: a wider O does not fit
//     the registers next to S), K streamed panel by panel through a 4-deep ring (S and PV are not overlapped here).
//     The N x N logits never leave the SM.
//     DV is the widest PV slice that ptxas fits with no spills (at DV = 192 it spills and serialises the wgmmas):
//       D = 384: DV = 128, 3 slices (S computed 3x), Q resident as 6 panels: 164,864 B of shared memory, 140 registers.
//       D = 512: DV = 128, 4 slices (4x), Q resident as 8 panels: 197,632 B, 140 registers.
//       D = 576: DV =  96, 6 slices (6x), Q resident as 9 panels: 205,824 B, 122 registers.
//       D = 960: DV = 160, 6 slices (6x), 154 registers. A resident Q tile (240 KiB) does not fit the 227 KiB a CTA
//         may have, so Q is streamed: each K-ring stage also carries the matching 64-column Q panel (16 KiB) on the
//         same mbarrier and is freed with it (140,288 B). Q is then re-read from L2 once per 64-key tile; the engine's
//         d = 960 layers have 16 or 64 tokens (a single tile) at the 32x32 / 64x64 latents.
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
constexpr int MAX_SMEM = 232448;   // dynamic shared memory a CTA may opt into on sm_90

// the single-head family (dpad = d > 192); the multi-head kernels use the 64 / 128 / 192 head slots
__host__ __device__ constexpr bool attn_wide(int dpad) { return dpad > 192; }

template <int DPAD, int DV>
struct AttnCfg {
  static constexpr int PANELS = DPAD / 64;
  static constexpr int QP_BYTES = AQ * 128;                 // one 64-column Q panel
  static constexpr int KP_BYTES = AKV * 64 * 2;            // one 64-column K panel
  static constexpr int V_TX = DV * AKV * 2;                 // one V^T tile [DV x 64 keys]
  static constexpr int V_BYTES = (V_TX + 1023) / 1024 * 1024;   // ring stage: swizzle atoms stay 1024-byte aligned
  // multi-head: two tiles of K panels, so S_{j+1}'s panels load while S_j's are still held
  static constexpr int KST = attn_wide(DPAD) ? 4 : (2 * PANELS < 4 ? 4 : 2 * PANELS);   // K panel ring depth
  static constexpr int VST = attn_wide(DPAD) ? 2 : 4;   // V^T ring depth: the producer loads K_{j+1} after V_j's slot frees
  // Q resident when it fits next to the rings, else streamed with the K panels (one Q panel per K-ring stage)
  static constexpr bool STREAM_Q = PANELS * QP_BYTES + KST * KP_BYTES + VST * V_BYTES + 1024 > MAX_SMEM - 256;
  static constexpr int Q_BYTES = STREAM_Q ? KST * QP_BYTES : PANELS * QP_BYTES;
  static constexpr int SMEM = Q_BYTES + KST * KP_BYTES + VST * V_BYTES + 1024;
  static_assert(SMEM <= MAX_SMEM - 256, "attention tile does not fit shared memory");   // 256: static mbarriers
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
// exp2 of x <= 0 on the FMA / integer pipes, for the share of the softmax exponentials that MUFU does not take.
// Cody-Waite split x = n + f with n = round(x) (the 1.5 * 2^23 shifter), f in [-1/2, 1/2]; 2^f by the cubic
// 1 + f (c1 + f (c2 + f c3)), minimax in relative error on [-1/2, 1/2]: |p / 2^f - 1| < 1.02e-4 < 2^-13, below the
// 2^-11 rounding of P to fp16. 2^n is added to the exponent field. x is clamped to -127: -inf (masked) and anything
// below gives n = -127, f = 0, p = 1 exactly, i.e. the bit pattern 0 = +0.0, as MUFU's flush-to-zero does.
__device__ __forceinline__ float poly_exp2(float x) {
  x = fmaxf(x, -127.f);
  const float t = x + 12582912.f;
  const float f = x - (t - 12582912.f);
  const float p = fmaf(fmaf(fmaf(0.05500893f, f, 0.24221095f), f, 0.6932829f), f, 1.0f);
  return __int_as_float(__float_as_int(p) + (__float_as_int(t) << 23));
}
__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
  const __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}
// named barriers 1 / 2: warpgroup w waits on 1 + w for its turn at the tensor cores and hands the turn on to the other
__device__ __forceinline__ void wg_turn_wait(int wg) { asm volatile("bar.sync %0, 256;" ::"r"(1 + wg) : "memory"); }
__device__ __forceinline__ void wg_turn_pass(int wg) { asm volatile("bar.arrive %0, 256;" ::"r"(2 - wg) : "memory"); }

// S fragment of one 64-key tile -> masked online softmax, exponentials left in s (fp32), l updated; returns the O
// rescale factors through al0 / al1. s[4c + e]: row qi0 (e < 2) or qi1, key kv0 + 8c + 2 t4 + (e & 1).
template <bool POLY>
__device__ __forceinline__ void softmax_tile(float (&s)[AKV / 2], const AttnArgs& p, int kv0, int q0, int qi0, int qi1,
                                             int t4, float& m0, float& m1, float& l0, float& l1, float& al0,
                                             float& al1) {
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
  al0 = (m0 == -INFINITY) ? 0.f : exp2f(m0 - mn0);   // nothing accumulated yet: O = 0, l = 0
  al1 = (m1 == -INFINITY) ? 0.f : exp2f(m1 - mn1);
  m0 = mn0;
  m1 = mn1;
  l0 *= al0;
  l1 *= al1;
  const float nm0 = (mn0 == -INFINITY) ? 0.f : -mn0;   // a fully masked row so far: exp2(-inf) = 0
  const float nm1 = (mn1 == -INFINITY) ? 0.f : -mn1;
#pragma unroll
  for (int c = 0; c < AKV / 8; ++c) {
    // POLY: the n8 blocks c = 3, 7 (one column pair in four) go to the FMA pipe, the rest to MUFU
    const bool poly = POLY && (c & 3) == 3;
    const float x0 = fmaf(s[4 * c], p.scale_log2, nm0), x1 = fmaf(s[4 * c + 1], p.scale_log2, nm0);
    const float x2 = fmaf(s[4 * c + 2], p.scale_log2, nm1), x3 = fmaf(s[4 * c + 3], p.scale_log2, nm1);
    s[4 * c] = poly ? poly_exp2(x0) : fast_exp2(x0);
    s[4 * c + 1] = poly ? poly_exp2(x1) : fast_exp2(x1);
    s[4 * c + 2] = poly ? poly_exp2(x2) : fast_exp2(x2);
    s[4 * c + 3] = poly ? poly_exp2(x3) : fast_exp2(x3);
    l0 += s[4 * c] + s[4 * c + 1];
    l1 += s[4 * c + 2] + s[4 * c + 3];
  }
}

// P (fp16) in the A-operand layout of wgmma: for key step kk, {row qi0 keys 2 t4 .. +1, row qi1 same, row qi0
// keys 8 + 2 t4 .. +1, row qi1 same} = the S fragments of n8 blocks 2 kk and 2 kk + 1
__device__ __forceinline__ void pack_p(uint32_t (&pa)[AKV / 16][4], const float (&s)[AKV / 2]) {
#pragma unroll
  for (int c = 0; c < AKV / 8; ++c) {
    pa[c >> 1][(c & 1) * 2] = pack_half2(s[4 * c], s[4 * c + 1]);
    pa[c >> 1][(c & 1) * 2 + 1] = pack_half2(s[4 * c + 2], s[4 * c + 3]);
  }
}

template <int DV>
__device__ __forceinline__ void rescale_o(float (&o)[DV / 2], float al0, float al1) {
#pragma unroll
  for (int c = 0; c < DV / 8; ++c) {
    o[4 * c] *= al0;
    o[4 * c + 1] *= al0;
    o[4 * c + 2] *= al1;
    o[4 * c + 3] *= al1;
  }
}

template <int DPAD, int DV>
__global__ void __launch_bounds__(ATT_THREADS, 1)
    attention_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                        const __grid_constant__ CUtensorMap tmV, const AttnArgs p) {
  using Cfg = AttnCfg<DPAD, DV>;
  constexpr bool WIDE = attn_wide(DPAD);
  constexpr bool STREAM_Q = Cfg::STREAM_Q;
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
      // tensor maps: Q / K {d, heads, rows, batch}, V^T {nkv, d, heads, batch}
      if constexpr (!STREAM_Q) {
        mbar_arrive_expect_tx(&q_full, Cfg::Q_BYTES);
        for (int pn = 0; pn < PANELS; ++pn) tma_load_4d(q_s + pn * (AQ * 128), &tmQ, &q_full, pn * 64, head, q0, b);
      }
      int ks = 0;
      uint32_t kph = 0;
      for (int j = 0; j < n_iter; ++j) {
        for (int pn = 0; pn < PANELS; ++pn) {
          mbar_wait_mma(&k_empty[ks], kph ^ 1);
          if constexpr (STREAM_Q) {   // the stage's Q panel rides on the K panel's barrier
            mbar_arrive_expect_tx(&k_full[ks], Cfg::KP_BYTES + Cfg::QP_BYTES);
            tma_load_4d(q_s + ks * Cfg::QP_BYTES, &tmQ, &k_full[ks], pn * 64, head, q0, b);
          } else {
            mbar_arrive_expect_tx(&k_full[ks], Cfg::KP_BYTES);
          }
          tma_load_4d(k_s + ks * Cfg::KP_BYTES, &tmK, &k_full[ks], pn * 64, head, j * AKV, b);
          if (++ks == KST) {
            ks = 0;
            kph ^= 1;
          }
        }
        const int vs = j % VST;
        mbar_wait_mma(&v_empty[vs], ((j / VST) & 1) ^ 1);
        mbar_arrive_expect_tx(&v_full[vs], Cfg::V_TX);
        tma_load_4d(v_s + vs * Cfg::V_BYTES, &tmV, &v_full[vs], j * AKV, dv0, head, b);
      }
    }
    __syncwarp();
  } else {
    const int wg = warp >> 2;
    const int t4 = lane & 3;
    const int qi0 = q0 + 64 * wg + 16 * (warp & 3) + (lane >> 2);   // fragment rows of this thread: qi0, qi0 + 8
    const int qi1 = qi0 + 8;
    // head dimension d < DPAD: columns d .. DPAD-1 of the Q / K panels are zero fill; only the 16-wide K steps that
    // hold real columns are issued for S
    const int ksteps = (p.d + 15) >> 4;
    const uint32_t q_addr = smem_u32(q_s) + static_cast<uint32_t>(wg * 64 * 128);
    float o[DV / 2];
#pragma unroll
    for (int i = 0; i < DV / 2; ++i) o[i] = 0.f;
    float s[AKV / 2];
#pragma unroll
    for (int i = 0; i < AKV / 2; ++i) s[i] = 0.f;
    uint32_t pa[AKV / 16][4];
    float m0 = -INFINITY, m1 = -INFINITY;   // running maxima (log2 domain) of rows qi0 / qi1
    float l0 = 0.f, l1 = 0.f;               // this thread's share of the row sums
    float al0, al1;
    int ks = 0;
    uint32_t kph = 0;
    if constexpr (!STREAM_Q) mbar_wait_mma(&q_full, 0);
    if constexpr (WIDE) {
      for (int j = 0; j < n_iter; ++j) {
        // ---- S = Q K^T over the K panels of this tile; each panel is handed back once its MMAs have completed
        wgmma_hold(s);
        int prev = -1;
#pragma unroll 1
        for (int pn = 0; pn < PANELS; ++pn) {
          mbar_wait_mma(&k_full[ks], kph);
          const uint32_t k_addr = smem_u32(k_s + ks * Cfg::KP_BYTES);
          const uint32_t qp_addr = STREAM_Q ? q_addr + ks * Cfg::QP_BYTES : q_addr + pn * Cfg::QP_BYTES;
          wgmma_fence();
#pragma unroll
          for (int kk = 0; kk < 4; ++kk)
            WgmmaSS<AKV>::mma(s, wg_desc(qp_addr + kk * 32), wg_desc(k_addr + kk * 32), (pn | kk) != 0);
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
        softmax_tile<false>(s, p, j * AKV, q0, qi0, qi1, t4, m0, m1, l0, l1, al0, al1);
        rescale_o<DV>(o, al0, al1);
        pack_p(pa, s);

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
    } else {
      // Every wgmma below is issued unconditionally (a data-dependent branch around one makes ptxas serialise them
      // all), hence the peeled first and last windows. S issues ceil16(DV) K steps: for DV = ceil8(d) that is
      // ceil16(d); where DV = DPAD the steps past d multiply the zero-filled panel columns.
      constexpr int KSTEPS = (DV + 15) / 16;
      auto issue_s = [&]() {   // S_j = Q K_j^T over the tile's panels (ring slots ks .. ks + PANELS - 1), one group
#pragma unroll
        for (int pn = 0; pn < PANELS; ++pn) {
          mbar_wait_mma(&k_full[ks + pn], kph);
          const uint32_t k_addr = smem_u32(k_s + (ks + pn) * Cfg::KP_BYTES);
#pragma unroll
          for (int kk = 0; kk < 4; ++kk)
            if (pn * 4 + kk < KSTEPS)
              WgmmaSS<AKV>::mma(s, wg_desc(q_addr + pn * (AQ * 128) + kk * 32), wg_desc(k_addr + kk * 32),
                                (pn | kk) != 0);
        }
        wgmma_commit();
      };
      auto release_k = [&]() {   // KST is a multiple of PANELS: a tile's panels never straddle the ring's end
        if (lane == 0)
#pragma unroll
          for (int pn = 0; pn < PANELS; ++pn) mbar_arrive(&k_empty[ks + pn]);
        ks += PANELS;
        if (ks == KST) {
          ks = 0;
          kph ^= 1;
        }
      };
      auto issue_pv = [&](int jv) {   // O += P_jv V_jv
        const int vs = jv % VST;
        mbar_wait_mma(&v_full[vs], (jv / VST) & 1);
        const uint32_t v_addr = smem_u32(v_s + vs * Cfg::V_BYTES);
#pragma unroll
        for (int kk = 0; kk < AKV / 16; ++kk) WgmmaRS<DV>::mma(o, pa[kk], wg_desc(v_addr + kk * 32), 1u);
        wgmma_commit();
      };
      // Turn order: warpgroup 1 hands warpgroup 0 the first turn; each warpgroup then takes n_iter + 1 turns and
      // passes on every one except warpgroup 1's last, so both named barriers end with no pending arrivals.
      if (wg == 1) wg_turn_pass(wg);
      wg_turn_wait(wg);
      wgmma_fence();
      issue_s();
      wg_turn_pass(wg);
      wgmma_wait<0>();
      wgmma_hold(s);
      release_k();
      softmax_tile<true>(s, p, 0, q0, qi0, qi1, t4, m0, m1, l0, l1, al0, al1);
      pack_p(pa, s);
      for (int j = 1; j < n_iter; ++j) {
        wg_turn_wait(wg);
        wgmma_hold(s);
        wgmma_hold(o);
        wgmma_fence();
        issue_s();
        issue_pv(j - 1);
        wg_turn_pass(wg);
        wgmma_wait<1>();   // S_j is done; PV_{j-1}, committed after it, may still run under the softmax
        wgmma_hold(s);
        release_k();
        softmax_tile<true>(s, p, j * AKV, q0, qi0, qi1, t4, m0, m1, l0, l1, al0, al1);
        wgmma_wait<0>();
        wgmma_hold(o);
        if (lane == 0) mbar_arrive(&v_empty[(j - 1) % VST]);
        rescale_o<DV>(o, al0, al1);
        pack_p(pa, s);
      }
      wg_turn_wait(wg);
      wgmma_hold(o);
      wgmma_fence();
      issue_pv(n_iter - 1);
      if (wg == 0) wg_turn_pass(wg);
      wgmma_wait<0>();
      wgmma_hold(o);
      if (lane == 0) mbar_arrive(&v_empty[(n_iter - 1) % VST]);
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

// Q / K as {d, heads, rows, batch} (head h of row r at element r * ld + h * hs), V^T as {nkv, d, heads, batch}
// (channel c of head h at row h * hs + c). The innermost extent is d, so a 64-wide panel box reads columns d .. 63 and
// a DV-row V^T box reads rows d .. DV-1 as zeros.
static int make_attn_maps(const sdb_attn_desc* d, int heads, int hd, int hs, uint32_t dv_box, CUtensorMap* tq,
                          CUtensorMap* tk, CUtensorMap* tv) {
  const uint64_t h = static_cast<uint64_t>(heads), dd = static_cast<uint64_t>(hd), e = 2;
  {
    uint64_t dims[4] = {dd, h, static_cast<uint64_t>(d->nq), static_cast<uint64_t>(d->batch)};
    uint64_t str[3] = {hs * e, static_cast<uint64_t>(d->ldq) * e, static_cast<uint64_t>(d->q_batch_stride) * e};
    uint32_t box[4] = {64, 1, AQ, 1};
    if (make_tmap_f16(tq, d->q, 4, dims, str, box)) return 1;
  }
  {
    uint64_t dims[4] = {dd, h, static_cast<uint64_t>(d->nkv), static_cast<uint64_t>(d->batch)};
    uint64_t str[3] = {hs * e, static_cast<uint64_t>(d->ldk) * e, static_cast<uint64_t>(d->k_batch_stride) * e};
    uint32_t box[4] = {64, 1, AKV, 1};
    if (make_tmap_f16(tk, d->k, 4, dims, str, box)) return 1;
  }
  {
    uint64_t dims[4] = {static_cast<uint64_t>(d->nkv), dd, h, static_cast<uint64_t>(d->batch)};
    uint64_t str[3] = {static_cast<uint64_t>(d->ldvt) * e, static_cast<uint64_t>(hs) * d->ldvt * e,
                       static_cast<uint64_t>(d->vt_batch_stride) * e};
    uint32_t box[4] = {AKV, dv_box, 1, 1};
    if (make_tmap_f16(tv, d->vt, 4, dims, str, box)) return 1;
  }
  return 0;
}

// PV width for head dim d in a dpad-column slot: ceil8(d) for the head dims of the engine's models, else the slot
// width; 0 where no instantiation exists (d > 160 in a 192 slot: PV at N = 192 next to S spills registers)
static uint32_t attn_dv(int dpad, int d) {
  const int dv = (d + 7) / 8 * 8;
  switch (dpad) {
    case 64: return dv <= 48 ? dv : 64;
    case 128: return (dv == 80 || dv == 96) ? dv : 128;
    default: return dv <= 160 ? 160 : 0;
  }
}

}  // namespace sdb

using namespace sdb;

extern "C" int sdb_attention(const sdb_attn_desc* d, sdb_stream_t stream) {
  if (d && ::sdb::plan_recording()) {
    const sdb_attn_desc c = *d;
    ::sdb::plan_record([c](cudaStream_t s_) { return sdb_attention(&c, s_); });
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  SDB_CHECK(d && d->q && d->k && d->vt && d->out, "sdb_attention: null pointer");
  // softmax_tile takes (row maximum of q.k) * scale as the maximum of the scaled logits
  SDB_CHECK(d->scale > 0 && isfinite(d->scale), "sdb_attention: scale must be positive and finite (got %g)", d->scale);
  CUtensorMap tq, tk, tv;
  AttnArgs p{};
  p.nq = d->nq;
  p.nkv = d->nkv;
  p.d = d->d;
  p.ldo = d->ldo;
  p.o_batch_stride = d->o_batch_stride;
  p.out = static_cast<__half*>(d->out);
  p.scale_log2 = d->scale * 1.4426950408889634f;
  if (d->dpad == 384 || d->dpad == 512 || d->dpad == 576 || d->dpad == 960) {
    // single-head d = dpad (AutoencoderKL AttnBlock at 512, num_heads-1 SpatialTransformers at 384 / 576 / 960):
    // q, k [B, n, d], vt [B, d, ldvt]
    const int dp = d->dpad;
    SDB_CHECK(d->d == dp && d->heads == 1 && !d->causal,
              "sdb_attention: dpad %d is the single-head d = %d kernel (got d %d, heads %d, causal %d)", dp, dp, d->d,
              d->heads, d->causal);
    SDB_CHECK(d->head_stride == 0 || d->head_stride == dp, "sdb_attention: dpad %d takes head_stride 0 or %d", dp, dp);
    SDB_CHECK(d->batch > 0 && d->nq > 0 && d->nkv > 0, "sdb_attention: bad sizes");
    SDB_CHECK(d->ldq % 8 == 0 && d->ldk % 8 == 0 && d->ldvt % 8 == 0 && d->ldo % 8 == 0 && d->o_batch_stride % 8 == 0,
              "sdb_attention: leading dims must be multiples of 8");
    const int dv = dp == 576 ? 96 : (dp == 960 ? 160 : 128);   // PV slice width: dp / dv slices, S recomputed per slice
    if (make_attn_maps(d, 1, dp, dp, dv, &tq, &tk, &tv)) return 1;
    p.heads = 1;
    p.causal = 0;
    dim3 grid((d->nq + AQ - 1) / AQ, dp / dv, d->batch);
    switch (dp) {
      case 384: return launch_attn<384, 128>(tq, tk, tv, p, grid, st);
      case 512: return launch_attn<512, 128>(tq, tk, tv, p, grid, st);
      case 576: return launch_attn<576, 96>(tq, tk, tv, p, grid, st);
      default: return launch_attn<960, 160>(tq, tk, tv, p, grid, st);
    }
  }
  SDB_CHECK(d->dpad == 64 || d->dpad == 128 || d->dpad == 192,
            "sdb_attention: dpad must be 64/128/192/384/512/576/960 (got %d)", d->dpad);
  SDB_CHECK(d->d > 0 && d->d <= d->dpad && d->d % 2 == 0, "sdb_attention: bad head dim %d", d->d);
  const int hs = d->head_stride ? d->head_stride : d->dpad;
  SDB_CHECK(hs >= d->d && hs % 8 == 0, "sdb_attention: head_stride %d must be >= d and a multiple of 8", hs);
  SDB_CHECK(d->batch > 0 && d->heads > 0 && d->nq > 0 && d->nkv > 0, "sdb_attention: bad sizes");
  SDB_CHECK(d->ldq % 8 == 0 && d->ldk % 8 == 0 && d->ldvt % 8 == 0, "sdb_attention: leading dims must be multiples of 8");
  SDB_CHECK(d->ldo % 2 == 0 && d->o_batch_stride % 2 == 0, "sdb_attention: output stride must be even");
  const uint32_t dv = attn_dv(d->dpad, d->d);
  SDB_CHECK(dv != 0, "sdb_attention: no kernel for head dim %d in dpad %d", d->d, d->dpad);
  if (make_attn_maps(d, d->heads, d->d, hs, dv, &tq, &tk, &tv)) return 1;
  p.heads = d->heads;
  p.causal = d->causal;
  dim3 grid((d->nq + AQ - 1) / AQ, d->heads, d->batch);
#define SDB_ATTN(DP, W) \
  if (d->dpad == (DP) && dv == (W)) return launch_attn<DP, W>(tq, tk, tv, p, grid, st);
  SDB_ATTN(64, 8) SDB_ATTN(64, 16) SDB_ATTN(64, 24) SDB_ATTN(64, 32) SDB_ATTN(64, 40) SDB_ATTN(64, 48) SDB_ATTN(64, 64)
  SDB_ATTN(128, 80) SDB_ATTN(128, 96) SDB_ATTN(128, 128)
  SDB_ATTN(192, 160)
#undef SDB_ATTN
  SDB_CHECK(false, "sdb_attention: no kernel for head dim %d in dpad %d", d->d, d->dpad);
  return 1;
}
