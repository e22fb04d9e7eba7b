// Host side of sdb_gemm: tile-shape model, tensor maps, epilogue-kind dispatch. The kernel lives in gemm_kernel.cuh and
// is instantiated per epilogue KIND in gemm_k0.cu / gemm_k1.cu / gemm_k2.cu (compiled in parallel).
#include "gemm_kernel.cuh"

namespace sdb {

// ------------------------------------------------------------------------------------------------ host side
struct Choice {
  int bn, cg, splits, csk;
};

struct Geometry {   // everything about a problem that does not depend on the tile choice
  long M;
  int k_iters, cpt;
  long m_tiles;
  int TW, TH, TN, tiles_x, tiles_y;
  int rps;
  bool geglu, want_stats, fast_possible;
  int sg;
};

static int pow2_divisor(int v, int cap) {
  int p = 1;
  while (p * 2 <= cap && v % (p * 2) == 0) p *= 2;
  return p;
}

// Statistics slots per sample (0: this tile choice cannot produce fused statistics)
static int stats_slots(const sdb_gemm_desc* d, const Geometry& g, const Choice& c, int* halves_out) {
  int halves = 1;
  if (g.sg <= 0 || d->n % g.sg != 0) return 0;
  if (!g.fast_possible || !d->out_f32 || g.geglu) return 0;   // statistics come from the staged fp32 tile of the TMA-store path
  if (c.splits > 1 && !c.csk) {   // workspace split-K: the second kernel produces them per 32-row block
    if (g.rps % 32 != 0 || d->n % 4 != 0) return 0;
    const int cb = (d->n % 160 == 0 && 160 % g.sg == 0) ? 160 : 128;
    if (cb % g.sg != 0) return 0;
    *halves_out = 1;
    return g.rps / 32;
  }
  if (c.bn % g.sg != 0) return 0;
  int T;
  if (d->taps == 1) {
    if (g.rps % 128 == 0) T = g.rps / 128;
    else if (g.rps == 64) { T = 1; halves = 2; }
    else return 0;
  } else {
    if (g.rps != d->h * d->w) return 0;
    T = g.tiles_x * g.tiles_y;                                       // one slot per spatial tile position
    if (g.TN == 1) halves = 1;                                       // TW * TH == 128: a tile lies inside one sample
    else if (g.TW * g.TH == 64 && g.TN == 2) halves = 2;             // 64-pixel tiles of two consecutive samples
    else return 0;
  }
  *halves_out = halves;
  return c.csk ? T * c.splits : T;
}

static bool choice_valid(const sdb_gemm_desc* d, const Geometry& g, const Choice& c) {
  if (!(c.bn == 32 || c.bn == 64 || c.bn == 128 || c.bn == 160 || c.bn == 256)) return false;
  if (c.cg == 2 && (c.bn < 128 || g.m_tiles < 2)) return false;
  if (g.geglu && (c.splits > 1 || (c.bn != 128 && c.bn != 256))) return false;
  if (c.splits < 1 || c.splits > g.k_iters) return false;
  if (c.csk) {
    const int ips = (g.k_iters + c.splits - 1) / c.splits;
    if ((g.k_iters + ips - 1) / ips != c.splits) return false;   // every CTA of the cluster needs a non-empty K slice
    if (!(c.splits == 2 || c.splits == 4) || c.splits * c.cg > 8 || !g.fast_possible || g.geglu) return false;
    if (g.k_iters / c.splits < 2) return false;
  } else if (c.splits > 1) {
    if (d->workspace == nullptr) return false;
    if (d->workspace_floats > 0 && static_cast<long>(c.splits) * g.M * d->n > d->workspace_floats) return false;
  }
  if (g.want_stats) {
    int h;
    if (stats_slots(d, g, c, &h) == 0) return false;
  }
  return true;
}

// Tile model used to pick (block_n, CTA pair, split-K). Every CTA computes one tile with its main loop and epilogue in
// sequence, one CTA per SM, so a launch is waves of (main loop + epilogue + pipeline fill). A main loop is bound by the
// tensor pipe (4*bn clk per 64-deep K step of a 128-row tile on an H100 SM) or by L2 -> SM operand traffic (~64 B/clk
// per SM, ~3000 B/clk chip-wide); a CTA pair halves the B bytes per CTA, split-K keeps tiles large at small M.
static double choice_cost(const sdb_gemm_desc* d, const Geometry& g, const Choice& c) {
  const int sms = sm_count();
  const long nt = (d->n + c.bn - 1) / c.bn;
  const long m_units = (g.m_tiles + c.cg - 1) / c.cg;
  const long units = m_units * nt * c.splits;            // CTA (pair) work items
  const long ctas = units * c.cg;
  const int iters = (g.k_iters + c.splits - 1) / c.splits;
  const double stage_bytes = 16384.0 + (c.bn / c.cg) * 128.0;
  long slots = c.csk ? std::max(1, sms / (c.splits * c.cg)) * (c.splits * c.cg) : (sms / c.cg) * c.cg;
  const long rounds = (ctas + slots - 1) / slots;
  const double t_tile = std::max(iters * 4.0 * c.bn, iters * stage_bytes / 64.0) + 1800.0 + 14.0 * c.bn + 3000.0;
  const double t_l2_chip = static_cast<double>(ctas) * iters * stage_bytes / 3000.0;
  double t = std::max(rounds * t_tile, t_l2_chip);
  t += 4000.0;                                  // launch
  if (c.csk) t += 2500.0 + 128.0 * c.bn * 4.0 * (c.splits - 1) / c.splits / 20.0;
  else if (c.splits > 1) t += 14000.0 + 8.0 * c.splits * g.M * d->n / (sms * 256.0);
  const long pad = nt * c.bn - d->n;             // zero-padded columns still cost MMA + B traffic
  if (pad > 0) t *= 1.0 + 0.5 * static_cast<double>(pad) / (nt * c.bn);
  return t;
}

static bool relu_family(int act) { return act == SDB_ACT_RELU || act == SDB_ACT_LEAKY_RELU; }

static int make_geometry(const sdb_gemm_desc* d, Geometry* g) {
  SDB_CHECK((d->act >= SDB_ACT_NONE && d->act <= SDB_ACT_GELU) || relu_family(d->act), "sdb_gemm: unknown activation %d",
            d->act);
  const void* srcs[MAX_SRC] = {d->a0, d->a1, d->a2, d->a3};
  const int chans[MAX_SRC] = {d->c0, d->c1, d->c2, d->c3};
  int nsrc = 0, chunks = 0;
  for (int i = 0; i < MAX_SRC; ++i) {
    if (srcs[i] == nullptr) break;
    // a width that is a multiple of 32 only takes ceil(c / 64) K steps: the A map keeps dims[0] = c, so TMA's
    // out-of-bounds fill supplies zeros for the channels c .. ceil64(c) - 1 of the last step
    SDB_CHECK(chans[i] > 0 && chans[i] % 32 == 0,
              "sdb_gemm: channel count of source %d must be a positive multiple of 64, or of 32 (tail zero-filled) (got %d)",
              i, chans[i]);
    ++nsrc;
    chunks += (chans[i] + 63) / 64;
  }
  for (int i = nsrc; i < MAX_SRC; ++i)
    SDB_CHECK(srcs[i] == nullptr && chans[i] == 0, "sdb_gemm: A sources must be contiguous (a%d/c%d)", i, i);
  g->M = static_cast<long>(d->nb) * d->h * d->w;
  SDB_CHECK(g->M < (1L << 31), "sdb_gemm: M too large");
  g->cpt = chunks;
  g->k_iters = d->taps * chunks;
  g->geglu = d->act == SDB_ACT_GEGLU;
  g->rps = d->rows_per_sample > 0 ? d->rows_per_sample : d->h * d->w;
  if (d->taps == 1) {
    g->TW = 128;
    g->TH = 1;
    g->TN = 1;
    g->tiles_x = static_cast<int>((g->M + 127) / 128);
    g->tiles_y = 1;
    g->m_tiles = g->tiles_x;
  } else {
    g->TW = pow2_divisor(d->w, 128);
    g->TH = pow2_divisor(d->h, 128 / g->TW);
    g->TN = 128 / (g->TW * g->TH);
    g->tiles_x = d->w / g->TW;
    g->tiles_y = (d->h + g->TH - 1) / g->TH;
    g->m_tiles = static_cast<long>(g->tiles_x) * g->tiles_y * ((d->nb + g->TN - 1) / g->TN);
  }
  g->want_stats = d->stats_out != nullptr;
  g->sg = d->stats_group > 0 ? d->stats_group : 1;
  const int n_out = g->geglu ? d->n / 2 : d->n;
  const int ldo = d->ldo > 0 ? d->ldo : n_out;
  const int ldf = d->ldf > 0 ? d->ldf : d->n;
  const int ldr = d->ldr > 0 ? d->ldr : d->n;
  auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  g->fast_possible = (n_out % 32 == 0) && (ldo % 8 == 0) && (!d->bias || al16(d->bias)) &&
                     (!d->film || (al16(d->film) && ldf % 4 == 0)) && (!d->residual || (al16(d->residual) && ldr % 4 == 0)) &&
                     (!d->out_f32 || al16(d->out_f32)) && (!d->out_f16 || al16(d->out_f16)) &&
                     (!d->out_f16_lo || al16(d->out_f16_lo));
  return 0;
}

// Resolve (block_n, pair, split-K) for a problem: explicit requests of the descriptor are honoured, the rest is picked
// by the tile model.
static int resolve_choice(const sdb_gemm_desc* d, const Geometry& g, Choice* out) {
  const int bns[] = {256, 160, 128, 64, 32};
  const int sps[] = {1, 2, 3, 4, 6, 8, 12, 16, 24, 32};
  int want_splits = d->splits;                      // >1 explicit, 0/1 none, -1 auto
  if (relu_family(d->act)) want_splits = 1;         // kind 4 runs unsplit (the split-K second pass has no ReLU)
  if (want_splits > g.k_iters) want_splits = g.k_iters;
  Choice best{0, 1, 1, 0};
  double best_t = 1e300;
  for (int bn : bns) {
    if (d->block_n > 0 && bn != d->block_n) continue;
    if (g.geglu && d->block_n <= 0 && bn != 128) continue;    // GEGLU weights are packed per tile: 128 unless told
    if (d->block_n <= 0 && bn > 32 && ((d->n + bn - 1) / bn) * bn - d->n >= bn / 2 && d->n > 32) continue;  // mostly padding
    for (int cg = 1; cg <= 2; ++cg) {
      if (d->pair == 1 && cg != 1) continue;
      if (d->pair == 2 && cg != 2) continue;
      for (int mode = 0; mode < 2; ++mode) {        // 0: workspace (or no) split-K, 1: cluster split-K
        if (d->splitk_mode == 1 && mode == 1) continue;
        if (d->splitk_mode == 2 && mode == 0 && want_splits != 0 && want_splits != 1 && want_splits != -1) continue;
        for (int spi : sps) {
          int sp = spi;
          if (want_splits > 1) {      // explicit factor: try exactly that one
            if (spi != 1) continue;
            sp = want_splits;
          }
          if (mode == 1 && sp == 1) continue;
          if ((want_splits == 0 || want_splits == 1) && sp != 1) continue;
          Choice c{bn, cg, sp, mode};
          if (!choice_valid(d, g, c)) continue;
          const double t = choice_cost(d, g, c);
          if (t < best_t) {
            best_t = t;
            best = c;
          }
        }
      }
    }
  }
  SDB_CHECK(best.bn != 0, "sdb_gemm: no valid tile configuration (block_n %d, pair %d, splits %d, mode %d%s)", d->block_n,
            d->pair, d->splits, d->splitk_mode, g.want_stats ? ", fused statistics requested" : "");
  *out = best;
  return 0;
}

}  // namespace sdb

using namespace sdb;

extern "C" int sdb_gemm_plan(const sdb_gemm_desc* d, int32_t* out) {
  SDB_CHECK(d && out, "sdb_gemm_plan: null argument");
  SDB_CHECK(d->taps == 1 || d->taps == 9, "sdb_gemm: taps must be 1 or 9 (got %d)", d->taps);
  Geometry g;
  if (make_geometry(d, &g)) return 1;
  Choice c;
  if (resolve_choice(d, g, &c)) return 1;
  int halves = 1;
  out[0] = c.bn;
  out[1] = c.cg;
  out[2] = c.splits;
  out[3] = c.splits > 1 ? (c.csk ? 2 : 1) : 0;
  out[4] = g.want_stats ? stats_slots(d, g, c, &halves) : 0;
  return 0;
}

extern "C" int sdb_gemm(const sdb_gemm_desc* d, sdb_stream_t stream) {
  if (d && ::sdb::plan_recording()) {
    const sdb_gemm_desc c = *d;
    ::sdb::plan_record([c](cudaStream_t s_) { return sdb_gemm(&c, s_); });
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  SDB_CHECK(d && d->a0 && d->b, "sdb_gemm: null operand");
  SDB_CHECK(d->taps == 1 || d->taps == 9, "sdb_gemm: taps must be 1 or 9 (got %d)", d->taps);
  const void* srcs[MAX_SRC] = {d->a0, d->a1, d->a2, d->a3};
  const int chans[MAX_SRC] = {d->c0, d->c1, d->c2, d->c3};
  SDB_CHECK(d->nb > 0 && d->h > 0 && d->w > 0 && d->n > 0, "sdb_gemm: bad dims");
  SDB_CHECK(d->out_f16 || d->out_f32, "sdb_gemm: no output");
  SDB_CHECK(!d->out_f16_lo || d->out_f16, "sdb_gemm: out_f16_lo needs out_f16");
  const int cstride = d->conv_stride > 1 ? d->conv_stride : 1;
  SDB_CHECK(cstride == 1 || (cstride == 2 && d->taps == 9), "sdb_gemm: conv_stride must be 1 or 2 (3x3 convs only)");
  SDB_CHECK(d->conv_shift == 0 || d->taps == 9, "sdb_gemm: conv_shift applies to 3x3 convs only");
  const int in_h = d->in_h > 0 ? d->in_h : d->h, in_w = d->in_w > 0 ? d->in_w : d->w;
  SDB_CHECK((in_h == d->h && in_w == d->w) || d->taps == 9, "sdb_gemm: in_h / in_w apply to 3x3 convs only");
  Geometry g;
  if (make_geometry(d, &g)) return 1;
  const bool geglu = g.geglu;
  if (geglu) {
    SDB_CHECK(d->n % 128 == 0, "sdb_gemm: GEGLU needs n %% 128 == 0");
    SDB_CHECK(!d->film && !d->residual && d->splits <= 1, "sdb_gemm: GEGLU epilogue excludes film/residual/split-K");
  }
  if (g.want_stats)
    SDB_CHECK(g.fast_possible && d->out_f32 && !geglu, "sdb_gemm: stats_out needs the TMA-store epilogue with an fp32 output");
  Choice ch;
  if (resolve_choice(d, g, &ch)) return 1;
  const int bn = ch.bn, splits_req = ch.splits;
  SDB_CHECK(!geglu || d->n % bn == 0, "sdb_gemm: GEGLU needs n %% block_n == 0");

  GemmArgs p{};
  int nsrc = 0;
  for (int i = 0; i < MAX_SRC && srcs[i]; ++i) ++nsrc;
  const long M = g.M;
  p.M = static_cast<int>(M);
  p.N = d->n;
  p.taps = d->taps;
  p.nsrc = nsrc;
  p.cb[0] = 0;
  for (int i = 0; i < nsrc; ++i) p.cb[i + 1] = p.cb[i] + (chans[i] + 63) / 64;
  for (int i = nsrc; i < MAX_SRC; ++i) p.cb[i + 1] = p.cb[nsrc];
  p.k_iters = g.k_iters;
  p.H = d->h;
  p.W = d->w;
  p.NB = d->nb;
  p.cstride = cstride;
  p.cshift = d->conv_shift;
  p.alpha = d->alpha == 0.f ? 1.f : d->alpha;
  p.bias = d->bias;
  p.film = d->film;
  p.ldf = d->ldf > 0 ? d->ldf : d->n;
  p.rows_per_sample = g.rps;
  p.residual = d->residual;
  p.ldr = d->ldr > 0 ? d->ldr : d->n;
  p.out_f16 = static_cast<__half*>(d->out_f16);
  p.out_f16_lo = static_cast<__half*>(d->out_f16_lo);
  p.out_f32 = d->out_f32;
  p.act = d->act;
  p.b_static = d->b_dynamic ? 0 : 1;
  const int n_out = geglu ? d->n / 2 : d->n;
  p.ldo = d->ldo > 0 ? d->ldo : n_out;
  p.lw = 0;
  p.lh = 0;
  while ((1 << p.lw) < g.TW) ++p.lw;
  while ((1 << p.lh) < g.TH) ++p.lh;
  p.TW = g.TW;
  p.TH = g.TH;
  p.TN = g.TN;
  p.tiles_x = g.tiles_x;
  p.tiles_y = g.tiles_y;
  const long m_tiles = g.m_tiles;

  p.iters_per_split = (p.k_iters + splits_req - 1) / splits_req;
  int splits = (p.k_iters + p.iters_per_split - 1) / p.iters_per_split;
  p.csk = (ch.csk && splits == splits_req && splits > 1) ? 1 : 0;
  if (ch.csk && !p.csk) {   // the K slices do not divide evenly enough: fall back to an unsplit launch
    splits = 1;
    p.iters_per_split = p.k_iters;
  }
  if (splits > 1 && !p.csk) {
    SDB_CHECK(d->workspace != nullptr, "sdb_gemm: split-K needs a workspace");
    SDB_CHECK(d->workspace_floats <= 0 || static_cast<long>(splits) * M * d->n <= d->workspace_floats,
              "sdb_gemm: split-K workspace too small");
    p.ws = d->workspace;
  }
  p.splits = splits;
  p.m_tiles = static_cast<int>(m_tiles);
  p.m_units = static_cast<int>((m_tiles + ch.cg - 1) / ch.cg);
  p.n_tiles = (d->n + bn - 1) / bn;
  SDB_CHECK(m_tiles * p.n_tiles * splits < (1L << 30), "sdb_gemm: too many tiles");

  // tensor maps
  TmapPack tm;
  for (int i = 0; i < nsrc; ++i) {
    const int c = chans[i];
    if (d->taps == 1) {
      uint64_t dims[4] = {static_cast<uint64_t>(c), static_cast<uint64_t>(M), 1, 1};
      uint64_t str[3] = {static_cast<uint64_t>(c) * 2, static_cast<uint64_t>(c) * 2 * M,
                         static_cast<uint64_t>(c) * 2 * M};
      uint32_t box[4] = {64, 128, 1, 1};
      if (make_tmap_f16(&tm.a[i], srcs[i], 4, dims, str, box)) return 1;
    } else {
      // the INPUT image; a stride-2 conv traverses it with element strides {1, 2, 2, 1}: a box of 2*TW x 2*TH input
      // positions delivers the TW x TH pixels one tap of the output tile needs
      uint64_t dims[4] = {static_cast<uint64_t>(c), static_cast<uint64_t>(in_w), static_cast<uint64_t>(in_h),
                          static_cast<uint64_t>(d->nb)};
      uint64_t str[3] = {static_cast<uint64_t>(c) * 2, static_cast<uint64_t>(c) * 2 * in_w,
                         static_cast<uint64_t>(c) * 2 * in_w * in_h};
      uint32_t box[4] = {64, static_cast<uint32_t>(p.TW * cstride), static_cast<uint32_t>(p.TH * cstride),
                         static_cast<uint32_t>(p.TN)};
      uint32_t est[4] = {1, static_cast<uint32_t>(cstride), static_cast<uint32_t>(cstride), 1};
      SDB_CHECK(box[1] <= 256 && box[2] <= 256, "sdb_gemm: strided box too large");
      if (make_tmap(&tm.a[i], srcs[i], 2, 128, 4, dims, str, box, est)) return 1;
    }
  }
  for (int i = nsrc; i < MAX_SRC; ++i) tm.a[i] = tm.a[0];
  {
    // B rows: taps * sum(ceil64(c_i)) columns, each source's padded tail zero; one source of one tap may be exactly
    // c wide (the tail step then reads TMA's out-of-bounds zeros, as for A)
    const uint64_t K = (nsrc == 1 && d->taps == 1) ? static_cast<uint64_t>(chans[0])
                                                    : static_cast<uint64_t>(d->taps) * g.cpt * 64;
    uint64_t dims[2] = {K, static_cast<uint64_t>(d->n)};
    uint64_t str[1] = {K * 2};
    uint32_t box[2] = {64, static_cast<uint32_t>(bn / ch.cg)};   // a CTA of a pair loads (and multicasts) half of the weight tile
    if (make_tmap_f16(&tm.b, d->b, 2, dims, str, box)) return 1;
  }
  // output maps for the TMA-store epilogue (fast path); otherwise the scalar transposed path is used
  auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  bool fast = g.fast_possible && (!p.ws || (d->n % 32 == 0 && al16(p.ws)));
  p.fast = fast ? 1 : 0;
  SDB_CHECK(!p.csk || fast, "sdb_gemm: cluster split-K needs the TMA-store epilogue");
  p.bw = d->taps == 1 ? 32 : std::min(p.TW, 32);
  p.bh = d->taps == 1 ? 1 : std::min(p.TH, 32 / p.bw);
  tm.o32 = tm.b;
  tm.o16 = tm.b;
  tm.o16lo = tm.b;
  tm.ows = tm.b;
  if (fast) {
    const uint32_t bnn = static_cast<uint32_t>(32 / (p.bw * p.bh));
    auto make_out = [&](CUtensorMap* m, const void* base, int elem, int ncols, long ld, int nsplit) -> int {
      uint64_t e = static_cast<uint64_t>(elem);
      uint64_t pitch = static_cast<uint64_t>(ld) * e;
      uint64_t dims[5], str[4];
      uint32_t box[5] = {32, static_cast<uint32_t>(p.bw), static_cast<uint32_t>(p.bh), bnn, 1};
      dims[0] = static_cast<uint64_t>(ncols);
      if (d->taps == 1) {
        dims[1] = static_cast<uint64_t>(M);
        dims[2] = 1;
        dims[3] = 1;
        str[0] = pitch;
        str[1] = pitch * M;
        str[2] = pitch * M;
      } else {
        dims[1] = static_cast<uint64_t>(d->w);
        dims[2] = static_cast<uint64_t>(d->h);
        dims[3] = static_cast<uint64_t>(d->nb);
        str[0] = pitch;
        str[1] = pitch * d->w;
        str[2] = pitch * d->w * d->h;
      }
      dims[4] = static_cast<uint64_t>(nsplit);
      str[3] = pitch * M;
      return make_tmap(m, base, elem, elem == 4 ? 128 : 64, 5, dims, str, box);
    };
    if (p.ws && make_out(&tm.ows, p.ws, 4, d->n, d->n, splits)) return 1;
    if (p.out_f32 && make_out(&tm.o32, p.out_f32, 4, n_out, p.ldo, 1)) return 1;
    if (p.out_f16 && make_out(&tm.o16, p.out_f16, 2, n_out, p.ldo, 1)) return 1;
    if (p.out_f16_lo && make_out(&tm.o16lo, p.out_f16_lo, 2, n_out, p.ldo, 1)) return 1;
  }
  // fused GroupNorm statistics: per-tile partial sums of the fp32 output, stored by the epilogue
  p.stats = nullptr;
  p.stats_halves = 1;
  p.stats_sg = g.sg;
  p.stats_tps = g.tiles_x * g.tiles_y;
  p.n_samples = static_cast<int>((M + p.rows_per_sample - 1) / p.rows_per_sample);
  if (d->stats_out) {
    Choice eff{bn, ch.cg, splits, p.csk};
    int halves = 1;
    const int T = stats_slots(d, g, eff, &halves);
    SDB_CHECK(T > 0, "sdb_gemm: this problem / tile shape cannot produce fused statistics (rows_per_sample %d, block_n %d, group %d)",
              p.rows_per_sample, bn, g.sg);
    p.stats = static_cast<float2*>(d->stats_out);
    p.stats_halves = halves;
    p.stats_T = T;
  }
  // bias + FiLM fold into a per-tile column table when each 64-row half of every tile belongs to one sample
  p.film_table = 0;
  if (p.film) {
    if (d->taps == 1) p.film_table = (p.rows_per_sample % 64 == 0) ? 1 : 0;
    else p.film_table = (p.TW * p.TH >= 64 && p.rows_per_sample == d->h * d->w) ? 1 : 0;
  }
  p.trace = trace_slot(8 + 8 * 160);
  {
    static int dbg = -1;
    if (dbg < 0) {
      const char* e = getenv("SDB_DBG");
      dbg = e ? atoi(e) : 0;
    }
    p.dbg = dbg;
  }

  // epilogue kind: the lean and GEGLU instantiations carry only the code their launches execute
  int kind = relu_family(d->act) ? 4 : 2;
  if (p.fast && d->act == SDB_ACT_GEGLU && !p.out_f32 && !p.out_f16_lo && !p.ws) kind = 1;
  else if (p.fast && d->act == SDB_ACT_NONE && (!p.film || p.film_table) && !(p.out_f32 && p.out_f16 && p.out_f16_lo)) kind = 0;
  if (kind == 0 && p.csk) kind = 3;
  int rc = kind == 0   ? launch_gemm_kind0(bn, ch.cg, tm, p, st)
           : kind == 1 ? launch_gemm_kind1(bn, ch.cg, tm, p, st)
           : kind == 3 ? launch_gemm_kind3(bn, ch.cg, tm, p, st)
           : kind == 4 ? launch_gemm_kind4(bn, ch.cg, tm, p, st)
                       : launch_gemm_kind2(bn, ch.cg, tm, p, st);
  if (rc) return rc;
  if (splits > 1 && !p.csk) {
    const bool vec = (p.N % 4 == 0) && (p.ldo % 4 == 0) && (!p.residual || p.ldr % 4 == 0) && (!p.film || p.ldf % 4 == 0);
    if (vec) {
      const bool wide = p.N % 160 == 0 && 160 % p.stats_sg == 0;
      // small outputs (the 8x8 / 16x16 levels: 128 x 1280 -> 32 blocks of 160 columns, 12 planes summed by each
      // thread: 10 us of pure latency on 32 SMs): 40-column blocks put four times as many SMs on the partial planes
      const bool narrow = wide && 40 % p.stats_sg == 0 &&
                          static_cast<long>(p.N / 160) * ((p.M + 31) / 32) < 2L * sm_count();
      const int cb = narrow ? 40 : (wide ? 160 : 128);
      dim3 grid((p.N + cb - 1) / cb, (p.M + 31) / 32);
      if (narrow) SDB_CUDA(launch_pdl(splitk_epilogue_kernel<10>, grid, dim3(80), 0, st, p, splits));
      else if (wide) SDB_CUDA(launch_pdl(splitk_epilogue_kernel<40>, grid, dim3(320), 0, st, p, splits));
      else SDB_CUDA(launch_pdl(splitk_epilogue_kernel<32>, grid, dim3(256), 0, st, p, splits));
    } else {
      SDB_CHECK(!p.stats, "sdb_gemm: stats_out with split-K needs n %% 4 == 0");
      size_t total = static_cast<size_t>(p.M) * p.N;
      int blocks = static_cast<int>(std::min<size_t>((total + 255) / 256, static_cast<size_t>(sm_count()) * 8));
      splitk_epilogue_scalar_kernel<<<blocks, 256, 0, st>>>(p, splits);
    }
    SDB_LAUNCH_CHECK();
  }
  return 0;
}
