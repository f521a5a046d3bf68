// Host drivers of the projection network's forward pass: the tensor-core stacks (tfl_cnn_tc.cu) with their padded
// activations, the fp32 graph executor (tfl_cnn.cu), and the two forwards the C ABI calls (tfl_api_cnn.cu).  No kernel
// lives here.  Every function that enqueues kernels returns how many it enqueued (what tfl_launch_count tallies); one
// that can fail returns < 0 after fail().
#include <algorithm>
#include <vector>

#include "tfl_api_internal.h"

int launch_tc_join(const float* const* l2, const ConvTcGeo* geo, const int* org, int zoff, int nbanks, bool add,
                   float* part, float* p_net, const std::vector<DevPtr<float>>& wj, const float* bias,
                   const float* tail, int split, const ConvTcGeo& g, cudaStream_t st, bool phases, const TcEpi& ep) {
  auto src_of = [&](int first, int n, int mode) {
    TcJoinSrc js = {};
    for (int k = 0; k < n; k++) {
      const int i = first + k;
      js.p[k] = l2[i];
      js.px[k] = geo[i].px; js.py[k] = geo[i].py; js.nz[k] = geo[i].nz; js.shift[k] = i; js.org[k] = org[i];
      js.phase[k] = phases && i > 0 ? 1 : 0;
    }
    js.zoff = zoff;
    js.n = n;
    js.part_mode = mode;
    js.partial = part;
    return js;
  };
  if (add) {
    launch_conv3_tc_join(src_of(0, nbanks, 0), p_net, wj[0].get(), bias, tail, split, g, st, ep);
    return 1;
  }
  for (int i = nbanks - 1; i >= 0; i--)
    launch_conv3_tc_join(src_of(i, 1, nbanks == 1 ? 0 : (i == nbanks - 1 ? 1 : (i > 0 ? 2 : 3))), p_net, wj[i].get(),
                         bias, tail, split, g, st, ep);
  return nbanks;
}

int cnn_ensure_act(tfl_ctx* ctx, tfl_cnn* m, const Geo& g) {
  if (m->act_geo.nb == g.nb && m->act_geo.nz == g.nz && m->act_geo.ny == g.ny && m->act_geo.nx == g.nx &&
      (m->nbanks == 1 || m->act_zoff == g.zoff))
    return 0;
  if (m->nbanks > 1 && !m->bank_dilate) {
    const int r = 1 << (m->nbanks - 1);
    if (ctx->slab && (g.nx % r || g.ny % r || g.gnz % r))
      return fail(ctx, "cnn: the z-slab's global grid %dx%dx%d is not divisible by 2^(banksNum-1) = %d", g.nx, g.ny,
                  g.gnz, r);
    if (!ctx->slab && (g.nx % r || g.ny % r || g.nz % r))
      return fail(ctx, "cnn: grid %dx%dx%d at bank split stage 1 is not divisible by 2^(banksNum-1) = %d", g.nx, g.ny,
                  g.nz, r);
    for (int i = 1, org = g.zoff; i < m->nbanks; i++) {
      org = (org + 1) >> 1;
      if (((g.zoff + g.nz) >> i) - org < 1)
        return fail(ctx, "cnn: the z-slab of %d planes holds no plane of bank %d", g.nz, i + 1);
    }
  }
  TFL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  m->act_gen++;
  m->act_geo = ConvTcGeo{};     // matches no grid until every buffer of the new one is in place
  for (DevPtr<float>& a : m->act) a.reset();
  m->bact.clear();
  m->bgeo.clear();
  m->borg.clear();
  m->part.reset();
  const ConvTcGeo ag = make_conv_tc_geo(g.nb, g.nz, g.ny, g.nx);
  for (DevPtr<float>& a : m->act)
    if (!(a = dev_zeros<float>(conv_tc_act_bytes(ag) / 4))) return fail(ctx, "cnn: cudaMalloc failed");
  for (int i = 1, org = g.zoff; i < m->nbanks; i++) {
    org = m->bank_dilate ? 0 : (org + 1) >> 1;     // dilated banks: whole grids only (cnn_slab_check)
    const ConvTcGeo bg = m->bank_dilate ? make_conv_tc_phase_geo(g.nb, g.nz, g.ny, g.nx, i)
                                        : make_conv_tc_geo(g.nb, ((g.zoff + g.nz) >> i) - org, g.ny >> i, g.nx >> i);
    m->bgeo.push_back(bg);
    m->borg.push_back(org);
    for (int q = 0; q < 3; q++)
      if (!keep(m->bact, dev_zeros<float>(conv_tc_act_bytes(bg) / 4))) return fail(ctx, "cnn: cudaMalloc failed");
  }
  if (m->nbanks > 1 && !m->bank_add && !(m->part = dev_alloc<float>((size_t)g.nb * g.nz * g.ny * g.nx * 8)))
    return fail(ctx, "cnn: cudaMalloc failed");
  m->act_geo = ag;
  m->act_zoff = g.zoff;
  return 0;
}

// Banked stack (split 1, join 3) on tensor cores: pyramid of the padded input, layers 1 and 2 of every bank at its
// own resolution, then the join layer reading the banks' layer-2 outputs with nearest indexing.  Dilated banks:
// the input copied into each bank's phase sub-grids, layers 1 and 2 as ordinary 3x3x3 layers on those (layer 1's
// voxels outside a short phase re-zeroed), and the join reading them through its phase index map.  'add': one launch
// summing the banks; 'concat': one launch per bank (N..2 into the fp32 partial sum, bank 1 last with the tail).
// p_net is wanted on the local planes [p_lo, p_hi): bank i's layers 1 and 2 run on the coarse planes the join reads
// from there (and the 3x3x3 stencil of layer 2 on those), the pyramid on all of the bank's planes.
static int run_conv_stack_banked(tfl_cnn* m, float* p_net, cudaStream_t st, int p_lo, int p_hi) {
  const ConvTcGeo& tg = m->act_geo;
  const int split = m->mode == 2 ? 1 : 0, nbk = m->nbanks, zoff = m->act_zoff;
  TcEpi act;                                  // relu6 (banked models with batch normalization run on the fp32 path)
  act.relu6 = m->nonlin == 3;
  const float* in[kTcMaxBanks];
  const float* l2[kTcMaxBanks];
  ConvTcGeo geo[kTcMaxBanks];
  int org[kTcMaxBanks];
  int launched = 0;
  in[0] = m->act[0].get();
  geo[0] = tg;
  org[0] = zoff;
  for (int i = 1; i < nbk; i++) {
    geo[i] = m->bgeo[i - 1];
    org[i] = m->borg[i - 1];
    float* dst = m->bact[3 * (i - 1)].get();
    if (m->bank_dilate) {
      // dilated bank i: the network input laid out as its 8^i phase sub-grids
      launch_tc_phase_copy(in[0], tg, dst, geo[i], i, m->tc_planes, st);
    } else {
      // coarse plane c pools the planes 2 c, 2 c + 1 of the level above (global indices): local 2 c + (org[i-1] & 1)
      launch_tc_pyramid(in[i - 1], geo[i - 1], dst, geo[i], org[i - 1] & 1, st, m->tc_planes);
    }
    launched += 1;
    in[i] = dst;
  }
  for (int i = 0; i < nbk; i++) {
    float* o1 = i == 0 ? m->act[1].get() : m->bact[3 * (i - 1) + 1].get();
    float* o2 = i == 0 ? m->act[2].get() : m->bact[3 * (i - 1) + 2].get();
    ConvTcGeo g1 = geo[i], g2 = geo[i];
    if (!m->bank_dilate) {
      // the join reads bank i at the coarse planes of the full-resolution planes [p_lo - 1, p_hi]
      const int c_lo = ((zoff + p_lo - 1) >> i) - org[i], c_hi = ((zoff + p_hi) >> i) - org[i] + 1;
      g2.z_lo = std::max(0, c_lo);     g2.z_hi = std::min(geo[i].nz, c_hi);
      g1.z_lo = std::max(0, c_lo - 1); g1.z_hi = std::min(geo[i].nz, c_hi + 1);
    }
    launch_conv3_tc(in[i], o1, nullptr, m->wBk[split][2 * i].get(), m->b[m->conv0[0] + i].get(), nullptr,
                    m->tc_planes, 0, split, g1, st, act);
    // a phase shorter than the sub-grid (d does not divide an axis): its extra voxels are padding for layer 2
    if (m->bank_dilate && i > 0 && ((tg.nx | tg.ny | tg.nz) & ((1 << i) - 1))) {
      launch_tc_phase_zero(o1, geo[i], i, tg, st);
      launched += 1;
    }
    launch_conv3_tc(o1, o2, nullptr, m->wBk[split][2 * i + 1].get(), m->b[m->conv0[1] + i].get(), nullptr, 2, 0,
                    split, g2, st, act);
    launched += 2;
    l2[i] = o2;
  }
  ConvTcGeo g3 = tg;
  g3.z_lo = std::max(0, p_lo);
  g3.z_hi = std::min(tg.nz, p_hi);
  return launched + launch_tc_join(l2, geo, org, zoff, nbk, m->bank_add, m->part.get(), p_net, m->wBj[split],
                                   m->b[m->conv0[2]].get(), m->tail.get(), split, g3, st, m->bank_dilate != 0, act);
}

int run_conv_stack(tfl_cnn* m, float* p_net, cudaStream_t st, int p_lo, int p_hi) {
  if (p_hi < 0) p_hi = m->act_geo.nz;
  if (m->nbanks > 1) return run_conv_stack_banked(m, p_net, st, p_lo, p_hi);
  const ConvTcGeo& tg = m->act_geo;
  const int split = m->mode == 2 ? 1 : 0;
  ConvTcGeo g1 = tg, g2 = tg, g3 = tg;
  g3.z_lo = std::max(0, p_lo);     g3.z_hi = std::min(tg.nz, p_hi);
  g2.z_lo = std::max(0, p_lo - 1); g2.z_hi = std::min(tg.nz, p_hi + 1);
  g1.z_lo = std::max(0, p_lo - 2); g1.z_hi = std::min(tg.nz, p_hi + 2);
  TcEpi e1, e2, e3;
  e1.relu6 = e2.relu6 = e3.relu6 = m->nonlin == 3;
  if (m->bn && !m->bn_batch) {
    // running statistics: BN1 / BN2 in the producing epilogues (after the activation, valid voxels only: the zero
    // padding of the next layer lies after BN), BN3 / BN4 folded into the tail at creation
    e1.ac = m->bn_ac[0].get();
    e2.ac = m->bn_ac[1].get();
  }
  float *a0 = m->act[0].get(), *a1 = m->act[1].get(), *a2 = m->act[2].get(), *tail = m->tail.get();
  const float *w1 = m->wBk[split][0].get(), *w2 = m->wBk[split][1].get(), *w3 = m->wBj[split][0].get();
  if (!m->bn_batch) {
    launch_conv3_tc(a0, a1, nullptr, w1, m->b[0].get(), nullptr, m->tc_planes, 0, split, g1, st, e1);
    launch_conv3_tc(a1, a2, nullptr, w2, m->b[1].get(), nullptr, 2, 0, split, g2, st, e2);
    launch_conv3_tc(a2, nullptr, p_net, w3, m->b[2].get(), tail, 2, 1, split, g3, st, e3);
    return 3;
  }
  // Batch statistics (whole grids only): each BN needs its layer's whole output first.  Layers 1 and 2: statistics
  // of the interior, then y = a x + c in place on it; layer 3 writes its output to act[1] (free again), and the tail
  // runs as two passes over it -- pass A accumulates BN4's statistics of h4 = act(w4 BN3(h3) + b4), pass B
  // recomputes h4 and writes p_net = w5 BN4(h4) + b5.
  double* part = m->bn_part.get();
  float* ac = m->bn_tcac.get();               // [4][2][8]
  const long long count = (long long)tg.nb * tg.nz * tg.ny * tg.nx;
  auto stats = [&](const float* buf, int l) {
    launch_tc_bn_stats(buf, tg, part, st);
    const float* wb = m->bn_wb[l].get();
    launch_bn_finalize(part, 8, count, wb, wb + 8, m->bn_eps[l], ac + 16 * l, nullptr, st);
  };
  launch_conv3_tc(a0, a1, nullptr, w1, m->b[0].get(), nullptr, m->tc_planes, 0, split, tg, st, e1);
  stats(a1, 0);
  launch_tc_bn_apply(a1, tg, ac, st);
  launch_conv3_tc(a1, a2, nullptr, w2, m->b[1].get(), nullptr, 2, 0, split, tg, st, e2);
  stats(a2, 1);
  launch_tc_bn_apply(a2, tg, ac + 16, st);
  launch_conv3_tc(a2, a1, nullptr, w3, m->b[2].get(), nullptr, 2, 0, split, tg, st, e3);
  stats(a1, 2);
  launch_tc_bn_tail(a1, tg, ac + 32, tail, e3.relu6, 0, part, nullptr, nullptr, st);
  launch_bn_finalize(part, 8, count, m->bn_wb[3].get(), m->bn_wb[3].get() + 8, m->bn_eps[3], ac + 48, nullptr, st);
  launch_tc_bn_tail(a1, tg, ac + 32, tail, e3.relu6, 1, nullptr, ac + 48, p_net, st);
  return 3 + 3 * 2 + 2 + 2 + 1;     // convolutions, stats() pairs, applies, tail passes, BN4's finalize
}

namespace {

// The tensor-core forward from a device `scale` on: the network input on gi's plane range (the divergence reads U1
// one plane up, so a z-slab stops short of its local end), the stack for p_net on the planes [p_lo, p_hi), the
// pressure skip, and the velocity update on g's plane range.  U1 is the wall-masked velocity; p_net a plain
// [b][z][y][x] scratch.  The model's activations are in place (cnn_ensure_act).
struct TcForward {
  const float* scale;
  float* p_net;
  Geo gi;
  int p_lo, p_hi;
};
int cnn_forward_tc(tfl_ctx* ctx, tfl_cnn* m, const CnnFields& f, const Geo& g, const TcForward& t) {
  cudaStream_t st = ctx->stream;
  const ConvTcGeo& tg = m->act_geo;
  launch_cnn_inputs_padded(f.p_div, f.U, f.flags, t.scale, m->act[0].get(), tg.px, tg.py, t.gi, st, m->in_sel,
                           m->tc_planes);
  int launched = 1 + run_conv_stack(m, t.p_net, st, t.p_lo, t.p_hi);
  if (m->skip) {
    launch_cnn_skip(t.p_net, f.p_div, t.scale, m->w_skip, g, st);
    launched += 1;
  }
  launch_cnn_finish(t.p_net, f.U, f.flags, t.scale, f.p_out, f.U_out, g, st);
  return launched + 1;
}

// The fp32 path's scratch in the arena, in pieces aligned to 256 bytes from `base`.  Over a null base only `bytes` is
// meaningful: what arena_reserve needs, 256 bytes beyond each piece (at least its alignment) and 768 more.
struct CnnScratch {
  float *U1, *x0, *actA, *actB, *scale;
  double* sums;        // the input scale's (sum, sum of squares) per batch entry
  double* bn_part;     // batch statistics: the partial sums and (a, c) of one BN module at a time
  float* bn_ac;
  float* actC;         // the third rotating buffer of the graphs that are not plain
  float* bank[kMaxBanks][3];
  size_t bytes;
};
CnnScratch cnn_scratch(const tfl_cnn* m, const Geo& g, char* base) {
  CnnScratch s = {};
  s.bytes = 3 * 256;
  size_t off = 0;
  auto take = [&](size_t bytes) {
    char* p = base ? base + off : nullptr;
    off = (off + bytes + 255) & ~(size_t)255;
    s.bytes += bytes + 256;
    return p;
  };
  const size_t cells = (size_t)g.n * g.nb;
  s.U1 = (float*)take(cells * 4 * g.nc);
  s.x0 = (float*)take(cells * 4 * m->in_ch);
  s.actA = (float*)take(cells * 4 * m->max_c);      // max_c covers max_rel (set at creation)
  s.actB = (float*)take(cells * 4 * m->max_c);
  s.scale = (float*)take(sizeof(float) * g.nb);
  s.sums = (double*)take(sizeof(double) * 2 * g.nb);
  s.bn_part = (double*)take(sizeof(double) * 2 * (kBnBlocks + 1) * m->bn_max_c);
  s.bn_ac = (float*)take(sizeof(float) * 2 * m->bn_max_c);
  if (m->plain) return s;
  s.actC = (float*)take((size_t)((double)cells * m->max_rel + 64) * 4);
  // Banks 2..N rotate through buffers of their own.  A multi-resolution bank i (0-based) holds 2^-d i of bank 1's
  // cells, and every activation of bank 1 fits max_rel; a dilated bank has bank 1's resolution and needs its own
  // largest activation, bank_rel (the joined banks live in bank 1's buffers).  A dilated stage is convolution ->
  // non-linearity -> pooling (no pixel shuffle), so its result can go back to the buffer its input came from, and two
  // buffers suffice: run_stage alternates them.
  for (int i = 1; i < m->nbanks; i++) {
    const double rel = m->bank_dilate ? m->bank_rel : m->max_rel / (double)(1LL << ((m->is3d ? 3 : 2) * i));
    for (int q = 0; q < (m->bank_dilate ? 2 : 3); q++)
      s.bank[i][q] = (float*)take((size_t)((double)cells * rel + 64) * 4);
    if (m->bank_dilate) s.bank[i][2] = s.bank[i][0];
  }
  return s;
}

// Grid g after up-sampling by u and pooling by q (z in 3-D only), as a whole grid of its own.
Geo resampled(Geo g, int u, int q) {
  g.nx = g.nx * u / q;
  g.ny = g.ny * u / q;
  if (g.is3d) g.nz = g.nz * u / q;
  g.n = (long long)g.nx * g.ny * g.nz;
  g.gnz = g.nz; g.zlo = 0; g.zhi = g.nz;
  return g;
}

// What one stage of one bank reads and where its result goes.
struct StageIo {
  const float* src;          // the stage's input
  float* const* bufs;        // the three rotating buffers the stage writes
  const float* keep;         // an input other banks still read, never written (may be null)
  float* dst;                // the stage's result goes there rather than to one of bufs (may be null)
  long long out_bstride;     // > 0: the result is written with this batch stride (floats), so that it lands in place in
                             // a concatenation of banks
  int dil;                   // dilation of the convolution
  float* other(const float* a) const {     // a buffer that holds neither a nor keep
    for (int q = 0; q < 3; q++) if (bufs[q] != a && bufs[q] != keep) return bufs[q];
    return bufs[0];
  }
};

// The executor of the 'tog' / 'yang' graphs and of every graph with banks, batch normalization or a non-linearity
// other than ReLU: conv (+ pixel shuffle) -> non-linearity -> pooling, layer by layer, on grids whose resolution
// follows the pooling / upsampling sizes (lib/model.lua:262-340).
struct Fp32Graph {
  tfl_ctx* ctx;
  const tfl_cnn* m;
  const CnnScratch& scr;
  float* bufs[3];                           // bank 1's (and the unbanked stages') rotating buffers
  const float* bank_in[kMaxBanks] = {};     // in the banked stages: every bank's current activation ...
  Geo bank_g[kMaxBanks];                    // ... and its grid

  // Channels of stage l's result (after the pixel shuffle).
  int stage_channels(int l) const {
    const int u = m->up[l];
    return m->cout[m->conv0[l]] / (u * u * (m->is3d ? u : 1));
  }
  int batch_norm(float* x, int ci, int chans, const Geo& gl, long long bstride);
  int run_stage(int ci, int l, const StageIo& io, Geo& gl, const float** result);
  int split_banks(int l, const float* in, const Geo& gl);
  int run_banked_stage(int l, const float* in);
  int join_banks(int l, const float** in, Geo* gl);
  int run(const float** in, const Geo& g);
};

// Convolution ci's batch normalization in place on x [nb][chans][gl.n], batch entries bstride floats apart.
int Fp32Graph::batch_norm(float* x, int ci, int chans, const Geo& gl, long long bstride) {
  cudaStream_t st = ctx->stream;
  if (!m->bn_batch) {
    launch_bn_apply(x, gl.nb, chans, gl.n, bstride, m->bn_ac[ci].get(), st);
    return 1;
  }
  launch_bn_stats(x, gl.nb, chans, gl.n, bstride, scr.bn_part, st);
  launch_bn_finalize(scr.bn_part, chans, (long long)gl.nb * gl.n, m->bn_wb[ci].get(), m->bn_wb[ci].get() + chans,
                     m->bn_eps[ci], scr.bn_ac, nullptr, st);
  launch_bn_apply(x, gl.nb, chans, gl.n, bstride, scr.bn_ac, st);
  return 3;
}

// One stage of one bank: convolution ci (+ pixel shuffle) -> non-linearity -> pooling (-> batch normalization) of
// stage l, on grid gl, which becomes the grid of the result.
int Fp32Graph::run_stage(int ci, int l, const StageIo& io, Geo& gl, const float** result) {
  cudaStream_t st = ctx->stream;
  const long long out_bstride = io.out_bstride;
  const int u = m->up[l], pl = m->pool[l];
  const int act = (l < m->n_layers - 1) ? m->nonlin : 0;     // element-wise: commutes with the shuffle
  int launched = 0;
  // per batch entry when the last operation of the stage writes with a batch stride (else one launch, b = 0)
  const int nloop_conv = (out_bstride > 0 && u == 1 && pl == 1) ? gl.nb : 1;
  float* o = (io.dst && u == 1 && pl == 1) ? io.dst : io.other(io.src);
  Geo gb = gl;
  gb.nb = gl.nb / nloop_conv;
  for (int b = 0; b < nloop_conv; b++) {
    if (launch_conv_direct(io.src + (long long)b * m->cin[ci] * gl.n, o + b * out_bstride, m->w[ci].get(),
                           m->b[ci].get(), m->cin[ci], m->cout[ci], m->ks[ci], act, gb, st, io.dil) < 0)
      return -fail(ctx, "cnn: unsupported layer shape cout=%d k=%d", m->cout[ci], m->ks[ci]);
    launched += 1;
  }
  const float* cur = o;
  int chans = m->cout[ci];
  if (u > 1) {
    chans = m->cout[ci] / (u * u * (gl.is3d ? u : 1));
    float* sh = (io.dst && pl == 1) ? io.dst : io.other(cur);
    const int nloop = (out_bstride > 0 && pl == 1) ? gl.nb : 1;
    const long long nin = (long long)m->cout[ci] * gl.n;
    for (int b = 0; b < nloop; b++)
      launch_pixel_shuffle(cur + b * nin, sh + b * out_bstride, gl.nb / nloop, chans, gl.nz, gl.ny, gl.nx, u, gl.is3d,
                           st);
    launched += nloop;
    gl = resampled(gl, u, 1);
    cur = sh;
  }
  if (pl > 1) {
    if (gl.nx % pl || gl.ny % pl || (gl.is3d && gl.nz % pl))
      return -fail(ctx, "cnn: grid %dx%dx%d is not divisible by the pooling size %d", gl.nx, gl.ny, gl.nz, pl);
    float* po = io.dst ? io.dst : io.other(cur);
    const int nloop = out_bstride > 0 ? gl.nb : 1;
    const long long nin = (long long)chans * gl.nx * gl.ny * gl.nz;
    for (int b = 0; b < nloop; b++)
      launch_pool(cur + b * nin, po + b * out_bstride, gl.nb / nloop * chans, gl.nz, gl.ny, gl.nx, pl, gl.is3d,
                  m->pool_is_max, st);
    launched += nloop;
    gl = resampled(gl, 1, pl);
    cur = po;
  }
  if (m->bn && l < m->n_layers - 1) {     // lib/model.lua:343-350: BN closes every stage but the last
    float* x = (float*)cur;               // one of this call's buffers, or a slot of one
    launched += batch_norm(x, ci, chans, gl, out_bstride > 0 ? out_bstride : (long long)chans * gl.n);
  }
  *result = cur;
  return launched;
}

// The banks' inputs at the split stage l, from the hidden layer `in` on grid gl.
int Fp32Graph::split_banks(int l, const float* in, const Geo& gl) {
  const int nbk = m->nbanks;
  bank_in[0] = in;
  bank_g[0] = gl;
  if (m->bank_dilate) {
    // Dilated banks (lib/model.lua:279-285): every bank reads the hidden layer as it is.
    for (int i = 1; i < nbk; i++) {
      bank_in[i] = in;
      bank_g[i] = gl;
    }
    return 0;
  }
  // Gaussian pyramid (lib/model.lua:276-289): bank i = 2x average pool of bank i-1.
  const int r = 1 << (nbk - 1);
  if (gl.nx % r || gl.ny % r || (gl.is3d && gl.nz % r))
    return -fail(ctx, "cnn: grid %dx%dx%d at bank split stage %d is not divisible by 2^(banksNum-1) = %d", gl.nx,
                 gl.ny, gl.nz, l + 1, r);
  for (int i = 1; i < nbk; i++) {
    const Geo& gi = bank_g[i - 1];
    launch_pool(bank_in[i - 1], scr.bank[i][0], gi.nb * m->cin[m->conv0[l]], gi.nz, gi.ny, gi.nx, 2, gi.is3d, 0,
                ctx->stream);
    bank_g[i] = resampled(gi, 1, 2);
    bank_in[i] = scr.bank[i][0];
  }
  return nbk - 1;
}

// Stage l of every bank, each through its own buffers; `in` is the hidden layer the banks were split from.
int Fp32Graph::run_banked_stage(int l, const float* in) {
  const int nbk = m->nbanks;
  const bool last = l == m->join - 1;
  // Dilated banks joined by 'concat' write their last stage straight into their channel slots of bank 1's
  // result; the shared input of the split stage stays intact until every bank has read it.
  const bool in_slot = m->bank_dilate && last && !m->bank_add;
  const float* shared = (m->bank_dilate && l == m->split) ? in : nullptr;
  // concat: bank 1's result is the first c_out channels of [nb][nbk c_out][n] at the join resolution (taken
  // before the stage runs: run_stage moves bank_g[0] to the stage's output grid)
  const int c_out = stage_channels(l), nb = bank_g[0].nb;
  const long long n_join = resampled(bank_g[0], m->up[l], m->pool[l]).n;
  int launched = 0;
  for (int i = 0; i < nbk; i++) {
    StageIo io = {bank_in[i], i == 0 ? bufs : scr.bank[i], shared, nullptr, 0, m->bank_dilate ? 1 << i : 1};
    if (last && (i == 0 || in_slot) && !m->bank_add && nb > 1) io.out_bstride = (long long)nbk * c_out * n_join;
    if (in_slot && i > 0) io.dst = (float*)bank_in[0] + (long long)i * c_out * n_join;
    const int k = run_stage(m->conv0[l] + i, l, io, bank_g[i], &bank_in[i]);
    if (k < 0) return k;
    launched += k;
  }
  return launched;
}

// After the banks' last stage l: their results joined into bank 1's, which becomes the hidden layer *in on *gl.
int Fp32Graph::join_banks(int l, const float** in, Geo* gl) {
  const int nbk = m->nbanks;
  const Geo& g1 = bank_g[0];
  int launched = 0;
  if (!m->bank_dilate)     // lib/model.lua:292-318: upsample banks 2..N, then JoinTable or CAddTable
    for (int i = 1; i < nbk; i++)
      if (bank_g[i].nx << i != g1.nx || bank_g[i].ny << i != g1.ny || (g1.is3d && bank_g[i].nz << i != g1.nz))
        return -fail(ctx, "cnn: bank %d does not upsample to the resolution of bank 1 (grid not divisible)", i + 1);
  // dilated banks (lib/model.lua:300-318) are at bank 1's resolution, and their 'concat' is already in place
  if (!m->bank_dilate || m->bank_add) {
    if (launch_bank_join(bank_in, nbk, (float*)bank_in[0], g1.nb, stage_channels(l), g1.nz, g1.ny, g1.nx, g1.is3d,
                         m->bank_add, ctx->stream, m->bank_dilate) < 0)
      return -fail(ctx, "cnn: bad bank count %d", nbk);
    launched = 1;
  }
  *in = bank_in[0];
  *gl = g1;
  return launched;
}

// Every stage of the graph from *in on grid g; *in becomes the network's output.
int Fp32Graph::run(const float** in, const Geo& g) {
  Geo gl = g;
  int launched = 0;
  auto ran = [&](int k) { launched += k; return k >= 0; };
  for (int l = 0; l < m->n_layers; l++) {
    if (m->nbanks == 1 || l < m->split || l >= m->join) {
      if (!ran(run_stage(m->conv0[l], l, {*in, bufs, nullptr, nullptr, 0, 1}, gl, in))) return -1;
      continue;
    }
    if (l == m->split && !ran(split_banks(l, *in, gl))) return -1;
    if (!ran(run_banked_stage(l, *in))) return -1;
    if (l == m->join - 1 && !ran(join_banks(l, in, &gl))) return -1;
  }
  if (gl.nx != g.nx || gl.ny != g.ny || gl.nz != g.nz)
    return -fail(ctx, "cnn: graph does not return to the input resolution");
  return launched;
}

// The fp32 forward from the network input on: f.U is the wall-masked velocity, scr.scale the input scale.
int cnn_project_fp32(tfl_ctx* ctx, const tfl_cnn* m, const CnnFields& f, const Geo& g, const CnnScratch& scr) {
  cudaStream_t st = ctx->stream;
  launch_cnn_inputs(f.p_div, f.U, f.flags, scr.scale, scr.x0, g, st, m->in_sel);
  ctx->launches += 1;
  const float* in = scr.x0;
  if (m->plain) {
    float* bufs[2] = {scr.actA, scr.actB};
    for (int l = 0; l < m->n_layers; l++) {
      float* o = bufs[l & 1];
      const int act = (l < m->n_layers - 1) ? 1 : 0;
      if (launch_conv_direct(in, o, m->w[l].get(), m->b[l].get(), m->cin[l], m->cout[l], m->ks[l], act, g, st) < 0)
        return fail(ctx, "cnn: unsupported layer shape cout=%d k=%d", m->cout[l], m->ks[l]);
      ctx->launches += 1;
      in = o;
    }
  } else {
    if (ctx->slab) return fail(ctx, "cnn: pooled / upsampled graphs run on whole grids only");
    Fp32Graph graph = {ctx, m, scr, {scr.actA, scr.actB, scr.actC}};
    const int k = graph.run(&in, g);
    if (k < 0) return 1;
    ctx->launches += k;
  }
  if (m->skip) {
    launch_cnn_skip((float*)in, f.p_div, scr.scale, m->w_skip, g, st);     // `in` is one of this call's scratch buffers
    ctx->launches += 1;
  }
  launch_cnn_finish(in, f.U, f.flags, scr.scale, f.p_out, f.U_out, g, st);
  ctx->launches += 1;
  return check_launch(ctx, "cnn_project");
}

}  // namespace

int cnn_project(tfl_ctx* ctx, tfl_cnn* m, const CnnFields& f, float threshold, const Geo& g, float* scale_out) {
  if (arena_reserve(ctx, cnn_scratch(m, g, nullptr).bytes)) return 1;
  const CnnScratch scr = cnn_scratch(m, g, ctx->arena.get());
  double* sums = scr.sums;
  cudaStream_t st = ctx->stream;
  TFL_CUDA(ctx, cudaMemsetAsync(sums, 0, sizeof(double) * 2 * g.nb, st));
  launch_cnn_mask_stats(f.U, f.flags, scr.U1, sums, g.zlo, g.zhi, g, st, m->norm_chan, f.p_div);
  ctx->launches += 1;
  if (m->norm_chan == kCnnStatDiv) {
    launch_cnn_div_stats(scr.U1, f.flags, sums, g.zlo, g.zhi, g, st);
    ctx->launches += 1;
  }
  launch_cnn_scale(sums, scr.scale, g.nb, m->norm_chan == kCnnStatU ? (long long)g.nc * g.n : g.n, threshold, st,
                   m->norm_func);
  ctx->launches += 1;
  const CnnFields f1 = {f.p_div, scr.U1, f.flags, f.p_out, f.U_out};     // from here on the velocity is the masked one
  if (m->mode > 0 && m->tc_ok && !ctx->slab) {
    if (cnn_ensure_act(ctx, m, g)) return 1;
    ctx->launches += cnn_forward_tc(ctx, m, f1, g, {scr.scale, scr.actA, g, 0, g.nz});
    if (check_launch(ctx, "cnn_project (tensor cores)")) return 1;
  } else if (cnn_project_fp32(ctx, m, f1, g, scr)) {
    return 1;
  }
  if (scale_out) {
    TFL_CUDA(ctx, cudaMemcpyAsync(scale_out, scr.scale, sizeof(float) * g.nb, cudaMemcpyDeviceToHost, st));
    TFL_CUDA(ctx, cudaStreamSynchronize(st));
  }
  return 0;
}

int cnn_project_from_sums(tfl_ctx* ctx, tfl_cnn* m, const CnnFields& f, const double* dev_sums, float threshold,
                          const Geo& g) {
  if (cnn_ensure_act(ctx, m, g)) return 1;
  const size_t cells = (size_t)g.n * g.nb;
  if (arena_reserve(ctx, carve_bytes({cells * 4, 4 * (size_t)g.nb}))) return 1;
  Carver cv(ctx);
  float* p_net = cv.take<float>(cells);
  float* scale = cv.take<float>(g.nb);
  // scale from the (already reduced) sums; the sample count is that of the GLOBAL grid.
  launch_cnn_scale(dev_sums, scale, g.nb, (long long)g.nc * g.nx * g.ny * g.gnz, threshold, ctx->stream);
  ctx->launches += 1;
  TcForward t = {scale, p_net, g, 0, g.nz};
  if (ctx->slab) {
    t.gi.zlo = (g.zoff == 0) ? 0 : 1;
    t.gi.zhi = (g.zoff + g.nz == g.gnz) ? g.nz : g.nz - 2;
    // the velocity update of the computed planes [zlo, zhi) reads p on [zlo - 1, zhi)
    t.p_lo = g.zlo - 1;
    t.p_hi = g.zhi;
  }
  ctx->launches += cnn_forward_tc(ctx, m, f, g, t);
  return check_launch(ctx, "cnn_project_from_sums");
}
