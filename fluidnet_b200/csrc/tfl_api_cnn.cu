// C ABI of the projection network (include/tfl.h): model creation, modes, the fp32 graph executor and the
// tensor-core stacks (tfl_cnn*.cu), and the test hooks of the tensor-core layers and of the fp32 kernels.
#include <string.h>
#include <algorithm>
#include <cmath>
#include <vector>

#include "tfl_api_internal.h"

constexpr int kMaxBanks = kMaxBankPtrs;     // banks a join kernel takes
constexpr char kSlabTcOnly[] =
    "the z-slab projection runs on the tensor-core path only (the 3-D 'default' graph, single-bank or with banks "
    "split at stage 1 and joined at stage 3, in mode 1 or 2)";
constexpr char kSlabDilate[] =
    "the z-slab projection does not run banksType 'dilate' (dilated banks run on whole grids only)";
constexpr char kSlabBatchNorm[] =
    "the z-slab projection does not run batch normalization (addBatchNorm models run on whole grids only)";
constexpr char kSlabDefaultInputs[] =
    "the z-slab projection takes the default input block only (inputChannels pDiv, div, flags; normalizeInput with "
    "'std' of UDiv; no addPressureSkip)";

constexpr int kTailFloats = 64 + 8 + 8 + 1;     // the fused 1x1x1 tail: w4[8][8], b4[8], w5[8], b5[1]

namespace {

// Appends p to v; false (and v unchanged) if p is empty, its upload having failed.
bool keep(std::vector<DevPtr<float>>& v, DevPtr<float> p) {
  if (!p) return false;
  v.push_back(std::move(p));
  return true;
}

// Packs a [8][cin][3][3][3] weight for launch_conv3_tc / launch_conv3_tc_join and uploads it.
DevPtr<float> upload_tc_weights(const float* w, int cin, int split) {
  std::vector<float> packed(conv_tc_b_floats(split));
  conv_tc_pack_weights(w, cin, split, packed.data());
  return upload(packed);
}

// A convolution weight in Torch layout [cout][cin][taps] re-laid out as the [cin][tap][cout] that
// launch_conv_direct and launch_conv_any read.
std::vector<float> relayout_conv_weights(const float* w, int cin, int cout, int taps) {
  std::vector<float> relaid((size_t)cin * taps * cout);
  for (int o = 0; o < cout; o++)
    for (int c = 0; c < cin; c++)
      for (int t = 0; t < taps; t++)
        relaid[((size_t)c * taps + t) * cout + o] = w[((size_t)o * cin + c) * taps + t];
  return relaid;
}

// Convolution wi's batch normalization (c channels) from norm->bn[wi] / eps[wi]: for batch statistics its weight and
// bias on the device, for running statistics y = a x + c with a = w / sqrt(running_var + eps), c = b - running_mean a
// (in double, rounded once).
void bn_running_affine(const tfl_cnn_norm* norm, int wi, int c, double* a, double* cc) {
  const float* p = norm->bn[wi];
  for (int ch = 0; ch < c; ch++) {
    a[ch] = (double)p[ch] / std::sqrt((double)p[3 * c + ch] + (double)norm->eps[wi]);
    cc[ch] = (double)p[c + ch] - (double)p[2 * c + ch] * a[ch];
  }
}
// What the model keeps on the device of convolution wi's batch normalization: bn_wb or bn_ac [2][c].
DevPtr<float> upload_bn(const tfl_cnn_norm* norm, bool batch, int wi, int c) {
  const float* p = norm->bn[wi];
  std::vector<float> h(2 * c);
  std::vector<double> a(c), cc(c);
  if (!batch) bn_running_affine(norm, wi, c, a.data(), cc.data());
  for (int ch = 0; ch < c; ch++) {
    h[ch] = batch ? p[ch] : (float)a[ch];
    h[c + ch] = batch ? p[c + ch] : (float)cc[ch];
  }
  return upload(h);
}

// A layer-1 weight [8][cin][3][3][3] zero-padded to [8][8][3][3][3] (the two-plane input of a set with UDiv).
std::vector<float> pad_cin8(const float* w, int cin) {
  std::vector<float> padded(8 * 8 * 27, 0.0f);
  for (int o = 0; o < 8; o++)
    memcpy(padded.data() + (size_t)o * 8 * 27, w + (size_t)o * cin * 27, (size_t)cin * 27 * 4);
  return padded;
}

// Bank i's 8-channel slice of a 'concat' join weight [8][8 nbanks][3][3][3] (one bank: the whole weight).
std::vector<float> concat_slice(const float* w, int nbanks, int i) {
  std::vector<float> slice(8 * 8 * 27);
  for (int o = 0; o < 8; o++)
    memcpy(slice.data() + (size_t)o * 8 * 27, w + ((size_t)o * 8 * nbanks + 8 * i) * 27, 8 * 27 * 4);
  return slice;
}

// The join layer of a banked stack (split 1, join 3) -> p_net on the output planes [g.z_lo, g.z_hi), reading bank
// i's layer-2 output l2[i] (geometry geo[i], 2^-i of bank 1's resolution) with nearest indexing.  z-slab: local
// full-resolution plane 0 is global plane zoff, bank i's local plane 0 its global coarse plane org[i] (whole grids:
// all 0).  'add': one launch summing the banks, weights wj[0]; 'concat': one launch per bank with its slice wj[i],
// banks N..2 writing / adding the fp32 partial sum `part`, bank 1 last adding it before the bias, ReLU and tail (one
// bank: no partial sum).  phases: banks 2..N are dilated banks held as phase sub-grids (geo[i] =
// make_conv_tc_phase_geo(.., i)) rather than multi-resolution banks.
void launch_tc_join(const float* const* l2, const ConvTcGeo* geo, const int* org, int zoff, int nbanks, bool add,
                    float* part, float* p_net, const std::vector<DevPtr<float>>& wj, const float* bias,
                    const float* tail, int split, const ConvTcGeo& g, cudaStream_t st, bool phases = false,
                    const TcEpi& ep = TcEpi()) {
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
  } else {
    for (int i = nbanks - 1; i >= 0; i--)
      launch_conv3_tc_join(src_of(i, 1, nbanks == 1 ? 0 : (i == nbanks - 1 ? 1 : (i > 0 ? 2 : 3))), p_net, wj[i].get(),
                           bias, tail, split, g, st, ep);
  }
}

// The whole-grid geometry of the fp32 test hooks, and their grid check and closing synchronisation.
Geo whole_grid(tfl_ctx* ctx, int nb, int nz, int ny, int nx, int is3d) {
  Geo g = {};
  g.nx = nx; g.ny = ny; g.nz = nz; g.gnz = nz; g.zoff = 0; g.zlo = 0; g.zhi = nz; g.nb = nb;
  g.is3d = is3d ? 1 : 0;
  g.nc = is3d ? 3 : 2;
  g.n = (long long)nx * ny * nz;
  g.faults = ctx->counters.get();
  return g;
}
bool bad_grid(int nb, int nz, int ny, int nx, int is3d) {
  return nb < 1 || nz < 1 || ny < 1 || nx < 1 || (!is3d && nz != 1) || (long long)nz * ny * nx >= (1LL << 31);
}
int finish_debug(tfl_ctx* ctx, const char* what) {
  const int rc = check_launch(ctx, what);
  const cudaError_t se = cudaStreamSynchronize(ctx->stream);
  if (rc) return rc;
  if (se != cudaSuccess) return fail(ctx, "%s: %s", what, cudaGetErrorString(se));
  if (conv_tc_take_z_fault(ctx->stream)) return fail(ctx, "%s: %s", what, kConvZStalled);
  return 0;
}

// Why the z-slab entry points refuse the model, or null if they run it.
const char* cnn_slab_refusal(const tfl_cnn* m) {
  if (m->bn) return kSlabBatchNorm;
  if (m->bank_dilate) return kSlabDilate;
  if (!m->default_inputs) return kSlabDefaultInputs;
  if (!m->tc_ok || m->mode == 0) return kSlabTcOnly;
  return nullptr;
}

}  // namespace

// The reach of a banked model, with s = 2^(banksNum-1) the coarsest bank's scale: p on the planes the velocity
// update reads (owned - 1 .. owned_hi - 1) needs the network input on 3 s + 1 planes below the owned ones and 3 s
// above (the coarse plane of the join's stencil end, two coarse 3x3x3 layers, the s fine planes a coarse plane
// pools, each at its worst alignment to the rank's boundary), the input reads U one plane up and the wall mask flags
// one plane down.  So the slab holds 3 s + 2 ghost planes on each interior side (the input is computed up to two
// planes short of the local end), which a halo of 2 margin + 2 provides from margin = 3 s / 2 on.
int cnn_slab_check(tfl_ctx* ctx, const tfl_cnn* m, int margin, int gnz, int ny, int nx, int zoff, int nz, int own_lo,
                   int own_hi) {
  if (const char* why = cnn_slab_refusal(m)) return fail(ctx, "slab: %s", why);
  if (m->nbanks == 1) return 0;
  const int need = tfl_slab_cnn_margin(m->nbanks), s = 1 << (m->nbanks - 1), depth = 3 * s + 2;
  if (margin < need)
    return fail(ctx, "slab: a %d-bank model needs a z-slab margin >= %d (tfl_slab_cnn_margin), got %d", m->nbanks,
                need, margin);
  if (gnz % s || ny % s || nx % s)
    return fail(ctx, "slab: the z-slab's global grid %dx%dx%d is not divisible by 2^(banksNum-1) = %d", nx, ny, gnz, s);
  if ((zoff > 0 && own_lo < depth) || (zoff + nz < gnz && nz - own_hi < depth))
    return fail(ctx, "slab: a %d-bank model needs %d ghost planes on each interior side of the z-slab (margin >= %d); "
                     "this one has %d below and %d above", m->nbanks, depth, need, own_lo, nz - own_hi);
  return 0;
}

// Tensor-core path: padded channels-last activations owned by the model (their zero borders
// must survive between calls, so they do not live in the shared arena).
// z-slab (g.zoff, g.gnz): bank i holds the global coarse planes [ceil(zoff / 2^i), floor((zoff + nz) / 2^i)).
// Dilated banks: bank i's buffers hold its 8^i phase sub-grids per batch entry (make_conv_tc_phase_geo).
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
static void run_conv_stack_banked(tfl_cnn* m, float* p_net, cudaStream_t st, int p_lo, int p_hi) {
  const ConvTcGeo& tg = m->act_geo;
  const int split = m->mode == 2 ? 1 : 0, nbk = m->nbanks, zoff = m->act_zoff;
  TcEpi act;                                  // relu6 (banked models with batch normalization run on the fp32 path)
  act.relu6 = m->nonlin == 3;
  const float* in[kTcMaxBanks];
  const float* l2[kTcMaxBanks];
  ConvTcGeo geo[kTcMaxBanks];
  int org[kTcMaxBanks];
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
    if (m->bank_dilate && i > 0 && ((tg.nx | tg.ny | tg.nz) & ((1 << i) - 1)))
      launch_tc_phase_zero(o1, geo[i], i, tg, st);
    launch_conv3_tc(o1, o2, nullptr, m->wBk[split][2 * i + 1].get(), m->b[m->conv0[1] + i].get(), nullptr, 2, 0,
                    split, g2, st, act);
    l2[i] = o2;
  }
  ConvTcGeo g3 = tg;
  g3.z_lo = std::max(0, p_lo);
  g3.z_hi = std::min(tg.nz, p_hi);
  launch_tc_join(l2, geo, org, zoff, nbk, m->bank_add, m->part.get(), p_net, m->wBj[split], m->b[m->conv0[2]].get(),
                 m->tail.get(), split, g3, st, m->bank_dilate != 0, act);
}

// The three 3x3x3 layers (+ fused 1x1x1 tail) on tensor cores: act[0] -> act[1] -> act[2] -> p_net.
// p_lo / p_hi: planes on which p_net is wanted (default all).  Layer l then only has to produce the planes the
// later layers' 3x3x3 stencils reach from there; on a z-slab that spares most of the ghost planes.
void run_conv_stack(tfl_cnn* m, float* p_net, cudaStream_t st, int p_lo, int p_hi) {
  if (p_hi < 0) p_hi = m->act_geo.nz;
  if (m->nbanks > 1) {
    run_conv_stack_banked(m, p_net, st, p_lo, p_hi);
    return;
  }
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
    return;
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
}

static const tfl_cnn_inputs kDefaultInputs = {1, 0, 1, 1, 0, 0, 0};

namespace {

// A model as the arguments of tfl_cnn_create_model_norm describe it, whichever creator it came through.
struct CnnSpec {
  int is_3d, n_layers;
  const int32_t *cin, *cout, *ksize, *pool, *up;     // pool / up may be null (all 1)
  int pool_is_max, nonlin_sigmoid;
  const float* const* weights;
  const float* const* biases;
  tfl_cnn_banks_ex banks = {1, 0, 0, 0, 0};          // num = 1: no banks
  bool banks_given = false;                           // the bank assertions of lib/model.lua hold whatever num is
  tfl_cnn_inputs inputs = kDefaultInputs;
  const tfl_cnn_norm* norm = nullptr;
};

void set_banks(CnnSpec& s, const tfl_cnn_banks_ex* banks) {
  if (!banks) return;
  s.banks = *banks;
  s.banks_given = true;
}
void set_banks(CnnSpec& s, const tfl_cnn_banks* banks) {
  if (!banks) return;
  const tfl_cnn_banks_ex ex = {banks->num, banks->split_stage, banks->join_stage, banks->aggregate_add, 0};
  set_banks(s, &ex);
}

// Convolutions of stage l: one per bank in the banked stages.
int stage_convs(const tfl_cnn* m, int l) { return (m->nbanks > 1 && l >= m->split && l < m->join) ? m->nbanks : 1; }

// Checks a spec, in one order whichever creator it came through, and fills in m's host-side description of the
// model.  Makes no CUDA call.
int cnn_validate(tfl_ctx* ctx, const CnnSpec& s, tfl_cnn** out, tfl_cnn* m) {
  const tfl_cnn_norm* norm = s.norm;
  if (norm && norm->relu6 && s.nonlin_sigmoid)
    return fail(ctx, "cnn: nonlinType is either 'relu6' or 'sigmoid', not both");
  if (norm && norm->batch_norm && (!norm->bn || !norm->eps))
    return fail(ctx, "cnn: addBatchNorm needs the batch normalization parameters (bn) and eps of every module");
  const tfl_cnn_banks_ex& banks = s.banks;
  if (banks.dilate != 0 && banks.dilate != 1)
    return fail(ctx, "cnn: banks dilate must be 0 ('mres') or 1 ('dilate') (got %d)", banks.dilate);
  const tfl_cnn_inputs& in = s.inputs;
  // lib/model.lua:27-150 and :357-361; checkYangSettings, lib/model_utils.lua:211-227.
  if (!in.p_div && !in.u_div && !in.div) return fail(ctx, "Are you sure you dont want any (U, div or p) fields?");
  if (!in.u_div && !in.div)
    return fail(ctx, "cnn: inputChannels needs UDiv or div: tfluids.VelocityUpdate takes UDiv, which the graph "
                     "selects only for them (lib/model.lua:69-72, :380)");
  if (in.normalize && in.norm_func != 0 && in.norm_func != 1) return fail(ctx, "Incorrect normalize input function");
  if (in.normalize && (in.norm_chan < 0 || in.norm_chan > 2)) return fail(ctx, "Incorrect normalize input channel.");
  if (in.normalize && in.norm_chan == 2 && !in.div)
    return fail(ctx, "cnn: normalizeInputChan 'div' needs inputChannels.div (lib/model.lua:108-116)");
  const int is_3d = s.is_3d, n_layers = s.n_layers;
  const int32_t *cin = s.cin, *cout_logical = s.cout, *ksize = s.ksize, *pool = s.pool, *up = s.up;
  if (!out || n_layers < 1 || !cin || !cout_logical || !ksize || !s.weights || !s.biases)
    return fail(ctx, "cnn: bad arguments");
  bool unit_sizes = true;     // no pooling, no upsampling
  for (int l = 0; l < n_layers; l++) unit_sizes = unit_sizes && (!pool || pool[l] == 1) && (!up || up[l] == 1);
  // 'yang' (lib/model.lua:228-239): osize {6, 6, 6, 1}, ksize {3, 1, 1, 1}
  const bool yang = n_layers == 4 && unit_sizes && cout_logical[0] == 6 && cout_logical[1] == 6 &&
                    cout_logical[2] == 6 && cout_logical[3] == 1 && ksize[0] == 3 && ksize[1] == 1 && ksize[2] == 1 &&
                    ksize[3] == 1;
  if (yang && !in.p_div) return fail(ctx, "ERROR: yang model must have pDiv input");
  if (yang && !in.div) return fail(ctx, "ERROR: yang model must have div input");
  if (yang && in.u_div) return fail(ctx, "ERROR: yang model must not have UDiv input");
  if (in.pressure_skip && (n_layers < 2 || ksize[n_layers - 1] != 1 || (up && up[n_layers - 1] != 1)))
    return fail(ctx, "cnn: addPressureSkip joins pDiv to the hidden layer before the last convolution at full "
                     "resolution, which needs a 1x1 last convolution without upsampling (lib/model.lua:357-361; "
                     "not 'tog')");
  if (s.banks_given) {     // the assertions of lib/model.lua:246-252 (checked whatever banksNum is)
    if (banks.num < 1) return fail(ctx, "cnn: banksNum >= 1 failed (got %d)", banks.num);
    if (!(banks.split_stage < banks.join_stage))
      return fail(ctx, "cnn: banksSplitStage < banksJoinStage failed (%d, %d)", banks.split_stage, banks.join_stage);
    if (banks.split_stage < 1 || banks.split_stage >= n_layers)
      return fail(ctx, "cnn: banksSplitStage >= 1 and banksSplitStage < #osize failed (%d, %d stages)",
                  banks.split_stage, n_layers);
    if (banks.join_stage < 1 || banks.join_stage >= n_layers)
      return fail(ctx, "cnn: banksJoinStage >= 1 and banksJoinStage < #osize failed (%d, %d stages)",
                  banks.join_stage, n_layers);
    if (banks.num > kMaxBanks) return fail(ctx, "cnn: at most %d banks are supported (got %d)", kMaxBanks, banks.num);
    // getConvLayer's assertion for banks 2..N, dilated by 2^(i-1) (lib/model_utils.lua:125)
    for (int l = banks.split_stage - 1; banks.dilate && banks.num > 1 && up && l < banks.join_stage - 1; l++)
      if (up[l] > 1) return fail(ctx, "upsampling not supported for dilated convolutions. (stage %d)", l + 1);
  }
  const int nbanks = banks.num;
  const int bsplit = nbanks > 1 ? banks.split_stage - 1 : 0, bjoin = nbanks > 1 ? banks.join_stage - 1 : 0;
  const int in_sel = (in.p_div ? kCnnInPDiv : 0) | (in.u_div ? kCnnInUDiv : 0) | (in.div ? kCnnInDiv : 0);
  const int in_ch = (in.p_div ? 1 : 0) + (in.u_div ? (is_3d ? 3 : 2) : 0) + (in.div ? 1 : 0) + 1;
  const bool skip = in.pressure_skip != 0;
  // Channels the convolution of layer l really emits: cout * up^d (ConvolutionUpsample, model_utils.lua:74-76).
  std::vector<int32_t> cout_conv(n_layers);
  bool plain = !s.nonlin_sigmoid;
  for (int l = 0; l < n_layers; l++) {
    const int u = up ? up[l] : 1, pl = pool ? pool[l] : 1;
    if (u < 1 || pl < 1) return fail(ctx, "cnn: pooling / upsampling sizes must be >= 1");
    if (u > 1 && pl > 1) return fail(ctx, "Pooling and upsampling in the same layer!");          // model.lua:326
    if (l == n_layers - 1 && pl != 1) return fail(ctx, "Pooling is not allowed in the last layer");  // model.lua:245
    cout_conv[l] = cout_logical[l] * u * u * (is_3d ? u : 1);
    if (u != 1 || pl != 1) plain = false;
  }
  const int32_t* cout = cout_conv.data();
  if (cout_logical[n_layers - 1] != 1) return fail(ctx, "Last layer osize must be 1 (pressure)");   // model.lua:244
  if (in_sel == (kCnnInPDiv | kCnnInDiv) && cin[0] != 3)
    return fail(ctx, "cnn: the first layer must take 3 channels (pDiv, div, occupancy)");
  if (cin[0] != in_ch)
    return fail(ctx, "cnn: the input block has %d channels (pDiv, UDiv, div, occupancy as selected), the first layer "
                     "takes %d", in_ch, cin[0]);
  // The last convolution's channels without the pressure skip's pDiv (its last input channel, lib/model.lua:357-361).
  std::vector<int32_t> cin_net(cin, cin + n_layers);
  if (skip) {
    if (cin[n_layers - 1] != cout_logical[n_layers - 2] + 1)
      return fail(ctx, "cnn: with addPressureSkip the last convolution takes cout[%d] + 1 = %d channels (got %d)",
                  n_layers - 2, cout_logical[n_layers - 2] + 1, cin[n_layers - 1]);
    cin_net[n_layers - 1] -= 1;
  }
  cin = cin_net.data();
  if (nbanks > 1) plain = false;
  const bool relu6 = norm && norm->relu6, bn = norm && norm->batch_norm;
  if (relu6 || bn) plain = false;     // the stage loop applies BN; relu6 is activation code 3
  m->bn = bn;
  m->bn_batch = bn && norm->batch_stats;
  m->in_sel = in_sel;
  m->in_ch = in_ch;
  m->norm_func = in.normalize ? (in.norm_func == 1 ? kCnnScaleNorm : kCnnScaleStd) : kCnnScaleOne;
  m->norm_chan = in.norm_chan == 1 ? kCnnStatPDiv : (in.norm_chan == 2 ? kCnnStatDiv : kCnnStatU);
  if (!in.normalize) m->norm_chan = kCnnStatU;
  m->skip = skip;
  m->default_inputs = in_sel == (kCnnInPDiv | kCnnInDiv) && m->norm_func == kCnnScaleStd && m->norm_chan == kCnnStatU &&
                      !skip;
  m->tc_planes = (in_sel & kCnnInUDiv) ? 2 : 1;
  m->plain = plain;
  m->pool_is_max = s.pool_is_max ? 1 : 0;
  m->nonlin = s.nonlin_sigmoid ? 2 : (relu6 ? 3 : 1);
  m->is3d = is_3d ? 1 : 0;
  m->n_layers = n_layers;
  m->nbanks = nbanks;
  m->split = bsplit;
  m->join = bjoin;
  m->bank_add = nbanks > 1 && banks.aggregate_add ? 1 : 0;
  m->bank_dilate = nbanks > 1 && banks.dilate ? 1 : 0;
  int wi = 0;     // index into weights / biases
  for (int l = 0; l < n_layers; l++) {
    if (l > 0 && nbanks > 1 && l == bjoin && !m->bank_add && cin[l] != nbanks * cout_logical[l - 1])
      return fail(ctx, "cnn: stage %d concatenates %d banks of %d channels, so it needs cin = %d (got %d)", l + 1,
                  nbanks, cout_logical[l - 1], nbanks * cout_logical[l - 1], cin[l]);
    if (l > 0 && !(nbanks > 1 && l == bjoin && !m->bank_add) && cin[l] != cout_logical[l - 1])
      return fail(ctx, "cnn: channel mismatch at layer %d", l);
    if (ksize[l] % 2 != 1) return fail(ctx, "convolution size must be odd");     // model_utils.lua:70
    m->pool.push_back(pool ? pool[l] : 1);
    m->up.push_back(up ? up[l] : 1);
    m->conv0.push_back(wi);
    for (int k = 0; k < stage_convs(m, l); k++, wi++) {
      m->cin.push_back(cin[l]); m->cout.push_back(cout[l]); m->ks.push_back(ksize[l]);
      if (bn && l < n_layers - 1) {
        if (!norm->bn[wi])
          return fail(ctx, "cnn: addBatchNorm: the batch normalization parameters of convolution %d are missing",
                      wi + 1);
        const float eps = norm->eps[wi];
        if (!(eps >= 0.0f))
          return fail(ctx, "cnn: batch normalization eps of convolution %d must be >= 0 (got %g)", wi + 1, eps);
        m->bn_eps.push_back(eps);
        m->bn_max_c = std::max(m->bn_max_c, (int)cout_logical[l]);
      }
    }
    if (cout[l] > m->max_c) m->max_c = cout[l];
  }
  {   // largest activation of the graph, in channels x cells-of-the-input-grid (banks 2..N have buffers of their
      // own, cnn_scratch; the joined banks are counted here)
    double rel = 1.0;
    m->max_rel = in_ch;      // the network input (pooled into, or shared by, the banks at stage 1)
    for (int l = 0; l < n_layers; l++) {
      if (nbanks > 1 && l == bjoin) m->max_rel = std::max(m->max_rel, rel * cin[l]);   // the joined banks
      if (nbanks > 1 && l >= bsplit && l < bjoin)     // one bank's activations (no upsampling in a dilated stage)
        m->bank_rel = std::max(m->bank_rel, rel * std::max(cout[l], cout_logical[l]));
      m->max_rel = std::max(m->max_rel, rel * cout[l]);                          // convolution output
      const int u = m->up[l], pl = m->pool[l];
      rel *= (double)u * u * (is_3d ? u : 1);
      m->max_rel = std::max(m->max_rel, rel * cout_logical[l]);                  // after the pixel shuffle
      rel /= (double)pl * pl * (is_3d ? pl : 1);
    }
    if (rel != 1.0) return fail(ctx, "cnn: pooling and upsampling do not return to the input resolution");
    if ((double)m->max_c < m->max_rel) m->max_c = (int)std::ceil(m->max_rel);
  }
  // Tensor-core eligibility: the 3-D 'default' graph (lib/model.lua:219-226), single-bank or with banks (either type)
  // split before stage 1 and joined before stage 3.
  static const int want[5][3] = {{0, 8, 3}, {8, 8, 3}, {8, 8, 3}, {8, 8, 1}, {8, 1, 1}};   // cin[0]: any input set
  m->tc_ok = is_3d && n_layers == 5 && !s.nonlin_sigmoid && !(bn && nbanks > 1) &&
             (nbanks == 1 || (bsplit == 0 && bjoin == 2 && nbanks <= kTcMaxBanks));
  for (int l = 0; m->tc_ok && l < 5; l++) {
    const int want_cin = l == 0 ? in_ch : (l == 2 && !m->bank_add) ? 8 * nbanks : want[l][0];
    m->tc_ok = m->pool[l] == 1 && m->up[l] == 1 && cin[l] == want_cin && cout[l] == want[l][1] && ksize[l] == want[l][2];
  }
  return 0;
}

// Puts the parameters of a model cnn_validate has described on the device: every convolution's weights, bias and
// batch normalization, and for the tensor cores the packed weights and the tail.  1 if a cudaMalloc or cudaMemcpy
// fails.
int cnn_upload(const CnnSpec& s, tfl_cnn* m) {
  const float* const* weights = s.weights;
  const float* const* biases = s.biases;
  const int n_layers = s.n_layers;
  for (int l = 0, wi = 0; l < n_layers; l++) {
    const int taps = (s.is_3d ? s.ksize[l] : 1) * s.ksize[l] * s.ksize[l];
    for (int k = 0; k < stage_convs(m, l); k++, wi++) {
      // the skip's layer is 1x1 with one output: its hidden channels' weights come first, pDiv's last
      if (m->skip && l == n_layers - 1) m->w_skip = weights[wi][m->cin[wi]];
      if (!keep(m->w, upload(relayout_conv_weights(weights[wi], m->cin[wi], m->cout[wi], taps))) ||
          !keep(m->b, upload(biases[wi], m->cout[wi])))
        return 1;
      if (m->bn && l < n_layers - 1 &&
          !keep(m->bn_batch ? m->bn_wb : m->bn_ac, upload_bn(s.norm, m->bn_batch, wi, s.cout[l])))
        return 1;
    }
  }
  if (!m->tc_ok) return 0;
  const int nbanks = m->nbanks, in_ch = m->in_ch, j0 = m->conv0[2], nj = m->bank_add ? 1 : nbanks;
  for (int split = 0; split < 2; split++) {
    for (int i = 0; i < nbanks; i++) {                 // layers 1 and 2 of bank i
      // layer 1: the input set on one float4 plane, or (with UDiv) on two with zero weights past in_ch
      const float* w1 = weights[m->conv0[0] + i];
      if (!keep(m->wBk[split], m->tc_planes == 1 ? upload_tc_weights(w1, in_ch, split)
                                                 : upload_tc_weights(pad_cin8(w1, in_ch).data(), 8, split)) ||
          !keep(m->wBk[split], upload_tc_weights(weights[m->conv0[1] + i], 8, split)))
        return 1;
    }
    for (int i = 0; i < nj; i++)
      if (!keep(m->wBj[split], upload_tc_weights(concat_slice(weights[j0], nj, i).data(), 8, split))) return 1;
  }
  std::vector<float> tail(kTailFloats);
  memcpy(tail.data(), weights[m->conv0[3]], 64 * 4);
  memcpy(tail.data() + 64, biases[m->conv0[3]], 8 * 4);
  memcpy(tail.data() + 72, weights[m->conv0[4]], 8 * 4);
  tail[80] = biases[m->conv0[4]][0];
  if (m->bn && !m->bn_batch) {
    // running statistics: BN3 (after layer 3's activation) into w4 / b4, BN4 (after layer 4's) into w5 / b5, exact in
    // real arithmetic: w4 (a3 h + c3) + b4 = (w4 a3) h + (b4 + w4 c3), w5 (a4 h + c4) + b5 = (w5 a4) h + (b5 + w5 c4)
    double a3[8], c3[8], a4[8], c4[8];
    bn_running_affine(s.norm, 2, 8, a3, c3);
    bn_running_affine(s.norm, 3, 8, a4, c4);
    double b5 = tail[80];
    for (int o = 0; o < 8; o++) {
      double b4 = tail[64 + o];
      for (int c = 0; c < 8; c++) {
        b4 += (double)tail[o * 8 + c] * c3[c];
        tail[o * 8 + c] = (float)((double)tail[o * 8 + c] * a3[c]);
      }
      tail[64 + o] = (float)b4;
      b5 += (double)tail[72 + o] * c4[o];
      tail[72 + o] = (float)((double)tail[72 + o] * a4[o]);
    }
    tail[80] = (float)b5;
  }
  if (m->bn_batch && (!(m->bn_part = dev_alloc<double>(2 * (kBnBlocks + 1) * 8)) ||
                      !(m->bn_tcac = dev_alloc<float>(4 * 16))))
    return 1;
  if (!(m->tail = upload(tail))) return 1;
  m->mode = 2;
  return 0;
}

// The one path of every creator: nothing reaches the device unless the spec is valid, and a failed upload frees what
// was uploaded before it.
int cnn_create(tfl_ctx* ctx, const CnnSpec& s, tfl_cnn** out) {
  std::unique_ptr<tfl_cnn> m(new tfl_cnn());
  if (cnn_validate(ctx, s, out, m.get())) return 1;
  if (cnn_upload(s, m.get())) return fail(ctx, "cnn: cudaMalloc failed");
  *out = m.release();
  return 0;
}

}  // namespace

extern "C" {

// ---------------------------------------------------------------------------------------
// CNN projection
// ---------------------------------------------------------------------------------------
int tfl_cnn_create(tfl_ctx* ctx, int is_3d, int n_layers, const int32_t* cin, const int32_t* cout,
                   const int32_t* ksize, const float* const* weights, const float* const* biases,
                   tfl_cnn** out) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  return cnn_create(ctx, {is_3d, n_layers, cin, cout, ksize, nullptr, nullptr, 0, 0, weights, biases}, out);
}

int tfl_cnn_create_graph(tfl_ctx* ctx, int is_3d, int n_layers, const int32_t* cin, const int32_t* cout,
                         const int32_t* ksize, const int32_t* pool, const int32_t* up, int pool_is_max,
                         int nonlin_sigmoid, const float* const* weights, const float* const* biases,
                         tfl_cnn** out) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  return cnn_create(ctx, {is_3d, n_layers, cin, cout, ksize, pool, up, pool_is_max, nonlin_sigmoid, weights, biases},
                    out);
}

int tfl_cnn_create_banked(tfl_ctx* ctx, int is_3d, int n_layers, const int32_t* cin, const int32_t* cout,
                          const int32_t* ksize, const int32_t* pool, const int32_t* up, int pool_is_max,
                          int nonlin_sigmoid, const tfl_cnn_banks* banks, const float* const* weights,
                          const float* const* biases, tfl_cnn** out) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  CnnSpec s = {is_3d, n_layers, cin, cout, ksize, pool, up, pool_is_max, nonlin_sigmoid, weights, biases};
  set_banks(s, banks);
  return cnn_create(ctx, s, out);
}

int tfl_cnn_create_model(tfl_ctx* ctx, int is_3d, int n_layers, const int32_t* cin, const int32_t* cout,
                         const int32_t* ksize, const int32_t* pool, const int32_t* up, int pool_is_max,
                         int nonlin_sigmoid, const tfl_cnn_banks* banks, const tfl_cnn_inputs* inputs,
                         const float* const* weights, const float* const* biases, tfl_cnn** out) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  CnnSpec s = {is_3d, n_layers, cin, cout, ksize, pool, up, pool_is_max, nonlin_sigmoid, weights, biases};
  set_banks(s, banks);
  if (inputs) s.inputs = *inputs;
  return cnn_create(ctx, s, out);
}

int tfl_cnn_create_model_ex(tfl_ctx* ctx, int is_3d, int n_layers, const int32_t* cin, const int32_t* cout,
                            const int32_t* ksize, const int32_t* pool, const int32_t* up, int pool_is_max,
                            int nonlin_sigmoid, const tfl_cnn_banks_ex* banks, const tfl_cnn_inputs* inputs,
                            const float* const* weights, const float* const* biases, tfl_cnn** out) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  CnnSpec s = {is_3d, n_layers, cin, cout, ksize, pool, up, pool_is_max, nonlin_sigmoid, weights, biases};
  set_banks(s, banks);
  if (inputs) s.inputs = *inputs;
  return cnn_create(ctx, s, out);
}

int tfl_cnn_create_model_norm(tfl_ctx* ctx, int is_3d, int n_layers, const int32_t* cin, const int32_t* cout,
                              const int32_t* ksize, const int32_t* pool, const int32_t* up, int pool_is_max,
                              int nonlin_sigmoid, const tfl_cnn_banks_ex* banks, const tfl_cnn_inputs* inputs,
                              const tfl_cnn_norm* norm, const float* const* weights, const float* const* biases,
                              tfl_cnn** out) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  CnnSpec s = {is_3d, n_layers, cin, cout, ksize, pool, up, pool_is_max, nonlin_sigmoid, weights, biases};
  set_banks(s, banks);
  if (inputs) s.inputs = *inputs;
  s.norm = norm;
  return cnn_create(ctx, s, out);
}

int tfl_cnn_set_mode(tfl_ctx* ctx, tfl_cnn* m, int mode) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!m || mode < 0 || mode > 2) return fail(ctx, "cnn_set_mode: bad arguments");
  if (mode > 0 && m->bn && m->nbanks > 1)
    return fail(ctx, "cnn_set_mode: banked models with batch normalization (addBatchNorm) run on the fp32 path; the "
                     "tensor-core path takes batch normalization on the single-bank 3-D 'default' graph");
  if (mode > 0 && m->nbanks > 1 && !m->tc_ok)
    return fail(ctx, "cnn_set_mode: the tensor-core path covers the 3-D 'default' architecture, single-bank or with "
                     "banks split at stage 1 and joined at stage 3; this banked model runs on the fp32 path");
  if (mode > 0 && !m->tc_ok)
    return fail(ctx, "cnn_set_mode: the tensor-core path covers the 3-D 'default' architecture only");
  m->mode = mode;
  return 0;
}
int tfl_cnn_get_mode(const tfl_cnn* m) { return m ? m->mode : -1; }

// Undocumented debugging hook (not in tfl.h): per-CTA phase timestamps of the tensor-core conv.
int tfl_debug_conv_timestamps(void* dev_buf) { conv_tc_set_debug((long long*)dev_buf); return 0; }

// Undocumented test hooks (not in tfl.h): one tensor-core 3x3x3 layer on caller-owned buffers.
// tfl_debug_conv_tc_layout: the padded pitches (px, py) of make_conv_tc_geo, so callers can lay out
// in / out ([nb][2 planes][nz+2][py][px] float4); p_net is plain [nb][nz][ny][nx].
int tfl_debug_conv_tc_layout(int nb, int nz, int ny, int nx, int32_t out[2]) {
  const ConvTcGeo g = make_conv_tc_geo(nb, nz, ny, nx);
  out[0] = g.px;
  out[1] = g.py;
  return 0;
}

// tfl_debug_conv3_tc: weights [8][cin][3][3][3] and bias [8] on the host, packed with conv_tc_pack_weights;
// tail (final layer only): w4[8][8], b4[8], w5[8], b5[1] as in tfl_cnn_create_graph.  Output planes
// [z_lo, z_hi) only.  Synchronises before returning.
int tfl_debug_conv3_tc(tfl_ctx* ctx, const float* in, float* out, float* p_net, const float* w_host,
                       const float* bias_host, const float* tail_host, int cin, int final_layer, int split,
                       int nb, int nz, int ny, int nx, int z_lo, int z_hi) {
  DeviceGuard guard_(ctx);
  if (!ctx) return 1;
  if (cin != 3 && cin != 8) return fail(ctx, "debug_conv3_tc: cin must be 3 or 8 (got %d)", cin);
  if (final_layer && cin != 8) return fail(ctx, "debug_conv3_tc: the final layer takes 8 channels");
  if (final_layer && (!tail_host || !p_net)) return fail(ctx, "debug_conv3_tc: the final layer needs tail and p_net");
  if (!final_layer && !out) return fail(ctx, "debug_conv3_tc: nil out");
  if (!in || !w_host || !bias_host) return fail(ctx, "debug_conv3_tc: nil argument");
  if (nb < 1 || nz < 1 || ny < 1 || nx < 1) return fail(ctx, "debug_conv3_tc: bad grid %dx%dx%dx%d", nb, nz, ny, nx);
  if (z_lo < 0 || z_hi > nz || z_lo >= z_hi) return fail(ctx, "debug_conv3_tc: z range [%d, %d) not in [0, %d]", z_lo, z_hi, nz);
  ConvTcGeo g = make_conv_tc_geo(nb, nz, ny, nx);
  g.z_lo = z_lo;
  g.z_hi = z_hi;
  const DevPtr<float> wB = upload_tc_weights(w_host, cin, split), bias = upload(bias_host, 8),
                      tail = final_layer ? upload(tail_host, kTailFloats) : DevPtr<float>();
  if (!wB || !bias || (final_layer && !tail)) return fail(ctx, "debug_conv3_tc: cudaMalloc failed");
  launch_conv3_tc(in, out, p_net, wB.get(), bias.get(), tail.get(), cin == 3 ? 1 : 2, final_layer, split, g,
                  ctx->stream);
  return finish_debug(ctx, "debug_conv3_tc");
}

// Undocumented test hook (not in tfl.h): caps the persistent grid of the z-streaming tensor-core convolution at
// `ctas` CTAs (0: one per SM), so that every CTA runs several work items back to back.
int tfl_debug_conv_tc_z_grid(int ctas) {
  conv_tc_set_z_grid(ctas);
  return 0;
}

// tfl_debug_conv3_tc_bn: one tensor-core 3x3x3 layer (not the final one) with the batch normalization of the
// projection network on caller-owned padded buffers (layout as tfl_debug_conv3_tc).  relu6: the epilogue clamps at 6;
// ep_ac_host ([2][8] a, c, may be NULL): running-statistics BN in the epilogue, y = a act(h) + c on the voxels
// written; batch = 1: then batch statistics over out's interior (launch_tc_bn_stats, launch_bn_finalize with
// bn_w_host / bn_b_host [8] (may be NULL: 1 / 0) and eps) and y = a x + c in place on the interior; stats_host
// ([8][2] mean, biased variance) and ac_host ([2][8]) receive what the finalize computed.  Synchronises.
int tfl_debug_conv3_tc_bn(tfl_ctx* ctx, const float* in, float* out, const float* w_host, const float* bias_host,
                          int cin, int split, int relu6, const float* ep_ac_host, int batch, const float* bn_w_host,
                          const float* bn_b_host, float eps, double* stats_host, float* ac_host, int nb, int nz, int ny,
                          int nx) {
  DeviceGuard guard_(ctx);
  if (!ctx) return 1;
  if (cin != 3 && cin != 8) return fail(ctx, "debug_conv3_tc_bn: cin must be 3 or 8 (got %d)", cin);
  if (!in || !out || !w_host || !bias_host || (batch && (!stats_host || !ac_host)))
    return fail(ctx, "debug_conv3_tc_bn: nil argument");
  if (bad_grid(nb, nz, ny, nx, 1) || !(eps >= 0.0f)) return fail(ctx, "debug_conv3_tc_bn: bad arguments");
  const ConvTcGeo g = make_conv_tc_geo(nb, nz, ny, nx);
  const DevPtr<float> wB = upload_tc_weights(w_host, cin, split), bias = upload(bias_host, 8),
                      ep = ep_ac_host ? upload(ep_ac_host, 16) : DevPtr<float>(),
                      bw = bn_w_host ? upload(bn_w_host, 8) : DevPtr<float>(),
                      bb = bn_b_host ? upload(bn_b_host, 8) : DevPtr<float>(), ac = dev_alloc<float>(16);
  const DevPtr<double> part = dev_alloc<double>(2 * (kBnBlocks + 1) * 8), stats = dev_alloc<double>(16);
  if (!wB || !bias || (ep_ac_host && !ep) || (bn_w_host && !bw) || (bn_b_host && !bb) || !ac || !part || !stats)
    return fail(ctx, "debug_conv3_tc_bn: cudaMalloc failed");
  TcEpi e;
  e.relu6 = relu6 ? 1 : 0;
  e.ac = ep.get();
  launch_conv3_tc(in, out, nullptr, wB.get(), bias.get(), nullptr, cin == 3 ? 1 : 2, 0, split, g, ctx->stream, e);
  if (batch) {
    launch_tc_bn_stats(out, g, part.get(), ctx->stream);
    launch_bn_finalize(part.get(), 8, (long long)nb * nz * ny * nx, bw.get(), bb.get(), eps, ac.get(), stats.get(),
                       ctx->stream);
    launch_tc_bn_apply(out, g, ac.get(), ctx->stream);
  }
  if (const int rc = finish_debug(ctx, "debug_conv3_tc_bn")) return rc;
  if (batch && (cudaMemcpy(stats_host, stats.get(), sizeof(double) * 16, cudaMemcpyDeviceToHost) != cudaSuccess ||
                cudaMemcpy(ac_host, ac.get(), 16 * 4, cudaMemcpyDeviceToHost) != cudaSuccess))
    return fail(ctx, "debug_conv3_tc_bn: copy failed");
  return 0;
}

// tfl_debug_conv3_tc_dilated: one tensor-core 3x3x3 layer (not the final one) dilated by 2^sh the way a dilated bank
// runs it: in (make_conv_tc_geo(nb, nz, ny, nx) layout, cin 3 on one float4 plane or 8 on two) is copied into phase
// sub-grids, the layer runs on those, layer-1 style re-zeroing of short phases follows, and the sub-grids are gathered
// back into the interior of out (same layout, 8 channels; nothing else of out is written).  Synchronises.
int tfl_debug_conv3_tc_dilated(tfl_ctx* ctx, const float* in, float* out, const float* w_host, const float* bias_host,
                               int cin, int split, int nb, int nz, int ny, int nx, int sh) {
  DeviceGuard guard_(ctx);
  if (!ctx) return 1;
  if (cin != 3 && cin != 8) return fail(ctx, "debug_conv3_tc_dilated: cin must be 3 or 8 (got %d)", cin);
  if (!in || !out || !w_host || !bias_host) return fail(ctx, "debug_conv3_tc_dilated: nil argument");
  if (sh < 0 || sh > 7 || bad_grid(nb, nz, ny, nx, 1))
    return fail(ctx, "debug_conv3_tc_dilated: bad grid %dx%dx%dx%d or dilation 2^%d", nb, nz, ny, nx, sh);
  const ConvTcGeo gf = make_conv_tc_geo(nb, nz, ny, nx), gs = make_conv_tc_phase_geo(nb, nz, ny, nx, sh);
  const DevPtr<float> wB = upload_tc_weights(w_host, cin, split), bias = upload(bias_host, 8),
                      sin = dev_zeros<float>(conv_tc_act_bytes(gs) / 4),
                      sout = dev_zeros<float>(conv_tc_act_bytes(gs) / 4);
  if (!wB || !bias || !sin || !sout) return fail(ctx, "debug_conv3_tc_dilated: cudaMalloc failed");
  const int planes = cin == 3 ? 1 : 2;
  launch_tc_phase_copy(in, gf, sin.get(), gs, sh, planes, ctx->stream);
  launch_conv3_tc(sin.get(), sout.get(), nullptr, wB.get(), bias.get(), nullptr, planes, 0, split, gs, ctx->stream);
  launch_tc_phase_zero(sout.get(), gs, sh, gf, ctx->stream);
  launch_tc_phase_gather(sout.get(), gs, out, gf, sh, ctx->stream);
  return finish_debug(ctx, "debug_conv3_tc_dilated");
}

// tfl_debug_conv3_tc_join: the join layer of a banked model (split 1, join 3) on caller-owned bank buffers.
// banks[i] (device) is bank i+1's layer-2 output in the padded layout of make_conv_tc_geo(nb, nz >> i, ny >> i,
// nx >> i); w_host [8][cin][3][3][3] with cin = 8 (add) or 8 nbanks (concat), bias [8], tail as in
// tfl_debug_conv3_tc.  Writes p_net [nb][nz][ny][nx].  Synchronises before returning.
static int debug_join_impl(tfl_ctx* ctx, const float* const* banks, int nbanks, int add, float* p_net,
                           const float* w_host, const float* bias_host, const float* tail_host, int split, int nb,
                           int nz, int ny, int nx, int zoff, const int32_t* bank_nz, const int32_t* bank_org, int z_lo,
                           int z_hi);

int tfl_debug_conv3_tc_join(tfl_ctx* ctx, const float* const* banks, int nbanks, int add, float* p_net,
                            const float* w_host, const float* bias_host, const float* tail_host, int split, int nb,
                            int nz, int ny, int nx) {
  DeviceGuard guard_(ctx);
  if (!ctx) return 1;
  if (nbanks < 1 || nbanks > kTcMaxBanks) return fail(ctx, "debug_conv3_tc_join: bad bank count %d", nbanks);
  const int r = 1 << (nbanks - 1);
  if (nb < 1 || nz < 1 || ny < 1 || nx < 1 || nz % r || ny % r || nx % r)
    return fail(ctx, "debug_conv3_tc_join: grid %dx%dx%dx%d is not divisible by %d", nb, nz, ny, nx, r);
  int32_t bnz[kTcMaxBanks], borg[kTcMaxBanks] = {};
  for (int i = 0; i < nbanks; i++) bnz[i] = nz >> i;
  return debug_join_impl(ctx, banks, nbanks, add, p_net, w_host, bias_host, tail_host, split, nb, nz, ny, nx, 0, bnz,
                         borg, 0, nz);
}

// tfl_debug_conv3_tc_join_slab: the same join on a z-slab.  p_net's local planes [0, nz) are the global planes
// zoff + z; bank i (i >= 1) holds bank_nz[i] planes from global coarse plane bank_org[i] on (bank_nz[0] and
// bank_org[0] are ignored: bank 1 is nz planes from zoff).  Writes the output planes [z_lo, z_hi) of p_net only.
int tfl_debug_conv3_tc_join_slab(tfl_ctx* ctx, const float* const* banks, int nbanks, int add, float* p_net,
                                 const float* w_host, const float* bias_host, const float* tail_host, int split,
                                 int nb, int nz, int ny, int nx, int zoff, const int32_t* bank_nz,
                                 const int32_t* bank_org, int z_lo, int z_hi) {
  DeviceGuard guard_(ctx);
  if (!ctx) return 1;
  if (nbanks < 1 || nbanks > kTcMaxBanks) return fail(ctx, "debug_conv3_tc_join_slab: bad bank count %d", nbanks);
  if (!bank_nz || !bank_org) return fail(ctx, "debug_conv3_tc_join_slab: nil argument");
  const int r = 1 << (nbanks - 1);
  if (nb < 1 || nz < 1 || ny < 1 || nx < 1 || ny % r || nx % r || zoff < 0)
    return fail(ctx, "debug_conv3_tc_join_slab: bad grid %dx%dx%dx%d", nb, nz, ny, nx);
  if (z_lo < 0 || z_hi > nz || z_lo >= z_hi) return fail(ctx, "debug_conv3_tc_join_slab: bad z range [%d, %d)", z_lo, z_hi);
  int32_t bnz[kTcMaxBanks], borg[kTcMaxBanks];
  bnz[0] = nz;
  borg[0] = zoff;
  for (int i = 1; i < nbanks; i++) {
    bnz[i] = bank_nz[i];
    borg[i] = bank_org[i];
    // the staged boxes may index ((z + zoff) >> i) - org for any z in [0, nz): inside the bank's padded planes
    const int lo = (zoff >> i) - borg[i], hi = ((zoff + nz - 1) >> i) - borg[i];
    if (bnz[i] < 1 || lo < -1 || hi > bnz[i])
      return fail(ctx, "debug_conv3_tc_join_slab: bank %d (%d planes from %d) does not cover the slab", i + 1, bnz[i],
                  borg[i]);
  }
  return debug_join_impl(ctx, banks, nbanks, add, p_net, w_host, bias_host, tail_host, split, nb, nz, ny, nx, zoff,
                         bnz, borg, z_lo, z_hi);
}

static int debug_join_impl(tfl_ctx* ctx, const float* const* banks, int nbanks, int add, float* p_net,
                           const float* w_host, const float* bias_host, const float* tail_host, int split, int nb,
                           int nz, int ny, int nx, int zoff, const int32_t* bank_nz, const int32_t* bank_org, int z_lo,
                           int z_hi) {
  if (!banks || !p_net || !w_host || !bias_host || !tail_host) return fail(ctx, "debug_conv3_tc_join: nil argument");
  ConvTcGeo g = make_conv_tc_geo(nb, nz, ny, nx);
  g.z_lo = z_lo;
  g.z_hi = z_hi;
  const int cin = add ? 8 : 8 * nbanks, nw = add ? 1 : nbanks;
  const DevPtr<float> bias = upload(bias_host, 8), tail = upload(tail_host, kTailFloats),
                      part = add ? DevPtr<float>() : dev_alloc<float>((size_t)nb * nz * ny * nx * 8);
  std::vector<DevPtr<float>> wj;
  bool ok = bias && tail && (add || part);
  for (int i = 0; ok && i < nw; i++)
    ok = keep(wj, upload_tc_weights(concat_slice(w_host, cin / 8, i).data(), 8, split));
  if (!ok) return fail(ctx, "debug_conv3_tc_join: cudaMalloc failed");
  ConvTcGeo geo[kTcMaxBanks];
  int org[kTcMaxBanks];
  for (int i = 0; i < nbanks; i++) {
    geo[i] = make_conv_tc_geo(nb, bank_nz[i], ny >> i, nx >> i);
    org[i] = bank_org[i];
  }
  launch_tc_join(banks, geo, org, zoff, nbanks, add, part.get(), p_net, wj, bias.get(), tail.get(), split, g,
                 ctx->stream);
  return finish_debug(ctx, "debug_conv3_tc_join");
}

// tfl_debug_tc_pyramid: one level of the bank pyramid on caller-owned padded buffers: in is
// make_conv_tc_geo(nb, nz_in, ny, nx), out make_conv_tc_geo(nb, nz_out, ny / 2, nx / 2); out's planes [z_lo, z_hi)
// pool in's planes 2 z + z_phase, 2 z + z_phase + 1.  Synchronises before returning.
static int debug_tc_pyramid_impl(tfl_ctx* ctx, const float* in, float* out, int nb, int nz_in, int ny, int nx,
                                 int nz_out, int z_phase, int z_lo, int z_hi, int planes) {
  if (!ctx) return 1;
  if (!in || !out) return fail(ctx, "debug_tc_pyramid: nil argument");
  if (nb < 1 || ny < 2 || nx < 2 || ny % 2 || nx % 2 || (z_phase != 0 && z_phase != 1) || z_lo < 0 || z_hi > nz_out ||
      z_lo >= z_hi || 2 * z_hi + z_phase > nz_in)
    return fail(ctx, "debug_tc_pyramid: bad arguments");
  ConvTcGeo go = make_conv_tc_geo(nb, nz_out, ny / 2, nx / 2);
  go.z_lo = z_lo;
  go.z_hi = z_hi;
  launch_tc_pyramid(in, make_conv_tc_geo(nb, nz_in, ny, nx), out, go, z_phase, ctx->stream, planes);
  return finish_debug(ctx, "debug_tc_pyramid");
}
int tfl_debug_tc_pyramid(tfl_ctx* ctx, const float* in, float* out, int nb, int nz_in, int ny, int nx, int nz_out,
                         int z_phase, int z_lo, int z_hi) {
  DeviceGuard guard_(ctx);
  return debug_tc_pyramid_impl(ctx, in, out, nb, nz_in, ny, nx, nz_out, z_phase, z_lo, z_hi, 1);
}
// tfl_debug_tc_pyramid2: the same level on both float4 planes (the input of a set with UDiv), all four channels of
// each pooled.
int tfl_debug_tc_pyramid2(tfl_ctx* ctx, const float* in, float* out, int nb, int nz_in, int ny, int nx, int nz_out,
                          int z_phase, int z_lo, int z_hi) {
  DeviceGuard guard_(ctx);
  return debug_tc_pyramid_impl(ctx, in, out, nb, nz_in, ny, nx, nz_out, z_phase, z_lo, z_hi, 2);
}

// tfl_debug_cnn_inputs_padded: the model's tensor-core input (launch_cnn_inputs_padded with its channel set and
// planes) from caller-owned device p_div [nb][n], U1 [nb][3][n] (already wall-masked), flags [nb][n] and the host
// scale [nb], into out (make_conv_tc_geo(nb, nz, ny, nx) layout).  Synchronises before returning.
int tfl_debug_cnn_inputs_padded(tfl_ctx* ctx, const tfl_cnn* m, const float* p_div, const float* U1,
                                const float* flags, const float* scale_host, float* out, int nb, int nz, int ny,
                                int nx) {
  DeviceGuard guard_(ctx);
  if (!ctx) return 1;
  if (!m || !p_div || !U1 || !flags || !scale_host || !out) return fail(ctx, "debug_cnn_inputs_padded: nil argument");
  if (!m->is3d || bad_grid(nb, nz, ny, nx, 1)) return fail(ctx, "debug_cnn_inputs_padded: bad grid or 2-D model");
  const DevPtr<float> scale = upload(scale_host, nb);
  if (!scale) return fail(ctx, "debug_cnn_inputs_padded: cudaMalloc failed");
  const ConvTcGeo tg = make_conv_tc_geo(nb, nz, ny, nx);
  launch_cnn_inputs_padded(p_div, U1, flags, scale.get(), out, tg.px, tg.py, whole_grid(ctx, nb, nz, ny, nx, 1),
                           ctx->stream, m->in_sel, m->tc_planes);
  return finish_debug(ctx, "debug_cnn_inputs_padded");
}

// Undocumented test hooks (not in tfl.h): the fp32 path's kernels (tfl_cnn.cu) on caller-owned device buffers, on
// the context's stream.  Each synchronises before returning.
// tfl_debug_conv_fp32: one convolution in [nb][cin][nz][ny][nx] -> out [nb][cout][nz][ny][nx] (nz = 1 in 2-D),
// weights [cout][cin][kz][k][k] (kz = k in 3-D, else 1) and bias [cout] on the host, re-laid out as
// tfl_cnn_create_graph does.  generic = 0: launch_conv_direct (the specialised kernel where the shape has one and its
// weights fit shared memory, else the generic one); generic = 1: the generic kernel.  *kernel: the kernel that ran,
// 1 direct or 2 generic.
static int debug_conv_fp32_impl(tfl_ctx* ctx, const float* in, float* out, const float* w_host, const float* bias_host,
                                int cin, int cout, int ks, int act, int is3d, int nb, int nz, int ny, int nx,
                                int generic, int dil, int32_t* kernel);
int tfl_debug_conv_fp32(tfl_ctx* ctx, const float* in, float* out, const float* w_host, const float* bias_host,
                        int cin, int cout, int ks, int act, int is3d, int nb, int nz, int ny, int nx, int generic,
                        int32_t* kernel) {
  DeviceGuard guard_(ctx);
  return debug_conv_fp32_impl(ctx, in, out, w_host, bias_host, cin, cout, ks, act, is3d, nb, nz, ny, nx, generic, 1,
                              kernel);
}
// tfl_debug_conv_fp32_dilated: the same with dilation dil >= 1 on every axis (padding dil (k-1)/2).
int tfl_debug_conv_fp32_dilated(tfl_ctx* ctx, const float* in, float* out, const float* w_host, const float* bias_host,
                                int cin, int cout, int ks, int act, int is3d, int nb, int nz, int ny, int nx,
                                int generic, int dil, int32_t* kernel) {
  DeviceGuard guard_(ctx);
  if (ctx && dil < 1) return fail(ctx, "debug_conv_fp32: bad dilation %d", dil);
  return debug_conv_fp32_impl(ctx, in, out, w_host, bias_host, cin, cout, ks, act, is3d, nb, nz, ny, nx, generic, dil,
                              kernel);
}
static int debug_conv_fp32_impl(tfl_ctx* ctx, const float* in, float* out, const float* w_host, const float* bias_host,
                                int cin, int cout, int ks, int act, int is3d, int nb, int nz, int ny, int nx,
                                int generic, int dil, int32_t* kernel) {
  if (!ctx) return 1;
  if (!in || !out || !w_host || !bias_host || !kernel) return fail(ctx, "debug_conv_fp32: nil argument");
  if (cin < 1 || cout < 1 || ks < 1 || ks % 2 != 1 || act < 0 || act > 2 || (generic != 0 && generic != 1))
    return fail(ctx, "debug_conv_fp32: bad layer cin=%d cout=%d k=%d act=%d generic=%d", cin, cout, ks, act, generic);
  if (bad_grid(nb, nz, ny, nx, is3d)) return fail(ctx, "debug_conv_fp32: bad grid %dx%dx%dx%d", nb, nz, ny, nx);
  const int taps = (is3d ? ks : 1) * ks * ks;
  const DevPtr<float> dw = upload(relayout_conv_weights(w_host, cin, cout, taps)), db = upload(bias_host, cout);
  if (!dw || !db) return fail(ctx, "debug_conv_fp32: cudaMalloc failed");
  const Geo g = whole_grid(ctx, nb, nz, ny, nx, is3d);
  const int ran = generic ? launch_conv_any(in, out, dw.get(), db.get(), cin, cout, ks, act, g, ctx->stream, dil)
                          : launch_conv_direct(in, out, dw.get(), db.get(), cin, cout, ks, act, g, ctx->stream, dil);
  if (const int rc = finish_debug(ctx, "debug_conv_fp32")) return rc;
  if (ran < 0) return fail(ctx, "debug_conv_fp32: no kernel for cout=%d k=%d", cout, ks);
  *kernel = ran;
  return 0;
}

// tfl_debug_pool: launch_pool, in [nbc][nz][ny][nx] -> out [nbc][nz / pz][ny / p][nx / p] (pz = p in 3-D, else 1);
// the grid must be divisible, as the graph executor checks before it pools.
int tfl_debug_pool(tfl_ctx* ctx, const float* in, float* out, int nbc, int nz, int ny, int nx, int p, int is3d,
                   int is_max) {
  DeviceGuard guard_(ctx);
  if (!ctx) return 1;
  if (!in || !out) return fail(ctx, "debug_pool: nil argument");
  if (p < 1 || bad_grid(nbc, nz, ny, nx, is3d) || nx % p || ny % p || (is3d && nz % p))
    return fail(ctx, "debug_pool: grid %dx%dx%dx%d does not pool by %d", nbc, nz, ny, nx, p);
  launch_pool(in, out, nbc, nz, ny, nx, p, is3d, is_max ? 1 : 0, ctx->stream);
  return finish_debug(ctx, "debug_pool");
}

// tfl_debug_pixel_shuffle: launch_pixel_shuffle, in [nb][n_out s^d][nz][ny][nx] -> out [nb][n_out][nz sz][ny s][nx s]
// (sz = s in 3-D, else 1).
int tfl_debug_pixel_shuffle(tfl_ctx* ctx, const float* in, float* out, int nb, int n_out, int nz, int ny, int nx,
                            int s, int is3d) {
  DeviceGuard guard_(ctx);
  if (!ctx) return 1;
  if (!in || !out) return fail(ctx, "debug_pixel_shuffle: nil argument");
  if (n_out < 1 || s < 1 || bad_grid(nb, nz, ny, nx, is3d))
    return fail(ctx, "debug_pixel_shuffle: bad arguments n_out=%d s=%d grid %dx%dx%dx%d", n_out, s, nb, nz, ny, nx);
  launch_pixel_shuffle(in, out, nb, n_out, nz, ny, nx, s, is3d, ctx->stream);
  return finish_debug(ctx, "debug_pixel_shuffle");
}

// tfl_debug_bank_join: launch_bank_join.  banks (host array of device pointers; banks[0] is not read) as in
// tfl_kernels.h; out [nb][nbanks c][nz][ny][nx] holding bank 1 in its first c channels ('concat', add = 0) or
// [nb][c][nz][ny][nx] holding bank 1 (add = 1).  The grid must be divisible by 2^(nbanks-1) (z in 3-D only).
int tfl_debug_bank_join(tfl_ctx* ctx, const float* const* banks, int nbanks, float* out, int nb, int c, int nz,
                        int ny, int nx, int is3d, int add) {
  DeviceGuard guard_(ctx);
  if (!ctx) return 1;
  if (nbanks < 2 || nbanks > kMaxBankPtrs) return fail(ctx, "debug_bank_join: bad bank count %d", nbanks);
  if (!banks || !out) return fail(ctx, "debug_bank_join: nil argument");
  for (int i = 1; i < nbanks; i++)
    if (!banks[i]) return fail(ctx, "debug_bank_join: nil bank %d", i + 1);
  const int r = 1 << (nbanks - 1);
  if (c < 1 || bad_grid(nb, nz, ny, nx, is3d) || nx % r || ny % r || (is3d && nz % r))
    return fail(ctx, "debug_bank_join: grid %dx%dx%dx%d is not divisible by %d", nb, nz, ny, nx, r);
  if (launch_bank_join(banks, nbanks, out, nb, c, nz, ny, nx, is3d, add ? 1 : 0, ctx->stream) < 0)
    return fail(ctx, "debug_bank_join: bad bank count %d", nbanks);
  return finish_debug(ctx, "debug_bank_join");
}

// tfl_debug_bn: batch normalization with batch statistics (launch_bn_stats, _finalize, _apply) in place on device x
// [nb][c][n] whose batch entries lie bstride floats apart; w_host / b_host [c] (may be NULL: 1 / 0).  stats_host
// ([c][2] doubles: mean, biased variance) and ac_host ([2][c] floats: a, c of y = a x + c) receive what the finalize
// computed.  Nothing but the nb c n values is written.
int tfl_debug_bn(tfl_ctx* ctx, float* x, int nb, int c, int64_t n, int64_t bstride, const float* w_host,
                 const float* b_host, float eps, double* stats_host, float* ac_host) {
  DeviceGuard guard_(ctx);
  if (!ctx) return 1;
  if (!x || !stats_host || !ac_host) return fail(ctx, "debug_bn: nil argument");
  if (nb < 1 || c < 1 || n < 1 || bstride < (int64_t)c * n || !(eps >= 0.0f)) return fail(ctx, "debug_bn: bad arguments");
  const DevPtr<float> w = w_host ? upload(w_host, c) : DevPtr<float>(),
                      b = b_host ? upload(b_host, c) : DevPtr<float>(), ac = dev_alloc<float>(2 * c);
  const DevPtr<double> part = dev_alloc<double>(2 * (kBnBlocks + 1) * c), stats = dev_alloc<double>(2 * c);
  if ((w_host && !w) || (b_host && !b) || !ac || !part || !stats) return fail(ctx, "debug_bn: cudaMalloc failed");
  launch_bn_stats(x, nb, c, n, bstride, part.get(), ctx->stream);
  launch_bn_finalize(part.get(), c, (long long)nb * n, w.get(), b.get(), eps, ac.get(), stats.get(), ctx->stream);
  launch_bn_apply(x, nb, c, n, bstride, ac.get(), ctx->stream);
  if (const int rc = finish_debug(ctx, "debug_bn")) return rc;
  if (cudaMemcpy(stats_host, stats.get(), sizeof(double) * 2 * c, cudaMemcpyDeviceToHost) != cudaSuccess ||
      cudaMemcpy(ac_host, ac.get(), 2 * c * 4, cudaMemcpyDeviceToHost) != cudaSuccess)
    return fail(ctx, "debug_bn: copy failed");
  return 0;
}

void tfl_cnn_destroy(tfl_ctx* ctx, tfl_cnn* m) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!m) return;
  if (ctx) cudaStreamSynchronize(ctx->stream);
  delete m;
}

// The fp32 path's scratch in the arena, in pieces aligned to 256 bytes from `base`.  Over a null base only `bytes` is
// meaningful: what arena_reserve needs, 256 bytes beyond each piece (at least its alignment) and 768 more.
struct CnnScratch {
  float *U1, *x0, *actA, *actB, *scale;
  double* bn_part;     // batch statistics: the partial sums and (a, c) of one BN module at a time
  float* bn_ac;
  float* actC;         // the third rotating buffer of the graphs that are not plain
  float* bank[kMaxBanks][3];
  size_t bytes;
};
static CnnScratch cnn_scratch(const tfl_cnn* m, const Geo& g, char* base) {
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

static int cnn_project_impl(tfl_ctx* ctx, tfl_cnn* m, const float* p_div, const float* U_div,
                            const float* flags, float* p_out, float* U_out, float threshold, const Geo& g,
                            const CnnScratch& scr, float** scale_dev_out) {
  float *U1 = scr.U1, *x0 = scr.x0, *actA = scr.actA, *actB = scr.actB, *scale = scr.scale;
  double* bn_part = scr.bn_part;
  float* bn_ac = scr.bn_ac;
  double* sums = ctx->dscratch.get() + 64;
  cudaStream_t st = ctx->stream;
  TFL_CUDA(ctx, cudaMemsetAsync(sums, 0, sizeof(double) * 2 * g.nb, st));
  launch_cnn_mask_stats(U_div, flags, U1, sums, g.zlo, g.zhi, g, st, m->norm_chan, p_div);
  if (m->norm_chan == kCnnStatDiv) {
    launch_cnn_div_stats(U1, flags, sums, g.zlo, g.zhi, g, st);
    ctx->launches += 1;
  }
  launch_cnn_scale(sums, scale, g.nb, m->norm_chan == kCnnStatU ? (long long)g.nc * g.n : g.n, threshold, st,
                   m->norm_func);
  if (m->mode > 0 && m->tc_ok && !ctx->slab) {
    if (cnn_ensure_act(ctx, m, g)) return 1;
    const ConvTcGeo& tg = m->act_geo;
    launch_cnn_inputs_padded(p_div, U1, flags, scale, m->act[0].get(), tg.px, tg.py, g, st, m->in_sel, m->tc_planes);
    float* p_net = actA;      // plain [b][z][y][x]
    run_conv_stack(m, p_net, st);
    if (m->skip) {
      launch_cnn_skip(p_net, p_div, scale, m->w_skip, g, st);
      ctx->launches += 1;
    }
    launch_cnn_finish(p_net, U1, flags, scale, p_out, U_out, g, st);
    ctx->launches += 7;
    if (scale_dev_out) *scale_dev_out = scale;
    return check_launch(ctx, "cnn_project (tensor cores)");
  }
  launch_cnn_inputs(p_div, U1, flags, scale, x0, g, st, m->in_sel);
  ctx->launches += 3;
  const float* in = x0;
  if (m->plain) {
    float* bufs[2] = {actA, actB};
    for (int l = 0; l < m->n_layers; l++) {
      float* o = bufs[l & 1];
      const int act = (l < m->n_layers - 1) ? 1 : 0;
      if (launch_conv_direct(in, o, m->w[l].get(), m->b[l].get(), m->cin[l], m->cout[l], m->ks[l], act, g, st) < 0)
        return fail(ctx, "cnn: unsupported layer shape cout=%d k=%d", m->cout[l], m->ks[l]);
      ctx->launches += 1;
      in = o;
    }
  } else {
    // 'tog' / 'yang' graphs: conv (+ pixel shuffle) -> non-linearity -> pooling, layer by layer, on grids
    // whose resolution follows the pooling / upsampling sizes (lib/model.lua:262-340, single bank).
    if (ctx->slab) return fail(ctx, "cnn: pooled / upsampled graphs run on whole grids only");
    float* bufs[3] = {actA, actB, scr.actC};
    // One stage of one bank: convolution ci (dilated by dil) (+ pixel shuffle) -> non-linearity -> pooling, on grid
    // gl, through the rotating buffers bb, never writing `keep` (an input other banks still read).  out_bstride > 0:
    // the stage's result is written with that batch stride (floats), so that it lands in place in a concatenation
    // of banks; dst (may be null): the stage's result goes there rather than to one of bb.
    auto run_stage = [&](int ci, int l, const float* src, float* const* bb, Geo& gl, long long out_bstride,
                         const float** result, int dil, const float* keep, float* dst) -> int {
      auto other = [&](const float* a) {
        for (int q = 0; q < 3; q++) if (bb[q] != a && bb[q] != keep) return bb[q];
        return bb[0];
      };
      const int u = m->up[l], pl = m->pool[l];
      const int act = (l < m->n_layers - 1) ? m->nonlin : 0;     // element-wise: commutes with the shuffle
      const int shuffled = m->cout[ci] / (u * u * (gl.is3d ? u : 1));
      // per batch entry when the last operation of the stage writes with a batch stride
      const int nloop_conv = (out_bstride > 0 && u == 1 && pl == 1) ? gl.nb : 1;
      float* o = (dst && u == 1 && pl == 1) ? dst : other(src);
      for (int b = 0; b < nloop_conv; b++) {
        Geo gb = gl;
        if (nloop_conv > 1) gb.nb = 1;
        const long long ioff = nloop_conv > 1 ? (long long)b * m->cin[ci] * gl.n : 0;
        const long long ooff = nloop_conv > 1 ? (long long)b * out_bstride : 0;
        if (launch_conv_direct(src + ioff, o + ooff, m->w[ci].get(), m->b[ci].get(), m->cin[ci], m->cout[ci],
                               m->ks[ci], act, gb, st, dil) < 0)
          return fail(ctx, "cnn: unsupported layer shape cout=%d k=%d", m->cout[ci], m->ks[ci]);
        ctx->launches += 1;
      }
      const float* cur = o;
      int chans = m->cout[ci];
      if (u > 1) {
        chans = shuffled;
        float* sh = (dst && pl == 1) ? dst : other(cur);
        const int nloop = (out_bstride > 0 && pl == 1) ? gl.nb : 1;
        const long long nin = (long long)m->cout[ci] * gl.n;
        for (int b = 0; b < nloop; b++) {
          launch_pixel_shuffle(cur + (nloop > 1 ? b * nin : 0), sh + (nloop > 1 ? b * out_bstride : 0),
                               nloop > 1 ? 1 : gl.nb, chans, gl.nz, gl.ny, gl.nx, u, gl.is3d, st);
          ctx->launches += 1;
        }
        gl.nx *= u; gl.ny *= u; if (gl.is3d) gl.nz *= u;
        cur = sh;
      }
      if (pl > 1) {
        if (gl.nx % pl || gl.ny % pl || (gl.is3d && gl.nz % pl))
          return fail(ctx, "cnn: grid %dx%dx%d is not divisible by the pooling size %d", gl.nx, gl.ny, gl.nz, pl);
        float* po = dst ? dst : other(cur);
        const int nloop = out_bstride > 0 ? gl.nb : 1;
        const long long nin = (long long)chans * gl.nx * gl.ny * gl.nz;
        for (int b = 0; b < nloop; b++) {
          launch_pool(cur + (nloop > 1 ? b * nin : 0), po + (nloop > 1 ? b * out_bstride : 0),
                      (nloop > 1 ? 1 : gl.nb) * chans, gl.nz, gl.ny, gl.nx, pl, gl.is3d, m->pool_is_max, st);
          ctx->launches += 1;
        }
        gl.nx /= pl; gl.ny /= pl; if (gl.is3d) gl.nz /= pl;
        cur = po;
      }
      gl.n = (long long)gl.nx * gl.ny * gl.nz;
      gl.gnz = gl.nz; gl.zlo = 0; gl.zhi = gl.nz;
      if (m->bn && l < m->n_layers - 1) {     // lib/model.lua:343-350: BN closes every stage but the last
        float* x = (float*)cur;               // one of this call's buffers, or a slot of one
        const long long bs = out_bstride > 0 ? out_bstride : (long long)chans * gl.n;
        const float* ac = m->bn_batch ? bn_ac : m->bn_ac[ci].get();
        if (m->bn_batch) {
          launch_bn_stats(x, gl.nb, chans, gl.n, bs, bn_part, st);
          launch_bn_finalize(bn_part, chans, (long long)gl.nb * gl.n, m->bn_wb[ci].get(), m->bn_wb[ci].get() + chans,
                             m->bn_eps[ci], bn_ac, nullptr, st);
          ctx->launches += 2;
        }
        launch_bn_apply(x, gl.nb, chans, gl.n, bs, ac, st);
        ctx->launches += 1;
      }
      *result = cur;
      return 0;
    };
    const int nbk = m->nbanks;
    const float* bank_in[kMaxBanks] = {};
    Geo bank_g[kMaxBanks];
    Geo gl = g;
    for (int l = 0; l < m->n_layers; l++) {
      if (nbk > 1 && l == m->split && m->bank_dilate) {
        // Dilated banks (lib/model.lua:279-285): every bank reads the hidden layer as it is.
        for (int i = 0; i < nbk; i++) {
          bank_in[i] = in;
          bank_g[i] = gl;
        }
      } else if (nbk > 1 && l == m->split) {
        // Gaussian pyramid (lib/model.lua:276-289): bank i = 2x average pool of bank i-1.
        const int r = 1 << (nbk - 1);
        if (gl.nx % r || gl.ny % r || (gl.is3d && gl.nz % r))
          return fail(ctx, "cnn: grid %dx%dx%d at bank split stage %d is not divisible by 2^(banksNum-1) = %d",
                      gl.nx, gl.ny, gl.nz, l + 1, r);
        bank_in[0] = in;
        bank_g[0] = gl;
        for (int i = 1; i < nbk; i++) {
          Geo gi = bank_g[i - 1];
          launch_pool(bank_in[i - 1], scr.bank[i][0], gi.nb * m->cin[m->conv0[l]], gi.nz, gi.ny, gi.nx, 2, gi.is3d, 0, st);
          ctx->launches += 1;
          gi.nx /= 2; gi.ny /= 2; if (gi.is3d) gi.nz /= 2;
          gi.n = (long long)gi.nx * gi.ny * gi.nz;
          gi.gnz = gi.nz; gi.zlo = 0; gi.zhi = gi.nz;
          bank_g[i] = gi;
          bank_in[i] = scr.bank[i][0];
        }
      }
      if (nbk > 1 && l >= m->split && l < m->join) {
        const bool last = l == m->join - 1;
        // Dilated banks joined by 'concat' write their last stage straight into their channel slots of bank 1's
        // result; the shared input of the split stage stays intact until every bank has read it.
        const bool in_slot = m->bank_dilate && last && !m->bank_add;
        const float* shared = (m->bank_dilate && l == m->split) ? in : nullptr;
        // concat: bank 1's result is the first c_out channels of [nb][nbk c_out][n] at the join resolution (taken
        // before the stage runs: run_stage moves bank_g[0] to the stage's output grid)
        const Geo gs = bank_g[0];
        const int c_out = m->cout[m->conv0[l]] / (m->up[l] * m->up[l] * (g.is3d ? m->up[l] : 1));
        const long long n_join = (long long)(gs.nx * m->up[l] / m->pool[l]) * (gs.ny * m->up[l] / m->pool[l]) *
                                 (g.is3d ? gs.nz * m->up[l] / m->pool[l] : gs.nz);
        for (int i = 0; i < nbk; i++) {
          const long long bstride = (last && (i == 0 || in_slot) && !m->bank_add && g.nb > 1)
                                        ? (long long)nbk * c_out * n_join : 0;
          float* dst = (in_slot && i > 0) ? (float*)bank_in[0] + (long long)i * c_out * n_join : nullptr;
          if (run_stage(m->conv0[l] + i, l, bank_in[i], i == 0 ? bufs : scr.bank[i], bank_g[i], bstride, &bank_in[i],
                        m->bank_dilate ? 1 << i : 1, shared, dst))
            return 1;
        }
        if (last && m->bank_dilate) {   // lib/model.lua:300-318: no upsampling; 'concat' is already in place
          if (m->bank_add) {
            const Geo& gj = bank_g[0];
            if (launch_bank_join(bank_in, nbk, (float*)bank_in[0], gj.nb, c_out, gj.nz, gj.ny, gj.nx, g.is3d, 1, st,
                                 1) < 0)
              return fail(ctx, "cnn: bad bank count %d", nbk);
            ctx->launches += 1;
          }
          in = bank_in[0];
          gl = bank_g[0];
        } else if (last) {   // lib/model.lua:292-318: upsample banks 2..N, then JoinTable or CAddTable
          const Geo& g1 = bank_g[0];
          for (int i = 1; i < nbk; i++)
            if (bank_g[i].nx << i != g1.nx || bank_g[i].ny << i != g1.ny || (g.is3d && bank_g[i].nz << i != g1.nz))
              return fail(ctx, "cnn: bank %d does not upsample to the resolution of bank 1 (grid not divisible)", i + 1);
          if (launch_bank_join(bank_in, nbk, (float*)bank_in[0], g1.nb, c_out, g1.nz, g1.ny, g1.nx, g.is3d,
                               m->bank_add, st) < 0)
            return fail(ctx, "cnn: bad bank count %d", nbk);
          ctx->launches += 1;
          in = bank_in[0];
          gl = g1;
        }
        continue;
      }
      if (run_stage(m->conv0[l], l, in, bufs, gl, 0, &in, 1, nullptr, nullptr)) return 1;
    }
    if (gl.nx != g.nx || gl.ny != g.ny || gl.nz != g.nz) return fail(ctx, "cnn: graph does not return to the input resolution");
  }
  if (m->skip) {
    launch_cnn_skip((float*)in, p_div, scale, m->w_skip, g, st);     // `in` is one of this call's scratch buffers
    ctx->launches += 1;
  }
  launch_cnn_finish(in, U1, flags, scale, p_out, U_out, g, st);
  ctx->launches += 1;
  if (scale_dev_out) *scale_dev_out = scale;
  return check_launch(ctx, "cnn_project");
}

int tfl_cnn_project(tfl_ctx* ctx, tfl_cnn* m, const tfl_grid* p_div, const tfl_grid* U_div,
                    const tfl_grid* flags, const tfl_grid* p_out, const tfl_grid* U_out, float threshold,
                    float* scale_out) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!m) return fail(ctx, "cnn is nil");
  if (check_scalar(ctx, flags, "flags") || check_scalar(ctx, p_div, "pDiv") || check_vel(ctx, U_div, flags) ||
      check_scalar(ctx, p_out, "p") || check_vel(ctx, U_out, flags))
    return 1;
  if (!same_spatial(flags, p_div) || !same_spatial(flags, p_out) || U_out->nc != U_div->nc)
    return fail(ctx, "Size mismatch");
  if ((U_div->nc == 3) != (m->is3d != 0)) return fail(ctx, "model / data dimensionality mismatch");
  if (ctx->slab) return fail(ctx, "cnn_project on a z-slab goes through the multi-GPU driver");
  Geo g;
  if (make_geo(ctx, flags, m->is3d, &g)) return 1;
  if (arena_reserve(ctx, cnn_scratch(m, g, nullptr).bytes)) return 1;
  float* scale_dev = nullptr;
  if (cnn_project_impl(ctx, m, p_div->data, U_div->data, flags->data, p_out->data, U_out->data, threshold, g,
                       cnn_scratch(m, g, ctx->arena.get()), &scale_dev))
    return 1;
  if (scale_out) {
    TFL_CUDA(ctx, cudaMemcpyAsync(scale_out, scale_dev, sizeof(float) * g.nb, cudaMemcpyDeviceToHost, ctx->stream));
    TFL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  }
  return 0;
}

// z-slab variant of model:forward, split around the one global reduction (the input scale):
//   tfl_cnn_stats              U1 = SetWallBcs mask * U on every local plane where the mask is
//                              computable, and (sum, sum of squares) over the OWNED planes into
//                              dev_sums[2 * nb] (device doubles the caller all-reduces, e.g. with NCCL);
//   tfl_cnn_project_from_sums  everything after the reduction.  The conv stack runs on the planes the
//                              owned ones need, which must lie at least 4 planes (a banked model:
//                              3 * 2^(banksNum-1) + 1, cnn_slab_check) away from a local end that is not
//                              a global end.
int tfl_cnn_stats(tfl_ctx* ctx, const tfl_grid* U_div, const tfl_grid* flags, const tfl_grid* U1,
                  double* dev_sums) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (check_scalar(ctx, flags, "flags") || check_vel(ctx, U_div, flags) || check_vel(ctx, U1, flags)) return 1;
  if (!dev_sums) return fail(ctx, "cnn_stats: nil sums");
  Geo g;
  if (make_geo(ctx, flags, U_div->nc == 3, &g)) return 1;
  Geo gw = g;
  if (ctx->slab) {
    gw.zlo = (g.zoff == 0) ? 0 : 1;
    gw.zhi = (g.zoff + g.nz == g.gnz) ? g.nz : g.nz - 1;
  }
  TFL_CUDA(ctx, cudaMemsetAsync(dev_sums, 0, sizeof(double) * 2 * g.nb, ctx->stream));
  launch_cnn_mask_stats(U_div->data, flags->data, U1->data, dev_sums, g.zlo, g.zhi, gw, ctx->stream);
  ctx->launches += 1;
  return check_launch(ctx, "cnn_stats");
}

int tfl_cnn_project_from_sums(tfl_ctx* ctx, tfl_cnn* m, const tfl_grid* p_div, const tfl_grid* U1,
                              const tfl_grid* flags, const double* dev_sums, const tfl_grid* p_out,
                              const tfl_grid* U_out, float threshold) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!m) return fail(ctx, "cnn is nil");
  if (const char* why = cnn_slab_refusal(m)) return fail(ctx, "cnn_project_from_sums: %s", why);
  if (!dev_sums) return fail(ctx, "cnn_project_from_sums: nil sums");
  if (check_scalar(ctx, flags, "flags") || check_scalar(ctx, p_div, "pDiv") || check_vel(ctx, U1, flags) ||
      check_scalar(ctx, p_out, "p") || check_vel(ctx, U_out, flags))
    return 1;
  Geo g;
  if (make_geo(ctx, flags, 1, &g)) return 1;
  if (ctx->slab && m->nbanks > 1 &&
      cnn_slab_check(ctx, m, ctx->slab_margin, g.gnz, g.ny, g.nx, g.zoff, g.nz, g.zlo, g.zhi))
    return 1;
  if (cnn_ensure_act(ctx, m, g)) return 1;
  const size_t cells = (size_t)g.n * g.nb;
  if (arena_reserve(ctx, carve_bytes({cells * 4, 4 * (size_t)g.nb}))) return 1;
  Carver cv(ctx);
  float* p_net = cv.take<float>(cells);
  float* scale = cv.take<float>(g.nb);
  cudaStream_t st = ctx->stream;
  // scale from the (already reduced) sums; the sample count is that of the GLOBAL grid.
  launch_cnn_scale(dev_sums, scale, g.nb, (long long)g.nc * g.nx * g.ny * g.gnz, threshold, st);
  Geo gi = g;            // the divergence reads U1 one plane up
  if (ctx->slab) {
    gi.zlo = (g.zoff == 0) ? 0 : 1;
    gi.zhi = (g.zoff + g.nz == g.gnz) ? g.nz : g.nz - 2;
  }
  const ConvTcGeo& tg = m->act_geo;
  launch_cnn_inputs_padded(p_div->data, U1->data, flags->data, scale, m->act[0].get(), tg.px, tg.py, gi, st);
  // the velocity update of the computed planes [zlo, zhi) reads p on [zlo - 1, zhi)
  if (ctx->slab) run_conv_stack(m, p_net, st, g.zlo - 1, g.zhi);
  else run_conv_stack(m, p_net, st);
  launch_cnn_finish(p_net, U1->data, flags->data, scale, p_out->data, U_out->data, g, st);
  ctx->launches += 6;
  return check_launch(ctx, "cnn_project_from_sums");
}

}  // extern "C"
