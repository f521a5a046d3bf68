// C ABI of the projection network (include/tfl.h): model creation, modes and the forward entry points.  The forward
// pass itself is in tfl_cnn_forward.cu, the test hooks in tfl_api_cnn_debug.cu.
#include <string.h>
#include <algorithm>
#include <cmath>
#include <vector>

#include "tfl_api_internal.h"

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

// Weight layouts the test hooks share (tfl_api_internal.h).
DevPtr<float> upload_tc_weights(const float* w, int cin, int split) {
  std::vector<float> packed(conv_tc_b_floats(split));
  conv_tc_pack_weights(w, cin, split, packed.data());
  return upload(packed);
}

std::vector<float> relayout_conv_weights(const float* w, int cin, int cout, int taps) {
  std::vector<float> relaid((size_t)cin * taps * cout);
  for (int o = 0; o < cout; o++)
    for (int c = 0; c < cin; c++)
      for (int t = 0; t < taps; t++)
        relaid[((size_t)c * taps + t) * cout + o] = w[((size_t)o * cin + c) * taps + t];
  return relaid;
}

std::vector<float> concat_slice(const float* w, int nbanks, int i) {
  std::vector<float> slice(8 * 8 * 27);
  for (int o = 0; o < 8; o++)
    memcpy(slice.data() + (size_t)o * 8 * 27, w + ((size_t)o * 8 * nbanks + 8 * i) * 27, 8 * 27 * 4);
  return slice;
}

namespace {

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

void tfl_cnn_destroy(tfl_ctx* ctx, tfl_cnn* m) {
  DeviceGuard guard_(ctx);
  NvtxRange range_(__func__);
  if (!m) return;
  if (ctx) cudaStreamSynchronize(ctx->stream);
  delete m;
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
  return cnn_project(ctx, m, {p_div->data, U_div->data, flags->data, p_out->data, U_out->data}, threshold, g,
                     scale_out);
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
  return cnn_project_from_sums(ctx, m, {p_div->data, U1->data, flags->data, p_out->data, U_out->data}, dev_sums,
                               threshold, g);
}

}  // extern "C"
