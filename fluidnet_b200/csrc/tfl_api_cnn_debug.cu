// Undocumented test hooks of the projection network (not in include/tfl.h): single tensor-core layers, the join and the
// pyramid on caller-owned buffers, and the fp32 path's kernels (tfl_cnn.cu).  Each synchronises before returning.
#include <vector>

#include "tfl_api_internal.h"

namespace {

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

}  // namespace

extern "C" {

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

}  // extern "C"
