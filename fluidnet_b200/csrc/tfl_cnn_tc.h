// Internal interface of the tensor-core convolution path (tfl_cnn_tc.cu).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

namespace tfl {

struct ConvTcGeo {
  int nb, nz, ny, nx;
  int px, py;             // padded pitches of the channels-last activation planes (x, y)
  int ntx, nty, ntz;      // CTA tiles of the one-shot box kernel (k_conv3_tc)
  int z_lo, z_hi;         // output planes of a launch (default: all; a z-slab computes only what its owned planes need)
};

ConvTcGeo make_conv_tc_geo(int nb, int nz, int ny, int nx);
// bytes of one activation buffer: [b][2 planes][nz+2][py][px] float4
size_t conv_tc_act_bytes(const ConvTcGeo& g);
int conv_tc_b_floats(int split);
void conv_tc_set_debug(long long* dev_buf);   // nullptr disables
// Test hook: caps the persistent grid of the z-streaming kernel at `ctas` CTAs (0: one per SM), so that every CTA
// runs several work items.
void conv_tc_set_z_grid(int ctas);
// 1 if a z-streaming launch on this device recorded a stalled pipeline (a bounded mbarrier wait ran out) since the
// last call, 0 otherwise; clears the record.  Synchronises `st`.
int conv_tc_take_z_fault(cudaStream_t st);
void conv_tc_pack_weights(const float* w /*[8][cin][3][3][3]*/, int cin, int split, float* out);
// The epilogue's options: relu6 = 1 clamps every non-linearity of the layer (and of the fused 1x1x1 tail) at 6
// (nn.ReLU6); ac (device, [2][8]: a then c; non-final layers only, may be null) applies y = a h + c per channel after
// the non-linearity -- batch normalization with running statistics -- to the voxels written, so the zero border stays
// zero.
struct TcEpi {
  const float* ac = nullptr;
  int relu6 = 0;
};
// in/out: padded channels-last activations; p_net: plain [b][z][y][x] (final layer only);
// tail (final layer): w4[8][8] (o, c), b4[8], w5[8], b5[1] on the device.
int launch_conv3_tc(const float* in, float* out, float* p_net, const float* wB, const float* bias,
                    const float* tail, int in_planes, int final_layer, int split, const ConvTcGeo& g,
                    cudaStream_t st, const TcEpi& ep = TcEpi());

// Join layer of the multi-resolution banks (lib/model.lua:292-318) on the tensor cores: the last 3x3x3 layer
// reads its 8 input channels as the sum over src[0..n) of bank src[k] upsampled nearest by 2^shift[k], staged
// straight from the bank's own padded buffer (geometry px / py / nz), so no full-resolution copy exists.
//   part_mode 0: bias, ReLU and the 1x1x1 tail -> p_net (as launch_conv3_tc with final_layer);
//   part_mode 1 / 2: write / add the x-tap-summed pre-activations to `partial` ([nb][nz][ny][nx][8] fp32), no
//                    bias, no tail (the other banks of a 'concat' join);
//   part_mode 3: add `partial` before the bias, then as part_mode 0.
// On a z-slab the full-resolution plane z (local) is global plane z + zoff, and local plane 0 of bank k is its
// global coarse plane org[k]: bank k is read at plane ((z + zoff) >> shift[k]) - org[k].  Whole grids: all zero.
// phase[k] = 1: bank k is a dilated bank at full resolution held as phase sub-grids (launch_tc_phase_copy, d =
// 2^shift[k]): the full-resolution voxel v is sub-grid voxel v >> shift[k] of batch entry (b, v & (d-1)).
constexpr int kTcMaxBanks = 8;
struct TcJoinSrc {
  const float* p[kTcMaxBanks];
  int px[kTcMaxBanks], py[kTcMaxBanks], nz[kTcMaxBanks], shift[kTcMaxBanks], org[kTcMaxBanks];
  int phase[kTcMaxBanks];
  int zoff;
  int n;
  int part_mode;
  float* partial;
};
int launch_conv3_tc_join(const TcJoinSrc& src, float* p_net, const float* wB, const float* bias, const float* tail,
                         int split, const ConvTcGeo& g, cudaStream_t st, const TcEpi& ep = TcEpi());

// Batch normalization with batch statistics on the padded layout (tfl_cnn.cu), all 8 channels of a 3x3x3 layer's
// output over its interior (nb nz ny nx voxels; the border is neither read nor written).  Partials as
// launch_bn_stats writes them (part [8][kBnBlocks + 1][2], fp64, fixed order), turned into ac [2][8] by
// launch_bn_finalize; launch_tc_bn_apply: x = a x + c in place on the interior.
void launch_tc_bn_stats(const float* buf, const ConvTcGeo& g, double* part, cudaStream_t st);
void launch_tc_bn_apply(float* buf, const ConvTcGeo& g, const float* ac, cudaStream_t st);
// The 1x1x1 tail of the 3-D 'default' graph with batch statistics, on layer 3's output `buf` (padded layout, already
// through its non-linearity): h4 = act(w4 (a3 h3 + c3) + b4) with ac3 = BN3's (a, c).  pass_b = 0 (pass A): only the
// per-channel partials of h4 into part, as launch_tc_bn_stats; pass_b = 1 (pass B): p_net = w5 (a4 h4 + c4) + b5 with
// ac4 = BN4's (a, c).  h4 is recomputed in pass B rather than stored.  tail: w4[8][8], b4[8], w5[8], b5[1] (device).
void launch_tc_bn_tail(const float* buf, const ConvTcGeo& g, const float* ac3, const float* tail, int relu6,
                       int pass_b, double* part, const float* ac4, float* p_net, cudaStream_t st);
// Bank pyramid on the padded channels-last layout: out's plane z = 2x2x2 average of in's planes 2 z + z_phase and
// 2 z + z_phase + 1 (interior, first float4 plane only: the 3 input channels and a zero fourth), for the output
// planes [gout.z_lo, gout.z_hi).  z_phase (0 or 1) aligns the pooling to the global grid on a z-slab whose
// fine level starts at an odd global plane.  Other planes and the borders of out are left as they are.
// planes = 2 (the input of a set with UDiv): both float4 planes, all four channels of each.
void launch_tc_pyramid(const float* in, const ConvTcGeo& gin, float* out, const ConvTcGeo& gout, int z_phase,
                       cudaStream_t st, int planes = 1);

// Phase decomposition of a dilated bank (banksType 'dilate', dilation d = 2^sh): a 3x3x3 convolution with dilation d
// on an nz x ny x nx grid is d^3 ordinary 3x3x3 convolutions, one on each sub-lattice {v = s d + r}, each zero-padded
// at its own border.  The sub-grids are batch entries e = ((b d + rz) d + ry) d + rx of make_conv_tc_phase_geo, of
// ceil(n / d) voxels per axis; a sub-grid voxel whose full-resolution voxel lies outside the grid (n % d != 0, or
// d > n) must read as zero.  launch_tc_phase_copy lays a padded full-resolution buffer (geometry gfull) out that way
// (zeros there); launch_tc_phase_zero zeroes those voxels of a layer's output (both planes) so that the next layer
// reads them as padding; launch_tc_phase_gather copies the sub-grids back to the interior of a full-resolution buffer
// (both planes).
ConvTcGeo make_conv_tc_phase_geo(int nb, int nz, int ny, int nx, int sh);
void launch_tc_phase_copy(const float* in, const ConvTcGeo& gfull, float* out, const ConvTcGeo& gsub, int sh,
                          int planes, cudaStream_t st);
void launch_tc_phase_zero(float* buf, const ConvTcGeo& gsub, int sh, const ConvTcGeo& gfull, cudaStream_t st);
void launch_tc_phase_gather(const float* in, const ConvTcGeo& gsub, float* out, const ConvTcGeo& gfull, int sh,
                            cudaStream_t st);

}  // namespace tfl
