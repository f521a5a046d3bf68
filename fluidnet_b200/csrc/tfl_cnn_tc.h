// Internal interface of the tensor-core convolution path (tfl_cnn_tc.cu).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

namespace tfl {

struct ConvTcGeo {
  int nb, nz, ny, nx;
  int px, py;             // padded pitches of the channels-last activation planes (x, y)
  int ntx, nty, ntz;      // CTA tiles
  int z_lo, z_hi;         // output planes of a launch (default: all; a z-slab computes only what its owned planes need)
};

ConvTcGeo make_conv_tc_geo(int nb, int nz, int ny, int nx);
// bytes of one activation buffer: [b][2 planes][nz+2][py][px] float4
size_t conv_tc_act_bytes(const ConvTcGeo& g);
int conv_tc_b_floats(int split);
void conv_tc_set_debug(long long* dev_buf);   // nullptr disables
void conv_tc_pack_weights(const float* w /*[8][cin][3][3][3]*/, int cin, int split, float* out);
// in/out: padded channels-last activations; p_net: plain [b][z][y][x] (final layer only);
// tail (final layer): w4[8][8] (o, c), b4[8], w5[8], b5[1] on the device.
int launch_conv3_tc(const float* in, float* out, float* p_net, const float* wB, const float* bias,
                    const float* tail, int in_planes, int final_layer, int split, const ConvTcGeo& g,
                    cudaStream_t st);

}  // namespace tfl
