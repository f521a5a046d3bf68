"""fluidnet_b200 -- H100-native Eulerian fluid step behind the tfluids operator surface.

The product is `libtfl.so` (hand-written sm_90a CUDA behind the C ABI in include/tfl.h).
This package is the thin host-side mirror of the reference's Lua interface
(torch/tfluids/init.lua, torch/lib/simulate.lua, torch/lib/model.lua) so that host code
written against `tfluids.*` keeps its call sites:

    from fluidnet_b200 import tfluids, simulate
    tfluids.advectScalar(dt, density, U, flags, 'maccormackOurs', None, False, 0.6)
    simulate.simulate(conf, mconf, batch, model)

PyTorch is used only for device memory and streams.  There is no CPU fallback: importing
`fluidnet_b200.tfluids` works without a GPU (so the ABI can be inspected), but every
operator raises if libtfl.so or a CUDA device is missing.
"""
__version__ = "0.1.0"
