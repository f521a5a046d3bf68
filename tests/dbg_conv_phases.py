import sys, os, numpy as np, torch, ctypes as C
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from fluidnet_b200 import synth, tfluids
from fluidnet_b200.model import ProjectionModel
n = 128
flags = torch.from_numpy(synth.make_flags(n, n, n, True, nb=1, geometry=True)).cuda()
U = torch.from_numpy(synth.make_smooth_velocity(flags.cpu().numpy(), True, amp=2.0)).cuda()
p = torch.zeros_like(flags)
gm = ProjectionModel.from_model(synth.make_model(True))
lib = tfluids.context().lib
for mode in ("tf32", "tf32x3"):
    gm.set_mode(mode)
    for _ in range(2):
        gm.forward((p, U, flags))
    torch.cuda.synchronize()
    buf = torch.zeros(8 * 4096, dtype=torch.int64, device="cuda")
    lib.tfl_debug_conv_timestamps(C.c_void_p(buf.data_ptr()))
    gm.forward((p, U, flags))
    torch.cuda.synchronize()
    lib.tfl_debug_conv_timestamps(C.c_void_p(0))
    d = buf.cpu().numpy().reshape(-1, 8)
    d = d[d[:, 0] != 0]
    t0 = d[:, 0]
    print(mode, "ctas", len(d))
    print("  load+sync   ", np.median(d[:, 1] - t0))
    print("  first commit", np.median(d[:, 2] - d[:, 1]))
    print("  all issued  ", np.median(d[:, 3] - d[:, 1]))
    print("  first full  ", np.median(d[:, 4] - d[:, 1]))
    print("  end         ", np.median(d[:, 5] - t0))
    # per SM concurrency: for SM 0 list start/end
    sm = d[:, 7]
    sel = d[sm == sm[0]]
    sel = sel[np.argsort(sel[:, 0])]
    base = sel[0, 0]
    print("  SM", sm[0], [(int(a - base), int(b - base)) for a, b in zip(sel[:8, 0], sel[:8, 5])])
