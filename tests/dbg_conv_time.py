import sys, os, numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from fluidnet_b200 import synth
from fluidnet_b200.model import ProjectionModel
n = int(sys.argv[1]) if len(sys.argv) > 1 else 128
flags = torch.from_numpy(synth.make_flags(n, n, n, True, nb=1, geometry=True)).cuda()
U = torch.from_numpy(synth.make_smooth_velocity(flags.cpu().numpy(), True, amp=2.0)).cuda()
p = torch.zeros_like(flags)
gm = ProjectionModel.from_model(synth.make_model(True))
for mode in ("fp32", "tf32", "tf32x3"):
    gm.set_mode(mode)
    for _ in range(3):
        gm.forward((p, U, flags))
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(10):
        gm.forward((p, U, flags))
    b.record()
    torch.cuda.synchronize()
    print("mode %-7s model:forward %.3f ms" % (mode, a.elapsed_time(b) / 10), flush=True)
