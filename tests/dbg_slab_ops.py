import os, sys, numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from fluidnet_b200 import tfluids
from fluidnet_b200.slab import SlabDecomposition
from slab_cases import convnet_problem
batch, mconf, mnp = convnet_problem(48)
tb = {k: torch.from_numpy(v).cuda() for k, v in batch.items()}
ctx = tfluids.context()
def cmp(name, got, want, d):
    g = d.owned(got); w = want[:, :, d.z0:d.z1]
    e = (g - w).abs()
    print("%-22s rank %d maxerr %.3e  bitexact %s" % (name, d.rank, e.max().item(), torch.equal(g, w)))
for rank in (0, 1):
    d = SlabDecomposition(48, rank, 2, 6)
    loc = {k: d.scatter(v) for k, v in tb.items()}
    def slab_on():
        ctx.set_slab(d.zoff, d.gnz, d.own_lo, d.own_hi)
    # advectVel
    Ug = tb["UDiv"].clone(); tfluids.advectVel(0.1, Ug, tb["flags"], "maccormackOurs", None, 0.6)
    Ul = loc["UDiv"].clone(); slab_on(); tfluids.advectVel(0.1, Ul, loc["flags"], "maccormackOurs", None, 0.6); ctx.clear_slab()
    cmp("advectVel", Ul, Ug, d)
    rg = tb["density"].clone(); tfluids.advectScalar(0.1, rg, tb["UDiv"], tb["flags"], "maccormackOurs", None, False, 0.6)
    rl = loc["density"].clone(); slab_on(); tfluids.advectScalar(0.1, rl, loc["UDiv"], loc["flags"], "maccormackOurs", None, False, 0.6); ctx.clear_slab()
    cmp("advectScalar", rl, rg, d)
    Ug = tb["UDiv"].clone(); tfluids.addBuoyancy(Ug, tb["flags"], tb["density"], [0, 0.3, 0.1], 0.1)
    Ul = loc["UDiv"].clone(); slab_on(); tfluids.addBuoyancy(Ul, loc["flags"], loc["density"], [0, 0.3, 0.1], 0.1); ctx.clear_slab()
    cmp("buoyancy", Ul, Ug, d)
    Ug = tb["UDiv"].clone(); tfluids.vorticityConfinement(Ug, tb["flags"], 0.3)
    Ul = loc["UDiv"].clone(); slab_on(); tfluids.vorticityConfinement(Ul, loc["flags"], 0.3); ctx.clear_slab()
    cmp("vorticity", Ul, Ug, d)
    Ug = tb["UDiv"].clone(); tfluids.setWallBcsForward(Ug, tb["flags"])
    Ul = loc["UDiv"].clone(); slab_on(); tfluids.setWallBcsForward(Ul, loc["flags"]); ctx.clear_slab()
    cmp("setWallBcs", Ul, Ug, d)
    dg = torch.empty_like(tb["flags"]); tfluids.velocityDivergenceForward(tb["UDiv"], tb["flags"], dg)
    dl = torch.empty_like(loc["flags"]); slab_on(); tfluids.velocityDivergenceForward(loc["UDiv"], loc["flags"], dl); ctx.clear_slab()
    cmp("divergence", dl, dg, d)
    Ug = tb["UDiv"].clone(); tfluids.velocityUpdateForward(Ug, tb["flags"], tb["density"])
    Ul = loc["UDiv"].clone(); slab_on(); tfluids.velocityUpdateForward(Ul, loc["flags"], loc["density"]); ctx.clear_slab()
    cmp("velocityUpdate", Ul, Ug, d)
    print("faults", ctx.trace_faults())
