"""Creation and destruction through the C ABI: every object the library hands out (context, model, host-buffer
simulation, step graph, z-slab simulation) is created, used and destroyed again and again in one process, in a
different destruction order each time, and gives the same bits every time; creators refuse bad grids before they
allocate; every destroyer accepts NULL."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle
from fluidnet_b200 import _lib, simulate, synth, tfluids
from scenes import plume_batch, step_mconf

pytestmark = pytest.mark.gpu

N = 32


def _ok(lib, ctx, rc, what):
    assert rc == 0, "%s: %s" % (what, lib.tfl_last_error(ctx).decode())


def _mconf(sim_method):
    return simulate.make_mconf(step_mconf(N, simMethod=sim_method, maxIter=20))


def test_host_sim_refuses_bad_grids():
    """nb = 0, nz = 0 and a 2-D grid with two planes are refused before anything is allocated."""
    lib = _lib.load()
    ctx = C.c_void_p()
    assert lib.tfl_create(C.byref(ctx), 0) == 0
    try:
        flags = np.ones(2 * N * N, np.float32)
        for nb, nz, is_3d in ((0, N, 1), (1, 0, 1), (1, 2, 0)):
            hs = C.c_void_p(16)                               # not NULL: the refusal must clear it
            rc = lib.tfl_host_sim_create(ctx, nb, nz, N, N, is_3d, flags.ctypes.data, None, None, None, None,
                                         C.byref(hs))
            assert rc != 0, (nb, nz, is_3d)
            assert "host_sim" in lib.tfl_last_error(ctx).decode(), (nb, nz, is_3d)
            assert not hs.value, (nb, nz, is_3d)
    finally:
        lib.tfl_destroy(ctx)


def test_destroyers_accept_null():
    lib = _lib.load()
    ctx = C.c_void_p()
    assert lib.tfl_create(C.byref(ctx), 0) == 0
    for c in (ctx, None):
        lib.tfl_cnn_destroy(c, None)
        lib.tfl_host_sim_destroy(c, None)
        lib.tfl_step_graph_destroy(c, None)
        lib.tfl_slab_sim_destroy(c, None)
    lib.tfl_destroy(ctx)
    lib.tfl_destroy(None)


def _cycle(lib, batch, layers, order):
    """One context and one of everything on it; returns p, U, density of the host-buffer steps, the replayed step
    graph and the z-slab step."""
    ctx = C.c_void_p()
    assert lib.tfl_create(C.byref(ctx), 0) == 0
    ok = lambda rc, what: _ok(lib, ctx, rc, what)           # noqa: E731
    stream = torch.cuda.Stream()
    ok(lib.tfl_set_stream(ctx, C.c_void_p(stream.cuda_stream)), "set_stream (torch)")
    assert lib.tfl_get_stream(ctx) == stream.cuda_stream
    ok(lib.tfl_set_stream(ctx, None), "set_stream (own)")
    own = lib.tfl_get_stream(ctx)
    assert own not in (None, stream.cuda_stream)
    ok(lib.tfl_set_stream(ctx, C.c_void_p(own)), "set_stream (its own stream, adopted)")   # stays owned and alive
    assert lib.tfl_get_stream(ctx) == own
    out = {}

    # a PCG solve: the context's PCG scratch is allocated here
    flags = torch.from_numpy(batch["flags"]).cuda()
    div = torch.from_numpy(synth.make_density(batch["flags"], seed=99) - np.float32(0.5)).cuda()
    p = torch.zeros_like(flags)
    torch.cuda.synchronize()
    res, its = C.c_float(), C.c_int()
    ok(lib.tfl_solve_linear_system_pcg(ctx, C.byref(tfluids._grid(p)), C.byref(tfluids._grid(flags)),
                                       C.byref(tfluids._grid(div)), 1, lib.tfl_precond_from_string(b"ic0"), 1e-4, 100,
                                       C.byref(res), C.byref(its)), "pcg")
    ok(lib.tfl_sync(ctx), "sync")

    # the 3-D 'default' model
    n = len(layers)
    ws = [np.ascontiguousarray(w, np.float32) for w, _ in layers]
    bs = [np.ascontiguousarray(b, np.float32) for _, b in layers]
    ints = lambda v: (C.c_int32 * n)(*v)                    # noqa: E731
    wp = (C.POINTER(C.c_float) * n)(*[w.ctypes.data_as(C.POINTER(C.c_float)) for w in ws])
    bp = (C.POINTER(C.c_float) * n)(*[b.ctypes.data_as(C.POINTER(C.c_float)) for b in bs])
    model = C.c_void_p()
    ok(lib.tfl_cnn_create(ctx, 1, n, ints([w.shape[1] for w in ws]), ints([w.shape[0] for w in ws]),
                          ints([w.shape[4] for w in ws]), wp, bp, C.byref(model)), "cnn_create")
    mc = _mconf("convnet")

    # two host-buffer steps
    keep = [np.ascontiguousarray(batch[k]) for k in ("flags", "UBC", "UBCInvMask", "densityBC", "densityBCInvMask")]
    hs = C.c_void_p()
    ok(lib.tfl_host_sim_create(ctx, 1, N, N, N, 1, *[a.ctypes.data for a in keep], C.byref(hs)), "host_sim_create")
    hp, hU, hd = (torch.from_numpy(batch[k].copy()).pin_memory() for k in ("pDiv", "UDiv", "density"))
    for _ in range(2):
        ok(lib.tfl_host_sim_step(ctx, hs, hp.data_ptr(), hU.data_ptr(), hd.data_ptr(), C.byref(mc), model), "host step")
    out["host"] = [t.numpy().copy() for t in (hp, hU, hd)]

    # one step, then the same step captured and replayed
    gb = {k: torch.from_numpy(v.copy()).cuda() for k, v in batch.items()}
    st = simulate.make_state(gb)
    torch.cuda.synchronize()
    ok(lib.tfl_simulate_step(ctx, C.byref(st), C.byref(mc), model), "simulate_step")
    graph = C.c_void_p()
    ok(lib.tfl_step_graph_create(ctx, C.byref(st), C.byref(mc), model, C.byref(graph)), "step_graph_create")
    ok(lib.tfl_step_graph_launch(ctx, graph), "step_graph_launch")
    ok(lib.tfl_sync(ctx), "sync")
    out["graph"] = [gb[k].cpu().numpy() for k in ("pDiv", "UDiv", "density")]

    # a world-1 z-slab simulation, one simMethod 'jacobi' step
    slab = C.c_void_p()
    ok(lib.tfl_slab_sim_create(ctx, N, N, N, 2, *[a.ctypes.data for a in keep], C.byref(slab)), "slab_sim_create")
    ok(lib.tfl_slab_sim_upload(ctx, slab, batch["pDiv"].ctypes.data, batch["UDiv"].ctypes.data,
                               batch["density"].ctypes.data), "slab upload")
    ok(lib.tfl_slab_sim_step(ctx, slab, C.byref(_mconf("jacobi")), None), "slab step")
    sp, sU, sd = (np.zeros_like(batch[k]) for k in ("pDiv", "UDiv", "density"))
    ok(lib.tfl_slab_sim_download(ctx, slab, sp.ctypes.data, sU.ctypes.data, sd.ctypes.data), "slab download")
    out["slab"] = [sp, sU, sd]

    destroy = {"model": lambda: lib.tfl_cnn_destroy(ctx, model), "host": lambda: lib.tfl_host_sim_destroy(ctx, hs),
               "graph": lambda: lib.tfl_step_graph_destroy(ctx, graph),
               "slab": lambda: lib.tfl_slab_sim_destroy(ctx, slab)}
    for name in order:
        destroy[name]()
    lib.tfl_destroy(ctx)
    return out


def test_repeated_create_use_destroy_gives_the_same_bits():
    """Five cycles of context, PCG solve, model, host-buffer steps, step graph and z-slab step, each torn down in
    another order with the context last: every call succeeds and the last cycle computes the first one's bits."""
    lib = _lib.load()
    batch = plume_batch(N, inflow=N / 128.0)
    layers = synth.make_model(True)["layers"]
    orders = [("model", "host", "graph", "slab"), ("slab", "graph", "host", "model"), ("graph", "model", "slab", "host"),
              ("host", "slab", "model", "graph"), ("model", "graph", "slab", "host")]
    runs = [_cycle(lib, batch, layers, order) for order in orders]
    for key, first in runs[0].items():
        for name, a, b in zip(("p", "U", "density"), first, runs[-1][key]):
            assert np.array_equal(a.view(np.int32), b.view(np.int32)), "%s %s differs between cycles" % (key, name)
