"""Deterministic synthetic inputs for parity tests and bench (SURVEY.md section 8d).

Host-side numpy only.  Flags follow the reference's `emptyDomain(bnd=1)`
(torch/tfluids/generic/tfluids.cc:136-172) plus optional solid geometry (a sphere of
radius N/8 centred at (N/2, N/3, N/2) and a 2-cell slab) to exercise line tracing and
wall boundary conditions.
"""
import numpy as np

FLUID, OBSTACLE, EMPTY, OUTFLOW, STICK = 1.0, 2.0, 4.0, 16.0, 128.0


def make_flags(nx, ny, nz, is3d=True, nb=1, geometry=True, exotic=False, seed=7):
    """[nb][1][nz][ny][nx] float32 flags. exotic=True sprinkles Empty / Outflow / Stick
    cells (never on the border) to exercise every branch of the wall/pressure stencils."""
    if not is3d:
        assert nz == 1
    f = np.full((nb, 1, nz, ny, nx), FLUID, np.float32)
    f[..., 0] = OBSTACLE
    f[..., -1] = OBSTACLE
    f[..., 0, :] = OBSTACLE
    f[..., -1, :] = OBSTACLE
    if is3d:
        f[:, :, 0] = OBSTACLE
        f[:, :, -1] = OBSTACLE
    if geometry:
        z, y, x = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
        n = max(nx, ny, nz)
        cz = nz // 2 if is3d else 0
        r2 = (x - nx // 2) ** 2 + (y - ny // 3) ** 2 + ((z - cz) ** 2 if is3d else 0)
        sphere = r2 <= (n / 8.0) ** 2
        slab = (y >= (2 * ny) // 3) & (y < (2 * ny) // 3 + 2) & (x >= nx // 4) & (x < nx // 2)
        f[:, 0][np.broadcast_to(sphere | slab, f[:, 0].shape)] = OBSTACLE
    if exotic:
        rs = np.random.RandomState(seed)
        inner = np.zeros(f.shape, bool)
        if is3d:
            inner[:, :, 2:-2, 2:-2, 2:-2] = True
        else:
            inner[:, :, :, 2:-2, 2:-2] = True
        r = rs.rand(*f.shape)
        f[inner & (r < 0.03)] = EMPTY
        f[inner & (r >= 0.03) & (r < 0.04)] = EMPTY + OUTFLOW
        f[inner & (r >= 0.04) & (r < 0.05)] = OBSTACLE + STICK
    return np.ascontiguousarray(f)


def make_velocity(flags, is3d=True, amp=2.0, seed=1234):
    """Uniform in [-amp, amp] cells/s per face (|u| dt <= 0.35 cell at amp=2, dt=0.1)."""
    nb, _, nz, ny, nx = flags.shape
    rs = np.random.RandomState(seed)
    nc = 3 if is3d else 2
    U = (rs.rand(nb, nc, nz, ny, nx).astype(np.float32) * 2.0 - 1.0) * np.float32(amp)
    return np.ascontiguousarray(U.astype(np.float32))


def make_smooth_velocity(flags, is3d=True, amp=2.0, seed=1234):
    """Band-limited velocity (a few random Fourier modes): exercises longer coherent
    traces than white noise does."""
    nb, _, nz, ny, nx = flags.shape
    rs = np.random.RandomState(seed)
    nc = 3 if is3d else 2
    z, y, x = np.meshgrid(np.arange(nz) / max(nz, 1), np.arange(ny) / ny, np.arange(nx) / nx,
                          indexing="ij")
    U = np.zeros((nb, nc, nz, ny, nx), np.float64)
    for b in range(nb):
        for c in range(nc):
            for _ in range(4):
                k = rs.randint(1, 4, size=3)
                ph = rs.rand(3) * 2 * np.pi
                U[b, c] += rs.randn() * np.sin(2 * np.pi * k[0] * x + ph[0]) * \
                    np.sin(2 * np.pi * k[1] * y + ph[1]) * np.cos(2 * np.pi * k[2] * z + ph[2])
    U *= amp / max(np.abs(U).max(), 1e-9)
    return np.ascontiguousarray(U.astype(np.float32))


def make_density(flags, seed=1235):
    rs = np.random.RandomState(seed)
    d = rs.rand(*flags.shape).astype(np.float32)
    d[(flags.astype(np.int32) & 1) == 0] = 0.0
    return np.ascontiguousarray(d)


def make_model(is3d=True, seed=4321, model_type="default", banks=None, inputs=None, batch_norm=None):
    """Random-init weights of a reference architecture (torch/lib/model.lua:164-226: 'default', 'tog',
    'yang'), Torch `reset` convention uniform +-1/sqrt(fan_in).  Inputs: pDiv, div, occupancy
    (lib/default_conf.lua:76-81).  'tog' layers carry pooling / ConvolutionUpsample sizes: the weights of
    an upsampling layer have cout * up^d output channels.
    banks: {"num", "split_stage", "join_stage", "aggregate"[, "type"]} (lib/model.lua:252-361); a banked stage's
    entry in "layers" is then a list of num (weight, bias) pairs, and a 'concat' join stage takes num x the channels.
    "type" ('mres' or 'dilate') is carried through; both types draw the same weights.
    inputs: the input-block keywords of model.ProjectionModel (inputChannels, normalizeInput*, addPressureSkip),
    kept under "inputs"; the first layer takes the selected channels, the last one more with addPressureSkip.
    batch_norm: {"train": bool[, "affine": bool (default True), "eps": float (default 1e-4)]} adds "batchNorm" in the
    form of model.ProjectionModel's keyword: per stage but the last (per bank of a banked stage) a weight in
    [0.5, 1.5) and a bias in [-0.5, 0.5) (None without affine), a running mean in [-0.5, 0.5) and a running variance
    in [0.05, 1.05), drawn after the weights from their own stream."""
    rs = np.random.RandomState(seed)
    extra = {}
    if model_type == "default":
        osize, ksize = ([8, 8, 8, 8, 1], [3, 3, 3, 1, 1]) if is3d else ([16, 16, 16, 16, 1], [3, 3, 3, 3, 1])
        psize = usize = [1] * 5
    elif model_type == "tog":
        if is3d:
            osize, ksize = [16, 16, 16, 16, 32, 32, 1], [3, 3, 3, 3, 1, 1, 3]
            psize, usize = [2, 2, 1, 1, 1, 1, 1], [1, 1, 1, 1, 1, 2, 2]
        else:
            osize, ksize = [16, 32, 32, 64, 64, 32, 1], [5, 5, 5, 5, 1, 1, 3]
            psize, usize = [2, 1, 1, 1, 1, 1, 1], [1, 1, 1, 1, 1, 1, 2]
        extra = {"pool": psize, "up": usize, "poolType": "avg"}
    elif model_type == "yang":
        osize, ksize = [6, 6, 6, 1], [3, 1, 1, 1]
        psize = usize = [1] * 4
        extra = {"nonlinType": "sigmoid"}
    else:
        raise ValueError(model_type)
    nbanks = banks["num"] if banks is not None else 1
    layers = []
    ch = {"pDiv": True, "UDiv": False, "div": True, "flags": True}
    ch.update((inputs or {}).get("inputChannels") or {})
    cin = int(ch["pDiv"]) + (3 if is3d else 2) * int(ch["UDiv"]) + int(ch["div"]) + int(ch["flags"])
    for stage, (cout, k, u) in enumerate(zip(osize, ksize, usize), start=1):
        if nbanks > 1 and stage == banks["join_stage"] and banks["aggregate"] == "concat":
            cin *= nbanks
        if stage == len(osize) and (inputs or {}).get("addPressureSkip"):
            cin += 1
        banked = nbanks > 1 and banks["split_stage"] <= stage < banks["join_stage"]
        kz = k if is3d else 1
        fan_in = cin * kz * k * k
        bound = 1.0 / np.sqrt(fan_in)
        ct = cout * u ** (3 if is3d else 2)
        convs = []
        for _ in range(nbanks if banked else 1):
            w = ((rs.rand(ct, cin, kz, k, k) * 2 - 1) * bound).astype(np.float32)
            b = ((rs.rand(ct) * 2 - 1) * bound).astype(np.float32)
            convs.append((np.ascontiguousarray(w), np.ascontiguousarray(b)))
        layers.append(convs if banked else convs[0])
        cin = cout
    out = {"is3D": is3d, "layers": layers}
    out.update(extra)
    if banks is not None:
        out["banks"] = dict(banks)
    if inputs is not None:
        out["inputs"] = dict(inputs)
    if batch_norm is not None:
        rb = np.random.RandomState(seed + 1)
        affine = batch_norm.get("affine", True)
        eps = float(batch_norm.get("eps", 1e-4))

        def entry(c):
            w = (0.5 + rb.rand(c)).astype(np.float32) if affine else None
            b = (rb.rand(c) - 0.5).astype(np.float32) if affine else None
            return {"weight": w, "bias": b, "running_mean": (rb.rand(c) - 0.5).astype(np.float32),
                    "running_var": (0.05 + rb.rand(c)).astype(np.float32), "eps": eps}
        bn_layers = []
        for cout, layer in zip(osize[:-1], layers[:-1]):
            bn_layers.append([entry(cout) for _ in layer] if isinstance(layer, list) else entry(cout))
        out["batchNorm"] = {"train": bool(batch_norm["train"]), "layers": bn_layers}
    return out
