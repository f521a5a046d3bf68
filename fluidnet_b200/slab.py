"""z-slab decomposition of ONE fluid domain across the GPUs of a node (SURVEY.md section 8e).

The reference is single-GPU; this is the multi-GPU path north_star asks for: rank r owns the planes
[z0, z1) of every field plus `halo` ghost planes on each interior side, the kernels of libtfl.so
are told where the local array sits in the global grid (tfl_set_slab: border tests, getDx, line
traces and interpolation clamps use GLOBAL coordinates), and ghost planes are refreshed with
neighbour send/recv pairs (torch.distributed, NCCL over NVLink on GPUs, gloo in the CPU tests)
before each phase whose stencil reaches across the cut:

    exchange U, density  (halo)   -> advectScalar, advectVel   (MacCormack fwd pass evaluated on
                                                                 owned +- margin planes, bwd on owned)
    exchange U, density  (4)      -> addBuoyancy on owned +- 3 planes, vorticityConfinement (-3 / +3)
    exchange U, p        (5)      -> CNN projection: wall mask + sum/sumsq on owned planes,
                                     all-reduce of the two sums (the input scale), conv stack on the
                                     whole local slab, velocity update on owned planes
                                     (banked models: 2 * cnn_margin(banksNum) + 1 planes; the halo
                                     then needs margin >= cnn_margin(banksNum))

simMethod 'jacobi' (no model) replaces the last phase: setWallBcsForward on the owned planes, then

    exchange U           (w)      -> divergence and Jacobi mask on owned +- (w - 1) planes
    Jacobi from p = 0 in blocks of up to `halo` sweeps (jacobi_schedule): after an exchange of p of
    width w a block's sweep s computes owned +- (w - 1 - s) planes, so one exchange serves a block;
    p starts at zero everywhere (no exchange before the first block), the last block leaves p right
    one plane below the owned ones for the velocity update on owned planes.

It has no reduction at all, so p, U and density equal the single-GPU step bit for bit.  'pcg' is not
decomposed (its IC(0) triangular solves sweep the whole domain in order).

There is no data-path collective other than those neighbour exchanges and the 2-double all-reduce.
A line trace or stencil that leaves the local slab (halo too small for the velocity) increments
the library's fault counter instead of reading out of bounds; `SlabSimulator.check()` raises.
"""
import contextlib
import ctypes as C

import torch
import torch.distributed as dist

from . import _lib


def jacobi_schedule(gnz, world, rank, margin, max_iter):
    """The Jacobi sweep schedule of one rank (tfl_slab_jacobi_schedule): ((first, past-last local plane with valid
    divergence and mask, width of the U exchange), [(sweeps, p exchange width before the block or 0, first /
    past-last local plane of the block's sweep 0, shrink at the bottom, shrink at the top), ...])."""
    lib = _lib.load()
    planes = (C.c_int32 * 3)()
    n = lib.tfl_slab_jacobi_schedule(gnz, world, rank, margin, max_iter, planes, None, 0)
    if n < 1:
        raise ValueError("no Jacobi schedule for gnz=%d world=%d rank=%d margin=%d maxIter=%d"
                         % (gnz, world, rank, margin, max_iter))
    raw = (C.c_int32 * (_lib.JACOBI_BLOCK_INTS * n))()
    lib.tfl_slab_jacobi_schedule(gnz, world, rank, margin, max_iter, planes, raw, n)
    k = _lib.JACOBI_BLOCK_INTS
    return tuple(planes), [tuple(raw[b * k:(b + 1) * k]) for b in range(n)]


def cnn_margin(banks_num):
    """The smallest slab margin a projection network with `banks_num` banks runs with (tfl_slab_cnn_margin): 2 for
    one bank, ceil(3 * 2^(banks_num-1) / 2) for more -- the coarsest bank's stencil reaches 3 * 2^(banks_num-1) + 2
    planes across a rank boundary, and the halo holds 2 * margin + 2."""
    m = _lib.load().tfl_slab_cnn_margin(int(banks_num))
    if m < 1:
        raise ValueError("no z-slab margin for %d banks (at most 8)" % banks_num)
    return m


def _resolve_margin(margin, banks):
    """margin=None -> the model's minimum (2 for a single bank); an explicit margin below it raises ValueError."""
    n = banks["num"] if banks else 1
    need = cnn_margin(n)
    if margin is None:
        return max(2, need)
    if n > 1 and margin < need:
        raise ValueError("a %d-bank model needs a z-slab margin >= %d (got %d)" % (n, need, margin))
    return margin


def _sim_method(mconf):
    """'convnet' or 'jacobi' and the sweep count (refuses what the slab step does not decompose)."""
    method = mconf.get("simMethod") or "convnet"
    if method == "pcg":
        raise ValueError("simMethod 'pcg' is not decomposed over z-slabs: the IC(0) triangular solves of its "
                         "preconditioner sweep the whole domain in order")
    if method not in ("convnet", "jacobi"):
        raise ValueError("mconf.simMethod (%s) is not a valid option" % method)
    iters = mconf.get("maxIter")
    if method == "jacobi" and iters is not None and int(iters) < 1:
        raise ValueError("At least 1 iteration is needed (maxIter < 1)")
    return method, int(iters or 100)


class SlabDecomposition:
    """Which global planes a rank owns / stores, and the halo exchange between neighbours."""

    def __init__(self, gnz, rank, world, halo):
        assert world >= 1 and 0 <= rank < world
        base, rem = divmod(gnz, world)
        sizes = [base + (1 if r < rem else 0) for r in range(world)]
        assert min(sizes) >= max(halo, 1), "slab thinner than the halo: use fewer ranks or a smaller halo"
        self.gnz, self.rank, self.world, self.halo = gnz, rank, world, halo
        self.z0 = sum(sizes[:rank])
        self.z1 = self.z0 + sizes[rank]
        self.lo_halo = min(halo, self.z0)                 # no ghost planes beyond the global ends
        self.hi_halo = min(halo, gnz - self.z1)
        self.zoff = self.z0 - self.lo_halo                # global index of local plane 0
        self.nz = (self.z1 - self.z0) + self.lo_halo + self.hi_halo
        self.own_lo = self.lo_halo
        self.own_hi = self.lo_halo + (self.z1 - self.z0)

    def scatter(self, t):
        """Local slab (owned + ghost planes) of a global [b][c][gnz][y][x] tensor."""
        return t[:, :, self.zoff:self.zoff + self.nz].contiguous()

    def owned(self, t):
        return t[:, :, self.own_lo:self.own_hi]

    def exchange(self, tensors, width, group=None):
        """Refresh `width` ghost planes on both sides of every tensor from the neighbours' owned
        planes.  One packed message per neighbour and direction."""
        if self.world == 1 or width == 0:
            return
        assert width <= self.halo
        ops, unpack = [], []

        def pack(a, b):
            return torch.cat([t[:, :, a:b].reshape(-1) for t in tensors])

        def plan(peer, send_rng, recv_rng):
            sbuf = pack(*send_rng)
            rbuf = torch.empty_like(sbuf)
            ops.append(dist.P2POp(dist.isend, sbuf, peer, group))
            ops.append(dist.P2POp(dist.irecv, rbuf, peer, group))
            unpack.append((rbuf, recv_rng))

        if self.rank > 0:                                  # lower neighbour: my first owned planes go down
            plan(self.rank - 1, (self.own_lo, self.own_lo + width), (self.own_lo - width, self.own_lo))
        if self.rank < self.world - 1:                     # upper neighbour
            plan(self.rank + 1, (self.own_hi - width, self.own_hi), (self.own_hi, self.own_hi + width))
        for req in dist.batch_isend_irecv(ops):
            req.wait()
        for rbuf, (a, b) in unpack:
            off = 0
            for t in tensors:
                view = t[:, :, a:b]
                n = view.numel()
                view.copy_(rbuf[off:off + n].view(view.shape))
                off += n


class SlabSimulator:
    """tfluids.simulate (simMethod 'convnet' or 'jacobi') for one domain split in z across the ranks of `group`."""

    def __init__(self, batch, mconf, model_layers, device, rank=None, world=None, margin=None, group=None,
                 jacobi_path=-1, banks=None, conv_mode=None):
        """batch: dict of GLOBAL torch CPU tensors (pDiv, UDiv, flags, density and the BC arrays),
        identical on every rank.  margin: planes a backward trace may reach (ceil(max|u| dt) + 1); None: the
        smallest the model runs with (cnn_margin), 2 for a single bank.
        model_layers: None for simMethod 'jacobi'.  jacobi_path: tfl_jacobi_slab_block's path (-1 automatic).
        banks / conv_mode: ProjectionModel's banks and, if given, its mode ('tf32' or 'tf32x3'; slabs run on the
        tensor cores only)."""
        from . import tfluids, model as fmodel
        self.tfluids = tfluids
        self.group = group
        self.rank = dist.get_rank(group) if rank is None else rank
        self.world = dist.get_world_size(group) if world is None else world
        self.mconf = dict(mconf)
        method, iters = _sim_method(self.mconf)
        self.jacobi = method == "jacobi"
        margin = _resolve_margin(margin, None if self.jacobi else banks)
        gnz = batch["flags"].shape[2]
        assert margin >= 2, "margin < 2 makes the halo narrower than the widest fixed exchange (5 planes)"
        self.dec = SlabDecomposition(gnz, self.rank, self.world, halo=2 * margin + 2)
        self.margin = margin
        self.device = torch.device(device)
        self.s = {k: self.dec.scatter(v).to(self.device) for k, v in batch.items() if v is not None}
        self.ctx = tfluids.context(self.device)
        if self.jacobi:
            self.model = None
            self.jsched = jacobi_schedule(gnz, self.world, self.rank, margin, iters)
            self.jacobi_path = jacobi_path
            self.div = torch.zeros_like(self.s["pDiv"])
            self.p2 = torch.zeros_like(self.s["pDiv"])
        else:
            self.model = fmodel.ProjectionModel(model_layers, True, device=self.device, banks=banks,
                                                normalizeInputThreshold=self.mconf.get("normalizeInputThreshold", 1e-5))
            if conv_mode is not None:
                self.model.set_mode(conv_mode)
        self.U1 = torch.empty_like(self.s["UDiv"])
        self.sums = torch.zeros(2, dtype=torch.float64, device=self.device)

    # -- helpers ---------------------------------------------------------------------------
    @contextlib.contextmanager
    def _slab(self, z_lo, z_hi):
        """Slab placement of the (shared, per-device) context for the enclosed calls only."""
        d = self.dec
        self.ctx.set_slab(d.zoff, d.gnz, z_lo, z_hi)
        try:
            self.ctx.check(self.ctx.lib.tfl_set_slab_margin(self.ctx.h, self.margin))
            yield
        finally:
            self.ctx.clear_slab()

    def _bc(self):
        t, s = self.tfluids, self.s
        if s.get("UBC") is not None:
            t.applyBC(s["UDiv"], s["UBCInvMask"], s["UBC"])
        if s.get("densityBC") is not None:
            t.applyBC(s["density"], s["densityBCInvMask"], s["densityBC"])

    def step(self):
        """One tfluids.simulate on this rank's slab; communication through torch.distributed."""
        for req in self.phases():
            if req[0] == "halo":
                self.dec.exchange(req[1], req[2], self.group)
            elif self.world > 1:
                dist.all_reduce(req[1], group=self.group)

    def phases(self):
        """The step as a generator that yields its communication requests -- ("halo", tensors,
        width) or ("sum", tensor) -- so that a driver can satisfy them with torch.distributed
        (`step`) or, in tests, between several slabs living in one process (`run_lockstep`)."""
        t, s, m, d = self.tfluids, self.s, self.mconf, self.dec
        p, U, flags, rho = s["pDiv"], s["UDiv"], s["flags"], s["density"]
        method, strength = m.get("advectionMethod"), m.get("maccormackStrength")
        yield ("halo", [U, rho], d.halo)
        with self._slab(d.own_lo, d.own_hi):
            t.advectScalar(m["dt"], rho, U, flags, method, None, False, strength)
            t.advectVel(m["dt"], U, flags, method, None, strength)
        self._bc()
        yield ("halo", [U, rho], 4)
        # Buoyancy / gravity are point-wise in U but vorticity confinement then reads U three planes across
        # the cut: apply them on those ghost planes too (buoyancy needs density one plane further).
        dx = 1.0 / max(d.gnz, flags.size(3), flags.size(4))
        f32 = lambda v: torch.tensor(float(v), dtype=torch.float32).item()
        g = m.get("gravity") or [0.0, 1.0, 0.0]
        with self._slab(d.own_lo - min(3, d.lo_halo), d.own_hi + min(3, d.hi_halo)):
            if (m.get("buoyancyScale") or 0) > 0:
                k = f32(-(dx / 4) * m["buoyancyScale"])
                t.addBuoyancy(U, flags, rho, [f32(f32(v) * k) for v in g], m["dt"])
            if (m.get("gravityScale") or 0) > 0:                      # lib/simulate.lua:229-233
                k = f32((-dx / 4) * m["gravityScale"])
                t.addGravity(U, flags, [f32(f32(v) * k) for v in g], m["dt"])
        if (m.get("vorticityConfinementAmp") or 0) > 0:
            with self._slab(d.own_lo, d.own_hi):
                t.vorticityConfinement(U, flags, dx * m["vorticityConfinementAmp"])
        if self.jacobi:
            with self._slab(d.own_lo, d.own_hi):
                t.setWallBcsForward(U, flags)
            self._bc()
            yield from self._jacobi(p, U, flags)
            self._bc()
            t.clamp(U, -1e6, 1e6)
            return
        self._bc()
        yield ("halo", [U, p], 2 * cnn_margin(self.model.banks["num"] if self.model.banks else 1) + 1)
        c, lib = self.ctx, self.ctx.lib
        with self._slab(d.own_lo, d.own_hi):
            c.use_current_stream()
            c.check(lib.tfl_cnn_stats(c.h, t._grid(U), t._grid(flags), t._grid(self.U1), C.c_void_p(self.sums.data_ptr())))
        yield ("sum", self.sums)
        with self._slab(d.own_lo, d.own_hi):
            c.use_current_stream()
            c.check(lib.tfl_cnn_project_from_sums(c.h, self.model.h, t._grid(p), t._grid(self.U1), t._grid(flags),
                                                  C.c_void_p(self.sums.data_ptr()), t._grid(p), t._grid(U),
                                                  float(self.model.threshold)))
        self._bc()
        t.clamp(U, -1e6, 1e6)

    def _jacobi(self, p, U, flags):
        """lib/simulate.lua:275-303 with pTol = 0 on this slab, in the blocks of jacobi_schedule."""
        t, d, c = self.tfluids, self.dec, self.ctx
        (plo, phi, u_width), blocks = self.jsched
        yield ("halo", [U], u_width)
        with self._slab(plo, phi):
            t.velocityDivergenceForward(U, flags, self.div)
        p.zero_()
        self.p2.zero_()
        bufs, done = [p, self.p2], 0
        for sweeps, width, zlo, zhi, shr_lo, shr_hi in blocks:
            if width:
                yield ("halo", [bufs[done & 1]], width)
            if sweeps:
                with self._slab(zlo, zhi):
                    c.use_current_stream()
                    c.check(c.lib.tfl_jacobi_slab_block(c.h, t._grid(bufs[done & 1]), t._grid(bufs[(done + 1) & 1]),
                                                        t._grid(flags), t._grid(self.div), 1, zlo, zhi, shr_lo, shr_hi,
                                                        sweeps, self.jacobi_path, None))
            done += sweeps
        if done & 1:
            p.copy_(self.p2)
        with self._slab(d.own_lo, d.own_hi):
            t.velocityUpdateForward(U, flags, p)

    def check(self):
        """Raises if any stencil / trace left the local slab since the last check."""
        f = torch.tensor([self.ctx.trace_faults()], dtype=torch.float64, device=self.device)
        if self.world > 1:
            dist.all_reduce(f, group=self.group)
        if f.item() != 0:
            raise RuntimeError("z-slab halo too small for the current velocities (%d faults): raise `margin`"
                               % int(f.item()))

    def gather(self, key):
        """Global tensor assembled from every rank's owned planes (on every rank, CPU)."""
        mine = self.dec.owned(self.s[key]).contiguous()
        if self.world == 1:
            return mine.cpu()
        sizes = [SlabDecomposition(self.dec.gnz, r, self.world, self.dec.halo) for r in range(self.world)]
        parts = [torch.empty(mine.shape[:2] + (q.z1 - q.z0,) + mine.shape[3:], dtype=mine.dtype, device=mine.device)
                 for q in sizes]
        dist.all_gather(parts, mine, group=self.group) if len({tuple(x.shape) for x in parts}) == 1 else \
            self._all_gather_uneven(parts, mine)
        return torch.cat([x.cpu() for x in parts], dim=2)

    def _all_gather_uneven(self, parts, mine):
        for r in range(self.world):
            if r == self.rank:
                parts[r].copy_(mine)
            dist.broadcast(parts[r], src=r, group=self.group)


class NativeSlabSimulator:
    """The same decomposition with everything inside libtfl.so (tfl_slab_sim_*): the context owns the NCCL
    communicator, the halo exchanges are ncclSend / ncclRecv straight on the field arrays, one C call per step.
    This is what a LuaJIT host would drive; torch.distributed is used here only to hand rank 0's NCCL id to the
    other ranks (any transport would do) and, in `gather`, by the tests.

    Without torch.distributed (`allgather` and `barrier` given, e.g. processes that share one GPU): no NCCL
    communicator, the IPC handles go through `allgather`, and peer memory is the only transport -- the constructor
    raises on every rank if any rank cannot map its neighbours' inboxes."""

    def __init__(self, batch, mconf, model_layers, device, rank=None, world=None, margin=None, group=None,
                 peer_halos=True, banks=None, conv_mode=None, model=None, allgather=None, barrier=None):
        """Arguments as SlabSimulator's (margin=None: the model's smallest, cnn_margin).  model: an existing
        ProjectionModel on `device` to run instead of one built from model_layers / banks.
        allgather(bytes or None) -> list over the ranks in rank order, and barrier(): replace torch.distributed (both
        or neither; rank and world must then be given)."""
        import numpy as np
        from . import tfluids, model as fmodel, simulate, _lib
        if (allgather is None) != (barrier is None):
            raise ValueError("NativeSlabSimulator: give allgather and barrier together")
        self._allgather, self._barrier = allgather, barrier
        if allgather is not None and (rank is None or world is None):
            raise ValueError("NativeSlabSimulator: without torch.distributed, rank and world must be given")
        if allgather is not None and world > 1 and not peer_halos:
            raise ValueError("NativeSlabSimulator: without torch.distributed there is no NCCL communicator; "
                             "the halos need peer memory (peer_halos=True)")
        self.group = group
        self.rank = dist.get_rank(group) if rank is None else rank
        self.world = dist.get_world_size(group) if world is None else world
        self.mconf = dict(mconf)
        method, _ = _sim_method(self.mconf)
        if model is not None:
            banks = model.banks
        margin = _resolve_margin(margin, None if method == "jacobi" else banks)
        self.device = torch.device(device)
        self.ctx = tfluids.context(self.device)
        lib = self.ctx.lib
        ident = [None]                        # NULL id: the context takes rank and world but makes no communicator
        if self.world > 1 and allgather is None:
            if self.rank == 0:
                buf = C.create_string_buffer(_lib.COMM_ID_BYTES)
                self.ctx.check(lib.tfl_comm_unique_id(self.ctx.h, buf))
                ident = [buf.raw]
            dist.broadcast_object_list(ident, src=0, group=group)
        self.ctx.check(lib.tfl_comm_init(self.ctx.h, ident[0], self.rank, self.world))
        self.mc = simulate.make_mconf(self.mconf)
        if method == "jacobi":
            self.model = None
        elif model is not None:
            self.model = model
        else:
            self.model = fmodel.ProjectionModel(model_layers, True, device=self.device, banks=banks,
                                                normalizeInputThreshold=self.mconf.get("normalizeInputThreshold", 1e-5))
        if self.model is not None and conv_mode is not None:
            self.model.set_mode(conv_mode)

        def host(key):
            t = batch.get(key)
            return None if t is None else np.ascontiguousarray(t.numpy() if isinstance(t, torch.Tensor) else t, np.float32)

        self.margin = margin
        self._shape = tuple(batch["flags"].shape)
        gnz, ny, nx = self._shape[2:]
        arrs = [host(k) for k in ("flags", "UBC", "UBCInvMask", "densityBC", "densityBCInvMask")]
        h = C.c_void_p()
        self.ctx.use_current_stream()
        self.ctx.check(lib.tfl_slab_sim_create(self.ctx.h, gnz, ny, nx, margin, *[a.ctypes.data if a is not None else None
                                                                                  for a in arrs], C.byref(h)))
        self.h = h
        self.ctx.check(lib.tfl_slab_sim_upload(self.ctx.h, self.h, host("pDiv").ctypes.data, host("UDiv").ctypes.data,
                                               host("density").ctypes.data))
        info = (C.c_int32 * 6)()
        lib.tfl_slab_sim_layout(self.h, None, info)
        self.zoff, self.nz, self.own_lo, self.own_hi, self.z0, self.z1 = list(info)
        # Halos over peer memory (CUDA IPC + NVLink) when every rank can map its neighbours; otherwise NCCL.
        self.halo_transport = "nccl"
        if self.world > 1 and allgather is not None:
            self._connect_without_dist()
        elif self.world > 1 and peer_halos:
            buf = C.create_string_buffer(_lib.IPC_HANDLE_BYTES)
            ok = lib.tfl_slab_sim_ipc_export(self.ctx.h, self.h, buf) == 0
            handles = [None] * self.world
            dist.all_gather_object(handles, buf.raw if ok else None, group=group)
            if all(h is not None for h in handles):
                ok = lib.tfl_slab_sim_ipc_connect(self.ctx.h, self.h, b"".join(handles)) == 0
            else:
                ok = False
            flags_ok = [None] * self.world
            dist.all_gather_object(flags_ok, bool(ok), group=group)      # also the barrier before the first step
            if all(flags_ok):
                self.halo_transport = "peer memory (CUDA IPC over NVLink)"
            elif ok:                                          # every rank must use the same transport
                self.ctx.check(lib.tfl_slab_sim_ipc_connect(self.ctx.h, self.h, None))

    def _connect_without_dist(self):
        """Peer memory with the handles moved by `allgather`.  There is no communicator to fall back on: an unconnected
        tfl_slab_sim_step would exchange nothing and reduce nothing, so every rank raises if any rank fails."""
        from ._lib import TflError
        lib = self.ctx.lib
        buf = C.create_string_buffer(_lib.IPC_HANDLE_BYTES)
        error = None
        if lib.tfl_slab_sim_ipc_export(self.ctx.h, self.h, buf) != 0:
            error = lib.tfl_last_error(self.ctx.h).decode()
        handles = self._allgather(None if error else buf.raw)
        failed = [(r, "no inbox handle") for r, h in enumerate(handles) if h is None]
        if not failed:                        # every rank learns every rank's error (the same list everywhere)
            if lib.tfl_slab_sim_ipc_connect(self.ctx.h, self.h, b"".join(handles)) != 0:
                error = lib.tfl_last_error(self.ctx.h).decode()
            failed = [(r, e) for r, e in enumerate(self._allgather(error)) if e]
        if failed:
            self.close()
            raise TflError("NativeSlabSimulator: peer memory refused (%s); without torch.distributed there is no "
                           "NCCL fallback, the halo exchanges would move nothing"
                           % "; ".join("rank %d: %s" % rf for rf in failed))
        self._barrier()                       # every rank is connected before any rank steps
        self.halo_transport = "peer memory (CUDA IPC)"

    def step(self):
        self.ctx.use_current_stream()
        self.ctx.check(self.ctx.lib.tfl_slab_sim_step(self.ctx.h, self.h, C.byref(self.mc),
                                                      self.model.h if self.model is not None else None))

    def exchange_stats(self):
        """(ms of the three halo exchanges and the all-reduce of the last step, bytes sent per exchange)."""
        ms, by = (C.c_float * 4)(), (C.c_int64 * 3)()
        self.ctx.check(self.ctx.lib.tfl_slab_sim_exchange_stats(self.ctx.h, self.h, ms, by))
        return list(ms), list(by)

    def jacobi_stats(self):
        """(count, ms, bytes sent) of the last step's p exchanges (simMethod 'jacobi')."""
        n, ms, by = C.c_int32(), C.c_float(), C.c_int64()
        self.ctx.check(self.ctx.lib.tfl_slab_sim_jacobi_stats(self.ctx.h, self.h, C.byref(n), C.byref(ms), C.byref(by)))
        return n.value, ms.value, by.value

    def set_jacobi_tolerance(self, p_tol):
        """pTol of later 'jacobi' steps (tfl_slab_sim_set_jacobi_tolerance): 0 is the fixed count of maxIter sweeps,
        > 0 solves to the tolerance as the whole-grid solveLinearSystemJacobiDevice does.  A SlabStepGraph keeps the
        tolerance it was captured with."""
        self.ctx.check(self.ctx.lib.tfl_slab_sim_set_jacobi_tolerance(self.ctx.h, self.h, float(p_tol)))

    def jacobi_status(self):
        """(residual, iterations) of the last step that solved to a tolerance, direct or replayed.  Synchronises."""
        res, it = C.c_float(), C.c_int32()
        self.ctx.check(self.ctx.lib.tfl_slab_sim_jacobi_status(self.ctx.h, self.h, C.byref(res), C.byref(it)))
        return res.value, it.value

    def check(self):
        """Raises if any stencil / trace left the local slab since the last check: on any rank, or without
        torch.distributed on this one."""
        f = torch.tensor([self.ctx.trace_faults()], dtype=torch.float64, device=self.device)
        if self.world > 1 and self._allgather is None:
            dist.all_reduce(f, group=self.group)
        if f.item() != 0:
            raise RuntimeError("z-slab halo too small for the current velocities (%d faults): raise `margin`"
                               % int(f.item()))

    def download(self):
        """Global numpy arrays holding THIS rank's owned planes (zeros elsewhere)."""
        import numpy as np
        b, _, gnz, ny, nx = self._shape
        p = np.zeros((1, 1, gnz, ny, nx), np.float32)
        U = np.zeros((1, 3, gnz, ny, nx), np.float32)
        d = np.zeros((1, 1, gnz, ny, nx), np.float32)
        self.ctx.check(self.ctx.lib.tfl_slab_sim_download(self.ctx.h, self.h, p.ctypes.data, U.ctypes.data, d.ctypes.data))
        return {"pDiv": p, "UDiv": U, "density": d}

    def gather(self, key):
        """Global tensor assembled from every rank's owned planes (on every rank, CPU)."""
        if self.world > 1 and self._allgather is not None:
            raise RuntimeError("NativeSlabSimulator.gather needs torch.distributed; without it each rank download()s "
                               "its owned planes and the host application assembles them")
        mine = torch.from_numpy(self.download()[key])
        if self.world > 1:
            t = mine.to(self.device)
            dist.all_reduce(t, group=self.group)          # owned planes are disjoint, the rest is zero
            mine = t.cpu()
        return mine

    def frame_recorder(self, slots=3, share=None, barrier=None):
        """A record.SlabFrameRecorder for this decomposition's global grid (collective; see there).  Without
        torch.distributed, share and barrier default to the simulator's allgather and barrier."""
        from .record import SlabFrameRecorder
        if self._allgather is not None:
            share = share or (lambda b: self._allgather(b)[0])
            barrier = barrier or self._barrier
        return SlabFrameRecorder(self._shape[2:], self.rank, self.world, slots, self.device, self.group, share, barrier)

    def monitor(self, capacity=64):
        """A monitor.SlabStepMonitor of this decomposition: each rank reduces its owned planes after a step, and the
        ranks' plane partials combine into the whole grid's divergence statistics (every rank records alike)."""
        from .monitor import SlabStepMonitor
        return SlabStepMonitor(self, capacity)

    def field(self, key):
        """The tfl_grid of this rank's local slab of `key` ('density' or 'pDiv'; owned and ghost planes, local plane 0
        at global plane self.zoff)."""
        st = _lib.State()
        self.ctx.check(self.ctx.lib.tfl_slab_sim_layout(self.h, C.byref(st), None))
        return getattr(st, {"density": "density", "pDiv": "p"}[key])

    def record(self, rec, writer, key="density"):
        """Collective: capture this rank's planes of `key` into `rec` (a frame_recorder) on the current stream, behind
        the steps enqueued so far; rank 0 writes the oldest frame to `writer` first if its ring is full."""
        self.ctx.use_current_stream()
        return rec.record_grid(self.field(key), self.zoff, writer)

    def close(self):
        """Free the slab and the communicator.  Without torch.distributed (world > 1) this is collective: every rank
        finishes its queued work and passes `barrier` before any rank frees its inbox (a neighbour's push may still be
        landing in it), and passes it again before going on (e.g. to map the inboxes of a new simulator)."""
        if self.h:
            collective = self._barrier is not None and self.world > 1
            if collective:
                torch.cuda.synchronize(self.device)
                self._barrier()
            self.ctx.lib.tfl_slab_sim_destroy(self.ctx.h, self.h)
            self.h = None
            if collective:
                self._barrier()
        self.ctx.lib.tfl_comm_destroy(self.ctx.h)


class SlabStepGraph:
    """One NativeSlabSimulator.step captured as a CUDA graph (tfl_slab_graph_*): `launch()` replays it, one launch per
    step.  Needs a non-default current stream, one earlier sim.step() and, with more than one rank, peer-memory
    exchanges (NCCL is not captured).  Every rank makes its own; the ranks still take the same steps, in any mix of
    sim.step() and launch()."""

    def __init__(self, sim):
        self.sim, self.ctx = sim, sim.ctx           # keep the captured simulator (and its model) alive
        self.ctx.use_current_stream()
        h = C.c_void_p()
        self.ctx.check(self.ctx.lib.tfl_slab_graph_create(self.ctx.h, sim.h, C.byref(sim.mc),
                                                          sim.model.h if sim.model is not None else None, C.byref(h)))
        self.h = h

    def launch(self):
        self.ctx.use_current_stream()
        self.ctx.check(self.ctx.lib.tfl_slab_graph_launch(self.ctx.h, self.h))

    def close(self):
        if self.h:
            self.ctx.lib.tfl_slab_graph_destroy(self.ctx.h, self.h)
            self.h = None


def run_lockstep(sims):
    """Advance several SlabSimulators of ONE decomposition that live in the same process (tests:
    the whole multi-rank logic on a single GPU).  Halo requests are served by direct copies between
    neighbouring slabs, sum requests by adding the partial sums."""
    sims = sorted(sims, key=lambda q: q.dec.rank)
    gens = [q.phases() for q in sims]
    while True:
        reqs = []
        for g in gens:
            try:
                reqs.append(next(g))
            except StopIteration:
                reqs.append(None)
        if all(r is None for r in reqs):
            return
        assert all(r is not None for r in reqs) and len({r[0] for r in reqs}) == 1
        if reqs[0][0] == "sum":
            total = sum(r[1].clone() for r in reqs)
            for r in reqs:
                r[1].copy_(total)
        else:
            width = reqs[0][2]
            for lo, hi in zip(range(len(sims) - 1), range(1, len(sims))):
                a, b = sims[lo].dec, sims[hi].dec
                for ta, tb in zip(reqs[lo][1], reqs[hi][1]):
                    tb[:, :, b.own_lo - width:b.own_lo].copy_(ta[:, :, a.own_hi - width:a.own_hi])
                    ta[:, :, a.own_hi:a.own_hi + width].copy_(tb[:, :, b.own_lo:b.own_lo + width])
