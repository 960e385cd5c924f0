"""Slab-decomposed MLS-MPM rollout: one big scene over several GPUs (BASELINE.json configs[4], SURVEY.md 8e).

The reference runs one `MPM_Simulator_WARP` on "cuda:0" (mpm_solver_warp.py:47); it has no multi-GPU path. This module
shards ONE simulation along x: rank r owns grid planes [x0, x1) and the particles whose stencil base plane
(`int(x/dx - 0.5)`, mpm_utils.py:344) lies there. One substep is

    scatter   every rank scatters its particles into its own full-size {mv, m} grid (g2p of the previous substep fused in)
    exchange  the partial sums of the planes two neighbours both touch are added: total = own + neighbour (on the CUDA backend
              inside the grid sweep of `finish`, straight from the neighbour's memory)
    finish    every rank normalises / applies the BCs on its owned + overlap planes

and every `migrate_every` substeps particles whose base plane left [x0, x1) move to the neighbour (packed records over
send/recv, live prefix of the bound arrays shrinks / grows). `slack` is how many planes a particle may drift outside
its slab between two migrations; the overlap with the right neighbour is [x1 - slack, x1 + 2 + slack) because a particle
touches planes base .. base+2. After the exchange both neighbours hold the COMPLETE sums on the overlap, so the grid
update there is computed redundantly and no second exchange is needed.

Two exchange mechanisms behind one orchestration:
  * `FusedSlabBackend` (the product): the exchange runs ON THE DEVICE. Every handle exposes an exchange buffer
    [flags][grid 0][grid 1]; neighbours map each other's buffers (cudaIpc over NVLink between processes). The grid sweep
    raises this rank's `scatter_done`, waits for the neighbours' (bounded) and adds their partial sums on the shared planes
    straight from their memory; the two grids alternate by substep parity so that a rank's own partial sums can stay in
    place while the neighbour reads them (no second handshake, no staging copy). scatter -> sweep chain in one CUDA graph
    per chunk of substeps; the host only steps in at migration check points (an 8-byte all-reduce; NCCL send/recv of packed
    records when particles really have to move).
  * host exchange (`planes` / `planes_add`): what the CPU test double (tests/slab_backends.py) implements, so that the
    orchestration — overlap ranges, migration, id bookkeeping — is exercised without a GPU, in one process and over gloo.

Restrictions (checked): slabs must be at least 2 + 2*slack planes wide; a particle that drifts more than `slack` planes
out of its slab between two migrations raises (migrate more often); boundary conditions that carry per-particle masks
(impulses, velocity translation / rotation) are not migrated and are rejected.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib


# ------------------------------------------------------------------------------------------- backends
class FusedSlabBackend:
    """One rank's solver (a `MPM_Simulator_WARP` shim created with `capacity` particles of which a prefix is live) on the
    default path, overlap exchange on the device."""
    device_exchange = True

    #: per-particle fields that migrate with a particle: (C-ABI field name, width)
    FIELDS = [("X", 3), ("V", 3), ("F", 9), ("F_TRIAL", 9), ("C", 9), ("STRESS", 9), ("R", 9), ("COV", 6), ("INIT_COV", 6),
              ("VOL", 1), ("MASS", 1), ("DENSITY", 1), ("MATERIAL", 1), ("SELECTION", 1), ("E", 1), ("NU", 1), ("MU", 1),
              ("LAM", 1), ("BULK", 1), ("YIELD", 1)]

    def __init__(self, solver, n_active: int):
        self.solver = solver
        self.lib = _lib.require_device()
        self.n_grid = int(solver.mpm_model.n_grid)
        self.capacity = int(solver.n_particles)
        self.device = solver._device
        self.inv_dx = float(solver.mpm_model.inv_dx)
        if solver._masks:
            raise ValueError("slab-decomposed runs do not migrate per-particle BC masks (impulses, velocity modifiers)")
        base, nbytes = C.c_void_p(), C.c_size_t()
        _lib.check(self.lib.pixie_mpm_exchange_buffer(solver._handle, C.byref(base), C.byref(nbytes)))
        self.xbuf, self.xbuf_bytes = base.value, nbytes.value
        self._opened = []
        self._active = -1
        self.set_active(n_active)

    # -- exchange set-up
    def export_handle(self) -> bytes:
        """64-byte cudaIpc handle of the exchange buffer, for a neighbour in another process."""
        buf = C.create_string_buffer(64)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pixie_ipc_export(C.c_void_p(self.xbuf), buf))
        return buf.raw

    def open_handle(self, handle: bytes) -> int:
        p = C.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pixie_ipc_open(C.create_string_buffer(handle, 64), C.byref(p)))
        self._opened.append(p.value)
        return p.value

    def attach(self, x0: int, x1: int, slack: int, left: Optional[int], right: Optional[int]):
        """Neighbours' exchange buffers as device pointers valid in this process (None at the domain ends)."""
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pixie_mpm_slab_attach(self.solver._handle, int(x0), int(x1), int(slack),
                                                       C.c_void_p(left) if left else None, C.c_void_p(right) if right else None))

    def close(self):
        for p in self._opened:
            self.lib.pixie_ipc_close(C.c_void_p(p))
        self._opened = []

    # -- substep phases (each only enqueues kernels)
    def _phase(self, ph: int, dt: float):
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pixie_mpm_slab_phase(self.solver._handle, ph, float(dt), _lib.stream(self.device)))

    def scatter(self, dt: float):
        self._phase(0, dt)

    def halo(self, dt: float):
        self._phase(1, dt)          # no launch on this backend: the overlap sums are formed inside the grid sweep (finish)

    def finish(self, dt: float, lo: int, hi: int):
        self._phase(2, dt)

    def step(self, n: int, dt: float):
        """`n` whole substeps (scatter and sweep chained on the device, replayed from a CUDA graph)."""
        self.solver.p2g2p_n(n, dt)

    def error(self) -> int:
        flag = C.c_int(0)
        with torch.cuda.device(self.device):
            torch.cuda.current_stream(self.device).synchronize()
            _lib.check(self.lib.pixie_mpm_slab_error(self.solver._handle, C.byref(flag)))
        return flag.value

    def excursion(self) -> torch.Tensor:
        """int32[1] on the device: planes by which the farthest particle's stencil base lies outside this slab (one small kernel
        over the sorted positions; no write-back of the particle fields, no host sync)."""
        out = torch.zeros(1, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self.lib.pixie_mpm_slab_excursion(self.solver._handle, _lib.ptr(out), _lib.stream(self.device)))
        return out

    # -- particles
    @property
    def active(self) -> int:
        return self._active

    def set_active(self, n: int, force: bool = False):
        """Live prefix length. `force` (after a migration, even when the count is unchanged: the SET changed) lets the
        library reset what depends on the particle set (graphs, leftovers on the shared planes)."""
        if n > self.capacity:
            raise RuntimeError(f"slab holds {n} particles but was created with capacity {self.capacity}")
        if n != self._active or force:
            _lib.check(self.lib.pixie_mpm_set_active_count(self.solver._handle, int(n)))
            self._active = int(n)

    def get(self, name: str) -> torch.Tensor:
        t = self.solver._t[name]           # syncs: results of the substeps so far are written back first
        return t.view(self.capacity, t.numel() // self.capacity)[: self._active]

    def records_at(self, index: torch.Tensor) -> torch.Tensor:
        """Records of the particles `index` only (migration touches a few thousand of them, not the whole slab);
        [len(index), W] float32, integer fields bit-cast, not converted."""
        cols = []
        for name, w in self.FIELDS:
            t = self.get(name)[index]
            cols.append(t.view(torch.float32) if t.dtype == torch.int32 else t)
        return torch.cat(cols, dim=1)

    def compact_and_append(self, keep_index: torch.Tensor, arrivals: Optional[torch.Tensor]):
        """Live prefix <- particles `keep_index` (in order) followed by the `arrivals` records."""
        n_keep = int(keep_index.shape[0])
        n_new = 0 if arrivals is None else int(arrivals.shape[0])
        old = self._active
        if n_keep + n_new > self.capacity:
            raise RuntimeError(f"slab would hold {n_keep + n_new} particles but was created with capacity {self.capacity}")
        c = 0
        for name, w in self.FIELDS:
            full = self.solver._t[name].view(self.capacity, w)
            if n_keep != old:
                full[:n_keep] = full[:old][keep_index]
            if n_new:
                src = arrivals[:, c:c + w].contiguous()
                full[n_keep:n_keep + n_new] = src.view(torch.int32) if full.dtype == torch.int32 else src
            c += w
        self.set_active(n_keep + n_new, force=(n_keep != old or n_new > 0))


# ------------------------------------------------------------------------------------------- orchestration
def slab_bounds(n_grid: int, world: int, rank: int) -> Tuple[int, int]:
    return rank * n_grid // world, (rank + 1) * n_grid // world


def balanced_slab_bounds(base_planes, n_grid: int, world: int, min_width: int) -> List[Tuple[int, int]]:
    """Plane ranges with (nearly) equal particle counts: cuts at the quantiles of the particles' stencil base planes, every
    slab at least `min_width` planes wide (>= 2 + 2*slack). Equal-width slabs leave most ranks idle when the particles
    occupy a fraction of the domain (BASELINE config 5: a 0.4-wide block in a 256^3 grid = 3 of 8 slabs)."""
    base = np.sort(np.asarray(base_planes).astype(np.int64))
    if world * min_width > n_grid:
        raise ValueError("domain too small for this many slabs")
    cuts = [0]
    for r in range(1, world):
        q = int(base[min(len(base) - 1, (len(base) * r) // world)]) if len(base) else r * n_grid // world
        lo = cuts[-1] + min_width                      # keep the previous slab wide enough ...
        hi = n_grid - (world - r) * min_width          # ... and room for the remaining ones
        cuts.append(max(lo, min(q, hi)))
    cuts.append(n_grid)
    return [(cuts[r], cuts[r + 1]) for r in range(world)]


class SlabRank:
    """Phase methods of one rank; a driver (`DistSlabDriver` or `LocalSlabCluster`) sequences them."""

    def __init__(self, backend, rank: int, world: int, slack: int = 1, migrate_every: int = 8, ids: Optional[torch.Tensor] = None,
                 bounds: Optional[Tuple[int, int]] = None, lazy_trigger: Optional[int] = None):
        """`lazy_trigger`: None migrates at every check point (every `migrate_every` substeps). An integer t (1 <= t <= slack)
        migrates only once some particle of SOME rank has its stencil base t or more planes outside its slab; until then
        the slack planes absorb the movers and a check point costs one small kernel + a 4-byte all-reduce."""
        self.b, self.rank, self.world, self.slack, self.migrate_every = backend, rank, world, slack, migrate_every
        if lazy_trigger is not None and not (1 <= lazy_trigger <= max(1, slack)):
            raise ValueError("lazy_trigger must lie in [1, slack]")
        self.lazy_trigger = lazy_trigger
        self.checks = self.migrations = 0
        n = backend.n_grid
        self.x0, self.x1 = bounds if bounds is not None else slab_bounds(n, world, rank)
        if world > 1 and (self.x1 - self.x0) < 2 + 2 * slack:
            raise ValueError(f"slab [{self.x0}, {self.x1}) is narrower than 2 + 2*slack = {2 + 2 * slack} planes")
        self.has_left, self.has_right = rank > 0, rank < world - 1
        # planes shared with the neighbours
        self.left_ov = (max(0, self.x0 - slack), min(n, self.x0 + 2 + slack)) if self.has_left else None
        self.right_ov = (max(0, self.x1 - slack), min(n, self.x1 + 2 + slack)) if self.has_right else None
        # planes this rank updates: owned + what its (drifted) particles can touch
        self.lo = max(0, self.x0 - slack) if self.has_left else 0
        self.hi = min(n, self.x1 + 2 + slack) if self.has_right else n
        self.steps = 0
        #: global particle ids travel with the records so results can be compared with a single-domain run
        self.ids = ids if ids is not None else torch.arange(backend.active, dtype=torch.int64)

    # -- substep phases
    def scatter(self, dt: float):
        self.b.scatter(dt)

    def snapshot(self):
        """Partial sums on the overlaps, taken BEFORE anything is added."""
        left = self.b.planes(*self.left_ov) if self.has_left else None
        right = self.b.planes(*self.right_ov) if self.has_right else None
        return left, right

    def snapshot_views(self):
        """Same without copies, for drivers that finish sending before they accumulate (backends without views copy)."""
        pv = getattr(self.b, "planes_view", self.b.planes)
        left = pv(*self.left_ov) if self.has_left else None
        right = pv(*self.right_ov) if self.has_right else None
        return left, right

    def accumulate(self, from_left, from_right):
        if self.has_left:
            self.b.planes_add(self.left_ov[0], self.left_ov[1], from_left)
        if self.has_right:
            self.b.planes_add(self.right_ov[0], self.right_ov[1], from_right)

    def finish(self, dt: float):
        self.b.finish(dt, self.lo, self.hi)
        self.steps += 1

    def due_for_migration(self) -> bool:
        return self.world > 1 and self.steps % self.migrate_every == 0

    def excursion(self) -> torch.Tensor:
        """int32[1]: planes by which this rank's farthest particle base lies outside [x0, x1) towards a neighbour."""
        if hasattr(self.b, "excursion"):
            return self.b.excursion()
        x = self.b.get("X")[:, 0]
        base = (x.to(torch.float32) * torch.tensor(self.b.inv_dx, dtype=torch.float32, device=x.device) - 0.5).to(torch.int32)
        e = torch.zeros(1, dtype=torch.int32, device=x.device)
        if base.numel():
            if self.has_left:
                e = torch.maximum(e, (self.x0 - base.min()).to(torch.int32).view(1))
            if self.has_right:
                e = torch.maximum(e, (base.max() - (self.x1 - 1)).to(torch.int32).view(1))
        return e

    def migration_needed(self, global_excursion: int) -> bool:
        """Decision at a check point from the max excursion over ALL ranks (every rank must take the same branch)."""
        self.checks += 1
        if global_excursion > self.slack:
            raise RuntimeError(f"slab rank {self.rank}: a particle drifted more than slack={self.slack} planes out of its slab "
                               f"between two migration checks; lower migrate_every or raise slack")
        need = self.lazy_trigger is None or global_excursion >= self.lazy_trigger
        self.migrations += int(need)
        return need

    # -- migration phases
    def check_device_error(self):
        """Device-exchange backends: raises if a neighbour never showed up or a particle out-ran the slack planes."""
        err = self.b.error() if hasattr(self.b, "error") else 0
        if err == 1:
            raise RuntimeError(f"slab rank {self.rank}: a neighbour did not reach the exchange (flag timeout)")
        if err == 2:
            raise RuntimeError(f"slab rank {self.rank}: a particle drifted more than slack={self.slack} planes out of "
                               f"[{self.x0}, {self.x1}) between two migrations; lower migrate_every or raise slack")

    def migrate_collect(self):
        """Splits the live particles into stay / to_left / to_right. Returns (stay_index, (rec, ids) left, (rec, ids) right)."""
        self.check_device_error()
        x = self.b.get("X")[:, 0]
        # base plane exactly as the kernels compute it: float32 product, truncation toward zero (mpm_utils.py:344-346)
        base = (x.to(torch.float32) * torch.tensor(self.b.inv_dx, dtype=torch.float32, device=x.device) - 0.5).to(torch.int32)
        # a particle further out than the slack planes has scattered into planes nobody exchanged or swept: its slab's
        # result is already wrong, so fail loudly instead of migrating it
        lo_ok = self.x0 - self.slack if self.has_left else -(1 << 30)
        hi_ok = self.x1 + self.slack if self.has_right else (1 << 30)
        if base.numel() and (int(base.min()) < lo_ok or int(base.max()) >= hi_ok):
            raise RuntimeError(f"slab rank {self.rank}: a particle drifted more than slack={self.slack} planes out of "
                               f"[{self.x0}, {self.x1}) between two migrations; lower migrate_every or raise slack")
        go_left = (base < self.x0) if self.has_left else torch.zeros_like(base, dtype=torch.bool)
        go_right = (base >= self.x1) if self.has_right else torch.zeros_like(base, dtype=torch.bool)
        stay_idx = torch.nonzero(~(go_left | go_right)).flatten()
        il, ir = torch.nonzero(go_left).flatten(), torch.nonzero(go_right).flatten()
        ids = self.ids.to(x.device)
        if hasattr(self.b, "records_at"):
            pack = lambda i: (self.b.records_at(i), ids[i])
        else:
            rec = self.b.records()
            pack = lambda i: (rec[i], ids[i])
        # a mover more than one slab away cannot be handed to a direct neighbour
        return stay_idx, pack(il), pack(ir)

    def migrate_apply(self, stay_idx, from_left, from_right):
        ids = self.ids.to(stay_idx.device)
        arrivals = [p for p in (from_left, from_right) if p is not None and p[0].shape[0] > 0]
        new_rec = torch.cat([p[0] for p in arrivals], dim=0) if arrivals else None
        if hasattr(self.b, "compact_and_append"):
            self.b.compact_and_append(stay_idx, new_rec)
        else:
            rec = self.b.records()[stay_idx]
            self.b.set_records(rec if new_rec is None else torch.cat([rec, new_rec.to(rec.dtype)], dim=0))
        self.ids = torch.cat([ids[stay_idx]] + [p[1].to(ids.device) for p in arrivals], dim=0)


class LocalSlabCluster:
    """All slabs in ONE process (tests, single-GPU emulation): the exchanges are plain hand-overs."""

    def __init__(self, ranks: Sequence[SlabRank]):
        self.ranks = list(ranks)
        self.device_exchange = bool(getattr(self.ranks[0].b, "device_exchange", False))
        if self.device_exchange:
            # same process: the neighbours' exchange buffers are plain device pointers; the phases of all slabs are
            # enqueued on one stream in order, so every flag a kernel waits for has already been raised
            for i, r in enumerate(self.ranks):
                r.b.attach(r.x0, r.x1, r.slack, self.ranks[i - 1].b.xbuf if r.has_left else None,
                           self.ranks[i + 1].b.xbuf if r.has_right else None)

    def substep(self, dt: float):
        R = self.ranks
        for r in R:
            r.scatter(dt)
        if self.device_exchange:
            for r in R:
                r.b.halo(dt)
        else:
            snaps = [r.snapshot() for r in R]
            for i, r in enumerate(R):
                from_left = snaps[i - 1][1] if r.has_left else None       # left neighbour's right overlap = my left overlap
                from_right = snaps[i + 1][0] if r.has_right else None
                r.accumulate(from_left, from_right)
        for r in R:
            r.finish(dt)
        if R[0].due_for_migration() and self._migration_needed():
            self._migrate()

    def _migrate(self):
        R = self.ranks
        parts = [r.migrate_collect() for r in R]
        for i, r in enumerate(R):
            from_left = parts[i - 1][2] if r.has_left else None
            from_right = parts[i + 1][1] if r.has_right else None
            r.migrate_apply(parts[i][0], from_left, from_right)

    def _migration_needed(self) -> bool:
        R = self.ranks
        if R[0].lazy_trigger is None:
            return all([r.migration_needed(0) for r in R])
        e = max(int(r.excursion().item()) for r in R)
        return all([r.migration_needed(e) for r in R])

    def gather(self, name: str) -> torch.Tensor:
        """Field `name` of every particle, ordered by global id."""
        vals = torch.cat([r.b.get(name).detach().cpu().to(torch.float64) for r in self.ranks], dim=0)
        ids = torch.cat([r.ids.cpu() for r in self.ranks], dim=0)
        out = torch.empty_like(vals)
        out[ids] = vals
        return out


class DistSlabDriver:
    """One rank of a `torch.distributed` job (NCCL on GPUs, gloo in the CPU tests)."""

    def __init__(self, rank_obj: SlabRank, group=None):
        import torch.distributed as dist
        self.r, self.dist, self.group = rank_obj, dist, group
        self._recv = None
        self.device_exchange = bool(getattr(rank_obj.b, "device_exchange", False))
        if self.device_exchange:
            # every rank publishes the cudaIpc handle of its exchange buffer; each maps its two neighbours' buffers
            r = rank_obj
            handles = [None] * r.world
            dist.all_gather_object(handles, r.b.export_handle(), group=group)
            left = r.b.open_handle(handles[r.rank - 1]) if r.has_left else None
            right = r.b.open_handle(handles[r.rank + 1]) if r.has_right else None
            r.b.attach(r.x0, r.x1, r.slack, left, right)
            dist.barrier(group=group)                    # nobody starts stepping before every buffer is mapped

    def run(self, n_substeps: int, dt: float):
        """`n_substeps` substeps; between migrations the device runs on its own (graph replays), the host only steps in every
        `migrate_every` substeps. Falls back to substep() for host-exchange backends."""
        r = self.r
        if not self.device_exchange:
            for _ in range(n_substeps):
                self.substep(dt)
            return
        done = 0
        while done < n_substeps:
            chunk = min(n_substeps - done, r.migrate_every - (r.steps % r.migrate_every))
            r.b.step(chunk, dt)
            r.steps += chunk
            done += chunk
            if r.due_for_migration():
                self._migrate()

    def _migration_needed(self) -> bool:
        """One 8-byte all-reduce per check point: [max excursion, max device error flag]. Every rank sees the same values,
        so a failure (a neighbour that never showed up, a particle beyond the slack planes) raises on ALL ranks instead of
        leaving the others waiting in a collective."""
        r = self.r
        e = r.excursion() if r.lazy_trigger is not None else None
        err = r.b.error() if hasattr(r.b, "error") else 0
        dev = e.device if e is not None else torch.device(getattr(r.b, "device", "cpu"))
        both = torch.zeros(2, dtype=torch.int32, device=dev)
        if e is not None:
            both[0:1] = e
        both[1] = err
        self.dist.all_reduce(both, op=self.dist.ReduceOp.MAX, group=self.group)
        ge, gerr = (int(v) for v in both.tolist())
        if gerr == 1:
            raise RuntimeError(f"slab rank {r.rank}: a rank waited for a neighbour that did not reach the exchange (flag timeout)")
        if gerr == 2:
            raise RuntimeError(f"slab rank {r.rank}: a particle drifted more than slack={r.slack} planes out of its slab between "
                               f"two migrations; lower migrate_every or raise slack")
        return r.migration_needed(ge)

    def _migrate(self):
        r = self.r
        if not self._migration_needed():
            return
        stay, go_left, go_right = r.migrate_collect()
        from_left, from_right = self._swap_var(go_left if r.has_left else None, go_right if r.has_right else None)
        r.migrate_apply(stay, from_left, from_right)

    def _swap(self, to_left: Optional[torch.Tensor], to_right: Optional[torch.Tensor], like_left=None, like_right=None, reuse=False):
        """Symmetric neighbour exchange. `like_*` give the shape of what is received (default: what is sent); with
        `reuse` they ARE the receive buffers."""
        dist, r = self.dist, self.r
        ops, from_left, from_right = [], None, None
        if r.has_left:
            from_left = like_left if reuse else torch.empty_like(to_left if like_left is None else like_left)
            ops += [dist.P2POp(dist.isend, to_left.contiguous(), r.rank - 1, self.group), dist.P2POp(dist.irecv, from_left, r.rank - 1, self.group)]
        if r.has_right:
            from_right = like_right if reuse else torch.empty_like(to_right if like_right is None else like_right)
            ops += [dist.P2POp(dist.isend, to_right.contiguous(), r.rank + 1, self.group), dist.P2POp(dist.irecv, from_right, r.rank + 1, self.group)]
        if ops:
            for w in dist.batch_isend_irecv(ops):
                w.wait()
        return from_left, from_right

    def _swap_var(self, to_left, to_right):
        """Variable-length record exchange: counts first, then the records, then the global ids."""
        r = self.r
        ref = to_left if to_left is not None else to_right
        dev, width, dtype = ref[0].device, ref[0].shape[1], ref[0].dtype
        cnt = lambda p: torch.tensor([p[0].shape[0]], dtype=torch.int64, device=dev)
        nl, nr = self._swap(cnt(to_left) if r.has_left else None, cnt(to_right) if r.has_right else None)
        nl = int(nl.item()) if r.has_left else 0
        nr = int(nr.item()) if r.has_right else 0
        rec_l, rec_r = self._swap(to_left[0] if r.has_left else None, to_right[0] if r.has_right else None,
                                  torch.empty((nl, width), dtype=dtype, device=dev), torch.empty((nr, width), dtype=dtype, device=dev))
        ids_l, ids_r = self._swap(to_left[1].to(dev) if r.has_left else None, to_right[1].to(dev) if r.has_right else None,
                                  torch.empty((nl,), dtype=torch.int64, device=dev), torch.empty((nr,), dtype=torch.int64, device=dev))
        return ((rec_l, ids_l) if r.has_left else None), ((rec_r, ids_r) if r.has_right else None)

    def substep(self, dt: float):
        r = self.r
        if self.device_exchange:
            r.b.scatter(dt); r.b.halo(dt); r.finish(dt)
            if r.due_for_migration():
                self._migrate()
            return
        r.scatter(dt)
        left, right = r.snapshot_views()
        if self._recv is None:          # overlap-plane receive buffers, allocated once
            self._recv = (torch.empty_like(left) if r.has_left else None, torch.empty_like(right) if r.has_right else None)
        from_left, from_right = self._swap(left, right, self._recv[0], self._recv[1], reuse=True)
        r.accumulate(from_left, from_right)
        r.finish(dt)
        if r.due_for_migration():
            self._migrate()

    def gather(self, name: str, dst: int = 0) -> Optional[torch.Tensor]:
        """Field `name` of every particle ordered by global id, on rank `dst` (None elsewhere)."""
        dist, r = self.dist, self.r
        vals = r.b.get(name).detach().cpu().to(torch.float64).contiguous()
        ids = r.ids.cpu()
        objs = [None] * r.world if r.rank == dst else None
        dist.gather_object((vals, ids), objs, dst=dst, group=self.group)
        if r.rank != dst:
            return None
        v = torch.cat([o[0] for o in objs], dim=0)
        i = torch.cat([o[1] for o in objs], dim=0)
        out = torch.empty_like(v)
        out[i] = v
        return out
