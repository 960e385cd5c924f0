"""MPM boundary conditions held to the reference at the comparisons that flip a node or a particle.

tests/golden/mpm_bc_edges_golden.npz was written by tests/golden/make_mpm_bc_edges_golden.py, which registers BCs
through the reference's own `MPM_Simulator_WARP` methods and runs its collide / `modify` closures and selection
kernels on the float32 stand-in of _fake_warp.py. Its cases sit on collider planes, cuboid faces, bounding-box
padding planes, time and reset windows, cylinder caps and walls and nested release boxes, and one float32 step either
side; the cases marked `disc` were found by search so that a fused multiply-add decides them differently.

  * CPU: oracle/mpm_ref.c (fp32) reproduces every node class and mask exactly; the product's host-side parameter
    arithmetic reproduces the stored float32 parameters bit for bit; the fused restatement of the predicates
    (tests/golden/mpm_bc_predicates.py) disagrees with the fixture on every `disc` case, so those cases bite.
  * GPU: a lattice of particles moving at the sentinel velocity u (C = 0, F_trial = I, jelly, g = 0, no damping) makes
    every node of the case's box massive with velocity u to a few float32 steps; one substep at the case's clock, then each node's
    class must equal the fixture's. The moving cuboid re-imports the particle state before every substep, so each
    substep starts from the sentinel state while the device clock and cuboid point advance.
"""
import json
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, HERE)

import mpm_bc_predicates as P  # noqa: E402

GOLD = np.load(os.path.join(HERE, "golden", "mpm_bc_edges_golden.npz"))
META = json.loads(bytes(GOLD["meta"]).decode())
CASES = META["grid"]
IDS = [c["name"] for c in CASES]
SEL = META["selection"]
f32 = np.float32


def _gold(i):
    return GOLD[f"grid/{i}/cls"]


def _expected(i):
    """What the oracle and the device must give: the stand-in's classes, except on the open-point case, where `modify`'s
    window is compared in double (see test_open_point_window_is_recorded)."""
    key = f"grid/{i}/cls_f64_window"
    return GOLD[key] if key in GOLD.files else _gold(i)


# ------------------------------------------------------------------------------------------ fixture sanity
def test_fixture_covers_the_edges():
    names = " ".join(IDS)
    for tag in ("plane_sticky", "plane_slip", "plane_separate", "plane_cut", "tilted_", "cuboid_face", "cuboid_fused",
                "cuboid_zero", "cuboid_huge", "bbox_lo", "bbox_hi", "window_collider", "window_cuboid", "window_bbox",
                "reset_dt0.0001_end0.0006_k21", "moving_cuboid"):
        assert tag in names, tag
    for i, c in enumerate(CASES):                       # every class the device must tell apart occurs somewhere
        assert (_gold(i) != P.UNKNOWN).all(), c["name"]
    seen = set(np.concatenate([_gold(i).ravel() for i in range(len(CASES))]).tolist())
    assert {P.PASS, P.ZERO, P.CUBOID, P.CUT} <= seen and len(seen - {P.PASS, P.ZERO, P.CUBOID, P.CUT}) >= 3, seen
    assert sum(c["disc"] for c in CASES) >= 30
    mv = _gold(IDS.index("moving_cuboid_n100"))
    sets = {tuple(np.flatnonzero(s == P.CUBOID)) for s in mv}
    assert len(sets) >= 10, "the moving cuboid should cross nodes many times"
    assert GOLD["sel/cyl_disc"].any() and GOLD["sel/rel_masks"].sum() > 0


# ------------------------------------------------------------------------------------------ restatement (CPU)
@pytest.mark.parametrize("i", range(len(CASES)), ids=IDS)
def test_unfused_restatement_matches_fixture(i):
    c = CASES[i]
    assert (P.restate_case(c, c["records"], fused=False) == _gold(i)).all()


@pytest.mark.parametrize("i", [i for i, c in enumerate(CASES) if c["disc"]], ids=[c["name"] for c in CASES if c["disc"]])
def test_fused_restatement_disagrees(i):
    """A device that contracts the BC predicates into FMAs decides these cases differently."""
    c = CASES[i]
    assert (P.restate_case(c, c["records"], fused=True) != _gold(i)).any()


def test_open_point_window_is_recorded():
    """Open modelling point: `modify` compares the Python-float clock with the float32 start time. The stand-in (NumPy 2)
    does it in float32; the device and the oracle do it in double. The fixture keeps both outcomes of one case whose start
    time rounds up from a substep's clock; if either convention changes, this test or the oracle / device tests fail."""
    opened = [i for i, c in enumerate(CASES) if c.get("open_point")]
    assert len(opened) == 1
    i = opened[0]
    c = CASES[i]
    assert (P.restate_case(c, c["records"], fused=False, window="f64") == _expected(i)).all()
    assert (_expected(i) != _gold(i)).any()
    for j, d in enumerate(CASES):
        if j != i:
            assert (_expected(j) == _gold(j)).all()


def test_fused_rotation_restatement_disagrees():
    """theta's sign on the half-plane dot(x - point, h2) = 0: the stand-in's velocities show it, and a fused dot product
    flips it on every fused-sensitive particle."""
    x, disc, pos = GOLD["sel/rot_x"], GOLD["sel/rot_disc"], GOLD["sel/rot_theta_pos"]
    point = SEL["rot"]["point"]
    assert (P.rotation_theta_positive(x, point, GOLD["sel/rot_h2"], fused=False) == pos).all()
    assert disc.sum() >= 10 and (~disc).sum() >= 4
    assert (P.rotation_theta_positive(x[disc], point, GOLD["sel/rot_h2"], fused=True) != pos[disc]).all()
    a1 = GOLD["sel/rot_v"].astype(np.float64) @ GOLD["sel/rot_h1"].astype(np.float64)
    assert ((a1 < 0) == pos).all()


def _rot_check(v, label):
    """Velocities of the rotation modifier against the stand-in's, and theta's sign on every half-plane particle."""
    want = GOLD["sel/rot_v"].astype(np.float64)
    v = np.asarray(v, np.float64).reshape(want.shape)
    err = np.abs(v - want).max() / np.abs(want).max()
    a1 = v @ GOLD["sel/rot_h1"].astype(np.float64)
    wrong = (a1 < 0) != GOLD["sel/rot_theta_pos"]
    assert not wrong.any(), f"{label}: theta's sign differs on {int(wrong.sum())} particles ({int(wrong[GOLD['sel/rot_disc']].sum())} fused-sensitive)"
    assert err < 1e-5, f"{label}: rel {err:.2e}"


def test_oracle_rotation_modifier():
    from oracle import mpm_ref as R
    x, c = GOLD["sel/rot_x"], SEL["rot"]
    o = R.MpmRef(len(x), 16, 2.0, "f32")
    o.set("X", x)
    o.set("SELECTION", np.ones(len(x)))            # not simulated: the modified velocity is what the substep leaves
    o.add_bc(R.BC_VROT, point=c["point"], normal=list(GOLD["sel/rot_normal"]), h1=list(GOLD["sel/rot_h1"]),
             h2=list(GOLD["sel/rot_h2"]), hhr=c["half_height_and_radius"], rotation_scale=c["rotation_scale"],
             translation_scale=c["translation_scale"], start_time=c["start_time"], end_time=c["end_time"],
             mask=np.ones(len(x), np.int32))
    o.time = 0.5
    o.step(1, 1e-4)
    _rot_check(o.get("V"), "oracle")


def test_fused_cylinder_restatement_disagrees():
    c = SEL["cyl"]
    x, disc = GOLD["sel/cyl_x"], GOLD["sel/cyl_disc"]
    hh, r = c["half_height_and_radius"]
    fus = P.select_cylinder(x[disc], c["point"], GOLD["sel/cyl_normal"], hh, r, fused=True)
    assert (fus != GOLD["sel/cyl_mask"][disc]).all()


# ------------------------------------------------------------------------------------------ C oracle (CPU)
def _oracle_case(c):
    from oracle import mpm_ref as R
    n, lim = c["n_grid"], c["grid_lim"]
    o = R.MpmRef(1, n, lim, "f32")
    o.set_params(g=(0.0, 0.0, 0.0), grid_v_damping_scale=1.0)
    o.set("X", np.full((1, 3), lim / 2))
    for r in c["records"]:
        o.add_bc(r["kind"], point=r["point"], normal=r["normal"], size=r["size"], velocity=r["velocity"],
                 start_time=r["start_time"], end_time=r["end_time"], surface_type=r["surface_type"], reset=r["reset"])
    o.time = P.clock(c["dt"], c["k"])
    nodes = P.box_nodes(c["lo"], c["hi"])
    sentinel = np.tile(np.array(list(c["u"]) + [1.0]), n ** 3)       # {m v, m} with m = 1 at every node
    out = []
    for _ in range(c["steps"]):
        o.planes_add(0, n, sentinel)
        o.finish(c["dt"], 0, n)
        vo = o.grid()[2]
        out.append(P.classify(vo[nodes[:, 0], nodes[:, 1], nodes[:, 2]], c["u"], velocity=c["vel"]))
    return np.stack(out)


@pytest.mark.parametrize("i", range(len(CASES)), ids=IDS)
def test_oracle_grid_decisions(i):
    assert (_oracle_case(CASES[i]) == _expected(i)).all()


def test_oracle_selections():
    from oracle import mpm_ref as R
    x = GOLD["sel/box_x"]
    o = R.MpmRef(len(x), 16, 2.0, "f32")
    o.set("X", x)
    for j, (p, s) in enumerate(SEL["box_params"]):
        assert (o.select_box(p, s) == GOLD["sel/box_masks"][j]).all()
    x = GOLD["sel/mat_x"]
    o = R.MpmRef(len(x), 16, 2.0, "f32")
    o.set("X", x)
    for b in SEL["mat_boxes"]:
        o.apply_additional_params(b["point"], b["size"], b["E"], b["nu"], b["density"], b["material"])
    assert (o.get("MATERIAL").astype(np.int32) == GOLD["sel/mat_material"]).all()
    x, c = GOLD["sel/cyl_x"], SEL["cyl"]
    o = R.MpmRef(len(x), 16, 2.0, "f32")
    o.set("X", x)
    mask = o.select_cylinder(c["point"], GOLD["sel/cyl_normal"], *c["half_height_and_radius"])
    assert (mask == GOLD["sel/cyl_mask"]).all()
    x = GOLD["sel/rel_x"]
    o = R.MpmRef(len(x), 16, 2.0, "f32")
    o.set("X", x)
    point = [1, 1, SEL["rel"]["end_position"]]
    for j, size in enumerate(GOLD["sel/rel_size"]):
        assert (o.select_box(point, size.astype(np.float64)) == GOLD["sel/rel_masks"][j]).all(), j


# ------------------------------------------------------------------------------------------ host-side parameters (CPU)
def _bits(a):
    return np.asarray(a, f32).view(np.uint32)


def test_collider_normal_bits():
    from pixie_b200.mpm_solver_warp import collider_normal
    got = np.stack([collider_normal(list(v)) for v in _normals_in()])
    assert (_bits(got) == _bits(GOLD["param/collider_normal"])).all()


def _normals_in():
    # the generator passes some normals as Python ints; as floats they give the same float32 bits (their squares and sums
    # are exact), so every normal is passed as float here
    vals = GOLD["param/normals_in"]
    out = []
    for v in vals:
        out.append([float(t) for t in v])
    return out


def test_rotation_axes_bits():
    from pixie_b200.mpm_solver_warp import rotation_axes
    for j, v in enumerate(_normals_in()):
        n, h1, h2 = rotation_axes(v)
        assert (_bits(n) == _bits(GOLD["param/rot_normal"][j])).all(), (j, v)
        assert (_bits(h1) == _bits(GOLD["param/rot_h1"][j])).all(), (j, v)
        assert (_bits(h2) == _bits(GOLD["param/rot_h2"][j])).all(), (j, v)


def test_release_layers_bits():
    from pixie_b200.mpm_solver_warp import release_layers
    for j, (a, b, e) in enumerate(GOLD["param/release_in"]):
        layers = release_layers([0, 1, 0], float(a), float(b), float(e))
        assert len(layers) == 50
        size = np.asarray([f32(s) for _, sz, _ in layers for s in sz], f32).reshape(50, 3)
        ends = np.asarray([f32(t) for _, _, t in layers], f32)
        assert (_bits(size) == _bits(GOLD["param/release_size"][j])).all(), j
        assert (_bits(ends) == _bits(GOLD["param/release_end_time"][j])).all(), j


def test_impulse_end_time_bits():
    from pixie_b200.mpm_solver_warp import impulse_end_time
    got = np.asarray([f32(impulse_end_time(float(s), float(d), int(k))) for s, d, k in GOLD["param/impulse_in"]], f32)
    assert (_bits(got) == _bits(GOLD["param/impulse_end_time"])).all()


# ------------------------------------------------------------------------------------------ device (GPU)
# m u / m on the device: where dx is inexact the lattice's weights differ from particle to particle, and the scatter sums
# them in its own order. The fp32 oracle stays within 3 float32 steps of u on these lattices; on an H100 the device's
# largest distance over all cases was 10 steps (each case prints its own, `-s`). u and the cut value are matched to 16
# steps: the classes stay apart by O(1) (u, 0.3 u, 0 and the cuboid velocity), and zeros and the cuboid velocity are
# matched exactly.
ULPS = 16


def _ulps_from(v, u):
    a = np.asarray(v, f32).view(np.int32).astype(np.int64)
    return np.abs(a - np.broadcast_to(np.asarray(u, f32), np.shape(v)).view(np.int32).astype(np.int64))

def _lattice(c):
    """Particle grid coordinates j + 0.75 (stencil base j) for every base whose stencil reaches the case's box."""
    n = c["n_grid"]
    dx = c["grid_lim"] / n
    axes = [(np.arange(max(lo - 1, 0), min(hi, n - 2)) + 0.75) * dx for lo, hi in zip(c["lo"], c["hi"])]
    return np.stack(np.meshgrid(*axes, indexing="ij"), -1).reshape(-1, 3).astype(f32)


class _SentinelState:
    def __init__(self, c):
        import torch
        self.x = torch.from_numpy(_lattice(c)).cuda()
        m = self.x.shape[0]
        self.v = torch.tensor(c["u"], dtype=torch.float32, device="cuda").repeat(m, 1).contiguous()
        self.C = torch.zeros(m, 3, 3, dtype=torch.float32, device="cuda")
        self.Ft = torch.eye(3, dtype=torch.float32, device="cuda").repeat(m, 1, 1).contiguous()

    def load(self, s):
        s.import_particle_x_from_torch(self.x)
        s.import_particle_v_from_torch(self.v)
        s.import_particle_C_from_torch(self.C)
        s.mpm_state.particle_F_trial = self.Ft.clone()


def _device_case(c):
    import torch
    from mpm_backends import device_grid_v
    from pixie_b200.mpm_solver_warp import MPM_Simulator_WARP
    n, lim = c["n_grid"], c["grid_lim"]
    st = _SentinelState(c)
    m = st.x.shape[0]
    s = MPM_Simulator_WARP(m, n_grid=n, grid_lim=lim, device="cuda:0")
    vol = torch.full((m,), (lim / n) ** 3 / 8, dtype=torch.float32, device="cuda")
    s.load_initial_data_from_torch(st.x, vol, n_grid=n, grid_lim=lim, device="cuda:0")
    s.set_parameters_dict(dict(material="jelly", E=1e4, nu=0.3, density=1000.0, g=[0.0, 0.0, 0.0], grid_v_damping_scale=1.0,
                               rpic_damping=0.0), device="cuda:0")
    s.finalize_mu_lam(device="cuda:0")
    for method, kw in c["bcs"]:
        getattr(s, method)(**kw)
    s.time = P.clock(c["dt"], c["k"])
    nodes = P.box_nodes(c["lo"], c["hi"])
    out = []
    for _ in range(c["steps"]):
        st.load(s)
        s.p2g2p(0, c["dt"], device="cuda:0")
        g = device_grid_v(s)[nodes[:, 0], nodes[:, 1], nodes[:, 2]]
        cls = P.classify(g, c["u"], velocity=c["vel"], ulps=ULPS)
        passed = cls == P.PASS
        if passed.any():
            print(f"{c['name']}: largest distance of a passed node from u: {int(_ulps_from(g[passed], c['u']).max())} float32 steps")
        out.append(cls)
    return np.stack(out)


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(len(CASES)), ids=IDS)
def test_device_grid_decisions(built_lib, cuda_dev, i):
    c = CASES[i]
    got, want = _device_case(c), _expected(i)
    bad = np.argwhere(got != want)
    nodes = P.box_nodes(c["lo"], c["hi"])
    assert len(bad) == 0, (f"{len(bad)} node decisions differ; first (substep, node, device, reference): " +
                           str([(int(k), nodes[j].tolist(), int(got[k, j]), int(want[k, j])) for k, j in bad[:6]]))


def _device_solver(x):
    import torch
    from pixie_b200.mpm_solver_warp import MPM_Simulator_WARP
    s = MPM_Simulator_WARP(len(x), n_grid=16, grid_lim=2.0, device="cuda:0")
    s.load_initial_data_from_torch(torch.from_numpy(x.copy()).cuda(), torch.ones(len(x), device="cuda"), n_grid=16,
                                   grid_lim=2.0, device="cuda:0")
    return s


@pytest.mark.gpu
def test_device_box_selections(built_lib, cuda_dev):
    s = _device_solver(GOLD["sel/box_x"])
    for p, sz in SEL["box_params"]:
        s.add_impulse_on_particles(force=[1.0, 0.0, 0.0], dt=1e-4, point=list(p), size=list(sz), num_dt=3, device="cuda:0")
        s.enforce_particle_velocity_translation(point=list(p), size=list(sz), velocity=[0.0, 0.0, 0.0], start_time=0.0,
                                                end_time=1.0, device="cuda:0")
    masks = [m.cpu().numpy() for m in s._masks]
    nb = len(SEL["box_params"])
    want = GOLD["sel/box_masks"]           # the reference lists the impulses first, then the modifiers
    for j in range(nb):
        assert (masks[2 * j] == want[j]).all() and (masks[2 * j + 1] == want[nb + j]).all(), j


@pytest.mark.gpu
def test_device_additional_params(built_lib, cuda_dev):
    s = _device_solver(GOLD["sel/mat_x"])
    s.set_parameters_dict(dict(material="jelly", E=3e5, nu=0.2, density=1000.0,
                               additional_material_params=[dict(b) for b in SEL["mat_boxes"]]), device="cuda:0")
    assert (s.mpm_state.particle_material.numpy().astype(np.int32) == GOLD["sel/mat_material"]).all()


@pytest.mark.gpu
def test_device_cylinder_selection(built_lib, cuda_dev):
    c = SEL["cyl"]
    s = _device_solver(GOLD["sel/cyl_x"])
    s.enforce_particle_velocity_rotation(point=c["point"], normal=c["normal"], half_height_and_radius=c["half_height_and_radius"],
                                         rotation_scale=1.0, translation_scale=0.0, start_time=0.0, end_time=1.0, device="cuda:0")
    got, want = s._masks[-1].cpu().numpy(), GOLD["sel/cyl_mask"]
    assert (got == want).all(), f"{int((got != want).sum())} particles differ, {int((got != want)[GOLD['sel/cyl_disc']].sum())} of them fused-sensitive"


@pytest.mark.gpu
def test_device_release_masks(built_lib, cuda_dev):
    s = _device_solver(GOLD["sel/rel_x"])
    s.release_particles_sequentially(**SEL["rel"])
    got = np.stack([m.cpu().numpy() for m in s._masks])
    assert (got == GOLD["sel/rel_masks"]).all()


@pytest.mark.gpu
def test_device_rotation_modifier(built_lib, cuda_dev):
    import torch
    x, c = GOLD["sel/rot_x"], SEL["rot"]
    s = _device_solver(x)
    s.enforce_particle_velocity_rotation(**c, device="cuda:0")
    assert (s._masks[-1].cpu().numpy() == 1).all()
    s.mpm_state.particle_selection = torch.ones(len(x), dtype=torch.int32, device="cuda")   # keeps the modified velocity
    s.time = 0.5
    s.p2g2p(0, 1e-4, device="cuda:0")
    _rot_check(s.mpm_state.particle_v.numpy(), "device")


# ------------------------------------------------------------------------------------------ moving cuboid, two slabs
@pytest.mark.gpu
def test_device_moving_cuboid_two_slabs(built_lib, cuda_dev):
    """The moving cuboid with the grid sweep split between two slabs on one device ([0, 50) and [50, 100) of the n_grid 100
    grid; the cuboid's nodes straddle plane 50). The set of nodes a cuboid sets to its velocity depends only on its point,
    its size and the predicate, not on the particle state, so the particles run freely here and each substep's set of
    nodes at exactly the cuboid velocity, read from the slab that owns the plane, must equal the fixture's."""
    import ctypes as C
    import torch
    from mpm_backends import device_grid_v
    from pixie_b200 import _lib
    from pixie_b200.mpm_slab import FusedSlabBackend, LocalSlabCluster, SlabRank
    from pixie_b200.mpm_solver_warp import MPM_Simulator_WARP
    i = IDS.index("moving_cuboid_n100")
    c = CASES[i]
    n, lim = c["n_grid"], c["grid_lim"]
    x = _lattice(c)
    N = len(x)
    base = (x[:, 0] * np.float32(n / lim) - np.float32(0.5)).astype(np.int32)
    bounds = [(0, 50), (50, 100)]
    lib = _lib.require_device()
    ranks = []
    for r, (lo, hi) in enumerate(bounds):
        idx = np.flatnonzero((base >= lo) & (base < hi))
        assert len(idx) > 100
        s = MPM_Simulator_WARP(N, n_grid=n, grid_lim=lim, device="cuda:0")
        m = len(idx)
        fields = dict(X=x[idx], V=np.tile(np.asarray(c["u"], f32), (m, 1)), F=np.tile(np.eye(3, dtype=f32), (m, 1, 1)),
                      F_TRIAL=np.tile(np.eye(3, dtype=f32), (m, 1, 1)), VOL=np.full(m, (lim / n) ** 3 / 8, f32),
                      DENSITY=np.full(m, 1000.0, f32), E=np.full(m, 1e4, f32), NU=np.full(m, 0.3, f32))
        for fid, arr in fields.items():
            s._t[fid].view(N, -1)[:m] = torch.from_numpy(arr.reshape(m, -1)).cuda()
        s._t["MATERIAL"].view(N, -1)[:m] = 0
        s._t["SELECTION"].view(N, -1)[:m] = 0
        s.mpm_model.gravitational_accelaration = (0.0, 0.0, 0.0)
        s.mpm_model.grid_v_damping_scale = 1.0
        s._push_params()
        _lib.check(lib.pixie_mpm_compute_mass(s._handle, s._stream()))
        _lib.check(lib.pixie_mpm_compute_mu_lam(s._handle, s._stream()))
        for method, kw in c["bcs"]:
            getattr(s, method)(**kw)
        ranks.append(SlabRank(FusedSlabBackend(s, m), r, 2, slack=1, migrate_every=2,
                              ids=torch.from_numpy(idx.astype(np.int64)), bounds=(lo, hi)))
    cl = LocalSlabCluster(ranks)
    nodes = P.box_nodes(c["lo"], c["hi"])
    want = _gold(i) == P.CUBOID
    vel = np.asarray(c["vel"], f32)
    for k in range(c["steps"]):
        cl.substep(c["dt"])
        torch.cuda.synchronize()
        got = np.zeros(len(nodes), bool)
        for rk in ranks:
            g = device_grid_v(rk.b.solver)[nodes[:, 0], nodes[:, 1], nodes[:, 2]]
            own = (nodes[:, 0] >= rk.x0) & (nodes[:, 0] < rk.x1)
            got |= own & (g == vel).all(1)
        assert (got == want[k]).all(), (f"substep {k}: nodes differ " +
                                         str([(nodes[j].tolist(), bool(got[j])) for j in np.flatnonzero(got != want[k])[:6]]))
    for rk in ranks:
        rk.check_device_error()
    assert want.any(1).sum() > 40 and (nodes[want.any(0), 0] < 50).any() and (nodes[want.any(0), 0] >= 50).any()


# ------------------------------------------------------------------------------------------ half-cell positions
HALF_NG = 19        # k = 1, 4 and ng - 3 = 16 are powers of two: there the fused base cell shifts (see below)


def _half_cell_positions(ng=HALF_NG):
    """float32 x with x * ng rounding to exactly k + 0.5 for k = 0, interior k and ng - 3. For k >= 1 the exact product lies
    just below k + 0.5, so a fused x * inv_dx - 0.5 gives a value below k, and truncates to base k - 1 (fx = 1.5), where the
    rounded product gives base k (fx = 0.5); both give the same weights. (The fused value can only land below k where the
    float32 spacing halves below k, i.e. where k is a power of two; elsewhere it rounds back to k.)"""
    out = {}
    for k in (0, 1, 4, ng - 3):
        x0 = f32((k + 0.5) / ng)
        got = []
        for j in range(-40, 41):
            x = x0
            for _ in range(abs(j)):
                x = np.nextafter(x, f32(np.inf) if j > 0 else f32(-np.inf))
            if f32(x * f32(ng)) == f32(k + 0.5) and (k == 0 or int(P.fma32(x, ng, -0.5)) == k - 1):
                got.append(f32(x))
        out[k] = np.asarray(got, f32)
    return out


def test_half_cell_positions_shift_the_fused_base_cell():
    pos = _half_cell_positions()
    for k, xs in pos.items():
        assert len(xs) >= 1, k
        for x in xs:
            assert int(f32(f32(x * f32(HALF_NG)) - f32(0.5))) == k            # the reference's rounded product: base k
            assert int(P.fma32(x, HALF_NG, -0.5)) == (k - 1 if k else 0)     # fused: base k - 1 (0 truncates toward 0)


def _half_cell_scene():
    import test_gpu_mpm_transfer as T
    sc = T.scene(1007, HALF_NG, "block", seed=17)
    rng = np.random.default_rng(17)
    pos = _half_cell_positions()
    choices = np.concatenate(list(pos.values()))
    pick = rng.random(sc["x"].shape) < 0.4
    sc["x"] = np.where(pick, rng.choice(choices, size=sc["x"].shape), sc["x"]).astype(f32)
    return sc


def _half_cell_compare(grid_v, particle, o64, o32, sc, label):
    """Against the fp32 oracle (the reference's arithmetic: base k, fx = 0.5), with the bound scales S of
    test_gpu_mpm_transfer.py and twice its constants (both sides round). The fp64 oracle is not the yardstick here: its
    exact product lies below k + 0.5, so it takes base k - 1 with fx just under 1.5 and reaches node k - 1 with a weight of
    order 2^-48, which float32 arithmetic never does (and the transfer bounds do not cover). Nodes the fp32 oracle leaves
    massless must stay massless on the device: velocity exactly 0."""
    import test_gpu_mpm_transfer as T
    n = sc["x"].shape[0]
    B = T.bounds(sc, o64, HALF_NG)
    m32 = o32.grid()[0].reshape(-1)
    v32 = o32.grid()[2].reshape(-1, 3)
    t = B["touched"] & (m32 > 0)
    ghost = B["touched"] & (m32 == 0)
    worst = {"grid_v": (np.abs(grid_v[t] - v32[t]) / (T.EPS * B["S_v"][t])).max()}
    bad = np.flatnonzero(ghost & (grid_v != 0).any(1))
    assert len(bad) == 0, (f"{label}: {len(bad)} of {int(ghost.sum())} nodes the float32 weights do not reach have a velocity, "
                           f"largest {np.abs(grid_v[bad]).max():.3g}; first nodes " +
                           str([np.unravel_index(j, (HALF_NG,) * 3) for j in bad[:4]]) + f" fp64 masses {o64.grid()[0].reshape(-1)[bad[:4]]}")
    for f, got in particle.items():
        got = np.asarray(got, np.float64).reshape(n, -1)
        worst[f] = (np.abs(got - o32.get(f).reshape(n, -1)) / (T.EPS * np.maximum(B[f].reshape(n, -1), 1e-30)))[B["judged"]].max()
    print(f"{label}: max err / (2^-23 S) against the fp32 oracle: " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))
    assert B["judged"].mean() > 0.9
    assert worst["grid_v"] <= 2 * T.K_GRID and max(worst[f] for f in particle) <= 2 * T.K_PART, worst


@pytest.mark.gpu
def test_device_half_cell_positions_match_the_reference_arithmetic(built_lib, cuda_dev):
    """Particles at x * inv_dx = k + 0.5 (k = 0, 1, 4, ng - 3) on some axes, one substep. A base cell computed from the
    unrounded product (k - 1, fx just under 1.5) gave node k - 1 a mass of ~1e-15 and velocities up to 1e5; the device
    must take the reference's base k and fx = 0.5, and leave that node massless."""
    import torch
    import test_gpu_mpm_transfer as T
    from mpm_backends import device_grid_v
    sc = _half_cell_scene()
    s = T.device(sc, HALF_NG, cuda_dev)
    o64, o32 = T.oracle(sc, HALF_NG, "f64"), T.oracle(sc, HALF_NG, "f32")
    s.p2g2p(0, T.DT)
    o64.step(1, T.DT); o32.step(1, T.DT)
    torch.cuda.synchronize()
    names = {"X": "particle_x", "V": "particle_v", "C": "particle_C", "F_TRIAL": "particle_F_trial"}
    _half_cell_compare(device_grid_v(s).reshape(-1, 3).astype(np.float64),
                       {f: getattr(s.mpm_state, k).numpy() for f, k in names.items()}, o64, o32, sc, "device")
