"""Particle-grid transfers of the MPM substep (p2g scatter, grid update, g2p gather) against the fp64 oracle at dense cells,
grid faces, ragged warps, partial selections and mixed materials, for every warp-aggregation width PIXIE_MPM_AGG.

One substep at a time: the device grid velocities (read through pixie_mpm_grid_ptrs) at every node a particle's stencil
touches, and the particles' x, v, C and F_trial after the gather, against `MpmRef(..., "f64")` run on the same
fp32-representable inputs. Bounds are err <= k * 2^-23 * S, with S the fp64 sum of the absolute contributions:
    node momentum:  sum_p |w| m (|v| + |C dpos|) + dt vol (|tau| + S_tau) |grad w|   (S_tau bounds the stress's own rounding)
    node velocity:  (S_mv + |v_node| sum_p |w| m) / |m_node| + dt |g|
                    (below a base cell of 0 the truncating base-cell rule gives weights of both signs, whose node masses
                    can nearly cancel)
    particle:       the gather of |v_node| + S_v over the stencil, with the weights of each output.
The multi-substep case runs fast particles through box growth, the re-sort at substep 100 and graph-replay boundaries, and
is judged like test_gpu_mpm.py::test_drift_vs_fp64_oracle: drift against fp64 next to the fp32 oracle's own drift.
"""
import itertools

import numpy as np
import pytest
import torch

from oracle import mpm_ref as R

EPS = 2.0 ** -23
DT = 1e-4
G = (0.0, 0.0, -9.8)
K_GRID, K_PART = 8.0, 8.0          # measured maxima of err / (2^-23 S) are printed and listed in the commit message


def scene(n, ng, layout, seed, selection=False):
    """Particles of one layout on an ng^3 grid over [0, 1)^3, every material id mixed within each warp."""
    rng = np.random.default_rng(seed)
    dx = 1.0 / ng
    if layout == "clump":                   # every particle in one base cell: whole warps form one run
        x = (np.array([7, 6, 5]) + 0.5 + rng.uniform(0.02, 0.98, (n, 3))) * dx
    elif layout == "faces":                 # stencils across every grid face: base < 0 and base >= ng - 2
        lo = rng.uniform(-1.45, 1.5, (n, 3)) * dx
        hi = 1.0 + rng.uniform(-2.5, 0.45, (n, 3)) * dx
        x = np.where(rng.random((n, 3)) < 0.5, lo, hi)
    else:                                   # `layout` particles per cell over a 4 x 4 x 4 block of cells
        x = (6.5 + rng.uniform(0, 4, (n, 3))) * dx
    x = x.astype(np.float32)
    F = (np.eye(3) + 0.05 * rng.standard_normal((n, 3, 3))).astype(np.float32)
    return dict(x=x, v=rng.standard_normal((n, 3)).astype(np.float32), C=(5 * rng.standard_normal((n, 3, 3))).astype(np.float32),
                F_trial=F, vol=(rng.uniform(0.5, 1.5, n) * dx ** 3 / 8).astype(np.float32),
                density=rng.uniform(500, 2000, n).astype(np.float32), E=(10 ** rng.uniform(4, 5.5, n)).astype(np.float32),
                nu=rng.uniform(0.1, 0.4, n).astype(np.float32), material=rng.integers(0, 7, n).astype(np.int32),
                selection=((rng.random(n) < 0.3) if selection else np.zeros(n, bool)).astype(np.int32),
                ys=(10 ** rng.uniform(2, 4, n)).astype(np.float32), bulk=(10 ** rng.uniform(4, 5, n)).astype(np.float32))


def _params():
    return dict(g=G, grid_v_damping_scale=1.1, rpic_damping=0.0, alpha=float(np.float32(R.friction_alpha(30.0))), hardening=1.0,
                xi=0.25, plastic_viscosity=8.0, softening=0.5)


def oracle(sc, ng, precision):
    n = sc["x"].shape[0]
    o = R.MpmRef(n, ng, 1.0, precision)
    for k, f in (("x", "X"), ("v", "V"), ("C", "C"), ("F_trial", "F_TRIAL"), ("vol", "VOL"), ("density", "DENSITY"),
                 ("E", "E"), ("nu", "NU"), ("material", "MATERIAL"), ("selection", "SELECTION"), ("ys", "YIELD"),
                 ("bulk", "BULK")):
        o.set(f, sc[k])
    o.compute_mass(); o.compute_mu_lam()
    o.set_params(**_params())
    return o


def device(sc, ng, dev):
    from pixie_b200.mpm_solver_warp import MPM_Simulator_WARP
    n = sc["x"].shape[0]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)     # noqa: E731
    s = MPM_Simulator_WARP(n)
    s.load_initial_data_from_torch(t(sc["x"]), t(sc["vol"]), None, n_grid=ng, grid_lim=1.0)
    p = _params()
    s.set_parameters_dict({"g": list(p["g"]), "grid_v_damping_scale": 1.1, "rpic_damping": 0.0, "friction_angle": 30.0,
                           "hardening": 1, "xi": p["xi"], "plastic_viscosity": p["plastic_viscosity"], "softening": p["softening"]})
    s.mpm_model.E, s.mpm_model.nu = t(sc["E"]), t(sc["nu"])
    s.mpm_model.yield_stress, s.mpm_model.bulk = t(sc["ys"]), t(sc["bulk"])
    s.mpm_state.particle_material = t(sc["material"])
    s.mpm_state.particle_selection = t(sc["selection"])
    s.reset_densities_and_update_masses(t(sc["density"]))
    s.finalize_mu_lam()
    s.import_particle_v_from_torch(t(sc["v"]))
    s.import_particle_C_from_torch(t(sc["C"]))
    s.mpm_state.particle_F_trial = t(sc["F_trial"])
    return s


def _stencil(x, ng):
    """Per particle and stencil offset: node index (-1 outside the grid), weight, grad weight, dpos (fp64, mpm_ref.c)."""
    g = x.astype(np.float64) * ng
    b = np.trunc(g - 0.5).astype(np.int64)
    fx = g - b
    w = np.stack([0.5 * (1.5 - fx) ** 2, 0.75 - (fx - 1.0) ** 2, 0.5 * (fx - 0.5) ** 2], -1)         # [n, 3 axes, 3]
    dw = np.stack([fx - 1.5, -2.0 * (fx - 1.0), fx - 0.5], -1)
    out = []
    for i, j, k in itertools.product(range(3), repeat=3):
        idx = b + np.array([i, j, k])
        ok = ((idx >= 0) & (idx < ng)).all(1)
        node = np.where(ok, (idx[:, 0] * ng + idx[:, 1]) * ng + idx[:, 2], -1)
        W = w[:, 0, i] * w[:, 1, j] * w[:, 2, k]
        dW = np.stack([dw[:, 0, i] * w[:, 1, j] * w[:, 2, k], w[:, 0, i] * dw[:, 1, j] * w[:, 2, k],
                       w[:, 0, i] * w[:, 1, j] * dw[:, 2, k]], 1) * ng
        dpos = (np.array([i, j, k]) - fx) / ng
        out.append((node, W, dW, dpos))
    return out


def bounds(sc, o64, ng):
    """Bound scales of the node velocities and of the particle outputs (fp64, from the inputs and the fp64 stresses)."""
    n = sc["x"].shape[0]
    act = sc["selection"] == 0
    m = (sc["density"].astype(np.float64) * sc["vol"])
    vol = sc["vol"].astype(np.float64)
    tau = o64.get("STRESS").reshape(n, 3, 3)
    E, nu = sc["E"].astype(np.float64), sc["nu"].astype(np.float64)
    mu, lam = E / (2 * (1 + nu)), E * nu / ((1 + nu) * (1 - 2 * nu))
    nf = np.sqrt((sc["F_trial"].astype(np.float64) ** 2).sum((1, 2)))
    s_tau = (2 * mu + 3 * lam + sc["bulk"]) * nf * (nf + np.sqrt(3))
    v, C = np.abs(sc["v"].astype(np.float64)), np.abs(sc["C"].astype(np.float64))
    nodes = ng ** 3
    S_mv, M = np.zeros((nodes, 3)), np.zeros(nodes)
    st = _stencil(sc["x"], ng)
    # (|W|: below base 0 the truncating base-cell rule puts fx outside [0.5, 1.5), where weights go negative)
    for node, W, dW, dpos in st:
        W = np.abs(W)
        ok = (node >= 0) & act
        contrib = (W * m)[:, None] * (v + np.einsum("nab,nb->na", C, np.abs(dpos))) + \
            DT * vol[:, None] * (np.einsum("nab,nb->na", np.abs(tau), np.abs(dW)) + s_tau[:, None] * np.abs(dW).sum(1, keepdims=True))
        np.add.at(S_mv, node[ok], contrib[ok])
        np.add.at(M, node[ok], (W * m)[ok])
    m64, _, vo = o64.grid()
    m64, vo = m64.reshape(nodes), vo.reshape(nodes, 3)
    # v = mv / m: the node mass carries a rounding of 2^-23 sum |w| m, which matters where weights of both signs nearly
    # cancel; nodes whose mass is within that reach of the 1e-15 cut-off (v = 0 below it) are not judged, nor are the
    # particles that gather from them
    settled = np.abs(m64 - 1e-15) > 64 * EPS * M
    touched = (M > 0) & settled
    with np.errstate(divide="ignore", invalid="ignore"):
        S_v = np.where(touched[:, None], (S_mv + np.abs(vo) * M[:, None]) / np.abs(m64)[:, None] + DT * np.abs(G), 0.0)
    # gather: v = sum w v_g, C = 4 inv_dx sum w v_g dpos^T, F_trial = (I + dt sum v_g grad w^T) F
    Sv_p, SC_p, SG_p = np.zeros((n, 3)), np.zeros((n, 3, 3)), np.zeros((n, 3, 3))
    judged = np.ones(n, bool)
    for node, W, dW, dpos in st:
        W = np.abs(W)
        ok = node >= 0
        judged &= ~(ok & (M[node] > 0) & ~settled[node])
        a = np.where(ok[:, None], np.abs(vo[node]) + S_v[node], 0.0)
        Sv_p += W[:, None] * a
        SC_p += 4 * ng * W[:, None, None] * a[:, :, None] * np.abs(dpos * ng)[:, None, :]
        SG_p += a[:, :, None] * np.abs(dW)[:, None, :]
    # F_trial = A F with F the return-mapped gradient: its rounding is of the order of ||F_trial||
    S_Ft = np.broadcast_to(nf[:, None, None] * (1 + DT * SG_p.sum(2, keepdims=True)), (n, 3, 3))
    return dict(touched=touched, judged=judged, S_v=S_v, X=np.abs(sc["x"]) + DT * Sv_p, V=Sv_p, C=SC_p, F_TRIAL=S_Ft)


def compare(s, o64, sc, ng, label):
    from mpm_backends import device_grid_v
    n = sc["x"].shape[0]
    B = bounds(sc, o64, ng)
    worst = {}
    vo = o64.grid()[2].reshape(-1, 3)
    gv = device_grid_v(s).reshape(-1, 3).astype(np.float64)
    t = B["touched"]
    assert np.isfinite(gv[t]).all()
    worst["grid_v"] = (np.abs(gv[t] - vo[t]) / (EPS * B["S_v"][t])).max()
    fields = {"X": "particle_x", "V": "particle_v", "C": "particle_C", "F_TRIAL": "particle_F_trial"}
    for f, name in fields.items():
        got = getattr(s.mpm_state, name).numpy().astype(np.float64).reshape(n, -1)
        ref = o64.get(f).reshape(n, -1)
        S = B[f].reshape(n, -1)
        assert np.isfinite(got).all(), f"{label}: {f} not finite"
        worst[f] = (np.abs(got - ref) / (EPS * np.maximum(S, 1e-30)))[B["judged"]].max()
    print(f"{label}: max err / (2^-23 S): " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()) +
          f"; {n - B['judged'].sum()} particles next to an unsettled node mass")
    assert B["judged"].mean() > 0.9
    assert worst["grid_v"] <= K_GRID, f"{label}: grid velocities {worst['grid_v']:.3g} > {K_GRID}"
    for f in fields:
        assert worst[f] <= K_PART, f"{label}: {f} {worst[f]:.3g} > {K_PART}"
    return worst


CASES = [(ppc, ppc * 64, "block", False) for ppc in (1, 8, 32, 64, 256)] + \
        [(0, n, "clump", False) for n in (1, 31, 33, 1007)] + [(0, 1007, "faces", False), (0, 1007, "faces", True),
                                                              (32, 2048, "block", True)]


def _run_case(monkeypatch, dev, agg, n, layout, selection, seed):
    monkeypatch.setenv("PIXIE_MPM_AGG", str(agg))          # read when the handle is created
    ng = 16
    sc = scene(n, ng, layout, seed, selection)
    s = device(sc, ng, dev)
    o = oracle(sc, ng, "f64")
    s.p2g2p(0, DT)
    o.step(1, DT)
    torch.cuda.synchronize()
    return compare(s, o, sc, ng, f"AGG={agg} n={n} {layout}{' selection' if selection else ''}")


@pytest.mark.gpu
@pytest.mark.parametrize("agg", [0, 1, 2, 3])
@pytest.mark.parametrize("ppc,n,layout,selection", CASES, ids=[f"{c[2]}{c[0] or ''}-n{c[1]}{'-sel' if c[3] else ''}" for c in CASES])
def test_one_substep_matches_fp64(built_lib, cuda_dev, monkeypatch, agg, ppc, n, layout, selection):
    _run_case(monkeypatch, cuda_dev, agg, n, layout, selection, seed=n + agg)


def test_bounds_hold_for_the_fp32_oracle():
    """The transfer bounds describe fp32 arithmetic: the fp32 oracle meets them against fp64 without a GPU."""
    ng = 16
    for n, layout, sel in ((2048, "block", True), (1007, "clump", False), (1007, "faces", True)):
        sc = scene(n, ng, layout, seed=n, selection=sel)
        o64, o32 = oracle(sc, ng, "f64"), oracle(sc, ng, "f32")
        o64.step(1, DT); o32.step(1, DT)
        B = bounds(sc, o64, ng)
        t = B["touched"]
        assert t.sum() > 8
        g32, g64 = o32.grid()[2].reshape(-1, 3), o64.grid()[2].reshape(-1, 3)
        worst = {"grid_v": (np.abs(g32[t] - g64[t]) / (EPS * B["S_v"][t])).max()}
        for f in ("X", "V", "C", "F_TRIAL"):
            worst[f] = (np.abs(o32.get(f) - o64.get(f)).reshape(n, -1) / (EPS * B[f].reshape(n, -1)))[B["judged"]].max()
        print(f"fp32 oracle n={n} {layout}: " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))
        assert worst["grid_v"] <= K_GRID and max(worst[f] for f in ("X", "V", "C", "F_TRIAL")) <= K_PART


@pytest.mark.gpu
def test_fast_particles_through_box_growth_and_resort(built_lib, cuda_dev):
    """20 m/s on a 64^3 grid over [0, 1)^3 crosses 0.128 cells per substep: the 2-node margin of the node box is gone after
    ~16 substeps, so the box must grow by atomics until the re-sort at substep 100; substep 150 lies past that re-sort and
    several graph replays."""
    ng, n = 64, 4000
    rng = np.random.default_rng(7)
    sc = scene(n, ng, "block", 7)
    sc["x"] = (np.array([0.2, 0.45, 0.45]) + rng.uniform(0, 0.1, (n, 3))).astype(np.float32)
    sc["v"] = (np.array([20.0, -3.0, 2.0]) + 0.1 * rng.standard_normal((n, 3))).astype(np.float32)
    sc["C"] = np.zeros((n, 3, 3), np.float32)
    sc["material"] = np.zeros(n, np.int32)
    s = device(sc, ng, cuda_dev)
    o64, o32 = oracle(sc, ng, "f64"), oracle(sc, ng, "f32")
    s.p2g2p(0, DT); s.p2g2p_n(149, DT)
    o64.step(150, DT); o32.step(150, DT)
    torch.cuda.synchronize()
    x = s.mpm_state.particle_x.numpy().astype(np.float64)
    assert (x[:, 0] - sc["x"][:, 0]).min() > 0.25                  # really travelled ~19 cells
    drift = np.abs(x - o64.get("X")).max()
    floor = np.abs(o32.get("X") - o64.get("X")).max()
    dv = np.abs(s.mpm_state.particle_v.numpy() - o64.get("V")).max()
    print(f"fast particles, 150 substeps: drift vs fp64 {drift:.3e}, fp32 oracle vs fp64 {floor:.3e}, |dv| {dv:.3e}")
    assert drift < 20 * floor + 1e-6
    assert dv < 1e-2
