"""Return maps, stresses and svd3 of the MPM substep against the fp64 oracle on adversarial deformation gradients.

One substep `p2g2p(0, dt)` starts with the launch that runs the return map and the stress of every particle on exactly the
bound `particle_F_trial` and writes `particle_F`, `particle_stress` and any change of `yield_stress` / `mu` / `lam`. The
fp64 build of oracle/mpm_ref.c (`MpmRef.stress_probe`, dt = 1e-4) computes the same quantities from the same
fp32-representable inputs.

Bounds have the form err <= k * 2^-23 * S per particle and output family, with
    S = (sum of |terms| of the output formula, in fp64) + (conditioning: max |change of the fp64 output| / 2^-23 over a few
        random perturbations of F_trial of relative size 2^-23, the backward error of an fp32 SVD).
The second term is what makes the bound hold on ill-conditioned inputs (near-equal or near-zero singular values, inverted F),
where any fp32 algorithm loses accuracy in proportion to the conditioning; it is computed with the branch decisions kept.
Particles whose branch decision (yield test, sand's dg <= 0 and tr > 0, damage's yield <= 0) lies within the rounding reach
of its boundary must match one of the two fp64 branch outcomes; all others must match the branch fp64 takes.
Where the fp64 stress itself is non-finite (Drucker-Prager on an un-returned inverted F, water with J <= 0) the device must
be non-finite in the same entries, and finite everywhere else.

`test_fp32_oracle_meets_the_same_bounds` holds the fp32 oracle (a different SVD: textbook Jacobi, exact square roots) to the
same bounds without a GPU: they describe fp32 arithmetic, not this kernel's algorithm.
"""
import numpy as np
import pytest
import torch

from oracle import mpm_ref as R

EPS = 2.0 ** -23
DT = 1e-4
MATERIALS = (0, 1, 2, 3, 4, 5, 6, 7, -1)
PARAMS = dict(alpha=float(np.float32(R.friction_alpha(30.0))), xi=0.25, softening=0.5, plastic_viscosity=8.0)   # fp32-exact
# k per output family: measured maxima of err / (2^-23 S) are in the module's printout and the commit message
K = {"F": 8.0, "stress": 16.0, "yield": 8.0, "R": 8.0}
K_MARGIN = 64.0           # rounding reach of a branch decision, in units of 2^-23 * (1 + its conditioning)
N_TRIALS = 3


def _rotations(rng, n):
    q, r = np.linalg.qr(rng.standard_normal((n, 3, 3)))
    q = q * np.sign(np.diagonal(r, axis1=1, axis2=2))[:, None, :]
    q[:, :, 2] *= np.linalg.det(q)[:, None]
    return q


def _dev_dirs(rng, n):
    d = rng.standard_normal((n, 3))
    d -= d.mean(1, keepdims=True)
    return d / np.linalg.norm(d, axis=1, keepdims=True)


def population(n, seed):
    """Adversarial F_trial families x every material id, with per-particle mu / lam / yield / bulk. Returns a dict of
    float32 / int32 arrays (the exact values both sides see) and the family label of each particle."""
    rng = np.random.default_rng(seed)
    fams = ["mild", "large", "equal3", "equal2", "near_equal", "cond", "near_singular", "rank_def", "inverted",
            "inverted_small", "clamp", "scale_small", "scale_large", "identity", "diag_unsorted", "zero_row",
            "yield_edge", "damage_edge", "damage", "sand_edge", "sand_tip"]
    fam = rng.integers(0, len(fams), n)
    E = 10 ** rng.uniform(3, 6, n)
    nu = rng.uniform(0.05, 0.45, n)
    mu = (E / (2 * (1 + nu))).astype(np.float32).astype(np.float64)
    lam = (E * nu / ((1 + nu) * (1 - 2 * nu))).astype(np.float32).astype(np.float64)
    mat = rng.choice(MATERIALS, n).astype(np.int32)
    ys = 2 * mu * 10 ** rng.uniform(-4, -0.5, n)
    r = rng.random(n)
    ys[(mat == 5) & (r < 0.05)] = 0.0                                     # damage path: yield <= 0 on entry
    ys[(mat == 5) & (r > 0.97)] = -1.0
    bulk = 10 ** rng.uniform(3, 6, n)
    sig = np.ones((n, 3))
    rot = np.ones(n, bool)
    u = lambda lo, hi: rng.uniform(lo, hi, n)                             # noqa: E731
    a, b, c = np.exp(u(-0.5, 0.5)), np.exp(u(-0.5, 0.5)), np.exp(u(-0.5, 0.5))
    sgn = rng.choice([-1.0, 1.0], n)
    kappa = 10 ** u(2, 4)
    choices = {
        "mild": 1 + 0.05 * rng.standard_normal((n, 3)),
        "large": np.exp(0.4 * rng.standard_normal((n, 3))),
        "equal3": np.stack([a, a, a], 1),
        "equal2": np.where((r < 0.5)[:, None], np.stack([a, a, b], 1), np.stack([a, b, b], 1)),
        "near_equal": a[:, None] * (1 + 10 ** u(-7, -3)[:, None] * rng.standard_normal((n, 3))),
        "cond": np.stack([np.ones(n), kappa ** -u(0, 1), 1 / kappa], 1) * a[:, None],
        "near_singular": np.stack([a, b, 10 ** u(-8, -4)], 1),
        "rank_def": np.where((r < 0.5)[:, None], np.stack([a, b, 0 * a], 1), np.stack([a, 0 * a, 0 * a], 1)),
        "inverted": np.stack([a, b, -u(0.05, 1.2)], 1),
        "inverted_small": np.stack([a, b, -(10 ** u(-4, -2))], 1),
        "clamp": np.stack([a, b, np.where(r < 0.5, 10 ** u(-3, -1.5), 0.01 * (1 + sgn * 10 ** u(-6, -2)))], 1),
        "scale_small": 1e-4 * (1 + 0.1 * rng.standard_normal((n, 3))),
        "scale_large": 1e3 * (1 + 0.1 * rng.standard_normal((n, 3))),
        "diag_unsorted": rng.permutation(np.stack([a, b * 0.5, c * 2.0], 1).T).T * rng.choice([-1.0, 1.0, 1.0, 1.0], (n, 3)),
        "yield_edge": np.exp(0.2 * rng.standard_normal((n, 3))),
        "damage_edge": np.exp(0.2 * rng.standard_normal((n, 3))),
        "damage": np.exp(0.2 * rng.standard_normal((n, 3))),
    }
    for i, name in enumerate(fams):
        if name in choices:
            sig[fam == i] = choices[name][fam == i]
    rot[np.isin(fam, [fams.index("identity"), fams.index("diag_unsorted")])] = False
    # sand: dg = hn + (3 lam + 2 mu) / (2 mu) tr alpha at 0 (edge), tr at 0 (tip)
    d, hn = _dev_dirs(rng, n), u(0.01, 0.3)
    coef = (3 * lam + 2 * mu) / (2 * mu)
    tr_edge = -hn / (coef * PARAMS["alpha"]) * (1 + sgn * 10 ** u(-7, -2))
    tr_tip = sgn * 10 ** u(-7, -3)
    for name, tr in (("sand_edge", tr_edge), ("sand_tip", tr_tip)):
        m = fam == fams.index(name)
        sig[m] = np.exp(hn[m, None] * d[m] + tr[m, None] / 3)
        mat[m] = 2
    F = np.einsum("nij,nj,nkj->nik", _rotations(rng, n), sig, _rotations(rng, n))
    F[~rot] = sig[~rot][:, :, None] * np.eye(3)[None]
    F[fam == fams.index("identity")] = np.eye(3)
    zr = fam == fams.index("zero_row")
    F[zr] = rng.standard_normal((zr.sum(), 3, 3))
    F[zr, rng.integers(0, 3)] = 0.0
    F = F.astype(np.float32)
    # yield stresses placed just either side of the yield surface of the rounded F (fp64)
    s64 = np.linalg.svd(F.astype(np.float64), compute_uv=False) * np.sign(np.linalg.det(F.astype(np.float64)))[:, None] ** np.array([0, 0, 1])
    e = np.log(np.maximum(s64, 0.01))
    h = np.linalg.norm(e - e.mean(1, keepdims=True), axis=1)
    near = 1 + sgn * 10 ** u(-7, -2)
    m = fam == fams.index("yield_edge")
    mat[m] = rng.choice([1, 3, 5], n)[m]
    ys[m] = np.where(mat[m] == 3, 2 * mu[m] * h[m] / np.sqrt(2.0 / 3.0), 2 * mu[m] * h[m]) * near[m]
    hp = h + 1e-6
    m = fam == fams.index("damage_edge")
    mat[m] = 5
    soft = PARAMS["softening"]
    ys[m] = (soft * h / (1 + soft * h / (2 * mu * hp)) * near)[m]
    m = fam == fams.index("damage")
    mat[m] = 5
    ys[m] = (soft * h * u(0.05, 0.9))[m]
    return dict(F=F, material=mat, mu=mu.astype(np.float32), lam=lam.astype(np.float32), ys=ys.astype(np.float32),
                bulk=bulk.astype(np.float32), family=np.array(fams)[fam])


def oracle_run(pop, precision, hardening, flip=0, F=None):
    n = pop["F"].shape[0]
    o = R.MpmRef(n, 16, 1.0, precision)
    o.set_params(hardening=float(hardening), **PARAMS)
    o.set("F_TRIAL", pop["F"] if F is None else F)
    o.set("MATERIAL", pop["material"]); o.set("MU", pop["mu"]); o.set("LAM", pop["lam"])
    o.set("YIELD", pop["ys"]); o.set("BULK", pop["bulk"])
    margins = o.stress_probe(flip)
    return dict(F=o.get("F").reshape(n, 9), stress=o.get("STRESS").reshape(n, 9), yield_=o.get("YIELD"), mu=o.get("MU"),
                lam=o.get("LAM"), margins=margins)


def _fro(A):
    return np.sqrt((A.reshape(A.shape[0], -1) ** 2).sum(1))


def _det_terms(F):
    F = F.reshape(-1, 3, 3)
    t = [F[:, 0, 0] * F[:, 1, 1] * F[:, 2, 2], F[:, 0, 1] * F[:, 1, 2] * F[:, 2, 0], F[:, 0, 2] * F[:, 1, 0] * F[:, 2, 1],
         F[:, 0, 2] * F[:, 1, 1] * F[:, 2, 0], F[:, 0, 0] * F[:, 1, 2] * F[:, 2, 1], F[:, 0, 1] * F[:, 1, 0] * F[:, 2, 2]]
    return np.abs(np.stack(t, 1)).sum(1)


def _term_sums(pop, ref, hardening):
    """Sum of |terms| of each output formula, per particle (fp64). The stress formulas count the rounding of their own
    inputs too: the singular values of F carry an absolute error of order 2^-23 ||F|| (so log sigma_k one of
    ||F|| / sigma_k), and J one of order 2^-23 times the sum of |terms| of the determinant."""
    n = pop["F"].shape[0]
    Ft = pop["F"].astype(np.float64)
    F = ref["F"].reshape(n, 3, 3)
    mat = pop["material"]
    mu, lam, bulk = np.abs(ref["mu"]), np.abs(ref["lam"]), np.abs(pop["bulk"].astype(np.float64))
    with np.errstate(all="ignore"):
        sv = np.linalg.svd(np.nan_to_num(F), compute_uv=False)
        J = np.linalg.det(F)
        nf = _fro(F)
        dJ = _det_terms(F)
        sc = np.maximum(sv, 0.01)
        e = np.abs(np.log(sc)) + nf[:, None] / sc                          # |log sigma| + its rounding reach
        l = np.abs(np.log(sv)) + nf[:, None] / sv
        s_fcr = 2 * mu * nf * (nf + np.sqrt(3)) + lam * (np.abs(J) + 1) * (np.abs(J) + 2 * dJ)
        s_stvk = nf * (2 * mu[:, None] * e + lam[:, None] * e.sum(1, keepdims=True)).sum(1)
        s_dp = nf * ((2 * mu[:, None] * l + lam[:, None] * l.sum(1, keepdims=True)) / sv * (1 + nf[:, None] / sv)).sum(1)
        aJ = np.abs(J)
        s_water = bulk * (aJ ** -0.1 + aJ) + bulk * (0.1 * aJ ** -1.1 + 1) * dJ
    S_stress = np.select([np.isin(mat, (0, 5)), np.isin(mat, (1, 3)), mat == 2, mat == 6], [s_fcr, s_stvk, s_dp, s_water], 0.0)
    # yield - softening |k h| (+ 2 mu xi dg): the plastic strain carries the rounding reach of the logs of F_trial
    st = np.linalg.svd(Ft, compute_uv=False)
    et = np.log(np.maximum(st, 0.01))
    strain = np.linalg.norm(et - et.mean(1, keepdims=True), axis=1) + (_fro(Ft)[:, None] / np.maximum(st, 0.01)).sum(1)
    mu_in, ys_in = np.abs(pop["mu"].astype(np.float64)), np.abs(pop["ys"].astype(np.float64))
    S_yield = ys_in + np.abs(ref["yield_"]) + (PARAMS["softening"] + hardening * 2 * PARAMS["xi"] * mu_in) * (strain + ys_in / (2 * mu_in))
    return {"F": _fro(Ft) + nf, "stress": S_stress, "yield_": S_yield}


def reference(pop, hardening, seed=0):
    """fp64 outcomes of every branch combination, the bound scales S and the near-boundary flags."""
    rng = np.random.default_rng(seed + 1)
    n = pop["F"].shape[0]
    outs = [oracle_run(pop, "f64", hardening, flip) for flip in range(4)]
    base = outs[0]
    Ft = pop["F"].astype(np.float64).reshape(n, 9)
    cond = {k: np.zeros(n) for k in ("F", "stress", "yield_")}
    cond_m = np.zeros((n, 2))
    scale = _fro(Ft)
    taken = lambda m: (m > 0).astype(int) @ np.array([1, 2])             # noqa: E731
    for _ in range(N_TRIALS):
        Z = rng.standard_normal((n, 9))
        Z *= (EPS * scale / np.linalg.norm(Z, axis=1))[:, None]
        Fp = (Ft + Z).reshape(n, 3, 3)
        runs = [oracle_run(pop, "f64", hardening, f, Fp) for f in range(4)]
        # the perturbed input on the branches the unperturbed one takes
        f_keep = taken(runs[0]["margins"]) ^ taken(base["margins"])
        t = {k: np.choose(f_keep[:, None], [r[k].reshape(n, -1) for r in runs]) for k in cond}
        t["margins"] = runs[0]["margins"]
        with np.errstate(all="ignore"):
            for k in cond:
                d = np.abs(t[k] - base[k].reshape(n, -1)).max(1) / EPS
                cond[k] = np.where(np.isfinite(d), np.maximum(cond[k], d), cond[k])
            dm = np.abs(t["margins"] - base["margins"]) / EPS
            cond_m = np.where(np.isfinite(dm), np.maximum(cond_m, dm), cond_m)
    S = []                                 # per branch combination: the term sums of that outcome + the conditioning
    for o in outs:
        t = _term_sums(pop, o, hardening)
        S.append({k: t[k] + cond[k] for k in cond})
    m = base["margins"]
    near = np.abs(m) <= K_MARGIN * EPS * (1 + cond_m)
    # allowed branch combinations per particle: flip bit b only where decision b is near its boundary
    allowed = np.stack([np.ones(n, bool), near[:, 0], near[:, 1], near[:, 0] & near[:, 1]], 1)
    # determinant sign settled (Hadamard-type bound of the fp32 determinant) or exactly zero by structure
    J = np.linalg.det(pop["F"].astype(np.float64))
    zero_line = (np.abs(pop["F"]).sum(1) == 0).any(1) | (np.abs(pop["F"]).sum(2) == 0).any(1)
    det_sure = (np.abs(J) > 64 * EPS * _det_terms(pop["F"].astype(np.float64))) | zero_line
    return dict(outs=outs, S=S, near=near, allowed=allowed, det_sure=det_sure)


def compare(pop, ref, got):
    """Largest err / (2^-23 S) per family over the allowed branch outcomes; asserts parity of non-finite entries and exact
    equality where the reference is exact (elastic branch F = F_trial, zero stress, unchanged / zeroed mu and lam)."""
    n = pop["F"].shape[0]
    mat = pop["material"]
    # the determinant's sign decides finiteness only for Drucker-Prager and water stress
    judged = ~np.isin(mat, (2, 6)) | ref["det_sure"]
    worst, report = {}, {}
    for key, k in (("F", "F"), ("stress", "stress"), ("yield_", "yield")):
        g = got[key].reshape(n, -1).astype(np.float64)
        ratio = np.full(n, np.inf)
        for flip in range(4):
            r = ref["outs"][flip][key].reshape(n, -1)
            with np.errstate(all="ignore"):
                fin = np.isfinite(r)
                e = np.where(fin, np.abs(g - r), 0.0).max(1)
                ok_nf = (np.isfinite(g) == fin).all(1)
                ratio_f = np.where(ok_nf, e / (EPS * np.maximum(ref["S"][flip][key], 1e-300)), np.inf)
                ratio_f = np.where((e == 0) & ok_nf, 0.0, ratio_f)
            ratio = np.where(ref["allowed"][:, flip], np.minimum(ratio, ratio_f), ratio)
        ratio = ratio[judged]
        bad = ratio > K[k]
        worst[k] = float(ratio.max())
        if bad.any():
            fam, mats = pop["family"][judged][bad], mat[judged][bad]
            report[k] = sorted({(f, int(m)) for f, m in zip(fam, mats)})[:12]
    for key in ("mu", "lam"):
        g = got[key].astype(np.float64)
        ok = np.zeros(n, bool)
        for flip in range(4):
            ok |= ref["allowed"][:, flip] & (g == ref["outs"][flip][key])
        if not ok.all():
            report[key] = sorted({(f, int(m)) for f, m in zip(pop["family"][~ok], mat[~ok])})[:12]
    return worst, report


def _check(pop, ref, got, label):
    worst, report = compare(pop, ref, got)
    print(f"{label}: max err / (2^-23 S): " + ", ".join(f"{k} {v:.3g} (bound {K[k]:g})" for k, v in worst.items()))
    assert not report, f"{label}: outside the bounds (family, material): {report}"
    return worst


def _families_are_exercised(pop, ref):
    base = ref["outs"][0]
    mat = pop["material"]
    m = base["margins"]
    taken = (m > 0) & np.isfinite(m)
    for mid in (1, 3, 5, 2):
        sel = mat == mid
        assert taken[sel, 0].any() and (~taken[sel, 0] & np.isfinite(m[sel, 0])).any(), f"material {mid}: both branches"
    assert (taken[mat == 2, 1]).any() and (~taken[mat == 2, 1] & np.isfinite(m[mat == 2, 1])).any()       # sand tr > 0
    assert ((mat == 5) & (base["mu"] == 0)).sum() > 10                     # damage zeroed mu / lam
    assert ((mat == 5) & (pop["ys"] <= 0)).sum() > 10
    assert ref["near"].any(0).all()                                        # particles at both kinds of boundary
    nf = ~np.isfinite(base["stress"]).all(1)
    assert (nf & (mat == 2) & ref["det_sure"]).sum() > 10 and (nf & (mat == 6) & ref["det_sure"]).sum() > 10
    assert np.isin(mat, (2, 6)).sum() > 0 and (ref["det_sure"] | ~np.isin(mat, (2, 6))).mean() > 0.97


@pytest.mark.parametrize("hardening", [0, 1])
def test_fp32_oracle_meets_the_same_bounds(hardening):
    pop = population(20_000, seed=10 + hardening)
    ref = reference(pop, hardening)
    _families_are_exercised(pop, ref)
    got = oracle_run(pop, "f32", hardening)
    _check(pop, ref, got, f"fp32 oracle, hardening {hardening}")


@pytest.mark.gpu
@pytest.mark.parametrize("hardening", [0, 1])
def test_return_maps_and_stresses_match_fp64(built_lib, cuda_dev, hardening):
    from pixie_b200.mpm_solver_warp import MPM_Simulator_WARP
    n = 100_000
    pop = population(n, seed=20 + hardening)
    ref = reference(pop, hardening)
    _families_are_exercised(pop, ref)
    dev = cuda_dev
    rng = np.random.default_rng(5)
    s = MPM_Simulator_WARP(n)
    x = torch.from_numpy(rng.uniform(0.3, 0.7, (n, 3)).astype(np.float32))
    s.load_initial_data_from_torch(x.to(dev), torch.full((n,), 1e-9).to(dev), None, n_grid=16, grid_lim=1.0)
    s.set_parameters_dict({"g": [0.0, 0.0, 0.0], "hardening": hardening, "xi": PARAMS["xi"], "softening": PARAMS["softening"],
                           "plastic_viscosity": PARAMS["plastic_viscosity"], "friction_angle": 30.0, "density": 1.0})
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)     # noqa: E731
    s.mpm_state.particle_material = t(pop["material"])
    s.mpm_state.particle_F_trial = t(pop["F"])
    s.mpm_model.mu, s.mpm_model.lam = t(pop["mu"]), t(pop["lam"])
    s.mpm_model.yield_stress, s.mpm_model.bulk = t(pop["ys"]), t(pop["bulk"])
    s.p2g2p(0, DT)
    torch.cuda.synchronize()
    got = dict(F=s.mpm_state.particle_F.numpy().reshape(n, 9), stress=s.mpm_state.particle_stress.numpy().reshape(n, 9),
               yield_=s.mpm_model.yield_stress.numpy(), mu=s.mpm_model.mu.numpy(), lam=s.mpm_model.lam.numpy())
    _check(pop, ref, got, f"device, hardening {hardening}")


def _polar_bound(F):
    """fp64 polar factor, its bound scale 1 + 2 ||F|| / (sigma_2 + sigma_3) and where it is defined (det F well above 0)."""
    F64 = F.astype(np.float64)
    U, sv, Vt = np.linalg.svd(F64)
    W = U @ Vt
    J = np.linalg.det(F64)
    ok = J > 64 * EPS * sv[:, 0] ** 3
    with np.errstate(divide="ignore"):
        S = 1 + 2 * _fro(F64) / (sv[:, 1] + sv[:, 2])
    return W, S, ok


def _check_rotations(Rm, F, label):
    n = F.shape[0]
    Rm = Rm.reshape(n, 3, 3).astype(np.float64).transpose(0, 2, 1)          # exported transposed (compute_R_from_F)
    assert np.isfinite(Rm).all(), f"{label}: non-finite R"
    orth = np.abs(np.einsum("nij,nkj->nik", Rm, Rm) - np.eye(3)).max()
    det = np.abs(np.linalg.det(Rm) - 1).max()
    W, S, ok = _polar_bound(F)
    ratio = (np.abs(Rm - W).reshape(n, 9).max(1) / (EPS * S))[ok]
    print(f"{label}: |R R^T - I| {orth:.2e}, |det R - 1| {det:.2e}, polar factor err / (2^-23 S) {ratio.max():.3g} "
          f"(bound {K['R']:g}) on {ok.sum()} of {n}")
    assert orth < 2e-6 and det < 2e-6
    assert ok.mean() > 0.6 and ratio.max() <= K["R"]


def test_fp32_oracle_rotations_meet_the_same_bounds():
    pop = population(20_000, seed=30)
    o = R.MpmRef(20_000, 16, 1.0, "f32")
    o.set("F_TRIAL", pop["F"])
    o.compute_R_from_F()
    _check_rotations(o.get("R").reshape(-1, 9), pop["F"], "fp32 oracle")


@pytest.mark.gpu
def test_svd3_rotation_matches_fp64_polar_factor(built_lib, cuda_dev):
    from pixie_b200.mpm_solver_warp import MPM_Simulator_WARP
    n = 100_000
    pop = population(n, seed=31)
    s = MPM_Simulator_WARP(n)
    s.mpm_state.particle_F_trial = torch.from_numpy(pop["F"]).to(cuda_dev)
    Rm = s.export_particle_R_to_torch().cpu().numpy()
    _check_rotations(Rm, pop["F"], "device")
