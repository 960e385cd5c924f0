/* ORACLE (test infrastructure, not product code): CPU restatement of the PhysGaussian MLS-MPM
 * substep the reference runs through NVIDIA Warp.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load
 * this library; pixie_b200/ never does.
 *
 * PINNED BY THE REFERENCE'S OWN SOURCE: the arithmetic of the reference lives in warp-lang==0.10.1 (pinned in
 * third_party/PhysGaussian/requirements.txt:4), which the reference neither vendors nor installs,
 * and the reference ships no tests or golden vectors for this path (SURVEY.md §4, §8c).  But its kernels are plain
 * Python syntax, so tests/golden/make_mpm_golden.py imports them from a checkout of the reference and EXECUTES them on a float32
 * `warp` stand-in (tests/golden/_fake_warp.py); the resulting fixture tests/golden/mpm_golden.npz (8 scenarios: every
 * material id, return map, stress model, BC closure, selection/setup/export kernel; 1- and 20-substep checkpoints)
 * is what tests/test_mpm_golden.py holds this file to (relative 5e-6 after one substep, masks / ids exact).
 * This file restates, statement by statement:
 *     third_party/PhysGaussian/mpm_solver_warp/mpm_utils.py        (kernels, :10-663)
 *     third_party/PhysGaussian/mpm_solver_warp/mpm_solver_warp.py  (p2g2p :514-637, BCs :749-1210)
 *     third_party/PhysGaussian/mpm_solver_warp/warp_utils.py       (structs :6-183)
 * Self-consistency tests stay (tests/test_oracle_mpm.py).  Still outside any pin: wp.svd3's own rounding (Warp
 * native/svd.h) — replaced here by a one-sided Jacobi SVD with the same output convention (U, V proper rotations,
 * |sigma| sorted descending, sign of det F on the last singular value); every use in the reference is of the
 * invariant form U f(Sigma) V^T.
 *
 * Compiled twice: -DREAL=float (the reference's precision) and -DREAL=double (drift reference).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#ifndef REAL
#define REAL float
#endif
typedef REAL real;

#ifdef _OPENMP
#include <omp.h>
#endif

#define RSQRT(x) ((real)sqrt((double)(x)))
#define RLOG(x) ((real)log((double)(x)))
#define REXP(x) ((real)exp((double)(x)))
#define RABS(x) ((real)fabs((double)(x)))
#define RMAX(a, b) ((a) > (b) ? (a) : (b))
#define RMIN(a, b) ((a) < (b) ? (a) : (b))

enum { F_X, F_V, F_F, F_FTRIAL, F_C, F_STRESS, F_R, F_COV, F_INITCOV, F_VOL, F_MASS, F_DENSITY, F_E, F_NU, F_MU,
       F_LAM, F_BULK, F_YIELD, F_MATERIAL, F_SELECTION, F_COUNT };
static const int kWidth[F_COUNT] = {3, 3, 9, 9, 9, 9, 9, 6, 6, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1};

enum { BC_SURFACE = 0, BC_CUBOID = 1, BC_BBOX = 2, BC_IMPULSE = 3, BC_VTRANS = 4, BC_VROT = 5 };

typedef struct {
    int kind;
    real point[3], normal[3], size[3], velocity[3];
    float start_time, end_time;   /* compared against float(time) in BOTH builds, like the Warp kernels */
    real friction;
    int surface_type, reset;
    real h1[3], h2[3], hhr[2], rotation_scale, translation_scale;
    int* mask;
} bc_t;

typedef struct {
    int n, n_grid;
    real grid_lim, dx, inv_dx;
    real* f[F_COUNT];          /* particle arrays (material / selection stored as int below) */
    int *material, *selection;
    real *grid_m, *grid_v_in, *grid_v_out;
    real g[3];
    real rpic_damping, grid_v_damping_scale, alpha, hardening, xi, plastic_viscosity, softening;
    int update_cov_with_F;
    double time;
    bc_t* bcs;
    int n_bc, cap_bc;
    int parallel_p2g;          /* 0: serial deterministic scatter (tests); 1: omp atomics (timing) */
} sim_t;

/* ------------------------------------------------------------------------------------- 3x3 helpers */
typedef struct { real m[9]; } m3;

static m3 m3_mul(const m3* a, const m3* b) {
    m3 c;
    for (int r = 0; r < 3; ++r)
        for (int k = 0; k < 3; ++k)
            c.m[3 * r + k] = a->m[3 * r] * b->m[k] + a->m[3 * r + 1] * b->m[3 + k] + a->m[3 * r + 2] * b->m[6 + k];
    return c;
}
static m3 m3_t(const m3* a) {
    m3 c;
    for (int r = 0; r < 3; ++r)
        for (int k = 0; k < 3; ++k) c.m[3 * r + k] = a->m[3 * k + r];
    return c;
}
static real m3_det(const m3* a) {
    return a->m[0] * (a->m[4] * a->m[8] - a->m[5] * a->m[7]) - a->m[1] * (a->m[3] * a->m[8] - a->m[5] * a->m[6]) +
           a->m[2] * (a->m[3] * a->m[7] - a->m[4] * a->m[6]);
}
static m3 m3_diag(real a, real b, real c) {
    m3 d;
    memset(&d, 0, sizeof(d));
    d.m[0] = a; d.m[4] = b; d.m[8] = c;
    return d;
}
/* U diag(s) V^T */
static m3 usvt(const m3* U, real s0, real s1, real s2, const m3* V) {
    m3 d = m3_diag(s0, s1, s2);
    m3 ud = m3_mul(U, &d);
    m3 vt = m3_t(V);
    return m3_mul(&ud, &vt);
}

/* wp.svd3 stand-in: one-sided Jacobi; exported for the tests as mpmref_svd3 */
static void svd3(const m3* F, m3* U, real* sig, m3* V) {
    real b[3][3], v[3][3];   /* columns */
    for (int c = 0; c < 3; ++c)
        for (int r = 0; r < 3; ++r) { b[c][r] = F->m[3 * r + c]; v[c][r] = (r == c) ? (real)1 : (real)0; }
    const real tol = (sizeof(real) == 4) ? (real)1e-15 : (real)1e-32;
    for (int sweep = 0; sweep < 12; ++sweep) {
        int rotated = 0;
        for (int p = 0; p < 2; ++p)
            for (int q = p + 1; q < 3; ++q) {
                real al = 0, be = 0, ga = 0;
                for (int r = 0; r < 3; ++r) { al += b[p][r] * b[p][r]; be += b[q][r] * b[q][r]; ga += b[p][r] * b[q][r]; }
                if (ga * ga <= tol * al * be || ga == 0) continue;
                rotated = 1;
                const real zeta = (be - al) / (2 * ga);
                const real t = (zeta >= 0 ? (real)1 : (real)-1) / (RABS(zeta) + RSQRT(1 + zeta * zeta));
                const real cs = 1 / RSQRT(1 + t * t), sn = cs * t;
                for (int r = 0; r < 3; ++r) {
                    const real bp = b[p][r], bq = b[q][r];
                    b[p][r] = cs * bp - sn * bq; b[q][r] = sn * bp + cs * bq;
                    const real vp = v[p][r], vq = v[q][r];
                    v[p][r] = cs * vp - sn * vq; v[q][r] = sn * vp + cs * vq;
                }
            }
        if (!rotated) break;
    }
    real n[3];
    for (int c = 0; c < 3; ++c) n[c] = b[c][0] * b[c][0] + b[c][1] * b[c][1] + b[c][2] * b[c][2];
    static const int order[3][2] = {{0, 1}, {0, 2}, {1, 2}};
    for (int k = 0; k < 3; ++k) {
        const int i = order[k][0], j = order[k][1];
        if (n[i] < n[j]) {
            real tn = n[i]; n[i] = n[j]; n[j] = tn;
            for (int r = 0; r < 3; ++r) {
                real tb = b[i][r]; b[i][r] = b[j][r]; b[j][r] = -tb;
                real tv = v[i][r]; v[i][r] = v[j][r]; v[j][r] = -tv;
            }
        }
    }
    const real s0 = RSQRT(n[0]), s1 = RSQRT(n[1]);
    real u0[3] = {1, 0, 0}, u1[3], u2[3];
    if (s0 > 0) for (int r = 0; r < 3; ++r) u0[r] = b[0][r] / s0;
    {
        real d = u0[0] * b[1][0] + u0[1] * b[1][1] + u0[2] * b[1][2];
        real w[3] = {b[1][0] - d * u0[0], b[1][1] - d * u0[1], b[1][2] - d * u0[2]};
        real nn = RSQRT(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
        if (!(nn > 0) || !(s1 > 0)) {
            if (RABS(u0[0]) < (real)0.9) { w[0] = 0; w[1] = -u0[2]; w[2] = u0[1]; }
            else { w[0] = -u0[2]; w[1] = 0; w[2] = u0[0]; }
            nn = RSQRT(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
        }
        for (int r = 0; r < 3; ++r) u1[r] = w[r] / nn;
    }
    u2[0] = u0[1] * u1[2] - u0[2] * u1[1];
    u2[1] = u0[2] * u1[0] - u0[0] * u1[2];
    u2[2] = u0[0] * u1[1] - u0[1] * u1[0];
    sig[0] = s0; sig[1] = s1;
    sig[2] = u2[0] * b[2][0] + u2[1] * b[2][1] + u2[2] * b[2][2];
    for (int r = 0; r < 3; ++r) {
        U->m[3 * r] = u0[r]; U->m[3 * r + 1] = u1[r]; U->m[3 * r + 2] = u2[r];
        V->m[3 * r] = v[0][r]; V->m[3 * r + 1] = v[1][r]; V->m[3 * r + 2] = v[2][r];
    }
}

/* ------------------------------------------------------------------------------------- constitutive */
/* kirchoff_stress_FCR, mpm_utils.py:10-17 */
static m3 stress_fcr(const m3* F, const m3* U, const m3* V, real J, real mu, real lam) {
    m3 Vt = m3_t(V), R = m3_mul(U, &Vt), Ft = m3_t(F), d, s;
    for (int i = 0; i < 9; ++i) d.m[i] = F->m[i] - R.m[i];
    s = m3_mul(&d, &Ft);
    for (int i = 0; i < 9; ++i) s.m[i] *= 2 * mu;
    const real p = lam * J * (J - 1);
    s.m[0] += p; s.m[4] += p; s.m[8] += p;
    return s;
}
/* kirchoff_stress_water, :20-28 */
static m3 stress_water(real J, real bulk) {
    const real pressure = -bulk * ((real)pow((double)J, -1.1) - 1);
    return m3_diag(J * pressure, J * pressure, J * pressure);
}
/* kirchoff_stress_StVK, :52-68 */
static m3 stress_stvk(const m3* F, const m3* U, const m3* V, const real* sg, real mu, real lam) {
    const real s0 = RMAX(sg[0], (real)0.01), s1 = RMAX(sg[1], (real)0.01), s2 = RMAX(sg[2], (real)0.01);
    const real e0 = RLOG(s0), e1 = RLOG(s1), e2 = RLOG(s2), tr = e0 + e1 + e2;
    m3 a = usvt(U, 2 * mu * e0 + lam * tr, 2 * mu * e1 + lam * tr, 2 * mu * e2 + lam * tr, V), Ft = m3_t(F);
    return m3_mul(&a, &Ft);
}
/* kirchoff_stress_drucker_prager, :71-86 */
static m3 stress_dp(const m3* F, const m3* U, const m3* V, const real* sg, real mu, real lam) {
    const real l0 = RLOG(sg[0]), l1 = RLOG(sg[1]), l2 = RLOG(sg[2]), tr = l0 + l1 + l2;
    m3 a = usvt(U, 2 * mu * l0 * (1 / sg[0]) + lam * tr * (1 / sg[0]), 2 * mu * l1 * (1 / sg[1]) + lam * tr * (1 / sg[1]),
                2 * mu * l2 * (1 / sg[2]) + lam * tr * (1 / sg[2]), V);
    m3 Ft = m3_t(F);
    return m3_mul(&a, &Ft);
}

/* von_mises_return_mapping (:89-135) and ..._with_damage (:138-191) */
static m3 return_von_mises(sim_t* s, int p, const m3* Ft, int with_damage) {
    m3 U, V; real so[3];
    svd3(Ft, &U, so, &V);
    real mu = s->f[F_MU][p], lam = s->f[F_LAM][p], ys = s->f[F_YIELD][p];
    const real g0 = RMAX(so[0], (real)0.01), g1 = RMAX(so[1], (real)0.01), g2 = RMAX(so[2], (real)0.01);
    real e0 = RLOG(g0), e1 = RLOG(g1), e2 = RLOG(g2);
    const real tr = e0 + e1 + e2, temp = tr / 3;
    const real t0 = 2 * mu * e0 + lam * tr, t1 = 2 * mu * e1 + lam * tr, t2 = 2 * mu * e2 + lam * tr;
    const real st = t0 + t1 + t2;
    const real c0 = t0 - st / 3, c1 = t1 - st / 3, c2 = t2 - st / 3;
    if (RSQRT(c0 * c0 + c1 * c1 + c2 * c2) > ys) {
        if (with_damage && ys <= 0) return *Ft;
        const real h0 = e0 - temp, h1 = e1 - temp, h2 = e2 - temp;
        const real hn = RSQRT(h0 * h0 + h1 * h1 + h2 * h2) + (real)1e-6;
        const real dg = hn - ys / (2 * mu);
        const real k = dg / hn;
        e0 -= k * h0; e1 -= k * h1; e2 -= k * h2;
        if (with_damage) {
            ys = ys - s->softening * RSQRT((k * h0) * (k * h0) + (k * h1) * (k * h1) + (k * h2) * (k * h2));
            s->f[F_YIELD][p] = ys;
            if (ys <= 0) { s->f[F_MU][p] = 0; s->f[F_LAM][p] = 0; }
        }
        m3 Fe = usvt(&U, REXP(e0), REXP(e1), REXP(e2), &V);
        if (s->hardening == 1) s->f[F_YIELD][p] = s->f[F_YIELD][p] + 2 * s->f[F_MU][p] * s->xi * dg;
        return Fe;
    }
    return *Ft;
}
/* viscoplasticity_return_mapping_with_StVK, :195-239 */
static m3 return_viscoplastic(sim_t* s, int p, const m3* Ft, real dt) {
    m3 U, V; real so[3];
    svd3(Ft, &U, so, &V);
    const real mu = s->f[F_MU][p];
    const real g0 = RMAX(so[0], (real)0.01), g1 = RMAX(so[1], (real)0.01), g2 = RMAX(so[2], (real)0.01);
    const real b0 = g0 * g0, b1 = g1 * g1, b2 = g2 * g2;
    const real e0 = RLOG(g0), e1 = RLOG(g1), e2 = RLOG(g2), tr = e0 + e1 + e2;
    const real h0 = e0 - tr / 3, h1 = e1 - tr / 3, h2 = e2 - tr / 3;
    const real s0 = 2 * mu * h0, s1 = 2 * mu * h1, s2 = 2 * mu * h2;
    const real sn = RSQRT(s0 * s0 + s1 * s1 + s2 * s2);
    const real y = sn - RSQRT((real)2 / (real)3) * s->f[F_YIELD][p];
    if (y > 0) {
        const real mu_hat = mu * (b0 + b1 + b2) / 3;
        const real snew = sn - y / (1 + s->plastic_viscosity / (2 * mu_hat * dt));
        const real r = snew / sn, k = 1 / (2 * mu);
        return usvt(&U, REXP(k * (r * s0) + tr / 3), REXP(k * (r * s1) + tr / 3), REXP(k * (r * s2) + tr / 3), &V);
    }
    return *Ft;
}
/* sand_return_mapping, :242-279 */
static m3 return_sand(sim_t* s, int p, const m3* Ft) {
    m3 U, V; real sg[3];
    svd3(Ft, &U, sg, &V);
    const real mu = s->f[F_MU][p], lam = s->f[F_LAM][p];
    const real e0 = RLOG(RMAX(RABS(sg[0]), (real)1e-14)), e1 = RLOG(RMAX(RABS(sg[1]), (real)1e-14)),
               e2 = RLOG(RMAX(RABS(sg[2]), (real)1e-14));
    const real tr = e0 + e1 + e2;
    const real h0 = e0 - tr / 3, h1 = e1 - tr / 3, h2 = e2 - tr / 3;
    const real hn = RSQRT(h0 * h0 + h1 * h1 + h2 * h2);
    const real dg = hn + (3 * lam + 2 * mu) / (2 * mu) * tr * s->alpha;
    if (dg <= 0) return *Ft;
    if (tr > 0) { m3 Vt = m3_t(&V); return m3_mul(&U, &Vt); }
    const real k = dg / hn;
    return usvt(&U, REXP(e0 - h0 * k), REXP(e1 - h1 * k), REXP(e2 - h2 * k), &V);
}

/* compute_stress_from_F_trial, :467-526 */
static void compute_stress(sim_t* s, int p, real dt) {
    if (s->selection[p] != 0) return;
    const int mat = s->material[p];
    m3 Ft, F;
    memcpy(Ft.m, s->f[F_FTRIAL] + 9 * (size_t)p, sizeof(Ft.m));
    if (mat == 1) F = return_von_mises(s, p, &Ft, 0);
    else if (mat == 2) F = return_sand(s, p, &Ft);
    else if (mat == 3) F = return_viscoplastic(s, p, &Ft, dt);
    else if (mat == 5) F = return_von_mises(s, p, &Ft, 1);
    else F = Ft;
    memcpy(s->f[F_F] + 9 * (size_t)p, F.m, sizeof(F.m));
    const real J = m3_det(&F);
    m3 U, V, tau; real sg[3];
    memset(&tau, 0, sizeof(tau));
    svd3(&F, &U, sg, &V);
    const real mu = s->f[F_MU][p], lam = s->f[F_LAM][p];
    if (mat == 0 || mat == 5) tau = stress_fcr(&F, &U, &V, J, mu, lam);
    if (mat == 1) tau = stress_stvk(&F, &U, &V, sg, mu, lam);
    if (mat == 2) tau = stress_dp(&F, &U, &V, sg, mu, lam);
    if (mat == 3) tau = stress_stvk(&F, &U, &V, sg, mu, lam);
    if (mat == 6) tau = stress_water(J, s->f[F_BULK][p]);
    m3 tt = m3_t(&tau);
    for (int i = 0; i < 9; ++i) tau.m[i] = (tau.m[i] + tt.m[i]) / 2;
    memcpy(s->f[F_STRESS] + 9 * (size_t)p, tau.m, sizeof(tau.m));
}

/* shared by p2g and g2p: base node, fractional offset, weights (mpm_utils.py:341-358, 416-434) */
typedef struct { int b[3]; real fx[3], w[3][3], dw[3][3]; } weights_t;
static weights_t bspline(const sim_t* s, const real* x) {
    weights_t W;
    for (int a = 0; a < 3; ++a) {
        const real g = x[a] * s->inv_dx;
        W.b[a] = (int)(g - (real)0.5);            /* wp.int: truncation toward zero */
        const real fx = g - (real)W.b[a];
        W.fx[a] = fx;
        const real wa = (real)1.5 - fx, wb = fx - (real)1.0, wc = fx - (real)0.5;
        W.w[a][0] = wa * wa * (real)0.5;
        W.w[a][1] = (real)0 - wb * wb + (real)0.75;
        W.w[a][2] = wc * wc * (real)0.5;
        W.dw[a][0] = fx - (real)1.5;
        W.dw[a][1] = (real)-2.0 * (fx - (real)1.0);
        W.dw[a][2] = fx - (real)0.5;
    }
    return W;
}

/* p2g_apic_with_stress, :338-394 */
static void p2g_particle(sim_t* s, int p, real dt) {
    if (s->selection[p] != 0) return;
    const int n = s->n_grid;
    const real* x = s->f[F_X] + 3 * (size_t)p;
    const real* v = s->f[F_V] + 3 * (size_t)p;
    const real* tau = s->f[F_STRESS] + 9 * (size_t)p;
    const real mass = s->f[F_MASS][p], vol = s->f[F_VOL][p];
    const weights_t W = bspline(s, x);
    real C[9];
    {
        const real* Cp = s->f[F_C] + 9 * (size_t)p;
        const real r = s->rpic_damping;
        for (int a = 0; a < 3; ++a)
            for (int b = 0; b < 3; ++b)
                C[3 * a + b] = ((real)1.0 - r) * Cp[3 * a + b] + r / (real)2.0 * (Cp[3 * a + b] - Cp[3 * b + a]);
        if (r < (real)-0.001) memset(C, 0, sizeof(C));
    }
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j)
            for (int k = 0; k < 3; ++k) {
                const int ix = W.b[0] + i, iy = W.b[1] + j, iz = W.b[2] + k;
                if (ix < 0 || iy < 0 || iz < 0 || ix >= n || iy >= n || iz >= n) continue;   /* reference: UB */
                const real dpos[3] = {((real)i - W.fx[0]) * s->dx, ((real)j - W.fx[1]) * s->dx, ((real)k - W.fx[2]) * s->dx};
                const real weight = W.w[0][i] * W.w[1][j] * W.w[2][k];
                const real dwt[3] = {W.dw[0][i] * W.w[1][j] * W.w[2][k] * s->inv_dx,
                                     W.w[0][i] * W.dw[1][j] * W.w[2][k] * s->inv_dx,
                                     W.w[0][i] * W.w[1][j] * W.dw[2][k] * s->inv_dx};
                const size_t node = ((size_t)ix * n + iy) * n + iz;
                real add[3];
                for (int a = 0; a < 3; ++a) {
                    const real sd = tau[3 * a] * dwt[0] + tau[3 * a + 1] * dwt[1] + tau[3 * a + 2] * dwt[2];
                    const real cd = C[3 * a] * dpos[0] + C[3 * a + 1] * dpos[1] + C[3 * a + 2] * dpos[2];
                    add[a] = weight * mass * (v[a] + cd) + dt * (-vol * sd);
                }
                const real am = weight * mass;
                if (s->parallel_p2g) {
                    for (int a = 0; a < 3; ++a) {
#pragma omp atomic
                        s->grid_v_in[3 * node + a] += add[a];
                    }
#pragma omp atomic
                    s->grid_m[node] += am;
                } else {
                    for (int a = 0; a < 3; ++a) s->grid_v_in[3 * node + a] += add[a];
                    s->grid_m[node] += am;
                }
            }
}

/* g2p, :412-463 (+ update_cov :315-335) */
static void g2p_particle(sim_t* s, int p, real dt) {
    if (s->selection[p] != 0) return;
    const int n = s->n_grid;
    real* x = s->f[F_X] + 3 * (size_t)p;
    const weights_t W = bspline(s, x);
    real nv[3] = {0, 0, 0}, nC[9], nF[9];
    memset(nC, 0, sizeof(nC));
    memset(nF, 0, sizeof(nF));
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j)
            for (int k = 0; k < 3; ++k) {
                const int ix = W.b[0] + i, iy = W.b[1] + j, iz = W.b[2] + k;
                real gv[3] = {0, 0, 0};
                if (!(ix < 0 || iy < 0 || iz < 0 || ix >= n || iy >= n || iz >= n)) {
                    const size_t node = ((size_t)ix * n + iy) * n + iz;
                    gv[0] = s->grid_v_out[3 * node]; gv[1] = s->grid_v_out[3 * node + 1]; gv[2] = s->grid_v_out[3 * node + 2];
                }
                const real dp[3] = {(real)i - W.fx[0], (real)j - W.fx[1], (real)k - W.fx[2]};
                const real weight = W.w[0][i] * W.w[1][j] * W.w[2][k];
                const real dwt[3] = {W.dw[0][i] * W.w[1][j] * W.w[2][k] * s->inv_dx,
                                     W.w[0][i] * W.dw[1][j] * W.w[2][k] * s->inv_dx,
                                     W.w[0][i] * W.w[1][j] * W.dw[2][k] * s->inv_dx};
                const real cw = weight * s->inv_dx * (real)4.0;
                for (int a = 0; a < 3; ++a) {
                    nv[a] = nv[a] + gv[a] * weight;
                    for (int b = 0; b < 3; ++b) {
                        nC[3 * a + b] = nC[3 * a + b] + (gv[a] * dp[b]) * cw;
                        nF[3 * a + b] = nF[3 * a + b] + gv[a] * dwt[b];
                    }
                }
            }
    real* v = s->f[F_V] + 3 * (size_t)p;
    for (int a = 0; a < 3; ++a) { v[a] = nv[a]; x[a] = x[a] + dt * nv[a]; }
    memcpy(s->f[F_C] + 9 * (size_t)p, nC, sizeof(nC));
    m3 A, F, Ft;
    for (int i = 0; i < 9; ++i) A.m[i] = nF[i] * dt;
    A.m[0] += 1; A.m[4] += 1; A.m[8] += 1;
    memcpy(F.m, s->f[F_F] + 9 * (size_t)p, sizeof(F.m));
    Ft = m3_mul(&A, &F);
    memcpy(s->f[F_FTRIAL] + 9 * (size_t)p, Ft.m, sizeof(Ft.m));
    if (s->update_cov_with_F) {
        real* cv = s->f[F_COV] + 6 * (size_t)p;
        m3 cn = {{cv[0], cv[1], cv[2], cv[1], cv[3], cv[4], cv[2], cv[4], cv[5]}}, G, a, b, Gt;
        memcpy(G.m, nF, sizeof(nF));
        Gt = m3_t(&G);
        a = m3_mul(&G, &cn);
        b = m3_mul(&cn, &Gt);
        real c1[9];
        for (int i = 0; i < 9; ++i) c1[i] = cn.m[i] + dt * (a.m[i] + b.m[i]);
        cv[0] = c1[0]; cv[1] = c1[1]; cv[2] = c1[2]; cv[3] = c1[4]; cv[4] = c1[5]; cv[5] = c1[8];
    }
}

/* grid_normalization_and_gravity :398-409, add_damping_via_grid :583-588, BC collide closures */
static void grid_node(sim_t* s, size_t idx, float time, real dt) {
    const int n = s->n_grid;
    const int gz = (int)(idx % n), gy = (int)((idx / n) % n), gx = (int)(idx / ((size_t)n * n));
    real* vo = s->grid_v_out + 3 * idx;
    vo[0] = vo[1] = vo[2] = 0;                                   /* zero_grid :295-300 */
    const real m = s->grid_m[idx];
    if (m > (real)1e-15) {
        const real inv = (real)1.0 / m;
        for (int a = 0; a < 3; ++a) vo[a] = s->grid_v_in[3 * idx + a] * inv + dt * s->g[a];
    }
    if (s->grid_v_damping_scale < (real)1.0)
        for (int a = 0; a < 3; ++a) vo[a] = vo[a] * s->grid_v_damping_scale;
    for (int k = 0; k < s->n_bc; ++k) {
        const bc_t* bc = &s->bcs[k];
        const int active = time >= bc->start_time && time < bc->end_time;
        if (bc->kind == BC_SURFACE) {                            /* mpm_solver_warp.py:785-840 */
            if (!active) continue;
            const real off[3] = {(real)gx * s->dx - bc->point[0], (real)gy * s->dx - bc->point[1], (real)gz * s->dx - bc->point[2]};
            const real dotp = off[0] * bc->normal[0] + off[1] * bc->normal[1] + off[2] * bc->normal[2];
            if (dotp < 0) {
                if (bc->surface_type == 0) { vo[0] = vo[1] = vo[2] = 0; }
                else if (bc->surface_type == 11) {
                    const real zz = (real)gz * s->dx;
                    if (zz < (real)0.4 || zz > (real)0.53) { vo[0] = vo[1] = vo[2] = 0; }
                    else { vo[0] = vo[0] * (real)0.3; vo[1] = (real)0.0 * (real)0.3; vo[2] = vo[2] * (real)0.3; }
                } else {
                    /* the projected / frictional velocity is computed and then discarded: :836-840 */
                    vo[0] = vo[1] = vo[2] = 0;
                }
            }
        } else if (bc->kind == BC_CUBOID) {                      /* :874-897 */
            if (active) {
                const real off[3] = {(real)gx * s->dx - bc->point[0], (real)gy * s->dx - bc->point[1], (real)gz * s->dx - bc->point[2]};
                if (RABS(off[0]) < bc->size[0] && RABS(off[1]) < bc->size[1] && RABS(off[2]) < bc->size[2])
                    for (int a = 0; a < 3; ++a) vo[a] = bc->velocity[a];
            } else if (bc->reset == 1) {
                if (time < bc->end_time + 15.0f * (float)dt) { vo[0] = vo[1] = vo[2] = 0; }
            }
        } else if (bc->kind == BC_BBOX) {                        /* :917-974 */
            if (!active) continue;
            const int pad = 3;
            if (gx < pad && vo[0] < 0) vo[0] = 0;
            if (gx >= n - pad && vo[0] > 0) vo[0] = 0;
            if (gy < pad && vo[1] < 0) vo[1] = 0;
            if (gy >= n - pad && vo[1] > 0) vo[1] = 0;
            if (gz < pad && vo[2] < 0) vo[2] = 0;
            if (gz >= n - pad && vo[2] > 0) vo[2] = 0;
        }
    }
}

/* pre-p2g particle operations: impulses, then velocity modifiers (mpm_solver_warp.py:528-547) */
static void particle_bcs(sim_t* s, int p, float time, real dt) {
    real* v = s->f[F_V] + 3 * (size_t)p;
    const real* x = s->f[F_X] + 3 * (size_t)p;
    for (int k = 0; k < s->n_bc; ++k) {
        const bc_t* bc = &s->bcs[k];
        if (bc->kind != BC_IMPULSE) continue;
        if (time >= bc->start_time && time < bc->end_time && bc->mask[p] == 1)        /* :1015-1027 */
            for (int a = 0; a < 3; ++a) v[a] = v[a] + (bc->velocity[a] / s->f[F_MASS][p]) * dt;
    }
    for (int k = 0; k < s->n_bc; ++k) {
        const bc_t* bc = &s->bcs[k];
        if (bc->kind == BC_VTRANS) {                                                    /* :1061-1073 */
            if (time >= bc->start_time && time < bc->end_time && bc->mask[p] == 1)
                for (int a = 0; a < 3; ++a) v[a] = bc->velocity[a];
        } else if (bc->kind == BC_VROT) {                                               /* :1137-1179 */
            if (time >= bc->start_time && time < bc->end_time && bc->mask[p] == 1) {
                const real off[3] = {x[0] - bc->point[0], x[1] - bc->point[1], x[2] - bc->point[2]};
                const real on = off[0] * bc->normal[0] + off[1] * bc->normal[1] + off[2] * bc->normal[2];
                const real h[3] = {off[0] - on * bc->normal[0], off[1] - on * bc->normal[1], off[2] - on * bc->normal[2]};
                const real hd = RSQRT(h[0] * h[0] + h[1] * h[1] + h[2] * h[2]);
                const real cosine = (off[0] * bc->h1[0] + off[1] * bc->h1[1] + off[2] * bc->h1[2]) / hd;
                real theta = (real)acos((double)cosine);
                if (!(off[0] * bc->h2[0] + off[1] * bc->h2[1] + off[2] * bc->h2[2] > 0)) theta = -theta;
                const real a1 = -hd * (real)sin((double)theta) * bc->rotation_scale;
                const real a2 = hd * (real)cos((double)theta) * bc->rotation_scale;
                const real av = bc->translation_scale;
                for (int a = 0; a < 3; ++a) v[a] = a1 * bc->h1[a] + a2 * bc->h2[a] + av * bc->normal[a];
            }
        }
    }
}

/* ------------------------------------------------------------------------------------- API */
sim_t* mpmref_create(int n, int n_grid, double grid_lim) {
    sim_t* s = (sim_t*)calloc(1, sizeof(sim_t));
    s->n = n; s->n_grid = n_grid; s->grid_lim = (real)grid_lim;
    s->dx = (real)(grid_lim / n_grid);
    s->inv_dx = (real)((double)n_grid / grid_lim);
    for (int i = 0; i < F_COUNT; ++i) s->f[i] = (real*)calloc((size_t)n * kWidth[i], sizeof(real));
    s->material = (int*)calloc(n, sizeof(int));
    s->selection = (int*)calloc(n, sizeof(int));
    const size_t nodes = (size_t)n_grid * n_grid * n_grid;
    s->grid_m = (real*)calloc(nodes, sizeof(real));
    s->grid_v_in = (real*)calloc(nodes * 3, sizeof(real));
    s->grid_v_out = (real*)calloc(nodes * 3, sizeof(real));
    s->grid_v_damping_scale = (real)1.1;
    {
        const double sin_phi = sin(25.0 / 180.0 * 3.14159265);
        s->alpha = (real)(sqrt(2.0 / 3.0) * 2.0 * sin_phi / (3.0 - sin_phi));
    }
    s->softening = (real)0.1;
    for (int p = 0; p < n; ++p) { real* F = s->f[F_FTRIAL] + 9 * (size_t)p; F[0] = F[4] = F[8] = 1; }   /* :263-277 */
    return s;
}
void mpmref_destroy(sim_t* s) {
    if (!s) return;
    for (int i = 0; i < F_COUNT; ++i) free(s->f[i]);
    for (int k = 0; k < s->n_bc; ++k) free(s->bcs[k].mask);
    free(s->bcs); free(s->material); free(s->selection); free(s->grid_m); free(s->grid_v_in); free(s->grid_v_out);
    free(s);
}
int mpmref_real_size(void) { return (int)sizeof(real); }
void mpmref_set(sim_t* s, int field, const double* data) {
    const size_t cnt = (size_t)s->n * kWidth[field];
    if (field == F_MATERIAL) for (size_t i = 0; i < cnt; ++i) s->material[i] = (int)data[i];
    else if (field == F_SELECTION) for (size_t i = 0; i < cnt; ++i) s->selection[i] = (int)data[i];
    else for (size_t i = 0; i < cnt; ++i) s->f[field][i] = (real)data[i];
}
void mpmref_get(sim_t* s, int field, double* out) {
    const size_t cnt = (size_t)s->n * kWidth[field];
    if (field == F_MATERIAL) for (size_t i = 0; i < cnt; ++i) out[i] = s->material[i];
    else if (field == F_SELECTION) for (size_t i = 0; i < cnt; ++i) out[i] = s->selection[i];
    else for (size_t i = 0; i < cnt; ++i) out[i] = (double)s->f[field][i];
}
void mpmref_get_grid(sim_t* s, double* m, double* v_in, double* v_out) {
    const size_t nodes = (size_t)s->n_grid * s->n_grid * s->n_grid;
    for (size_t i = 0; i < nodes; ++i) m[i] = s->grid_m[i];
    for (size_t i = 0; i < 3 * nodes; ++i) { v_in[i] = s->grid_v_in[i]; v_out[i] = s->grid_v_out[i]; }
}
void mpmref_set_params(sim_t* s, const double* g, double rpic, double damping, double alpha, double hardening, double xi,
                       double plastic_viscosity, double softening, int update_cov, int parallel_p2g) {
    for (int a = 0; a < 3; ++a) s->g[a] = (real)g[a];
    s->rpic_damping = (real)rpic; s->grid_v_damping_scale = (real)damping; s->alpha = (real)alpha;
    s->hardening = (real)hardening; s->xi = (real)xi; s->plastic_viscosity = (real)plastic_viscosity;
    s->softening = (real)softening; s->update_cov_with_F = update_cov; s->parallel_p2g = parallel_p2g;
}
void mpmref_set_time(sim_t* s, double t) { s->time = t; }
double mpmref_get_time(sim_t* s) { return s->time; }
/* vals: point3 normal3 size3 velocity3 start end friction h1_3 h2_3 hhr2 rot trans = 25 doubles */
void mpmref_add_bc(sim_t* s, int kind, const double* vals, int surface_type, int reset, const int* mask) {
    if (s->n_bc == s->cap_bc) { s->cap_bc = s->cap_bc ? 2 * s->cap_bc : 8; s->bcs = (bc_t*)realloc(s->bcs, s->cap_bc * sizeof(bc_t)); }
    bc_t* b = &s->bcs[s->n_bc++];
    memset(b, 0, sizeof(*b));
    b->kind = kind; b->surface_type = surface_type; b->reset = reset;
    for (int a = 0; a < 3; ++a) {
        b->point[a] = (real)vals[a]; b->normal[a] = (real)vals[3 + a]; b->size[a] = (real)vals[6 + a];
        b->velocity[a] = (real)vals[9 + a]; b->h1[a] = (real)vals[15 + a]; b->h2[a] = (real)vals[18 + a];
    }
    b->start_time = (float)vals[12]; b->end_time = (float)vals[13]; b->friction = (real)vals[14];
    b->hhr[0] = (real)vals[21]; b->hhr[1] = (real)vals[22]; b->rotation_scale = (real)vals[23]; b->translation_scale = (real)vals[24];
    if (mask) { b->mask = (int*)malloc(s->n * sizeof(int)); memcpy(b->mask, mask, s->n * sizeof(int)); }
}
void mpmref_compute_mu_lam(sim_t* s) {          /* compute_mu_lam_from_E_nu, mpm_utils.py:282-288 */
    for (int p = 0; p < s->n; ++p) {
        const real E = s->f[F_E][p], nu = s->f[F_NU][p];
        s->f[F_MU][p] = E / ((real)2.0 * ((real)1.0 + nu));
        s->f[F_LAM][p] = E * nu / (((real)1.0 + nu) * ((real)1.0 - (real)2.0 * nu));
    }
}
void mpmref_compute_mass(sim_t* s) {            /* get_float_array_product, warp_utils.py:233-241 */
    for (int p = 0; p < s->n; ++p) s->f[F_MASS][p] = s->f[F_DENSITY][p] * s->f[F_VOL][p];
}
void mpmref_compute_cov_from_F(sim_t* s) {      /* compute_cov_from_F, mpm_utils.py:529-553 */
    for (int p = 0; p < s->n; ++p) {
        m3 F, c0, a, Ft, c;
        memcpy(F.m, s->f[F_FTRIAL] + 9 * (size_t)p, sizeof(F.m));
        const real* ic = s->f[F_INITCOV] + 6 * (size_t)p;
        const real cc[9] = {ic[0], ic[1], ic[2], ic[1], ic[3], ic[4], ic[2], ic[4], ic[5]};
        memcpy(c0.m, cc, sizeof(cc));
        a = m3_mul(&F, &c0); Ft = m3_t(&F); c = m3_mul(&a, &Ft);
        real* o = s->f[F_COV] + 6 * (size_t)p;
        o[0] = c.m[0]; o[1] = c.m[1]; o[2] = c.m[2]; o[3] = c.m[4]; o[4] = c.m[5]; o[5] = c.m[8];
    }
}
void mpmref_compute_bulk(sim_t* s) {            /* compute_bulk, mpm_utils.py:290-293 */
    for (int p = 0; p < s->n; ++p) s->f[F_BULK][p] = s->f[F_LAM][p] + (real)(2. / 3.) * s->f[F_MU][p];
}
void mpmref_compute_R_from_F(sim_t* s) {        /* compute_R_from_F, mpm_utils.py:556-579 */
    for (int p = 0; p < s->n; ++p) {
        m3 F, U, V, Vt, R, Rt; real sg[3];
        memcpy(F.m, s->f[F_FTRIAL] + 9 * (size_t)p, sizeof(F.m));
        svd3(&F, &U, sg, &V);
        if (m3_det(&U) < 0) { U.m[2] = -U.m[2]; U.m[5] = -U.m[5]; U.m[8] = -U.m[8]; }
        if (m3_det(&V) < 0) { V.m[2] = -V.m[2]; V.m[5] = -V.m[5]; V.m[8] = -V.m[8]; }
        Vt = m3_t(&V); R = m3_mul(&U, &Vt); Rt = m3_t(&R);
        memcpy(s->f[F_R] + 9 * (size_t)p, Rt.m, sizeof(Rt.m));
    }
}
/* apply_additional_params, mpm_utils.py:591-610: box = point3 size3 E nu density material */
void mpmref_apply_additional_params(sim_t* s, const double* box) {
    const real pt[3] = {(real)box[0], (real)box[1], (real)box[2]}, sz[3] = {(real)box[3], (real)box[4], (real)box[5]};
    for (int p = 0; p < s->n; ++p) {
        const real* x = s->f[F_X] + 3 * (size_t)p;
        if (x[0] > pt[0] - sz[0] && x[0] < pt[0] + sz[0] && x[1] > pt[1] - sz[1] && x[1] < pt[1] + sz[1] &&
            x[2] > pt[2] - sz[2] && x[2] < pt[2] + sz[2]) {
            s->f[F_E][p] = (real)box[6]; s->f[F_NU][p] = (real)box[7]; s->f[F_DENSITY][p] = (real)box[8];
            s->material[p] = (int)box[9];
        }
    }
}
/* selection_add_impulse_on_particles / selection_enforce_particle_velocity_translation, mpm_utils.py:613-645 */
void mpmref_select_box(sim_t* s, const double* point, const double* size, int* mask) {
    for (int p = 0; p < s->n; ++p) {
        const real* x = s->f[F_X] + 3 * (size_t)p;
        int in = 1;
        for (int a = 0; a < 3; ++a) in = in && (RABS(x[a] - (real)point[a]) < (real)size[a]);
        mask[p] = in;
    }
}
/* selection_enforce_particle_velocity_cylinder, mpm_utils.py:648-663 */
void mpmref_select_cylinder(sim_t* s, const double* point, const double* normal, double half_height, double radius, int* mask) {
    const real nn[3] = {(real)normal[0], (real)normal[1], (real)normal[2]};
    for (int p = 0; p < s->n; ++p) {
        const real* x = s->f[F_X] + 3 * (size_t)p;
        const real off[3] = {x[0] - (real)point[0], x[1] - (real)point[1], x[2] - (real)point[2]};
        const real on = off[0] * nn[0] + off[1] * nn[1] + off[2] * nn[2];
        const real h[3] = {off[0] - on * nn[0], off[1] - on * nn[1], off[2] - on * nn[2]};
        const real hd = RSQRT(h[0] * h[0] + h[1] * h[1] + h[2] * h[2]);
        mask[p] = (RABS(on) < (real)half_height && hd < (real)radius) ? 1 : 0;
    }
}
void mpmref_svd3(const double* F9, double* U9, double* sig3, double* V9) {
    m3 F, U, V; real sg[3];
    for (int i = 0; i < 9; ++i) F.m[i] = (real)F9[i];
    svd3(&F, &U, sg, &V);
    for (int i = 0; i < 9; ++i) { U9[i] = U.m[i]; V9[i] = V.m[i]; }
    for (int i = 0; i < 3; ++i) sig3[i] = sg[i];
}
void mpmref_stress_of_F(sim_t* s, int p) { compute_stress(s, p, (real)1e-4); }

/* one p2g2p (mpm_solver_warp.py:514-637) */
static void substep(sim_t* s, double dt_d) {
    const real dt = (real)dt_d;
    const float time = (float)s->time;      /* wp kernels receive `time` as fp32 */
    const int n = s->n;
    const size_t nodes = (size_t)s->n_grid * s->n_grid * s->n_grid;
    memset(s->grid_m, 0, nodes * sizeof(real));
    memset(s->grid_v_in, 0, 3 * nodes * sizeof(real));
#pragma omp parallel for schedule(static)
    for (int p = 0; p < n; ++p) { particle_bcs(s, p, time, dt); compute_stress(s, p, dt); }
    if (s->parallel_p2g) {
#pragma omp parallel for schedule(static)
        for (int p = 0; p < n; ++p) p2g_particle(s, p, dt);
    } else {
        for (int p = 0; p < n; ++p) p2g_particle(s, p, dt);
    }
#pragma omp parallel for schedule(static)
    for (long long i = 0; i < (long long)nodes; ++i) grid_node(s, (size_t)i, time, dt);
    for (int k = 0; k < s->n_bc; ++k) {                       /* modify(): :899-905, host-side doubles */
        bc_t* bc = &s->bcs[k];
        if (bc->kind == BC_CUBOID && s->time >= (double)bc->start_time && s->time < (double)bc->end_time)
            for (int a = 0; a < 3; ++a) bc->point[a] = (real)((double)bc->point[a] + dt_d * (double)bc->velocity[a]);
    }
#pragma omp parallel for schedule(static)
    for (int p = 0; p < n; ++p) g2p_particle(s, p, dt);
    s->time = s->time + dt_d;
}
void mpmref_step(sim_t* s, int n_substeps, double dt) {
    for (int i = 0; i < n_substeps; ++i) substep(s, dt);
}
/* ---- split substep for slab-decomposed runs (test double of pixie_mpm_substep_scatter / _finish; the reference has
 *      no multi-GPU path, SURVEY.md 8e). The caller owns the zero-invariant: planes outside the finished range
 *      keep whatever was scattered into them. */
void mpmref_set_active(sim_t* s, int n_active) { s->n = n_active; }
void mpmref_scatter(sim_t* s, double dt_d) {
    const real dt = (real)dt_d;
    const float time = (float)s->time;
    for (int p = 0; p < s->n; ++p) { particle_bcs(s, p, time, dt); compute_stress(s, p, dt); }
    for (int p = 0; p < s->n; ++p) p2g_particle(s, p, dt);
}
void mpmref_finish(sim_t* s, double dt_d, int x_begin, int x_end) {
    const real dt = (real)dt_d;
    const float time = (float)s->time;
    const size_t plane = (size_t)s->n_grid * s->n_grid;
    for (size_t i = (size_t)x_begin * plane; i < (size_t)x_end * plane; ++i) grid_node(s, i, time, dt);
    for (int k = 0; k < s->n_bc; ++k) {
        bc_t* bc = &s->bcs[k];
        if (bc->kind == BC_CUBOID && s->time >= (double)bc->start_time && s->time < (double)bc->end_time)
            for (int a = 0; a < 3; ++a) bc->point[a] = (real)((double)bc->point[a] + dt_d * (double)bc->velocity[a]);
    }
    for (int p = 0; p < s->n; ++p) g2p_particle(s, p, dt);
    memset(s->grid_m + (size_t)x_begin * plane, 0, (size_t)(x_end - x_begin) * plane * sizeof(real));
    memset(s->grid_v_in + 3 * (size_t)x_begin * plane, 0, 3 * (size_t)(x_end - x_begin) * plane * sizeof(real));
    s->time = s->time + dt_d;
}
/* planes [a, b) of the scatter target as {mv.x, mv.y, mv.z, m} per node (the CUDA grid layout) */
void mpmref_planes_get(sim_t* s, int a, int b, double* out) {
    const size_t plane = (size_t)s->n_grid * s->n_grid;
    for (size_t i = (size_t)a * plane, k = 0; i < (size_t)b * plane; ++i, ++k) {
        out[4 * k] = s->grid_v_in[3 * i]; out[4 * k + 1] = s->grid_v_in[3 * i + 1]; out[4 * k + 2] = s->grid_v_in[3 * i + 2];
        out[4 * k + 3] = s->grid_m[i];
    }
}
void mpmref_planes_add(sim_t* s, int a, int b, const double* in) {
    const size_t plane = (size_t)s->n_grid * s->n_grid;
    for (size_t i = (size_t)a * plane, k = 0; i < (size_t)b * plane; ++i, ++k) {
        s->grid_v_in[3 * i] += (real)in[4 * k]; s->grid_v_in[3 * i + 1] += (real)in[4 * k + 1]; s->grid_v_in[3 * i + 2] += (real)in[4 * k + 2];
        s->grid_m[i] += (real)in[4 * k + 3];
    }
}
void mpmref_set_num_threads(int n) {
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}
int mpmref_num_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}
