// Standalone test of the U-Net's memory-bound kernels (unet_kernels.cu) against fp64 host references:
//   moments    per-(item, channel) sum and sum of squares; variance of offset data (|mean| / sigma up to 100)
//   norm_act   LN / GN / none x activation x lo layout, written into a channel slice of a wider buffer, plus the raw copy
//   upsample2  nearest x2 with the fp16 hi / lo split
//   attention  softmax(q k^T / sqrt(C)) v with logits up to +-60
// The fp16 `hi` must be within 1 fp16 ulp of the fp64 value, hi + lo must reconstruct it to the precision of the lo
// format, and each E5M2 byte must decode to within 2^-3 of its target (see store_hi_lo_t).
//   usage: unet_kernels_test      exit status 0 iff every check passes
#include "unet_kernels.cuh"
#include "conv3d_igemm.cuh"   // kF8Shift

#include <cuda_fp8.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <string>
#include <vector>

using namespace pixie;

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); exit(2); } } while (0)

static int n_run = 0, n_fail = 0;
static void result(const std::string& name, bool ok, const char* detail) {
    ++n_run; n_fail += !ok;
    printf("[%s] %s %s\n", name.c_str(), ok ? "PASS" : "FAIL", detail);
    fflush(stdout);
}

template <typename T> static T* to_dev(const std::vector<T>& h) {
    T* d = nullptr;
    CK(cudaMalloc(&d, h.size() * sizeof(T)));
    CK(cudaMemcpy(d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice));
    return d;
}
template <typename T> static std::vector<T> to_host(const T* d, size_t n) {
    std::vector<T> h(n);
    CK(cudaMemcpy(h.data(), d, n * sizeof(T), cudaMemcpyDeviceToHost));
    return h;
}
static float h2f(__half h) { return __half2float(h); }
static float e5m2f(uint8_t b) { return __half2float(__half(__nv_cvt_fp8_to_halfraw(b, __NV_E5M2))); }
static double ulp16(double f) {                      // fp16 ulp at |f| (subnormal spacing below 2^-14)
    const double a = std::fabs(f);
    return a < std::ldexp(1.0, -14) ? std::ldexp(1.0, -24) : std::ldexp(1.0, (int)std::floor(std::log2(a)) - 10);
}

// Checks of one stored value f (fp64) against its fp16 hi and the lo companion; `lo` points at the start of the lo buffer
// (fp16 elements for lo_mode 0, bytes laid out as in store_hi_lo_t for lo_mode 1), idx is the element index of f.
struct SplitCheck {
    double hi_ulps = 0, lo_rel = 0, e5_rel = 0;
    size_t bad = 0;
    void add(double f, __half hi, const void* lo, int lo_mode, size_t idx, double hi_tol_abs) {
        const double h = h2f(hi);
        const double u = std::fabs(h - f) / ulp16(f);
        hi_ulps = std::max(hi_ulps, u);
        if (std::fabs(h - f) > ulp16(f) + hi_tol_abs) ++bad;
        if (!lo) return;
        if (lo_mode == 0) {
            // fp16 lo carries f - hi to 11 bits: |hi + lo - f| <= 2^-11 |f - hi| + the kernel's fp32 error
            const double l = h2f(reinterpret_cast<const __half*>(lo)[idx]);
            const double e = std::fabs(h + l - f), tol = std::ldexp(std::fabs(f - h), -11) + 4e-7 * std::fabs(f) + hi_tol_abs;
            lo_rel = std::max(lo_rel, e / std::max(std::fabs(f), 1e-30));
            if (e > tol) ++bad;
        } else {
            const uint8_t* row = reinterpret_cast<const uint8_t*>(lo) + 2 * (idx & ~(size_t)63) + (idx & 63);
            const double up = std::ldexp(1.0, kF8Shift), down = 1.0 / up;
            const double t1 = (f - h) * up, t2 = f * down;
            const double d1 = e5m2f(row[0]), d2 = e5m2f(row[64]);
            // E5M2 keeps 2 mantissa bits: 2^-3 relative, plus half its smallest subnormal (2^-17) and the kernel's fp32 error
            const double e1 = std::fabs(d1 - t1), e2 = std::fabs(d2 - t2);
            e5_rel = std::max({e5_rel, e1 / std::max(std::fabs(t1), 1e-30), e2 / std::max(std::fabs(t2), 1e-30)});
            if (e1 > std::ldexp(std::fabs(t1), -3) + std::ldexp(1.0, -17) + (4e-7 * std::fabs(f) + hi_tol_abs) * up) ++bad;
            if (e2 > std::ldexp(std::fabs(t2), -3) + std::ldexp(1.0, -17)) ++bad;
        }
    }
    std::string str() const {
        char b[160];
        snprintf(b, sizeof(b), "hi max %.2f ulp, hi+lo rel %.2e, e5m2 rel %.3f, bad=%zu", hi_ulps, lo_rel, e5_rel, bad);
        return b;
    }
};

// ------------------------------------------------------------------------------------------------ moments
static void test_moments() {
    std::mt19937 g(1);
    std::normal_distribution<double> nd;
    for (int C : {32, 64, 256, 1024})
        for (int V : {1000, 4097})
            for (double ratio : {0.0, 100.0}) {
                const int NB = 2;
                std::vector<float> x((size_t)NB * V * C);
                std::vector<double> mu(NB * C), sg(NB * C);
                for (int i = 0; i < NB * C; ++i) {
                    sg[i] = 0.5 + std::uniform_real_distribution<double>(0, 1)(g);
                    mu[i] = ratio * sg[i] * (i % 2 ? 1 : -1);
                }
                for (int nb = 0; nb < NB; ++nb)
                    for (int v = 0; v < V; ++v)
                        for (int c = 0; c < C; ++c) x[((size_t)nb * V + v) * C + c] = (float)(mu[nb * C + c] + sg[nb * C + c] * nd(g));
                float* dx = to_dev(x);
                double* ds = nullptr;
                CK(cudaMalloc(&ds, (size_t)NB * C * 2 * sizeof(double)));
                CK(cudaMemset(ds, 0, (size_t)NB * C * 2 * sizeof(double)));
                const int rc = launch_moments(dx, NB, V, C, ds, 0);
                CK(cudaDeviceSynchronize());
                const auto st = to_host(ds, (size_t)NB * C * 2);
                double mean_err = 0, var_err = 0;
                for (int nb = 0; nb < NB; ++nb)
                    for (int c = 0; c < C; ++c) {
                        double s = 0;
                        for (int v = 0; v < V; ++v) s += x[((size_t)nb * V + v) * C + c];
                        const double m = s / V;
                        double q = 0;
                        for (int v = 0; v < V; ++v) { const double d = x[((size_t)nb * V + v) * C + c] - m; q += d * d; }
                        const double var = q / V;
                        const double gm = st[((size_t)nb * C + c) * 2] / V, gv = st[((size_t)nb * C + c) * 2 + 1] / V - gm * gm;
                        mean_err = std::max(mean_err, std::fabs(gm - m) / std::sqrt(var));
                        var_err = std::max(var_err, std::fabs(gv - var) / var);
                    }
                // the normaliser uses mean and variance in fp32: 1e-5 of sigma and of the variance is far below that
                const bool ok = rc == 0 && mean_err < 1e-5 && var_err < 1e-5;
                char d[160];
                snprintf(d, sizeof(d), "max |mean err|/sigma %.2e, max var rel err %.2e (bounds 1e-5)", mean_err, var_err);
                result("moments_C" + std::to_string(C) + "_V" + std::to_string(V) + "_mean" + std::to_string((int)ratio) + "sigma", ok, d);
                cudaFree(dx); cudaFree(ds);
            }
}

// ------------------------------------------------------------------------------------------------ norm_act
static double act_ref(double v, int act) {
    if (act == kActLeaky) return v > 0 ? v : 0.02 * v;
    if (act == kActSiLU) return v / (1.0 + std::exp(-v));
    return v;
}

static void test_norm_act() {
    std::mt19937 g(2);
    std::uniform_real_distribution<float> ud(-1.f, 1.f);
    const int NB = 2, sp = 6, V = sp * sp * sp, C = 64;
    const int ld = 192, c0 = 64, raw_ld = 128, raw_c0 = 64;      // a 64-channel slice of wider buffers
    const char* mode_name[] = {"none", "ln", "gn"};
    const char* act_name[] = {"id", "leaky", "silu"};
    std::vector<float> x((size_t)NB * V * C);
    for (size_t i = 0; i < x.size(); ++i) x[i] = 3.f * ud(g) + 0.5f * (float)((i % C) % 5);
    std::vector<float> gam_v(V), bet_v(V), gam_c(C), bet_c(C);
    for (auto& v : gam_v) v = 1.f + 0.2f * ud(g);
    for (auto& v : bet_v) v = 0.2f * ud(g);
    for (auto& v : gam_c) v = 1.f + 0.2f * ud(g);
    for (auto& v : bet_c) v = 0.2f * ud(g);
    std::vector<double> stats((size_t)NB * C * 2, 0.0);
    for (int nb = 0; nb < NB; ++nb)
        for (int v = 0; v < V; ++v)
            for (int c = 0; c < C; ++c) {
                const double a = x[((size_t)nb * V + v) * C + c];
                stats[((size_t)nb * C + c) * 2] += a;
                stats[((size_t)nb * C + c) * 2 + 1] += a * a;
            }
    float *dx = to_dev(x), *dgv = to_dev(gam_v), *dbv = to_dev(bet_v), *dgc = to_dev(gam_c), *dbc = to_dev(bet_c);
    double* dst = to_dev(stats);
    const size_t n_dst = (size_t)NB * V * ld, n_raw = (size_t)NB * V * raw_ld;
    __half *d_hi, *d_lo, *d_raw, *d_rawlo;
    CK(cudaMalloc(&d_hi, n_dst * 2)); CK(cudaMalloc(&d_lo, n_dst * 2));
    CK(cudaMalloc(&d_raw, n_raw * 2)); CK(cudaMalloc(&d_rawlo, n_raw * 2));
    for (int mode : {kNormNone, kNormLN, kNormGN})
        for (int groups : (mode == kNormGN ? std::vector<int>{32, 16, 8} : std::vector<int>{1}))   // cg = 2, 4, 8
            for (int act : {kActNone, kActLeaky, kActSiLU})
                for (int lom : {-1, 0, 1}) {                     // -1: no lo tensor
                    CK(cudaMemset(d_hi, 0x5A, n_dst * 2)); CK(cudaMemset(d_lo, 0x5A, n_dst * 2));
                    CK(cudaMemset(d_raw, 0x5A, n_raw * 2)); CK(cudaMemset(d_rawlo, 0x5A, n_raw * 2));
                    NormArgs a;
                    a.x = dx; a.V = V; a.C = C; a.mode = mode; a.groups = groups; a.act = act; a.eps = 1e-5f;
                    a.stats = mode == kNormNone ? nullptr : dst;
                    a.gamma = mode == kNormLN ? dgv : dgc; a.beta = mode == kNormLN ? dbv : dbc;
                    a.lo_mode = lom < 0 ? 0 : lom;
                    a.dst = d_hi; a.dst_lo = lom < 0 ? nullptr : d_lo; a.dst_ld = ld; a.dst_c0 = c0;
                    a.raw_dst = d_raw; a.raw_lo = lom < 0 ? nullptr : d_rawlo; a.raw_ld = raw_ld; a.raw_c0 = raw_c0;
                    const int rc = launch_norm_act(a, NB, 0);
                    CK(cudaDeviceSynchronize());
                    const auto hi = to_host(d_hi, n_dst), lo = to_host(d_lo, n_dst), raw = to_host(d_raw, n_raw), rawlo = to_host(d_rawlo, n_raw);
                    SplitCheck sc, rc_raw;
                    const int cg = mode == kNormGN ? C / groups : 1;
                    for (int nb = 0; nb < NB; ++nb)
                        for (int v = 0; v < V; ++v)
                            for (int c = 0; c < C; ++c) {
                                const double xv = x[((size_t)nb * V + v) * C + c];
                                double y = xv;
                                if (mode != kNormNone) {
                                    double s = 0, q = 0;
                                    const int gc0 = c / cg * cg;
                                    for (int k = 0; k < cg; ++k) { s += stats[((size_t)nb * C + gc0 + k) * 2]; q += stats[((size_t)nb * C + gc0 + k) * 2 + 1]; }
                                    const double n = (double)V * cg, m = s / n, var = q / n - m * m;
                                    const double gm = mode == kNormLN ? gam_v[v] : gam_c[c], bt = mode == kNormLN ? bet_v[v] : bet_c[c];
                                    y = (xv - m) / std::sqrt(var + 1e-5) * gm + bt;
                                }
                                const double f = act_ref(y, act);
                                const size_t i = ((size_t)nb * V + v) * ld + c0 + c, ir = ((size_t)nb * V + v) * raw_ld + raw_c0 + c;
                                sc.add(f, hi[i], lom < 0 ? nullptr : lo.data(), a.lo_mode, i, 1e-6 * (1 + std::fabs(f)));
                                rc_raw.add(xv, raw[ir], lom < 0 ? nullptr : rawlo.data(), a.lo_mode, ir, 0.0);
                                if (__half_as_ushort(raw[ir]) != __half_as_ushort(__float2half_rn((float)xv))) ++rc_raw.bad;
                            }
                    // the neighbouring channel slices (and, without a lo tensor, the whole lo buffer) stay untouched
                    size_t touched = 0;
                    auto untouched = [](__half h) { return __half_as_ushort(h) == 0x5A5A; };
                    for (size_t r = 0; r < (size_t)NB * V; ++r) {
                        for (int c = 0; c < ld; ++c) {
                            const bool mine = c >= c0 && c < c0 + C;
                            if (!mine && !untouched(hi[r * ld + c])) ++touched;
                            if ((!mine || lom < 0) && !untouched(lo[r * ld + c])) ++touched;
                        }
                        for (int c = 0; c < raw_ld; ++c) {
                            const bool mine = c >= raw_c0 && c < raw_c0 + C;
                            if (!mine && !untouched(raw[r * raw_ld + c])) ++touched;
                            if ((!mine || lom < 0) && !untouched(rawlo[r * raw_ld + c])) ++touched;
                        }
                    }
                    const bool ok = rc == 0 && sc.bad == 0 && rc_raw.bad == 0 && touched == 0;
                    char d[400];
                    snprintf(d, sizeof(d), "out: %s | raw: %s | outside the slices: %zu", sc.str().c_str(), rc_raw.str().c_str(), touched);
                    result(std::string("norm_act_") + mode_name[mode] + (mode == kNormGN ? "_cg" + std::to_string(C / groups) : "") + "_" +
                           act_name[act] + "_lo" + (lom < 0 ? "none" : lom == 0 ? "fp16" : "e5m2"), ok, d);
                }
    cudaFree(dx); cudaFree(dgv); cudaFree(dbv); cudaFree(dgc); cudaFree(dbc); cudaFree(dst);
    cudaFree(d_hi); cudaFree(d_lo); cudaFree(d_raw); cudaFree(d_rawlo);
}

// ------------------------------------------------------------------------------------------------ upsample2
static void test_upsample2() {
    std::mt19937 g(3);
    std::uniform_real_distribution<float> ud(-4.f, 4.f);
    const int NB = 2, C = 64;
    for (int sp : {1, 3, 6})
        for (int lom : {-1, 0, 1}) {
            const int S = 2 * sp;
            std::vector<float> x((size_t)NB * sp * sp * sp * C);
            for (auto& v : x) v = ud(g);
            float* dx = to_dev(x);
            const size_t n = (size_t)NB * S * S * S * C;
            __half *dy, *dlo;
            CK(cudaMalloc(&dy, n * 2)); CK(cudaMalloc(&dlo, n * 2));
            CK(cudaMemset(dy, 0x5A, n * 2)); CK(cudaMemset(dlo, 0x5A, n * 2));
            const int rc = launch_upsample2(dx, dy, lom < 0 ? nullptr : dlo, lom < 0 ? 0 : lom, NB, sp, C, 0);
            CK(cudaDeviceSynchronize());
            const auto y = to_host(dy, n), lo = to_host(dlo, n);
            SplitCheck sc;
            size_t not_exact = 0;
            for (int nb = 0; nb < NB; ++nb)
                for (int d = 0; d < S; ++d)
                    for (int h = 0; h < S; ++h)
                        for (int w = 0; w < S; ++w)
                            for (int c = 0; c < C; ++c) {
                                const float f = x[((((size_t)nb * sp + d / 2) * sp + h / 2) * sp + w / 2) * C + c];
                                const size_t i = ((((size_t)nb * S + d) * S + h) * S + w) * C + c;
                                not_exact += __half_as_ushort(y[i]) != __half_as_ushort(__float2half_rn(f));
                                sc.add(f, y[i], lom < 0 ? nullptr : lo.data(), lom < 0 ? 0 : lom, i, 0.0);
                            }
            size_t touched = 0;
            if (lom < 0) for (auto h : lo) touched += __half_as_ushort(h) != 0x5A5A;
            char d[300];
            snprintf(d, sizeof(d), "hi not bit-exact: %zu | %s | lo written without a lo tensor: %zu", not_exact, sc.str().c_str(), touched);
            result("upsample2_sp" + std::to_string(sp) + "_lo" + (lom < 0 ? "none" : lom == 0 ? "fp16" : "e5m2"),
                   rc == 0 && not_exact == 0 && sc.bad == 0 && touched == 0, d);
            cudaFree(dx); cudaFree(dy); cudaFree(dlo);
        }
}

// ------------------------------------------------------------------------------------------------ attention
static void test_attention() {
    std::mt19937 g(4);
    std::normal_distribution<float> nd;
    const int NB = 2;
    for (int C : {64, 256})
        for (int T : {1, 27, 216, 512}) {
            std::vector<float> qkv((size_t)NB * T * 3 * C);
            for (auto& v : qkv) v = nd(g);
            // scale q and k so that the largest |logit| = |q.k| / sqrt(C) is 60
            double mx = 0;
            for (int nb = 0; nb < NB; ++nb)
                for (int t = 0; t < T; ++t)
                    for (int s = 0; s < T; ++s) {
                        double l = 0;
                        for (int c = 0; c < C; ++c) l += (double)qkv[((size_t)nb * T + t) * 3 * C + c] * qkv[((size_t)nb * T + s) * 3 * C + C + c];
                        mx = std::max(mx, std::fabs(l) / std::sqrt((double)C));
                    }
            const float k = (float)std::sqrt(60.0 / mx);
            for (int nb = 0; nb < NB; ++nb)
                for (int t = 0; t < T; ++t)
                    for (int c = 0; c < 2 * C; ++c) qkv[((size_t)nb * T + t) * 3 * C + c] *= k;
            float* dq = to_dev(qkv);
            const size_t n = (size_t)NB * T * C;
            for (int lom : {0, 1}) {
                __half *dy, *dlo;
                CK(cudaMalloc(&dy, n * 2)); CK(cudaMalloc(&dlo, n * 2));
                const int rc = launch_attention(dq, dy, dlo, lom, NB, T, C, 0);
                CK(cudaDeviceSynchronize());
                const auto y = to_host(dy, n), lo = to_host(dlo, n);
                SplitCheck sc;
                double max_logit = 0;
                for (int nb = 0; nb < NB; ++nb)
                    for (int t = 0; t < T; ++t) {
                        std::vector<double> l(T);
                        double m = -1e300;
                        for (int s = 0; s < T; ++s) {
                            double acc = 0;
                            for (int c = 0; c < C; ++c) acc += (double)qkv[((size_t)nb * T + t) * 3 * C + c] * qkv[((size_t)nb * T + s) * 3 * C + C + c];
                            l[s] = acc / std::sqrt((double)C);
                            m = std::max(m, l[s]);
                            max_logit = std::max(max_logit, std::fabs(l[s]));
                        }
                        double z = 0;
                        for (int s = 0; s < T; ++s) { l[s] = std::exp(l[s] - m); z += l[s]; }
                        for (int c = 0; c < C; ++c) {
                            double o = 0;
                            for (int s = 0; s < T; ++s) o += l[s] * qkv[((size_t)nb * T + s) * 3 * C + 2 * C + c];
                            // fp32 logits of magnitude 60 carry ~1e-5 absolute error into the weights
                            sc.add(o / z, y[((size_t)nb * T + t) * C + c], lo.data(), lom, ((size_t)nb * T + t) * C + c, 1e-4);
                        }
                    }
                char d[300];
                snprintf(d, sizeof(d), "max |logit| %.1f | %s", max_logit, sc.str().c_str());
                result("attention_C" + std::to_string(C) + "_T" + std::to_string(T) + (lom ? "_loe5m2" : "_lofp16"), rc == 0 && sc.bad == 0, d);
                cudaFree(dy); cudaFree(dlo);
            }
            cudaFree(dq);
        }
}

int main() {
    test_moments();
    test_norm_act();
    test_upsample2();
    test_attention();
    printf("SUMMARY run=%d fail=%d\n", n_run, n_fail);
    return n_fail ? 1 : 0;
}
