// Standalone test of the wgmma implicit-GEMM conv (not part of the product library). Every case goes through the same host
// planner the U-Net executor uses, and every checked output element is compared with an fp64 host reference of exactly the
// products the kernel is asked to compute, under a per-element bound set by fp32 (and E5M2) accumulation:
//     |got - ref| <= kTau * S + kTau8 * S8,
//     S  = sum |a_i w_i| over the fp16 products + |bias| + |residual|,   S8 = sum |a1 w1| + |a2 w2| over the E5M2 products.
// The split-precision modes are also checked against the exact product a*w of the un-rounded operands. A few large cases
// are timed as well.
//   usage: conv_test [case-filter-substring]      exit status 0 iff every selected case passes
#include "conv3d_igemm.cuh"

#include <cuda_fp8.h>
#include <omp.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <random>
#include <string>
#include <vector>

using namespace pixie;

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); exit(2); } } while (0)

// Per-element error bound (see the header comment). Measured on an H100 SXM (80 GB HBM3, 400 W power limit) over all
// cases: max err/S = 2^-20.67 (fp16 cases) and 2^-21.15 (fp16x3 cases), so kTau has 1.6x headroom. Every E5M2 element
// was within kTau * S alone (max (err - kTau S)/S8 = 0): kTau8 is the allowance for the narrower accumulation of E5M2
// products (DESIGN.md, "E5M2 before fp16"), about 2^-12 of their magnitude, not a measured error.
constexpr double kTau = 1.0 / (1 << 20);
constexpr double kTau8 = 1.0 / (1 << 12);
// The host reference checks every voxel up to this many multiply-adds per case, else the tile-edge sample below.
constexpr double kFullCheckMacs = 2e8;
// Least improvement of fp16x3 over a single fp16 pass, both measured against the exact a*w. The main pass's own fp32
// accumulation error bounds it: measured 635x at K = 128, 96-123x at K = 1728, 61x at K = 6912 (split-K) on the H100.
constexpr double kX3Gain = 32.0;

enum { kF16 = 0, kX3 = 1, kE5 = 2 };                 // numerics: one fp16 pass / three fp16 passes (hi, lo, w_lo) / fp16 + E5M2
enum { kNoStats = 0, kChanStats = 1, kScalarStats = 2 };
static const char* const kPrecName[] = {"fp16", "fp16x3", "fp16e5"};
static const char* const kStatsName[] = {"none", "channel", "scalar"};

struct Case {
    std::string tag, name;
    int NB = 1, Dout = 16, stride = 1;
    std::vector<int> srcC;                 // channels (padded to 64) per source
    std::vector<int> srcCreal;
    std::vector<std::pair<int, int>> segs; // (src, ks)
    int Cout = 64;
    bool bias = true, residual = false, planar = false;
    int split_k = 1, block_n = 0, td = 0;  // 0: the planner chooses
    int nv = 0;                            // channel-major voxel tile; 0: the planner chooses
    bool forced = false;                   // block_n and td (voxel-major) or nv (channel-major) are forced: the plan must use them
    bool want_split = false;               // the planner must choose split-K
    bool timing = false;
    int prec = kF16;
    int stats = kChanStats;                // statistics requested from the epilogue
    int launch_nb = 0;                     // > 0: planned for NB items, launched for this many (as the executor does)
};

struct Totals {
    int n_run = 0, n_fail = 0;
    double r = 0, rx3 = 0, r8 = 0;         // max err/S (fp16 cases, fp16x3 cases), max (err - kTau S)/S8 (E5M2 cases)
    std::string r_case, rx3_case, r8_case;
    double e5_ratio = 1e30, x3_ratio = 1e30;   // min over cases of (single fp16 pass error) / (corrected error), vs a*w
    std::map<std::string, int> inst;           // kernel instance ("vm(block_n,TD)" or "cm(NV)") -> cases that ran on it
    std::map<std::string, int> tags;
};

static float frand(std::mt19937& g) { return std::uniform_real_distribution<float>(-1.f, 1.f)(g); }
static float f16r(float v) { return __half2float(__float2half(v)); }
static uint8_t e5m2(float v) { return (uint8_t)__nv_cvt_float_to_fp8(v, __NV_SATFINITE, __NV_E5M2); }
static float e5m2f(uint8_t b) { return __half2float(__half(__nv_cvt_fp8_to_halfraw(b, __NV_E5M2))); }

static bool run_case(const Case& c, int* d_err, Totals& T) {
    std::mt19937 gen(1234);
    const int Do = c.Dout, Di = c.Dout * c.stride, NB = c.NB, nl = c.launch_nb ? c.launch_nb : c.NB;
    const size_t vin = (size_t)Di * Di * Di, vout = (size_t)Do * Do * Do;
    const int nsrc = (int)c.srcC.size(), nseg = (int)c.segs.size();
    const float up = (float)(1 << kF8Shift), down = 1.0f / up;
    std::vector<void*> dev;
    auto dmalloc = [&](size_t bytes) { void* p = nullptr; CK(cudaMalloc(&p, bytes)); dev.push_back(p); return p; };
    auto upload = [&](const void* h, size_t bytes) { void* p = dmalloc(bytes); CK(cudaMemcpy(p, h, bytes, cudaMemcpyHostToDevice)); return p; };

    ConvDesc d;
    d.NB = NB; d.D = d.H = d.W = Do; d.stride = c.stride; d.Cout = c.Cout;
    d.Cout_pad = (c.Cout + 15) / 16 * 16;
    d.split_k = c.split_k; d.block_n = c.block_n; d.td = c.td; d.nv = c.nv; d.out_planar = c.planar;

    // ---- activations, built the way the executor's normalise kernel stores them. Host copies are the decoded operands:
    // Ah = fp16(a), Al = fp16(a - Ah) (fp16x3), A1 = e5m2((a - Ah) 2^s), A2 = e5m2(a 2^-s) (fp16e5), At = a.
    std::vector<std::vector<float>> Ah(nsrc), Al(nsrc), A1(nsrc), A2(nsrc), At(nsrc);
    std::vector<ConvSrc> companions;       // companion of source s is source s + nsrc
    for (int s = 0; s < nsrc; ++s) {
        const int C = c.srcC[s];
        const size_t n = (size_t)NB * vin * C;
        std::vector<__half> hi(n), lo;
        std::vector<uint8_t> pair;
        Ah[s].resize(n); At[s].resize(n);
        if (c.prec == kX3) { lo.resize(n); Al[s].resize(n); }
        if (c.prec == kE5) { pair.assign(2 * n, 0); A1[s].resize(n); A2[s].resize(n); }
        for (size_t v = 0; v < (size_t)NB * vin; ++v)
            for (int ch = 0; ch < C; ++ch) {
                const size_t i = v * C + ch;
                const float a = ch < c.srcCreal[s] ? frand(gen) : 0.f;
                hi[i] = __float2half(a);
                Ah[s][i] = __half2float(hi[i]);
                At[s][i] = a;
                if (c.prec == kX3) { lo[i] = __float2half(a - Ah[s][i]); Al[s][i] = __half2float(lo[i]); }
                if (c.prec == kE5) {
                    uint8_t* row = &pair[(v * C + (size_t)(ch & ~63)) * 2];
                    row[ch & 63] = e5m2((a - Ah[s][i]) * up);
                    row[64 + (ch & 63)] = e5m2(a * down);
                    A1[s][i] = e5m2f(row[ch & 63]);
                    A2[s][i] = e5m2f(row[64 + (ch & 63)]);
                }
            }
        d.srcs.push_back({(const __half*)upload(hi.data(), n * 2), C, Di, Di, Di});
        if (c.prec == kX3) companions.push_back({(const __half*)upload(lo.data(), n * 2), C, Di, Di, Di});
        if (c.prec == kE5) companions.push_back({(const __half*)upload(pair.data(), 2 * n), C, Di, Di, Di});
    }
    for (const auto& s : companions) d.srcs.push_back(s);

    // ---- weights: torch layout for the packer; host copies [co][tap][ci] of the decoded operands, as for the activations
    std::vector<std::vector<float>> hw(nseg), Wh(nseg), Wl(nseg), W1(nseg), W2(nseg), Wt(nseg);
    std::vector<const float*> wptr;
    std::vector<int> cin_real;
    for (int g = 0; g < nseg; ++g) {
        const int src = c.segs[g].first, ks = c.segs[g].second, kv = ks * ks * ks, cin = c.srcCreal[src];
        const size_t n = (size_t)c.Cout * cin * kv;
        const float sc = 1.0f / std::sqrt((float)cin * kv);
        hw[g].resize(n);
        for (auto& x : hw[g]) x = c.prec == kF16 ? f16r(frand(gen) * sc) : frand(gen) * sc;
        auto seg = [&](int sidx, int wlo, int f8, int lo) {
            d.segs.push_back({sidx, ks, wlo, f8, lo});
            wptr.push_back(hw[g].data()); cin_real.push_back(cin);
        };
        seg(src, 0, 0, 0);                                // a_hi * w_hi
        if (c.prec == kX3) { seg(src + nsrc, 0, 0, 1); seg(src, 1, 0, 0); }   // a_lo * w_hi, a_hi * w_lo (emit_conv's order)
        if (c.prec == kE5) seg(src + nsrc, 0, 1, 0);      // a_lo * w + a * w_lo in E5M2
        Wh[g].resize(n); Wt[g].resize(n);
        if (c.prec == kX3) Wl[g].resize(n);
        if (c.prec == kE5) { W1[g].resize(n); W2[g].resize(n); }
        for (int co = 0; co < c.Cout; ++co)
            for (int ci = 0; ci < cin; ++ci)
                for (int t = 0; t < kv; ++t) {
                    const float w = hw[g][((size_t)co * cin + ci) * kv + t], wh = f16r(w);
                    const size_t j = ((size_t)co * kv + t) * cin + ci;
                    Wh[g][j] = wh; Wt[g][j] = w;
                    if (c.prec == kX3) Wl[g][j] = f16r(w - wh);
                    if (c.prec == kE5) { W1[g][j] = e5m2f(e5m2(w * down)); W2[g][j] = e5m2f(e5m2((w - wh) * up)); }
                }
    }
    std::vector<__half> packed;
    conv_pack_weights(d, wptr, cin_real, packed);
    d.weights = (const __half*)upload(packed.data(), packed.size() * 2);

    std::vector<float> h_bias(c.Cout), h_res;
    for (auto& x : h_bias) x = frand(gen);
    if (c.bias) d.bias = (const float*)upload(h_bias.data(), c.Cout * 4);
    const size_t item = vout * c.Cout;                   // output floats per batch item (out_ld == Cout)
    if (c.residual) {
        h_res.resize((size_t)NB * item);
        for (auto& x : h_res) x = frand(gen);
        d.residual = (const float*)upload(h_res.data(), h_res.size() * 4);
    }
    // the output holds the launched items only, followed by a guard band that must stay untouched (as long as the planned
    // items, so that a launch writing all of them stays inside this allocation)
    const size_t out_elems = (size_t)nl * item, guard = std::max<size_t>(item * std::max(1, NB - nl), 16384);
    float* d_out = (float*)dmalloc((out_elems + guard) * 4);
    CK(cudaMemset(d_out, 0xFF, out_elems * 4));          // NaN pattern: unwritten outputs are caught
    CK(cudaMemset(d_out + out_elems, 0xA5, guard * 4));
    d.out = d_out; d.out_ld = c.Cout;
    double* d_stats = (double*)dmalloc((size_t)NB * c.Cout * 2 * sizeof(double));
    CK(cudaMemset(d_stats, 0, (size_t)NB * c.Cout * 2 * sizeof(double)));
    d.stats = c.stats != kNoStats ? d_stats : nullptr;
    d.stats_scalar = c.stats == kScalarStats;

    auto cleanup = [&]() { for (void* p : dev) cudaFree(p); };
    CK(cudaMemset(d_err, 0, sizeof(int)));
    ConvPlan plan;
    char err[256] = {0};
    if (conv_plan_create(d, d_err, plan, err, sizeof(err))) {
        printf("[%s] FAIL plan: %s\n", c.name.c_str(), err);
        cleanup();
        return false;
    }
    const std::string inst = plan.channel_major ? "cm(" + std::to_string(plan.p.TH * plan.p.TW) + ")"
                                                : "vm(" + std::to_string(plan.p.block_n) + "," + std::to_string(plan.p.TD) + ")";
    printf("[%s] %s NB=%d launched=%d plan_grid=%d smem=%d %s bn=%d TD=%d TW=%d TH=%d w_stages=%d s_stages=%d phases=%d split=%d stats=%s%s\n",
           c.name.c_str(), kPrecName[c.prec], NB, nl, plan.grid, plan.smem_bytes, inst.c_str(), plan.p.block_n, plan.p.TD, plan.p.TW, plan.p.TH,
           plan.p.w_stages, plan.p.s_stages, plan.p.n_phases, plan.p.split_k, kStatsName[c.stats], plan.fused_stats ? " (fused)" : "");
    fflush(stdout);
    bool plan_ok = true;
    const std::string want = c.nv ? "cm(" + std::to_string(c.nv) + ")"
                                  : "vm(" + std::to_string(c.block_n) + "," + std::to_string(c.td) + ")";
    if (c.forced && inst != want) {
        printf("[%s] forced %s but the plan uses %s\n", c.name.c_str(), want.c_str(), inst.c_str());
        plan_ok = false;
    }
    if (c.want_split && plan.p.split_k == 1) { printf("[%s] expected a split-K plan\n", c.name.c_str()); plan_ok = false; }

    const int lrc = conv_plan_launch(plan, nl, 0);
    const cudaError_t se = cudaDeviceSynchronize();
    int h_err = 0;
    cudaMemcpy(&h_err, d_err, sizeof(int), cudaMemcpyDeviceToHost);
    if (lrc || se != cudaSuccess || h_err) {
        printf("[%s] FAIL launch=%d sync=%s pipeline_timeout_flag=%d\n", c.name.c_str(), lrc, cudaGetErrorString(se), h_err);
        if (se != cudaSuccess) { printf("sticky CUDA error, stopping\n"); exit(3); }
        conv_plan_destroy(plan);
        cleanup();
        return false;
    }
    T.inst[inst]++;

    if (c.timing) {
        cudaEvent_t e0, e1;
        cudaEventCreate(&e0); cudaEventCreate(&e1);
        for (int i = 0; i < 3; ++i) conv_plan_launch(plan, nl, 0);
        const int iters = 20;
        float ms = 0;
        if (getenv("CONV_TEST_COLD")) {
            // cold launches: a 512 MB memset (evicts L2 and the instruction caches' backing lines) before every timed launch
            static void* scrub = nullptr;
            if (!scrub) CK(cudaMalloc(&scrub, 512u << 20));
            for (int i = 0; i < iters; ++i) {
                CK(cudaMemsetAsync(scrub, i, 512u << 20, 0));
                cudaEventRecord(e0);
                conv_plan_launch(plan, nl, 0);
                cudaEventRecord(e1);
                CK(cudaEventSynchronize(e1));
                float t = 0; cudaEventElapsedTime(&t, e0, e1); ms += t;
            }
        } else {
            cudaEventRecord(e0);
            for (int i = 0; i < iters; ++i) conv_plan_launch(plan, nl, 0);
            cudaEventRecord(e1);
            CK(cudaEventSynchronize(e1));
            cudaEventElapsedTime(&ms, e0, e1);
        }
        ms /= iters;
        const double flops = 2.0 * nl * vout * c.Cout * (double)conv_k_total(d);
        printf("[%s] TIME %.3f ms  %.1f TFLOP/s (padded-K flops)\n", c.name.c_str(), ms, flops / ms * 1e-9);
        cudaEventDestroy(e0); cudaEventDestroy(e1);
    }

    std::vector<float> h_out(out_elems + guard);
    CK(cudaMemcpy(h_out.data(), d_out, h_out.size() * 4, cudaMemcpyDeviceToHost));
    size_t guard_bad = 0;
    {
        const uint8_t* gb = reinterpret_cast<const uint8_t*>(h_out.data() + out_elems);
        for (size_t i = 0; i < guard * 4; ++i) guard_bad += gb[i] != 0xA5;
    }
    {
        // FNV-1a over the output bytes, so that two builds can be compared bit for bit. Plain stores after a fixed MMA order
        // make it reproducible; split-K reduces with red.add in arrival order, so its outputs (and the statistics) are not.
        uint64_t hash = 1469598103934665603ull;
        const uint8_t* ob = reinterpret_cast<const uint8_t*>(h_out.data());
        for (size_t i = 0; i < out_elems * 4; ++i) hash = (hash ^ ob[i]) * 1099511628211ull;
        printf("[%s] OUTHASH %016llx%s\n", c.name.c_str(), (unsigned long long)hash,
               plan.p.split_k > 1 ? " (split-K: not deterministic)" : "");
    }

    // ---- voxels to check: all, or (large cases) every voxel on an edge of its tile (at least two of its d, h, w on the
    // first or last index of the tile or of the volume) plus random ones
    double kreal = 0;
    for (const auto& sg : c.segs) kreal += (double)sg.second * sg.second * sg.second * c.srcCreal[sg.first];
    std::vector<size_t> vs;
    if ((double)nl * vout * c.Cout * kreal <= kFullCheckMacs) {
        for (size_t v = 0; v < (size_t)nl * vout; ++v) vs.push_back(v);
    } else {
        auto edge = [&](int x, int t) { return x % t == 0 || x % t == t - 1 || x == Do - 1; };
        std::mt19937 g2(99);
        for (size_t v = 0; v < (size_t)nl * vout; ++v) {
            const int w = (int)(v % Do), h = (int)(v / Do % Do), dd = (int)(v / ((size_t)Do * Do) % Do);
            const int n_edge = edge(dd, plan.p.TD) + edge(h, plan.p.TH) + edge(w, plan.p.TW);
            if (n_edge >= 2 || g2() % 4096 == 0) vs.push_back(v);
        }
    }

    struct Acc {
        double max_err = 0, max_ref = 0, max_bar = 0, r = 0, r8 = 0, true_err = 0, f16_err = 0;
        size_t bad = 0, nan = 0;
    };
    Acc tot;
#pragma omp parallel
    {
        Acc a;
#pragma omp for schedule(dynamic, 8)
        for (long long si = 0; si < (long long)vs.size(); ++si) {
            const size_t v = vs[si], loc = v % vout;
            const int ow = (int)(loc % Do), oh = (int)(loc / Do % Do), od = (int)(loc / ((size_t)Do * Do));
            const int nb = (int)(v / vout);
            for (int co = 0; co < c.Cout; ++co) {
                double ref = c.bias ? h_bias[co] : 0.0, S = std::fabs(ref), S8 = 0, tru = ref, f16 = ref;
                for (int g = 0; g < nseg; ++g) {
                    const int src = c.segs[g].first, ks = c.segs[g].second, pad = ks / 2, kv = ks * ks * ks;
                    const int cin = c.srcCreal[src], C = c.srcC[src];
                    for (int kd = 0; kd < ks; ++kd)
                        for (int kh = 0; kh < ks; ++kh)
                            for (int kw = 0; kw < ks; ++kw) {
                                const int id = od * c.stride + kd - pad, ih = oh * c.stride + kh - pad, iw = ow * c.stride + kw - pad;
                                if (id < 0 || ih < 0 || iw < 0 || id >= Di || ih >= Di || iw >= Di) continue;
                                const size_t xo = ((((size_t)nb * Di + id) * Di + ih) * Di + iw) * C;
                                const size_t wo = ((size_t)co * kv + (kd * ks + kh) * ks + kw) * cin;
                                const float *ah = &Ah[src][xo], *wh = &Wh[g][wo];
                                if (c.prec == kF16) {
                                    for (int ci = 0; ci < cin; ++ci) {
                                        const double p = (double)ah[ci] * wh[ci];
                                        ref += p; S += std::fabs(p);
                                    }
                                    continue;
                                }
                                const float *at = &At[src][xo], *wt = &Wt[g][wo];
                                if (c.prec == kX3) {
                                    const float *al = &Al[src][xo], *wl = &Wl[g][wo];
                                    for (int ci = 0; ci < cin; ++ci) {
                                        const double p0 = (double)ah[ci] * wh[ci], p1 = (double)al[ci] * wh[ci], p2 = (double)ah[ci] * wl[ci];
                                        ref += p0 + p1 + p2; S += std::fabs(p0) + std::fabs(p1) + std::fabs(p2);
                                        f16 += p0; tru += (double)at[ci] * wt[ci];
                                    }
                                } else {
                                    const float *a1 = &A1[src][xo], *a2 = &A2[src][xo], *w1 = &W1[g][wo], *w2 = &W2[g][wo];
                                    for (int ci = 0; ci < cin; ++ci) {
                                        const double p0 = (double)ah[ci] * wh[ci], p1 = (double)a1[ci] * w1[ci], p2 = (double)a2[ci] * w2[ci];
                                        ref += p0 + p1 + p2; S += std::fabs(p0); S8 += std::fabs(p1) + std::fabs(p2);
                                        f16 += p0; tru += (double)at[ci] * wt[ci];
                                    }
                                }
                            }
                }
                const size_t oidx = c.planar ? ((size_t)nb * c.Cout + co) * vout + loc : v * c.Cout + co;
                if (c.residual) { const double r = h_res[oidx]; ref += r; tru += r; f16 += r; S += std::fabs(r); }
                const double got = h_out[oidx];
                if (std::isnan(got)) { ++a.nan; continue; }
                const double e = std::fabs(got - ref), bar = kTau * S + kTau8 * S8;
                if (e > bar) {
                    if (a.bad++ < 3) printf("   mismatch nb=%d d=%d h=%d w=%d co=%d: got %.9g ref %.9g err %.3e bar %.3e\n", nb, od, oh, ow, co, got, ref, e, bar);
                }
                if (c.prec == kE5) { if (S8 > 0) a.r8 = std::max(a.r8, std::max(0.0, e - kTau * S) / S8); }
                else if (S > 0) a.r = std::max(a.r, e / S);
                if (c.prec != kF16) {
                    a.true_err = std::max(a.true_err, std::fabs(got - tru));
                    a.f16_err = std::max(a.f16_err, std::fabs(f16 - tru));
                }
                a.max_err = std::max(a.max_err, e);
                a.max_ref = std::max(a.max_ref, std::fabs(ref));
                a.max_bar = std::max(a.max_bar, bar);
            }
        }
#pragma omp critical
        {
            tot.max_err = std::max(tot.max_err, a.max_err); tot.max_ref = std::max(tot.max_ref, a.max_ref);
            tot.max_bar = std::max(tot.max_bar, a.max_bar); tot.r = std::max(tot.r, a.r); tot.r8 = std::max(tot.r8, a.r8);
            tot.true_err = std::max(tot.true_err, a.true_err); tot.f16_err = std::max(tot.f16_err, a.f16_err);
            tot.bad += a.bad; tot.nan += a.nan;
        }
    }

    // ---- fused statistics: per-(item, channel) sum and sum of squares of the outputs; nothing for items not launched
    size_t stats_bad = 0;
    if (plan.fused_stats && !c.timing) {
        std::vector<double> h_stats((size_t)NB * c.Cout * 2);
        CK(cudaMemcpy(h_stats.data(), d_stats, h_stats.size() * sizeof(double), cudaMemcpyDeviceToHost));
        const bool scalar = c.stats == kScalarStats;
        for (int nb = 0; nb < NB; ++nb) {
            double ts = 0, tq = 0, gts = 0, gtq = 0;
            for (int co = 0; co < c.Cout; ++co) {
                const double gs = h_stats[((size_t)nb * c.Cout + co) * 2], gq = h_stats[((size_t)nb * c.Cout + co) * 2 + 1];
                if (nb >= nl) { stats_bad += (gs != 0 || gq != 0); continue; }
                double s = 0, q = 0;
                for (size_t v = 0; v < vout; ++v) { const double x = h_out[((size_t)nb * vout + v) * c.Cout + co]; s += x; q += x * x; }
                ts += s; tq += q; gts += gs; gtq += gq;
                if (scalar) {
                    if (co > 0 && (gs != 0 || gq != 0)) ++stats_bad;      // totals live in channel 0's slot only
                    continue;
                }
                if (std::fabs(gs - s) > 1e-3 * (1 + std::fabs(s)) + 1e-4 * std::sqrt(q * vout) || std::fabs(gq - q) > 1e-4 * (1 + q)) {
                    if (stats_bad < 3) printf("   stats mismatch nb=%d co=%d: sum %g vs %g, sumsq %g vs %g\n", nb, co, gs, s, gq, q);
                    ++stats_bad;
                }
            }
            if (nb < nl && scalar && (std::fabs(gts - ts) > 1e-5 * std::sqrt(tq * vout * c.Cout) + 1e-6 || std::fabs(gtq - tq) > 1e-6 * (1 + tq))) {
                printf("   scalar stats mismatch nb=%d: sum %.9g vs %.9g, sumsq %.9g vs %.9g\n", nb, gts, ts, gtq, tq);
                ++stats_bad;
            }
        }
    }

    bool acc_ok = true;
    if (c.prec != kF16) {
        const double need = c.prec == kE5 ? 4.0 : kX3Gain, ratio = tot.f16_err / std::max(tot.true_err, 1e-300);
        acc_ok = ratio >= need;
        printf("[%s] vs exact a*w: corrected %.3e, single fp16 pass %.3e, improvement %.1fx (need >= %.0fx)\n", c.name.c_str(),
               tot.true_err, tot.f16_err, ratio, need);
        double& worst = c.prec == kE5 ? T.e5_ratio : T.x3_ratio;
        worst = std::min(worst, ratio);
    }
    if (c.prec == kF16 && tot.r > T.r) { T.r = tot.r; T.r_case = c.name; }
    if (c.prec == kX3 && tot.r > T.rx3) { T.rx3 = tot.r; T.rx3_case = c.name; }
    if (tot.r8 > T.r8) { T.r8 = tot.r8; T.r8_case = c.name; }
    const bool pass = plan_ok && acc_ok && tot.bad == 0 && tot.nan == 0 && stats_bad == 0 && guard_bad == 0;
    printf("[%s] %s checked=%zu/%zu voxels max_err=%.3e max_bar=%.3e max_ref=%.3f err/S=%.3e err8/S8=%.3e bad=%zu nan=%zu stats_bad=%zu guard_bad=%zu\n",
           c.name.c_str(), pass ? "PASS" : "FAIL", vs.size(), (size_t)nl * vout, tot.max_err, tot.max_bar, tot.max_ref, tot.r, tot.r8,
           tot.bad, tot.nan, stats_bad, guard_bad);
    fflush(stdout);
    conv_plan_destroy(plan);
    cleanup();
    return pass;
}

int main(int argc, char** argv) {
    const char* filter = argc > 1 ? argv[1] : "";
    std::vector<Case> cases;
    // one source of Cin channels (all real), one segment
    auto add = [&](const char* tag, const std::string& name, int NB, int Do, int stride, int Cin, int ks, int Cout, int prec = kF16) -> Case& {
        Case c;
        c.tag = tag; c.name = name; c.NB = NB; c.Dout = Do; c.stride = stride;
        c.srcC = {Cin}; c.srcCreal = {Cin}; c.segs = {{0, ks}}; c.Cout = Cout; c.prec = prec;
        cases.push_back(c);
        return cases.back();
    };
    // the concatenated input of an output block: a 3x3x3 conv over `a` plus the 1x1 skip conv over the raw input `b`
    auto add_cat = [&](const char* tag, const std::string& name, int NB, int Do, int Ca, int Cb, int Cout, int prec) -> Case& {
        Case& c = add(tag, name, NB, Do, 1, Ca, 3, Cout, prec);
        c.srcC = {Ca, Cb}; c.srcCreal = {Ca, Cb}; c.segs = {{0, 3}, {1, 1}};
        return c;
    };

    // ---- basic shapes
    add("base", "gemm1x1_64_64_d16", 1, 16, 1, 64, 1, 64).bias = false;
    add("base", "gemm1x1_128_32_d16", 1, 16, 1, 128, 1, 32);
    add("base", "conv3_64_64_d16", 1, 16, 1, 64, 3, 64).bias = false;
    { Case& c = add("base", "conv3_64_64_d16_td1", 1, 16, 1, 64, 3, 64); c.td = 1; }
    { Case& c = add("base", "conv3_32pad_64_d16", 2, 16, 1, 64, 3, 64); c.srcCreal = {32}; }
    { Case& c = add("base", "conv3_cat_skip_d16", 1, 16, 1, 128, 3, 64); c.srcC = c.srcCreal = {128, 64, 64};
      c.segs = {{0, 3}, {1, 1}, {2, 1}}; c.residual = true; }
    add("base", "conv3_128_128_d16", 1, 16, 1, 128, 3, 128).residual = true;
    { Case& c = add("base", "conv3_256_256_d8_splitk", 1, 8, 1, 256, 3, 256); c.residual = true; c.split_k = 0; c.want_split = true; }
    add("base", "conv3_s2_64_64_d16to8", 1, 8, 2, 64, 3, 64);
    add("base", "conv3_s2_64_64_d32to16", 1, 16, 2, 64, 3, 64);
    add("base", "head_64_3_planar_d16", 1, 16, 1, 64, 3, 3).planar = true;
    add("base", "qkv_256_768_d8", 1, 8, 1, 256, 1, 768);
    add("base", "conv3_256_256_d4", 1, 4, 1, 256, 3, 256).split_k = 0;
    // ---- fp16 + E5M2 corrections
    add("e5", "x2_gemm1x1_128_64_d16", 1, 16, 1, 128, 1, 64, kE5);
    add("e5", "x2_conv3_64_64_d16", 1, 16, 1, 64, 3, 64, kE5).residual = true;
    add("e5", "x2_conv3_128_128_d16", 2, 16, 1, 128, 3, 128, kE5);
    add("e5", "x2_conv3_s2_64_64_d16to8", 1, 8, 2, 64, 3, 64, kE5);
    add("e5", "x2_conv3_256_256_d8_splitk", 1, 8, 1, 256, 3, 256, kE5).split_k = 0;
    // ---- three fp16 passes on hi / lo split operands
    add("x3", "x3_gemm1x1_128_64_d16", 1, 16, 1, 128, 1, 64, kX3);
    add("x3", "x3_conv3_64_64_d16", 1, 16, 1, 64, 3, 64, kX3).residual = true;
    add("x3", "x3_conv3_s2_64_64_d16to8", 2, 8, 2, 64, 3, 64, kX3);
    add_cat("x3", "x3_cat_skip_128_64_d12", 2, 12, 64, 128, 64, kX3);
    add("x3", "x3_conv3_256_256_d8_splitk", 1, 8, 1, 256, 3, 256, kX3).split_k = 0;
    add("x3", "x3_head_64_3_planar_d16_splitk", 2, 16, 1, 64, 3, 3, kX3).planar = true;
    cases.back().split_k = 0; cases.back().want_split = true;

    // ---- every voxel-major kernel instance, forced, on a 3x3x3 stride-1, a stride-2 and a 1x1 conv with 48 output channels
    // (a partial channel tile), in fp16 and with E5M2
    const struct { const char* kind; int stride, ks, Cin; } kinds[] = {{"c3", 1, 3, 64}, {"s2", 2, 3, 64}, {"1x1", 1, 1, 128}};
    for (int prec : {kF16, kE5})
        for (int bn : {16, 32})
            for (int td : {1, 2, 4}) {
                const std::string sfx = "_bn" + std::to_string(bn) + "_td" + std::to_string(td) + (prec == kE5 ? "_e5" : "");
                for (const auto& k : kinds) {
                    Case& c = add("instance", std::string("inst_") + k.kind + sfx, 1, 8, k.stride, k.Cin, k.ks, 48, prec);
                    c.block_n = bn; c.td = td; c.forced = true;
                }
            }
    // ---- every channel-major instance, forced: the same three kinds with 96 output channels (a partial channel tile) in
    // fp16 and with E5M2, then at 9^3 (ragged sides for every tile, a last tile with one plane): concatenated sources with the
    // fused skip and a residual, split-K, a short batch, each statistics mode
    for (int nv : {64, 128, 256}) {
        const std::string sn = "_nv" + std::to_string(nv);
        auto force = [&](Case& c) { c.nv = nv; c.forced = true; return &c; };
        for (int prec : {kF16, kE5})
            for (const auto& k : kinds)
                force(add("instance", std::string("cm_") + k.kind + sn + (prec == kE5 ? "_e5" : ""), 1, 8, k.stride, k.Cin, k.ks, 96, prec));
        force(add_cat("instance", "cm_cat_skip_res_d9" + sn, 2, 9, 64, 128, 64, kE5))->residual = true;
        { Case* c = force(add("instance", "cm_splitk_res_d9" + sn, 1, 9, 1, 128, 3, 128, kE5)); c->split_k = 3; c->residual = true;
          c->want_split = true; }
        { Case* c = force(add("instance", "cm_short_d9" + sn + "_nb3_launch2", 3, 9, 1, 64, 3, 64)); c->launch_nb = 2; c->residual = true; }
        force(add("instance", "cm_scalar_stats_d9" + sn, 2, 9, 1, 64, 3, 64, kE5))->stats = kScalarStats;
        force(add("instance", "cm_no_stats_s2_d9" + sn, 1, 9, 2, 64, 3, 64))->stats = kNoStats;
        force(add("instance", "cm_x3_1x1_d9" + sn, 2, 9, 1, 128, 1, 64, kX3));
    }

    // ---- ragged geometry: the grid sides the U-Net reaches at grid_size 24 / 48, partial depth and channel tiles
    for (int D : {3, 6, 12, 24}) add("ragged", "r_conv3_64_64_d" + std::to_string(D), D <= 6 ? 2 : 1, D, 1, 64, 3, 64);
    for (int D : {3, 6, 12}) add("ragged", "r_conv3_64_64_d" + std::to_string(D) + "_e5", 2, D, 1, 64, 3, 64, kE5).residual = true;
    add("ragged", "r_s2_64_64_d6to3", 2, 3, 2, 64, 3, 64);
    add("ragged", "r_s2_64_64_d12to6", 1, 6, 2, 64, 3, 64);
    add("ragged", "r_s2_64_64_d12to6_e5", 2, 6, 2, 64, 3, 64, kE5);
    { Case& c = add("ragged", "r_td4_d6_tde2", 2, 6, 1, 64, 3, 32); c.block_n = 32; c.td = 4; c.forced = true; }
    { Case& c = add("ragged", "r_td4_d6_tde2_e5", 1, 6, 1, 64, 3, 32, kE5); c.block_n = 32; c.td = 4; c.forced = true; }
    add("ragged", "r_cout8_d12", 1, 12, 1, 64, 3, 8);
    add("ragged", "r_cout80_d12", 1, 12, 1, 64, 3, 80).residual = true;
    add("ragged", "r_cout192_d6", 2, 6, 1, 128, 3, 192);
    add("ragged", "r_cout80_d6_e5", 1, 6, 1, 64, 3, 80, kE5);
    add_cat("ragged", "r_block_e5_cat_skip_128_64_d12", 2, 12, 64, 128, 64, kE5);          // 4 slots, fused statistics
    { Case& c = add("ragged", "r_head_e5_planar_splitk_d16", 2, 16, 1, 64, 3, 3, kE5); c.planar = true; c.split_k = 0; c.want_split = true; }
    { Case& c = add("ragged", "r_head_e5_planar_splitk_d24", 1, 24, 1, 64, 3, 3, kE5); c.planar = true; c.split_k = 0; c.want_split = true; }

    // ---- short batches: planned for 3 items, launched for fewer into an output that holds only those
    for (int nl : {1, 2}) {
        const std::string s = "_nb3_launch" + std::to_string(nl);
        { Case& c = add("short", "sb_conv3_64_64_d8" + s, 3, 8, 1, 64, 3, 64); c.launch_nb = nl; c.residual = true; }
        { Case& c = add("short", "sb_conv3_64_64_d8_split4" + s, 3, 8, 1, 64, 3, 64); c.launch_nb = nl; c.split_k = 4; c.want_split = true; }
        { Case& c = add("short", "sb_head_planar_splitk_d16" + s, 3, 16, 1, 64, 3, 3, kE5); c.launch_nb = nl; c.planar = true;
          c.split_k = 0; c.want_split = true; }
        { Case& c = add("short", "sb_s2_e5_scalar_d12to6" + s, 3, 6, 2, 64, 3, 64, kE5); c.launch_nb = nl; c.stats = kScalarStats; }
    }

    // ---- statistics modes of the epilogue
    add("stats", "st_scalar_conv3_64_64_d12", 2, 12, 1, 64, 3, 64).stats = kScalarStats;
    add("stats", "st_none_conv3_64_64_d12", 2, 12, 1, 64, 3, 64).stats = kNoStats;
    add_cat("stats", "st_scalar_e5_cat_skip_d12", 2, 12, 64, 128, 64, kE5).stats = kScalarStats;
    add("stats", "st_none_x3_conv3_d6", 2, 6, 1, 64, 3, 64, kX3).stats = kNoStats;

    // ---- 64^3: several tiles per CTA and batch-item boundaries crossed (tile-edge sample), timed
    auto add_t = [&](const std::string& name, int NB, int Cin, int ks, int Cout, int prec) {
        Case& c = add("timing", name, NB, 64, 1, Cin, ks, Cout, prec);
        c.timing = true;
        return &c;
    };
    add_t("T_x2_conv3_64_64_d64_nb2", 2, 64, 3, 64, kE5);
    add_t("T_x2_conv3_128_64_d64", 1, 128, 3, 64, kE5)->residual = true;
    add_t("T_x3_conv3_64_64_d64", 1, 64, 3, 64, kX3);
    add_t("T_x2_conv3_128_128_d64", 1, 128, 3, 128, kE5);
    add_t("T_conv3_64_64_d64", 1, 64, 3, 64, kF16);
    add_t("T_conv3_128_64_d64", 1, 128, 3, 64, kF16)->residual = true;
    add_t("T_conv3_128_128_d64", 1, 128, 3, 128, kF16);
    add_t("T_gemm1x1_512_128_d64", 1, 512, 1, 128, kF16);
    {
        Case& c = add("timing", "T_conv3_64_64_d32", 1, 32, 1, 64, 3, 64); c.timing = true;
        Case& c2 = add("timing", "T_conv3_256_256_d8", 1, 8, 1, 256, 3, 256); c2.timing = true; c2.split_k = 0;
        Case& c3 = add("timing", "T_conv3_128_128_d16", 1, 16, 1, 128, 3, 128); c3.timing = true; c3.split_k = 0;
    }

    int* d_err = nullptr;
    CK(cudaMalloc(&d_err, sizeof(int)));
    Totals T;
    for (const Case& c : cases) {
        if (filter[0] && c.name.find(filter) == std::string::npos) continue;
        ++T.n_run;
        T.tags[c.tag]++;
        if (!run_case(c, d_err, T)) ++T.n_fail;
    }

    // every instance the planner can select: voxel-major (block_n, TD) and channel-major NV
    printf("INSTANCES: cases");
    int missing = 0;
    std::vector<std::string> all;
    for (int bn : {16, 32})
        for (int td : {1, 2, 4}) all.push_back("vm(" + std::to_string(bn) + "," + std::to_string(td) + ")");
    for (int nv : {64, 128, 256}) all.push_back("cm(" + std::to_string(nv) + ")");
    for (const auto& k : all) {
        const auto it = T.inst.find(k);
        const int n = it == T.inst.end() ? 0 : it->second;
        printf("  %s: %d", k.c_str(), n);
        missing += n == 0;
    }
    printf("\n");
    if (!filter[0] && missing) { printf("FAIL: %d kernel instance(s) not run\n", missing); ++T.n_fail; }
    printf("CASES by kind:");
    for (const auto& kv : T.tags) printf("  %s: %d", kv.first.c_str(), kv.second);
    printf("\n");
    printf("TAU  max err/S over fp16 cases = %.3e = 2^%.2f (%s); kTau = 2^%.2f\n", T.r, std::log2(T.r), T.r_case.c_str(), std::log2(kTau));
    printf("TAU  max err/S over fp16x3 cases = %.3e = 2^%.2f (%s); kTau = 2^%.2f\n", T.rx3, std::log2(T.rx3), T.rx3_case.c_str(),
           std::log2(kTau));
    printf("TAU8 max (err - kTau S)/S8 over E5M2 cases = %.3e = 2^%.1f (%s); kTau8 = 2^%.0f\n", T.r8, std::log2(T.r8),
           T.r8_case.c_str(), std::log2(kTau8));
    if (T.e5_ratio < 1e30) printf("E5M2 worst improvement over a single fp16 pass vs a*w: %.1fx (need >= 4)\n", T.e5_ratio);
    if (T.x3_ratio < 1e30) printf("FP16X3 worst improvement over a single fp16 pass vs a*w: %.1fx (need >= %.0f)\n", T.x3_ratio, kX3Gain);
    printf("SUMMARY run=%d fail=%d\n", T.n_run, T.n_fail);
    cudaFree(d_err);
    return T.n_fail ? 1 : 0;
}
