// wgmma implicit-GEMM Conv3d for sm_90a: kernel + host planning. See conv3d_igemm.cuh.
#include "conv3d_igemm.cuh"
#include "ptx.cuh"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>

#include <cuda_fp8.h>

namespace pixie {

using namespace ptx;

namespace {

constexpr int kMaxWStages = 4;          // voxel-major: up to 2 phase stages; channel-major: up to 4 kd units
constexpr int kMaxSStages = 8;
constexpr int kConsumerWarps = 8;          // two warpgroups, 64 accumulator rows each
constexpr int kProducerWarp = 8;

struct SmemCtrl {
    uint64_t wfull[kMaxWStages];
    uint64_t wempty[kMaxWStages];
    uint64_t sfull[kMaxSStages];
    uint64_t sempty[kMaxSStages];
    int abort_flag;
};

constexpr int kCtlBarrierBytes = 512;     // SmemCtrl
// channel-major epilogue: per consumer warpgroup, a staging chunk of kCmChunk voxels x 64 channels (rows padded to 68 floats:
// the fragment writes hit 32 distinct banks, the 16-byte row reads stay aligned)
constexpr int kCmChunk = 16;
constexpr int kCmStageLd = 68;
constexpr int kCmStageFloats = kCmChunk * kCmStageLd;
constexpr int kStatsMaxC = 256;
// statistics rows: [2][stats_ld] floats (sum, sum of squares) shared by the consumer warps (shared-memory atomics)

struct TileCoord {
    int nb, d0, h0, w0, n0, ph_begin, ph_end, split, tde;
};

// Tile coordinates of work item `wi`: unsigned 32-bit divisions only, and none at all for the split-K bookkeeping of
// unsplit convolutions (this sits on the critical path of every role once per tile).
__device__ __forceinline__ TileCoord decode_tile(const ConvKernelParams& p, int wi) {
    TileCoord t;
    unsigned rest = (unsigned)wi;
    if (p.split_k == 1) {
        t.split = 0; t.ph_begin = 0; t.ph_end = p.n_phases;
    } else {
        const unsigned sk = (unsigned)p.split_k;
        t.split = (int)(rest % sk);
        rest /= sk;
        t.ph_begin = (int)(((unsigned)t.split * (unsigned)p.n_phases) / sk);            // n_phases * split_k < 2^31 (checked at plan time)
        t.ph_end = (int)((((unsigned)t.split + 1u) * (unsigned)p.n_phases) / sk);
    }
    const unsigned nt = rest % (unsigned)p.n_tiles;
    unsigned m = rest / (unsigned)p.n_tiles;
    const unsigned tw = m % (unsigned)p.tiles_w;
    m /= (unsigned)p.tiles_w;
    const unsigned th = m % (unsigned)p.tiles_h;
    m /= (unsigned)p.tiles_h;
    const unsigned td = m % (unsigned)p.tiles_d;
    t.nb = (int)(m / (unsigned)p.tiles_d);
    t.d0 = (int)td * p.TD;
    t.h0 = (int)th * p.TH;
    t.w0 = (int)tw * p.TW;
    t.n0 = (int)nt * p.block_n;
    t.tde = min(p.TD, p.D - t.d0);
    return t;
}

// One wgmma group: four K steps of 32 bytes (16 fp16 or 32 E5M2 values) of D[64 x N] += A[64 x K] * B[N x K]^T, both
// operands K-major SW128 rows in shared memory. Voxel-major: A = slab rows (voxels), B = weight rows (N = block_n output
// channels). Channel-major: A = weight rows (64 output channels), B = slab rows (N = the tile's voxels of one plane).
// Branch-free between fence and commit: ptxas serialises wgmma on any branch in between.
template <int N, bool F8>
__device__ __forceinline__ void mma_block(float* acc, uint32_t a, uint32_t b) {
    wgmma_fence();
#pragma unroll
    for (int k4 = 0; k4 < 4; ++k4) {
        const uint64_t da = make_sw128_desc(a + 32u * k4), db = make_sw128_desc(b + 32u * k4);
        if (F8) {
            if (N == 16) wgmma_e5m2_n16(acc, da, db);
            if (N == 32) wgmma_e5m2_n32(acc, da, db);
            if (N == 64) wgmma_e5m2_n64(acc, da, db);
            if (N == 128) wgmma_e5m2_n128(acc, da, db);
            if (N == 256) wgmma_e5m2_n256(acc, da, db);
        } else {
            if (N == 16) wgmma_f16_n16(acc, da, db);
            if (N == 32) wgmma_f16_n32(acc, da, db);
            if (N == 64) wgmma_f16_n64(acc, da, db);
            if (N == 128) wgmma_f16_n128(acc, da, db);
            if (N == 256) wgmma_f16_n256(acc, da, db);
        }
    }
    wgmma_commit();
}

// wgmma.wait_group with a run-time count (the instruction takes an immediate)
__device__ __forceinline__ void wgmma_wait_n(int n) {
    switch (n) {
        case 0: wgmma_wait<0>(); break;
        case 1: wgmma_wait<1>(); break;
        case 2: wgmma_wait<2>(); break;
        case 3: wgmma_wait<3>(); break;
        case 4: wgmma_wait<4>(); break;
        case 5: wgmma_wait<5>(); break;
        case 6: wgmma_wait<6>(); break;
        case 7: wgmma_wait<7>(); break;
        case 8: wgmma_wait<8>(); break;
        case 9: wgmma_wait<9>(); break;
        default: wgmma_wait<0>(); break;
    }
}

// Position in a ring of stages: the stage and the parity of its barriers' current phase.
struct RingPos {
    int stage = 0, parity = 0;
    __device__ __forceinline__ void advance(int n_stages) {
        if (++stage == n_stages) { stage = 0; parity ^= 1; }
    }
};

// Stages whose MMAs may still be in flight (-1: none). release() hands them back to the producer, one lane per consumer
// warp arriving on their empty barriers, once the wgmma groups that read them have retired.
struct PendingStages {
    int s = -1, w = -1;
    __device__ __forceinline__ void release(SmemCtrl* ctl, int lane) {
        if (lane == 0) {
            if (s >= 0) mbar_arrive(&ctl->sempty[s]);
            if (w >= 0) mbar_arrive(&ctl->wempty[w]);
        }
        s = -1; w = -1;
    }
};

// Fused output statistics of the consumer threads: per-channel sums gather in the CTA's shared-memory rows, scalar totals
// (p.stats_scalar) in each thread's fp64 registers. Both fold into the global fp64 accumulators of batch item `nb` when the
// consumers reach a tile of another item, and after their last tile.
struct ConvStats {
    float* rows;                 // [2][p.stats_ld]: sum, sum of squares
    int nb = -1;
    double tot_s = 0.0, tot_q = 0.0;

    __device__ __forceinline__ void flush(const ConvKernelParams& p, int lane) {
        if (p.stats_scalar) {
            // totals go to channel 0's slot; the LayerNorm consumer sums the [Cout][2] row anyway
#pragma unroll
            for (int off = 16; off >= 1; off >>= 1) {
                tot_s += __shfl_xor_sync(0xffffffffu, tot_s, off);
                tot_q += __shfl_xor_sync(0xffffffffu, tot_q, off);
            }
            if (lane == 0) {
                atomicAdd(p.stats + (size_t)nb * p.Cout * 2, tot_s);
                atomicAdd(p.stats + (size_t)nb * p.Cout * 2 + 1, tot_q);
            }
            tot_s = 0.0; tot_q = 0.0;
            return;
        }
        // both consumer warpgroups: fold the block's partial sums into the global fp64 accumulators
        asm volatile("bar.sync 1, 256;" ::: "memory");
        for (int ch = threadIdx.x; ch < p.Cout; ch += 256) {
            atomicAdd(p.stats + ((size_t)nb * p.Cout + ch) * 2, (double)rows[ch]);
            atomicAdd(p.stats + ((size_t)nb * p.Cout + ch) * 2 + 1, (double)rows[p.stats_ld + ch]);
            rows[ch] = 0.f;
            rows[p.stats_ld + ch] = 0.f;
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
    }
    // before the epilogue of a tile of batch item item_nb
    __device__ __forceinline__ void enter(const ConvKernelParams& p, int item_nb, int lane) {
        if (nb != item_nb) {
            if (nb >= 0) flush(p, lane);
            nb = item_nb;
        }
    }
};

// Dynamic shared memory of both kernels: w_stages weight stages, s_stages slab stages, the control block (SmemCtrl in
// kCtlBarrierBytes), the epilogue staging (channel-major), then the statistics rows (iff p.stats).
struct ConvSmem {
    uint8_t* w;
    uint8_t* s;
    SmemCtrl* ctl;
    float* stage;
    float* stats;
};

// Carves the dynamic shared memory (stage_floats of epilogue staging), initialises the barriers, prefetches the tensor maps
// and clears the statistics rows; ends with a block-wide barrier.
__device__ __forceinline__ ConvSmem conv_prologue(const ConvKernelParams& p, int stage_floats, int n_threads) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    // dynamic smem base is only guaranteed 16 B aligned by the ABI: align manually to 1024 B
    uint8_t* smem = reinterpret_cast<uint8_t*>(
        (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
    ConvSmem m;
    m.w = smem;
    m.s = smem + (size_t)p.w_stages * p.w_stage_bytes;
    m.ctl = reinterpret_cast<SmemCtrl*>(m.s + (size_t)p.s_stages * p.s_stage_bytes);
    m.stage = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(m.ctl) + kCtlBarrierBytes);
    m.stats = m.stage + stage_floats;
    // plans without alignment slack (p.smem_slack == 0) rely on the 1 KB-aligned dynamic smem base that kernels without
    // static shared memory get in practice; verified here, failing loudly through the error flag instead of corrupting smem
    const bool smem_misaligned = (p.smem_slack == 0) && (smem != smem_raw);

    if (threadIdx.x == 0) {
        for (int i = 0; i < kMaxWStages; ++i) { mbar_init(&m.ctl->wfull[i], 1); mbar_init(&m.ctl->wempty[i], kConsumerWarps); }
        for (int i = 0; i < kMaxSStages; ++i) { mbar_init(&m.ctl->sfull[i], 1); mbar_init(&m.ctl->sempty[i], kConsumerWarps); }
        m.ctl->abort_flag = smem_misaligned ? 1 : 0;
        fence_barrier_init();
    }
    if ((threadIdx.x >> 5) == kProducerWarp && (threadIdx.x & 31) == 0) {
        for (int i = 0; i < kConvMaxSrc; ++i) prefetch_tmap(&p.tmA[i]);
        prefetch_tmap(&p.tmB);
    }
    if (p.stats != nullptr && !p.stats_scalar)
        for (int i = threadIdx.x; i < 2 * p.stats_ld; i += n_threads) m.stats[i] = 0.f;
    __syncthreads();
    return m;
}

// Once every role has left its loop: a CTA whose pipeline aborted (timeout, or misaligned shared memory) reports itself.
__device__ __forceinline__ void conv_report_abort(const ConvKernelParams& p, const SmemCtrl* ctl) {
    __syncthreads();
    if (threadIdx.x == 0 && ctl->abort_flag && p.err_flag) atomicExch(p.err_flag, 1 + (int)blockIdx.x);
}

// One input slab (input plane pl) of a phase, for this warpgroup's 64 rows: the slab feeds output planes d = pl - kd for the
// kd taps of the phase, each through n_kh row-shifted views (kh taps). The accumulator of plane d is acc[d]. Returns the
// number of wgmma groups committed.
template <int BN, int TD>
__device__ __forceinline__ int issue_slab(float (&acc)[TD][BN / 2], uint32_t a_addr, uint32_t w_addr, int pl, int d_min, int d_max,
                                          int n_kd, int n_kh, int TW, bool f8) {
    int groups = 0;
#pragma unroll
    for (int d = 0; d < TD; ++d) {
        if (d < d_min || d > d_max) continue;                 // warpgroup-uniform
        const int kd = pl - d;
        for (int kh = 0; kh < n_kh; ++kh) {
            const uint32_t a = a_addr + (uint32_t)(kh * TW * 128);
            const uint32_t b = w_addr + (uint32_t)(conv_wtile(0, n_kd, kh, kd) * BN * 128);
            if (f8) mma_block<BN, true>(acc[d], a, b);
            else mma_block<BN, false>(acc[d], a, b);
            ++groups;
        }
    }
    return groups;
}

// TMA producer loop (one warp; one elected lane issues). Per tile and phase, the tde + n_kd - 1 input-plane slabs go into the
// slab ring and the phase's weight tiles into the weight ring in units of kUnitKd kd taps (kWholePhase: all n_kd taps, one
// unit), unit u loaded just before slab u. Inside a unit over kd_lo .. kd_hi the tiles sit in the packed order, kh major,
// then kd = kd_hi .. kd_lo.
constexpr int kWholePhase = 0;

template <int kUnitKd>
__device__ __forceinline__ void produce_tiles(const ConvKernelParams& p, SmemCtrl* ctl, uint8_t* w_smem, uint8_t* s_smem,
                                              volatile int* abort_flag, int total_items) {
    RingPos wring, sring;
    bool ok = true;
    for (int wi = blockIdx.x; wi < total_items && ok; wi += gridDim.x) {
        const TileCoord t = decode_tile(p, wi);
        for (int ph = t.ph_begin; ph < t.ph_end && ok; ++ph) {
            const ConvPhase P = p.phases[ph];
            const int n_kd = P.n_kd, n_kh = P.n_kh, nplanes = t.tde + n_kd - 1;
            const int unit_kd = kUnitKd ? kUnitKd : n_kd, n_units = kUnitKd ? n_kd / kUnitKd : 1;
            const uint32_t slab_bytes = (uint32_t)p.slab_rows[P.src] * 128u, unit_bytes = (uint32_t)(n_kh * unit_kd * p.block_n * 128);
            const CUtensorMap* tm = &p.tmA[P.src];
            const int cw = t.w0 * p.stride + P.dw, ch = t.h0 * p.stride + P.dh0, cd = t.d0 * p.stride + P.dd0;
#pragma unroll 1
            for (int pl = 0; pl < nplanes && ok; ++pl) {
                if (pl < n_units) {
                    ok = mbar_wait(&ctl->wempty[wring.stage], wring.parity ^ 1, abort_flag);
                    if (!ok) break;
                    if (elect_one()) {
                        mbar_expect_tx(&ctl->wfull[wring.stage], unit_bytes);
                        uint8_t* wdst = w_smem + (size_t)wring.stage * p.w_stage_bytes;
                        const int kd_lo = pl * unit_kd, kd_hi = kd_lo + unit_kd - 1;
#pragma unroll 1
                        for (int kh = 0; kh < n_kh; ++kh)
                            for (int kd = kd_hi; kd >= kd_lo; --kd)
                                tma_load_2d(wdst + (size_t)conv_wtile(0, unit_kd, kh, kd - kd_lo) * p.block_n * 128, &p.tmB,
                                            &ctl->wfull[wring.stage], conv_wtile(P.wtile_base, n_kd, kh, kd) * 64, t.n0);
                    }
                    wring.advance(p.w_stages);
                }
                ok = mbar_wait(&ctl->sempty[sring.stage], sring.parity ^ 1, abort_flag);
                if (!ok) break;
                if (elect_one()) {
                    mbar_expect_tx(&ctl->sfull[sring.stage], slab_bytes);
                    tma_load_5d(s_smem + (size_t)sring.stage * p.s_stage_bytes, tm, &ctl->sfull[sring.stage], (int)P.c0, cw, ch,
                                cd + pl * p.stride, t.nb);
                }
                sring.advance(p.s_stages);
            }
        }
    }
}

}  // namespace

template <int BN, int TD>
__global__ void __launch_bounds__(kConvThreads, 1)
conv3d_igemm_kernel(const __grid_constant__ ConvKernelParams p) {
    const ConvSmem sm = conv_prologue(p, 0, kConvThreads);
    SmemCtrl* ctl = sm.ctl;
    volatile int* abort_flag = &ctl->abort_flag;
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int total_items = conv_work_items(p.NB, p.tiles_d, p.tiles_h, p.tiles_w, p.n_tiles, p.split_k);
    const bool do_stats = p.stats != nullptr;
    const bool scalar_stats = do_stats && p.stats_scalar;     // consumer only needs the per-item totals (LayerNorm)

    if (warp == kProducerWarp) {
        // ================================================================ TMA producer (warp-uniform, one elected lane issues)
        produce_tiles<kWholePhase>(p, ctl, sm.w, sm.s, abort_flag, total_items);
    } else {
        // ================================================================ consumers: MMA + epilogue (warpgroups 0 and 1)
        // Each warpgroup owns rows 64 g .. 64 g + 63 of the 128-voxel plane tile and the TD plane accumulators of those rows in
        // registers. A slab stage is released one slab late (once only the current slab's wgmma groups are pending) so
        // that the tensor cores always have the next slab's MMAs queued behind the current ones.
        const int g = warp >> 2, wq = warp & 3;
        float acc[TD][BN / 2];
        RingPos wring, sring;
        const uint32_t w_base0 = smem_u32(sm.w), s_base0 = smem_u32(sm.s) + (uint32_t)(g * 64 * 128);
        bool ok = true;
        const long long DHW = (long long)p.D * p.H * p.W;
        ConvStats stats{sm.stats};
        // accumulator rows of this thread (the two rows of the wgmma fragment)
        int th2[2], tw2[2];
#pragma unroll
        for (int r2 = 0; r2 < 2; ++r2) {
            const int r = g * 64 + wq * 16 + (lane >> 2) + 8 * r2;
            th2[r2] = r / p.TW; tw2[r2] = r % p.TW;
        }
        const int cq = (lane & 3) * 2;

        for (int wi = blockIdx.x; wi < total_items && ok; wi += gridDim.x) {
            const TileCoord t = decode_tile(p, wi);
#pragma unroll
            for (int d = 0; d < TD; ++d)
#pragma unroll
                for (int j = 0; j < BN / 2; ++j) acc[d][j] = 0.f;
            PendingStages pend;
            int prev_f8 = -1;                   // operand type of the previous phase of this tile
            for (int ph = t.ph_begin; ph < t.ph_end && ok; ++ph) {
                const ConvPhase P = p.phases[ph];
                const int n_kd = P.n_kd, n_kh = P.n_kh;
                const bool f8 = P.f8 != 0;
                // wgmma groups of different shapes (E5M2 k32, fp16 k16) in flight on the same accumulators: drain at the switch
                if (prev_f8 >= 0 && prev_f8 != (int)f8) wgmma_wait<0>();
                prev_f8 = (int)f8;
                ok = mbar_wait(&ctl->wfull[wring.stage], wring.parity, abort_flag);
                if (!ok) break;
                const uint32_t w_addr = w_base0 + (uint32_t)(wring.stage * p.w_stage_bytes);
                const int nplanes = t.tde + n_kd - 1;
                for (int pl = 0; pl < nplanes && ok; ++pl) {
                    ok = mbar_wait(&ctl->sfull[sring.stage], sring.parity, abort_flag);
                    if (!ok) break;
                    const int d_min = max(0, pl - (n_kd - 1)), d_max = min(t.tde - 1, pl);
                    const int groups = issue_slab<BN, TD>(acc, s_base0 + (uint32_t)(sring.stage * p.s_stage_bytes), w_addr, pl, d_min,
                                                          d_max, n_kd, n_kh, p.TW, f8);
                    wgmma_wait_n(groups);          // the previous slab's MMAs have retired
                    pend.release(ctl, lane);
                    pend.s = sring.stage;
                    sring.advance(p.s_stages);
                }
                pend.w = wring.stage;
                wring.advance(p.w_stages);
                if (p.w_stages == 1) { wgmma_wait<0>(); pend.release(ctl, lane); }   // the producer needs this stage for the next phase
            }
            wgmma_wait<0>();
            pend.release(ctl, lane);
#pragma unroll
            for (int d = 0; d < TD; ++d)
#pragma unroll
                for (int j = 0; j < BN / 2; ++j) fence_operand(acc[d][j]);
            if (!ok) break;

            // ---------------------------------------------------------------- epilogue from registers
            if (do_stats) stats.enter(p, t.nb, lane);
            const bool first_split = (t.split == 0);
            const bool use_bias = first_split && p.bias != nullptr;
            const bool use_res = first_split && p.residual != nullptr;
#pragma unroll
            for (int d = 0; d < TD; ++d) {
                if (d >= t.tde) break;
#pragma unroll
                for (int r2 = 0; r2 < 2; ++r2) {
                    const int hh = t.h0 + th2[r2], ww = t.w0 + tw2[r2];
                    const bool row_ok = (hh < p.H) && (ww < p.W);
                    const long long vox = ((long long)(t.d0 + d) * p.H + hh) * p.W + ww;   // inside batch item
#pragma unroll
                    for (int j8 = 0; j8 < BN / 8; ++j8) {
                        const int ch = t.n0 + j8 * 8 + cq;
                        float& a0 = acc[d][j8 * 4 + r2 * 2];
                        float& a1 = acc[d][j8 * 4 + r2 * 2 + 1];
                        const bool ok0 = row_ok && ch < p.Cout, ok1 = row_ok && ch + 1 < p.Cout;
                        float v0 = a0, v1 = a1;
                        if (use_bias) {
                            if (ok0) v0 += __ldg(p.bias + ch);
                            if (ok1) v1 += __ldg(p.bias + ch + 1);
                        }
                        if (p.out_planar) {
                            const long long i0 = ((long long)t.nb * p.Cout + ch) * DHW + vox;
                            if (ok0) {
                                if (use_res) v0 += p.residual[i0];
                                if (p.atomic_out) atomicAdd(p.out + i0, v0); else p.out[i0] = v0;
                            }
                            if (ok1) {
                                if (use_res) v1 += p.residual[i0 + DHW];
                                if (p.atomic_out) atomicAdd(p.out + i0 + DHW, v1); else p.out[i0 + DHW] = v1;
                            }
                        } else if (ok0) {
                            const long long base = ((long long)t.nb * DHW + vox) * p.out_ld + p.out_c0 + ch;
                            if (ok1 && (base & 1) == 0) {
                                if (use_res) {
                                    const float2 rv = __ldg(reinterpret_cast<const float2*>(p.residual + base));
                                    v0 += rv.x; v1 += rv.y;
                                }
                                if (p.atomic_out) red_add_v2(p.out + base, v0, v1);
                                else *reinterpret_cast<float2*>(p.out + base) = make_float2(v0, v1);
                            } else {
                                if (use_res) { v0 += p.residual[base]; if (ok1) v1 += p.residual[base + 1]; }
                                if (p.atomic_out) { atomicAdd(p.out + base, v0); if (ok1) atomicAdd(p.out + base + 1, v1); }
                                else { p.out[base] = v0; if (ok1) p.out[base + 1] = v1; }
                            }
                        }
                        a0 = ok0 ? v0 : 0.f;       // final values (zero where invalid) for the statistics
                        a1 = ok1 ? v1 : 0.f;
                    }
                }
            }
            if (do_stats) {
                if (scalar_stats) {
                    float s = 0.f, q2 = 0.f;
#pragma unroll
                    for (int d = 0; d < TD; ++d)
#pragma unroll
                        for (int j = 0; j < BN / 2; ++j) { s += acc[d][j]; q2 = fmaf(acc[d][j], acc[d][j], q2); }
                    stats.tot_s += (double)s; stats.tot_q += (double)q2;
                } else {
                    // per column: this thread's rows and planes, then the 8 lanes holding the same columns
#pragma unroll
                    for (int j8 = 0; j8 < BN / 8; ++j8)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            float s = 0.f, q2 = 0.f;
#pragma unroll
                            for (int d = 0; d < TD; ++d)
#pragma unroll
                                for (int r2 = 0; r2 < 2; ++r2) {
                                    const float v = acc[d][j8 * 4 + r2 * 2 + e];
                                    s += v; q2 = fmaf(v, v, q2);
                                }
#pragma unroll
                            for (int off = 4; off <= 16; off <<= 1) {
                                s += __shfl_xor_sync(0xffffffffu, s, off);
                                q2 += __shfl_xor_sync(0xffffffffu, q2, off);
                            }
                            const int ch = t.n0 + j8 * 8 + cq + e;
                            if (lane < 4 && ch < p.Cout) {
                                atomicAdd(stats.rows + ch, s);
                                atomicAdd(stats.rows + p.stats_ld + ch, q2);
                            }
                        }
                }
            }
        }
        if (do_stats && stats.nb >= 0 && ok) stats.flush(p, lane);
    }

    conv_report_abort(p, ctl);
}

// Channel-major instance: D[co][vox] = W[co][k] * S[vox][k]^T. A tile is 64 output channels x NV voxels (TH x TW of one plane)
// x 2 planes; consumer warpgroup g owns output plane d0 + g, so one wgmma is m64 nNV (n256 for 16 x 16 tiles) and a slab
// still feeds both warpgroups through its kd taps. The weight rows of a phase are the A operand, the slab rows the B operand;
// the phase table, producer, slab ring and barriers are those of the voxel-major kernel, but the weight ring holds one kd tap
// per unit. The accumulator is NV / 2 registers per thread: the producer warpgroup hands its registers to the two consumer
// warpgroups (setmaxnreg).
template <int NV>
__global__ void __launch_bounds__(kConvCmThreads, 1)
conv3d_igemm_cm_kernel(const __grid_constant__ ConvKernelParams p) {
    constexpr int TW = NV == 64 ? 8 : 16;
    const ConvSmem sm = conv_prologue(p, 2 * kCmStageFloats, kConvCmThreads);
    SmemCtrl* ctl = sm.ctl;
    volatile int* abort_flag = &ctl->abort_flag;
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int total_items = conv_work_items(p.NB, p.tiles_d, p.tiles_h, p.tiles_w, p.n_tiles, p.split_k);
    const bool do_stats = p.stats != nullptr;
    const bool scalar_stats = do_stats && p.stats_scalar;

    if (warp >= kProducerWarp) {
        // ================================================================ producer warpgroup: one warp issues the TMA loads
        // NV = 256 needs 232 consumer registers (a 128-register accumulator); narrower tiles leave the producer more
        setmaxnreg_dec<NV == 256 ? 40 : 56>();
        if (warp == kProducerWarp) produce_tiles<1>(p, ctl, sm.w, sm.s, abort_flag, total_items);
    } else {
        // ================================================================ consumers: warpgroup g computes plane d0 + g
        setmaxnreg_inc<NV == 256 ? 232 : 216>();
        const int g = warp >> 2, wq = warp & 3, wt = threadIdx.x & 127;
        float acc[NV / 2];
        RingPos wring, sring;
        const uint32_t w_base0 = smem_u32(sm.w), s_base0 = smem_u32(sm.s);
        bool ok = true;
        ConvStats stats{sm.stats};
        // epilogue read-out: this thread's channel quad and voxel row inside a staged chunk
        const int q4 = wt & 15, vr = wt >> 4;
        float* stage = sm.stage + g * kCmStageFloats;

        for (int wi = blockIdx.x; wi < total_items && ok; wi += gridDim.x) {
            const TileCoord t = decode_tile(p, wi);
#pragma unroll
            for (int j = 0; j < NV / 2; ++j) acc[j] = 0.f;
            const bool has_plane = g < t.tde;   // warpgroup-uniform
            PendingStages pend;
            int prev_f8 = -1;
            for (int ph = t.ph_begin; ph < t.ph_end && ok; ++ph) {
                const ConvPhase P = p.phases[ph];
                const int n_kd = P.n_kd, n_kh = P.n_kh;
                const bool f8 = P.f8 != 0;
                if (prev_f8 >= 0 && prev_f8 != (int)f8) wgmma_wait<0>();
                prev_f8 = (int)f8;
                // weight unit kd of this phase sits in ring stage w0 + kd (mod w_stages); slab pl is the last user of unit
                // pl - tde + 1 (the plane-1 warpgroup reads unit kd at slab kd + 1), which is released with that slab
                const int w0 = wring.stage;
                const int nplanes = t.tde + n_kd - 1;
                for (int pl = 0; pl < nplanes && ok; ++pl) {
                    if (pl < n_kd) {
                        ok = mbar_wait(&ctl->wfull[wring.stage], wring.parity, abort_flag);
                        if (!ok) break;
                        wring.advance(p.w_stages);
                    }
                    ok = mbar_wait(&ctl->sfull[sring.stage], sring.parity, abort_flag);
                    if (!ok) break;
                    const int kd = pl - g;
                    int groups = 0;
                    if (has_plane && kd >= 0 && kd < n_kd) {
                        int wsk = w0 + kd;
                        if (wsk >= p.w_stages) wsk -= p.w_stages;
                        const uint32_t w_addr = w_base0 + (uint32_t)(wsk * p.w_stage_bytes);
                        const uint32_t s_addr = s_base0 + (uint32_t)(sring.stage * p.s_stage_bytes);
                        for (int kh = 0; kh < n_kh; ++kh) {
                            const uint32_t a = w_addr + (uint32_t)(conv_wtile(0, 1, kh, 0) * 64 * 128);
                            const uint32_t b = s_addr + (uint32_t)(kh * TW * 128);
                            if (f8) mma_block<NV, true>(acc, a, b);
                            else mma_block<NV, false>(acc, a, b);
                            ++groups;
                        }
                    }
                    wgmma_wait_n(groups);          // the previous slab's MMAs have retired
                    pend.release(ctl, lane);
                    pend.s = sring.stage;
                    const int kd_done = pl - t.tde + 1;
                    if (kd_done >= 0) {
                        pend.w = w0 + kd_done;
                        if (pend.w >= p.w_stages) pend.w -= p.w_stages;
                    }
                    sring.advance(p.s_stages);
                }
            }
            wgmma_wait<0>();
            pend.release(ctl, lane);
#pragma unroll
            for (int j = 0; j < NV / 2; ++j) fence_operand(acc[j]);
            if (!ok) break;

            // ---------------------------------------------------------------- epilogue through shared memory
            // The fragment holds 2 channels x NV / 4 voxels per thread; it is staged in chunks of kCmChunk voxels x 64
            // channels so that every output row is written (and the residual read) as 16-byte vectors.
            if (do_stats) stats.enter(p, t.nb, lane);
            if (!has_plane) continue;
            const bool first_split = (t.split == 0);
            const int ch = t.n0 + 4 * q4;
            const bool ch_ok = ch < p.Cout;      // Cout % 4 == 0 (plan)
            float4 bias4 = make_float4(0.f, 0.f, 0.f, 0.f);
            if (first_split && p.bias != nullptr && ch_ok)
                bias4 = make_float4(__ldg(p.bias + ch), __ldg(p.bias + ch + 1), __ldg(p.bias + ch + 2), __ldg(p.bias + ch + 3));
            const bool use_res = first_split && p.residual != nullptr;
            const long long plane_base = ((long long)t.nb * p.D + t.d0 + g) * p.H;
            float st_s[4] = {0.f, 0.f, 0.f, 0.f}, st_q[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int c = 0; c < NV / kCmChunk; ++c) {
#pragma unroll
                for (int jj = 0; jj < kCmChunk / 8; ++jj)
#pragma unroll
                    for (int r2 = 0; r2 < 2; ++r2)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int row = wq * 16 + (lane >> 2) + 8 * r2, v = jj * 8 + (lane & 3) * 2 + e;
                            stage[v * kCmStageLd + row] = acc[(c * (kCmChunk / 8) + jj) * 4 + r2 * 2 + e];
                        }
                asm volatile("bar.sync %0, 128;" ::"r"(2 + g) : "memory");
#pragma unroll
                for (int k = 0; k < kCmChunk / 8; ++k) {
                    const int v = vr + 8 * k, vt = c * kCmChunk + v;
                    const int hh = t.h0 + vt / TW, ww = t.w0 + vt % TW;
                    float4 x = *reinterpret_cast<const float4*>(stage + v * kCmStageLd + 4 * q4);
                    if (ch_ok && hh < p.H && ww < p.W) {
                        const long long base = ((plane_base + hh) * p.W + ww) * p.out_ld + p.out_c0 + ch;
                        x.x += bias4.x; x.y += bias4.y; x.z += bias4.z; x.w += bias4.w;
                        if (use_res) {
                            const float4 rv = __ldg(reinterpret_cast<const float4*>(p.residual + base));
                            x.x += rv.x; x.y += rv.y; x.z += rv.z; x.w += rv.w;
                        }
                        if (p.atomic_out) red_add_v4(p.out + base, x.x, x.y, x.z, x.w);
                        else *reinterpret_cast<float4*>(p.out + base) = x;
                        st_s[0] += x.x; st_s[1] += x.y; st_s[2] += x.z; st_s[3] += x.w;
                        st_q[0] = fmaf(x.x, x.x, st_q[0]); st_q[1] = fmaf(x.y, x.y, st_q[1]);
                        st_q[2] = fmaf(x.z, x.z, st_q[2]); st_q[3] = fmaf(x.w, x.w, st_q[3]);
                    }
                }
                asm volatile("bar.sync %0, 128;" ::"r"(2 + g) : "memory");
            }
            if (do_stats) {
                if (scalar_stats) {
                    stats.tot_s += (double)(st_s[0] + st_s[1] + st_s[2] + st_s[3]);
                    stats.tot_q += (double)(st_q[0] + st_q[1] + st_q[2] + st_q[3]);
                } else {
                    // lanes q4 and q4 + 16 of a warp hold the same channels: one shuffle, then shared atomics
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        st_s[i] += __shfl_xor_sync(0xffffffffu, st_s[i], 16);
                        st_q[i] += __shfl_xor_sync(0xffffffffu, st_q[i], 16);
                    }
                    if (lane < 16 && ch_ok) {
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            atomicAdd(stats.rows + ch + i, st_s[i]);
                            atomicAdd(stats.rows + p.stats_ld + ch + i, st_q[i]);
                        }
                    }
                }
            }
        }
        if (do_stats && stats.nb >= 0 && ok) stats.flush(p, lane);
    }

    conv_report_abort(p, ctl);
}

// =====================================================================================  host side

int conv_k_total(const ConvDesc& d) {
    int k = 0;
    for (const auto& s : d.segs) k += s.ks * s.ks * s.ks * d.srcs[s.src].C;
    return k;
}

// Source slots: a (source, kernel-size class) pair needs its own tensor map because the TMA box
// height differs (TH+2 rows for in-slab kh taps vs TH rows).  Slot i of the returned table is used
// as ConvPhase::src.
struct SrcSlot { int src; int n_kh; };

static std::vector<SrcSlot> conv_src_slots(const ConvDesc& d) {
    std::vector<SrcSlot> slots;
    for (const auto& s : d.segs) {
        const int n_kh = (s.ks == 3 && d.stride == 1) ? 3 : 1;
        bool found = false;
        for (const auto& sl : slots) found |= (sl.src == s.src && sl.n_kh == n_kh);
        if (!found) slots.push_back({s.src, n_kh});
    }
    return slots;
}

static int conv_slot_of(const std::vector<SrcSlot>& slots, int src, int n_kh) {
    for (size_t i = 0; i < slots.size(); ++i)
        if (slots[i].src == src && slots[i].n_kh == n_kh) return (int)i;
    return -1;
}

// One phase as the host enumerates it: the kernel's ConvPhase and the segment it belongs to. The phase's n_kh x n_kd taps
// are kernel taps (P.dd0 + pad + kd, P.dh0 + pad + kh, P.dw + pad), pad = ks / 2 of the segment; tap (kh, kd) sits in packed
// weight tile conv_wtile(P.wtile_base, P.n_kd, kh, kd).
struct PhaseRec {
    ConvPhase P;
    int seg;
};

// The phases of `d` in the kernel's order. Weight tiles are numbered segment by segment, then chunk, kw (and kh, kd for
// stride-2 taps), before the phases are reordered: residual phases first, E5M2 ones before fp16 ones. The tensor cores do
// not round the fp32 accumulation to nearest (and accumulate E5M2 products with a narrower mantissa still), so small
// correction terms added to accumulators that already hold the main partial sums lose their low bits at every K step;
// started from zero they keep their precision, and the main fp16 phases then accumulate on top.
static std::vector<PhaseRec> conv_phase_records(const ConvDesc& d) {
    std::vector<PhaseRec> recs;
    const auto slots = conv_src_slots(d);
    int wtile = 0;
    for (int si = 0; si < (int)d.segs.size(); ++si) {
        const auto& s = d.segs[si];
        const int chunks = d.srcs[s.src].C / 64;
        // stride-1 3x3x3: one phase per (chunk, kw) holding all 9 (kd, kh) taps; otherwise one phase per tap
        const int n_k = (s.ks == 3 && d.stride == 1) ? 3 : 1, n_ph = s.ks / n_k, pad = s.ks / 2;
        for (int c = 0; c < chunks; ++c)
            for (int kw = 0; kw < s.ks; ++kw)
                for (int kh = 0; kh < n_ph; ++kh)
                    for (int kd = 0; kd < n_ph; ++kd) {
                        ConvPhase P{};
                        P.src = (int8_t)conv_slot_of(slots, s.src, n_k);
                        P.dw = (int8_t)(kw - pad);
                        P.dh0 = (int8_t)(kh - pad);
                        P.dd0 = (int8_t)(kd - pad);
                        P.n_kh = (int8_t)n_k;
                        P.n_kd = (int8_t)n_k;
                        P.c0 = (int16_t)(c * 64);
                        P.wtile_base = wtile;
                        P.f8 = s.f8;
                        wtile += n_k * n_k;
                        recs.push_back({P, si});
                    }
    }
    auto rank = [&](const PhaseRec& r) {   // 0 E5M2 residual, 1 fp16 residual, 2 the main fp16 products
        const auto& s = d.segs[r.seg];
        return s.f8 ? 0 : (s.lo || s.wlo) ? 1 : 2;
    };
    std::stable_sort(recs.begin(), recs.end(), [&](const PhaseRec& a, const PhaseRec& b) { return rank(a) < rank(b); });
    return recs;
}

std::vector<ConvPhase> conv_build_phases(const ConvDesc& d) {
    std::vector<ConvPhase> ph;
    for (const auto& r : conv_phase_records(d)) ph.push_back(r.P);
    return ph;
}

void conv_pack_weights(const ConvDesc& d, const std::vector<const float*>& seg_weights,
                       const std::vector<int>& seg_cin_real, std::vector<__half>& packed) {
    const int K = conv_k_total(d);
    packed.assign((size_t)d.Cout_pad * K, __float2half(0.f));
    const float up = (float)(1 << kF8Shift), down = 1.0f / up;
    auto e5m2 = [](float v) { return (uint8_t)__nv_cvt_float_to_fp8(v, __NV_SATFINITE, __NV_E5M2); };
    for (const auto& r : conv_phase_records(d)) {
        const ConvPhase& P = r.P;
        const auto& s = d.segs[r.seg];
        const int cin = seg_cin_real[r.seg];
        const int ks = s.ks, kv = ks * ks * ks, pad = ks / 2;
        const float* w = seg_weights[r.seg];   // [Cout][cin][kd][kh][kw]
        for (int kh = 0; kh < P.n_kh; ++kh)
            for (int kd = 0; kd < P.n_kd; ++kd) {
                const int tile = conv_wtile(P.wtile_base, P.n_kd, kh, kd);
                const int tap = ((P.dd0 + pad + kd) * ks + P.dh0 + pad + kh) * ks + P.dw + pad;
                for (int co = 0; co < d.Cout; ++co) {
                    // an f8 tile is 128 bytes per row: [e5m2(w / 2^s) x 64 | e5m2((w - fp16(w)) * 2^s) x 64]
                    uint8_t* row8 = reinterpret_cast<uint8_t*>(&packed[(size_t)co * K + (size_t)tile * 64]);
                    for (int cil = 0; cil < 64; ++cil) {
                        const int ci = P.c0 + cil;
                        if (ci >= cin) continue;
                        float v = w[((size_t)co * cin + ci) * kv + tap];
                        if (s.f8) {
                            row8[cil] = e5m2(v * down);
                            row8[64 + cil] = e5m2((v - __half2float(__float2half(v))) * up);
                            continue;
                        }
                        if (s.wlo) v = v - __half2float(__float2half(v));
                        packed[(size_t)co * K + (size_t)tile * 64 + cil] = __float2half(v);
                    }
                }
            }
    }
}

// Voxel-major instance for (block_n, TD); the plan guarantees block_n in {16, 32}, TD in {1, 2, 4}.
static ConvKernelFn conv_kernel_for(int bn, int td) {
    switch (bn * 8 + td) {
        case 16 * 8 + 1: return conv3d_igemm_kernel<16, 1>;
        case 16 * 8 + 2: return conv3d_igemm_kernel<16, 2>;
        case 16 * 8 + 4: return conv3d_igemm_kernel<16, 4>;
        case 32 * 8 + 1: return conv3d_igemm_kernel<32, 1>;
        case 32 * 8 + 2: return conv3d_igemm_kernel<32, 2>;
        default: return conv3d_igemm_kernel<32, 4>;
    }
}

// Channel-major instance for NV voxels per plane tile (64, 128 or 256).
static ConvKernelFn conv_cm_kernel_for(int nv) {
    switch (nv) {
        case 64: return conv3d_igemm_cm_kernel<64>;
        case 128: return conv3d_igemm_cm_kernel<128>;
        default: return conv3d_igemm_cm_kernel<256>;
    }
}

// ---- driver entry point for tensor-map encoding (no link-time dependency on libcuda)
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                    const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
    static PFN_encodeTiled fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_encodeTiled>(p);
    }
    return fn;
}


static int encode_a_maps(const ConvDesc& d, ConvKernelParams& p, PFN_encodeTiled enc, char* err, int errlen) {
    const auto slots = conv_src_slots(d);
    for (size_t i = 0; i < slots.size(); ++i) {
        const ConvSrc& s = d.srcs[slots[i].src];
        cuuint64_t gdim[5] = {(cuuint64_t)s.C, (cuuint64_t)s.Win, (cuuint64_t)s.Hin, (cuuint64_t)s.Din, (cuuint64_t)d.NB};
        cuuint64_t gstr[4] = {(cuuint64_t)s.C * 2, (cuuint64_t)s.Win * s.C * 2,
                              (cuuint64_t)s.Hin * s.Win * s.C * 2, (cuuint64_t)s.Din * s.Hin * s.Win * s.C * 2};
        cuuint32_t box[5] = {64, (cuuint32_t)(p.TW * d.stride), (cuuint32_t)((p.TH + slots[i].n_kh - 1) * d.stride), 1, 1};
        cuuint32_t estr[5] = {1, (cuuint32_t)d.stride, (cuuint32_t)d.stride, 1, 1};
        CUresult r = enc(&p.tmA[i], CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, (void*)s.ptr, gdim, gstr, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { snprintf(err, errlen, "cuTensorMapEncodeTiled(A%zu) failed: %d", i, (int)r); return 1; }
    }
    for (size_t i = slots.size(); i < (size_t)kConvMaxSrc; ++i) p.tmA[i] = p.tmA[0];
    return 0;
}

int conv_plan_retarget(const ConvDesc& d, ConvPlan& plan, char* err, int errlen) {
    PFN_encodeTiled enc = get_encode_fn();
    if (!enc) { snprintf(err, errlen, "cuTensorMapEncodeTiled unavailable"); return 1; }
    return encode_a_maps(d, plan.p, enc, err, errlen);
}

// Channel-major geometry: 64 output channels x NV voxels (TH x TW of one plane) x TD = 2 planes. A weight stage holds one kd
// tap of a phase (its n_kh tiles). Returns an error message or nullptr.
static const char* cm_geometry(const ConvDesc& d, int sms, int max_kh, ConvKernelParams& p) {
    int nv = d.nv;
    if (nv && nv != 64 && nv != 128 && nv != 256) return "bad nv";
    if (!nv) {
        // voxel tile: 16 x 16, 8 x 16 or 8 x 8 of one plane. Wave quantisation: a persistent grid of `sms` CTAs finishes in
        // ceil(tiles/sms) rounds; prefer the tile with the best last-round fill times the share of real voxels, each halving
        // of NV costing ~7 % (more weight and slab traffic per MAC, narrower MMAs)
        double best = -1.0;
        for (int v : {256, 128, 64}) {
            if (v != 64 && d.W < 16) continue;
            const int tw = v == 64 ? 8 : 16, th = v / tw;
            const int tx = (d.W + tw - 1) / tw, ty = (d.H + th - 1) / th;
            const long long tiles = conv_work_items(d.NB, (d.D + 1) / 2, ty, tx, (d.Cout_pad + 63) / 64, 1);
            const long long rounds = (tiles + sms - 1) / sms;
            const double sc = (double)tiles / (double)(rounds * sms) * (double)d.W * d.H / (double)(tx * tw * ty * th) *
                              std::pow(0.93, v == 256 ? 0 : v == 128 ? 1 : 2);
            if (sc > best) { best = sc; nv = v; }
        }
    }
    p.TW = nv == 64 ? 8 : 16;
    p.TH = nv / p.TW;
    p.TD = 2;
    p.block_n = 64;
    p.w_stage_bytes = max_kh * p.block_n * 128;
    return nullptr;
}

// Channel-major stages: a phase holds all n_kd of its weight units at its middle slab, and the next phase's first unit must
// find a free stage while the last one is still in use when n_kd == 1; slab stages first (up to 6), then spare units.
static bool cm_stages(const ConvKernelParams& p, int max_kd, int avail, int& ws, int& ss) {
    ws = std::max(2, max_kd);
    if (ws * p.w_stage_bytes + 2 * p.s_stage_bytes > avail) return false;
    ss = std::min(std::min(kMaxSStages, 6), (avail - ws * p.w_stage_bytes) / p.s_stage_bytes);
    ws = std::min(kMaxWStages, (avail - ss * p.s_stage_bytes) / p.w_stage_bytes);
    return true;
}

// Voxel-major geometry: 128 voxels (TH x TW of one plane) x TD planes x block_n output channels. A weight stage holds all
// taps of a phase. Returns an error message or nullptr.
static const char* vm_geometry(const ConvDesc& d, int sms, bool any3, int max_taps, ConvKernelParams& p) {
    p.TW = (d.W >= 16) ? 16 : 8;
    p.TH = 128 / p.TW;
    // N tile: 16 or 32; columns past Cout_pad are zero-filled by the weight TMA and never stored
    int bn = d.block_n;
    if (bn == 0) bn = d.Cout_pad > 16 ? 32 : 16;
    if (bn != 16 && bn != 32) return "bad block_n";

    // TD: output planes per tile. Their accumulators live in the consumer warpgroups' registers: TD * block_n <= 128
    // fp32 columns (64 registers per thread).
    int td = d.td ? d.td : std::min(4, 128 / bn);
    td = std::max(1, std::min(td, d.D));
    if (!any3 && !d.td) td = std::min(td, 2);    // no plane re-use without kd taps: smaller tiles, more CTAs (unless forced)
    if (td == 3) td = 2;                // the kernel is instantiated for TD = 1, 2, 4
    if (td * bn > 128) return "TD*block_n exceeds the register accumulator budget (128)";
    if (!d.td && td > 1) {
        // wave quantisation: prefer the plane count with the better last-round fill
        auto fill = [&](int t) {
            const long long tiles = conv_work_items(d.NB, (d.D + t - 1) / t, (d.H + p.TH - 1) / p.TH, (d.W + p.TW - 1) / p.TW,
                                                    (d.Cout_pad + bn - 1) / bn, 1);
            const long long rounds = (tiles + sms - 1) / sms;
            return (double)tiles / (double)(rounds * sms) * (t == td ? 1.0 : 0.93);   // halving TD costs ~7 % more slab traffic
        };
        if (fill(td / 2) > fill(td)) td /= 2;
    }
    p.TD = td;
    p.block_n = bn;
    p.w_stage_bytes = max_taps * bn * 128;
    return nullptr;
}

// Voxel-major stages: two whole-phase weight stages when they fit beside two slab stages, else one; then up to 6 slab stages.
static bool vm_stages(const ConvKernelParams& p, int avail, int& ws, int& ss) {
    ws = (2 * p.w_stage_bytes + 2 * p.s_stage_bytes <= avail) ? 2 : 1;
    if (ws * p.w_stage_bytes + 2 * p.s_stage_bytes > avail) return false;
    ss = std::min(std::min(kMaxSStages, 6), (avail - ws * p.w_stage_bytes) / p.s_stage_bytes);
    return true;
}

int conv_plan_create(const ConvDesc& d, int* d_err_flag, ConvPlan& plan, char* err, int errlen) {
    auto fail = [&](const char* m) { snprintf(err, errlen, "conv_plan_create: %s", m); return 1; };
    PFN_encodeTiled enc = get_encode_fn();
    if (!enc) return fail("cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
    if (d.srcs.empty() || d.segs.empty()) return fail("no sources/segments");
    for (const auto& s : d.srcs)
        if (s.C % 64) return fail("source channels must be a multiple of 64");
    if (d.Cout_pad % 16 || d.Cout_pad < d.Cout) return fail("Cout_pad must be a multiple of 16 >= Cout");

    ConvKernelParams& p = plan.p;
    memset(&p, 0, sizeof(p));
    p.NB = d.NB; p.D = d.D; p.H = d.H; p.W = d.W; p.stride = d.stride;
    p.Cout = d.Cout;
    const int out_ld = d.out_ld ? d.out_ld : d.Cout;

    const auto slots = conv_src_slots(d);
    if ((int)slots.size() > kConvMaxSrc) return fail("too many (source, tap-class) slots");
    const std::vector<ConvPhase> phases = conv_build_phases(d);
    p.n_phases = (int)phases.size();
    int max_taps = 1, max_kh = 1, max_kd = 1;
    bool any3 = false;
    for (const auto& P : phases) {
        max_taps = std::max(max_taps, P.n_kh * P.n_kd);
        max_kh = std::max(max_kh, (int)P.n_kh);
        max_kd = std::max(max_kd, (int)P.n_kd);
        any3 |= (P.n_kh == 3);
    }

    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);

    // Orientation. Channel-major puts 64 output channels on the wgmma M side and up to 256 voxels on N: the widest MMA, the
    // least shared-memory operand traffic per MAC and a phase's weights reused over up to 512 voxels. It needs outputs of at
    // least 64 channels (M is 64 wide) written as 16-byte NDHWC vectors; the narrow heads and the projector, which would
    // leave most of M empty, and planar outputs take the voxel-major kernel.
    plan.channel_major = d.Cout >= 64 && d.Cout % 4 == 0 && !d.out_planar && out_ld % 4 == 0 && d.out_c0 % 4 == 0 &&
                         reinterpret_cast<uintptr_t>(d.out) % 16 == 0 && reinterpret_cast<uintptr_t>(d.residual) % 16 == 0;
    const char* bad = plan.channel_major ? cm_geometry(d, sms, max_kh, p) : vm_geometry(d, sms, any3, max_taps, p);
    if (bad) return fail(bad);
    p.n_tiles = (d.Cout_pad + p.block_n - 1) / p.block_n;
    p.tiles_w = (d.W + p.TW - 1) / p.TW;
    p.tiles_h = (d.H + p.TH - 1) / p.TH;
    p.tiles_d = (d.D + p.TD - 1) / p.TD;

    // split-K
    const int items = conv_work_items(d.NB, p.tiles_d, p.tiles_h, p.tiles_w, p.n_tiles, 1);
    int split = d.split_k;
    if (split <= 0) {
        split = 1;
        while (items * split < 120 && split * 2 <= p.n_phases && split < 64) split *= 2;
    }
    split = std::max(1, std::min(split, p.n_phases));
    if ((long long)p.n_phases * (split + 1) >= (1ll << 31)) return fail("too many phases for the split-K bookkeeping");
    p.split_k = split;
    p.atomic_out = split > 1;
    plan.needs_zero = split > 1;

    // shared memory plan
    for (size_t i = 0; i < slots.size(); ++i) p.slab_rows[i] = p.TW * (p.TH + slots[i].n_kh - 1);
    int max_rows = 0;
    for (size_t i = 0; i < slots.size(); ++i) max_rows = std::max(max_rows, p.slab_rows[i]);
    p.s_stage_bytes = max_rows * 128;
    // control block: barriers + per-warp statistics rows; the 1 KB alignment slack is dropped when exactly that buys
    // another slab stage (the kernel then verifies the base alignment itself)
    plan.fused_stats = d.stats != nullptr && split == 1 && d.Cout <= kStatsMaxC && !d.out_planar;
    p.stats_ld = (d.Cout + 31) / 32 * 32;
    const int stats_bytes = plan.fused_stats ? 2 * p.stats_ld * 4 : 0;
    const int ctl_core = kCtlBarrierBytes + (plan.channel_major ? 2 * kCmStageFloats * 4 : 0) + stats_bytes;
    auto plan_stages = [&](int slack, int& ws, int& ss) {
        const int avail = 227 * 1024 - ctl_core - slack;
        return plan.channel_major ? cm_stages(p, max_kd, avail, ws, ss) : vm_stages(p, avail, ws, ss);
    };
    int ws1 = 0, ss1 = 0, ws0 = 0, ss0 = 0;
    const bool ok1 = plan_stages(1024, ws1, ss1), ok0 = plan_stages(0, ws0, ss0);
    if (!ok0) return fail("tile does not fit in shared memory");
    if (ok1 && ws1 >= ws0 && ss1 >= ss0) { p.smem_slack = 1024; p.w_stages = ws1; p.s_stages = ss1; }
    else { p.smem_slack = 0; p.w_stages = ws0; p.s_stages = ss0; }
    const int ctl_bytes = ctl_core + p.smem_slack;
    plan.smem_bytes = p.w_stages * p.w_stage_bytes + p.s_stages * p.s_stage_bytes + ctl_bytes;

    if (encode_a_maps(d, p, enc, err, errlen)) return 1;
    {
        const int K = conv_k_total(d);
        cuuint64_t gdim[2] = {(cuuint64_t)K, (cuuint64_t)d.Cout_pad};
        cuuint64_t gstr[1] = {(cuuint64_t)K * 2};
        cuuint32_t box[2] = {64, (cuuint32_t)p.block_n};
        cuuint32_t estr[2] = {1, 1};
        CUresult r = enc(&p.tmB, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void*)d.weights, gdim, gstr, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { snprintf(err, errlen, "cuTensorMapEncodeTiled(B) failed: %d", (int)r); return 1; }
    }

    if (cudaMalloc(&plan.d_phases, phases.size() * sizeof(ConvPhase)) != cudaSuccess) return fail("cudaMalloc phases");
    cudaMemcpy(plan.d_phases, phases.data(), phases.size() * sizeof(ConvPhase), cudaMemcpyHostToDevice);
    p.phases = plan.d_phases;

    p.bias = d.bias; p.residual = d.residual; p.out = d.out;
    p.out_ld = out_ld; p.out_c0 = d.out_c0; p.out_planar = d.out_planar;
    p.err_flag = d_err_flag;
    p.stats = plan.fused_stats ? d.stats : nullptr;
    p.stats_scalar = d.stats_scalar ? 1 : 0;
    plan.out_item_bytes = d.out_planar ? (size_t)d.Cout * d.D * d.H * d.W * 4
                                       : (size_t)d.D * d.H * d.W * p.out_ld * 4;

    plan.grid = std::min(items * split, sms);

    plan.kernel = plan.channel_major ? conv_cm_kernel_for(p.TH * p.TW) : conv_kernel_for(p.block_n, p.TD);
    plan.threads = plan.channel_major ? kConvCmThreads : kConvThreads;
    if (cudaFuncSetAttribute(plan.kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) != cudaSuccess)
        return fail("cudaFuncSetAttribute(max dynamic smem)");
    return 0;
}

void conv_plan_destroy(ConvPlan& plan) {
    if (plan.d_phases) cudaFree(plan.d_phases);
    plan.d_phases = nullptr;
}

int conv_plan_launch(const ConvPlan& plan, int nb, cudaStream_t stream) {
    if (nb < 1 || nb > plan.p.NB) return (int)cudaErrorInvalidValue;
    ConvKernelParams p = plan.p;
    p.NB = nb;
    const int grid = std::min(plan.grid, conv_work_items(nb, p.tiles_d, p.tiles_h, p.tiles_w, p.n_tiles, p.split_k));
    // split-K accumulates with red.add: only the channel slice written by this conv may be cleared when out_ld > Cout, so
    // callers with sliced outputs must not use split-K. `out` holds the launched items only: clear those.
    if (plan.needs_zero) cudaMemsetAsync(p.out, 0, plan.out_item_bytes * (size_t)nb, stream);
    plan.kernel<<<grid, plan.threads, plan.smem_bytes, stream>>>(p);
    return (int)cudaGetLastError();
}

}  // namespace pixie
