// Implicit-GEMM 3-D convolution on Hopper tensor cores (wgmma, sm_90a), host-side description.
//
// Replaces, for the U-Net path, every torch.nn.Conv3d / Conv1d call of the reference
// (third_party/Wavelet-Generation/models/module/diffusion_network.py:69-71, 91, 208-209, 571-581,
//  663, 674, 687-694, 776, 872) with one persistent, warp-specialised kernel.
//
// Data layout: activations are NDHWC fp16 (the layout voxelize.py:86,111 already writes to disk),
// weights are packed per "phase" (see below) as fp16 [Cout_pad][K] with K contiguous, accumulation
// is fp32 in registers, outputs are fp32 (NDHWC, or NCDHW planar for the network head).
//
// GEMM view, two orientations chosen by the planner from the output shape:
//  * channel-major (every output of 64 or more channels): M = 64 output channels, N = NV voxels of one d-plane (TH x TW =
//    8 x 8, 8 x 16 or 16 x 16), K = taps x input channels in chunks of 64. The two consumer warpgroups take the two planes of
//    a TD = 2 tile (NV / 2 fp32 accumulator registers per thread) and write their outputs through shared memory; a producer
//    warpgroup issues the TMA loads and hands its registers to them.
//  * voxel-major (narrow outputs: the network heads, the 32-channel projector; planar outputs): M = output voxels (tile = TD planes x TH x
//    TW, TH*TW = 128 rows per accumulator), N = output channels (BLOCK_N of 16 or 32 per CTA tile). Each of the two consumer
//    warpgroups computes 64 of the 128 rows for all TD planes and writes them out itself; one producer warp issues the TMA loads.
//
// The K loop is organised in PHASES so that shared memory, not L2, serves the tap re-use:
//   phase = (source tensor, 64-channel chunk, kw)  for 3x3x3 stride-1 convolutions.
// For one phase the CTA marches over the TD+2 input planes of its tile; every plane slab ((TH+2) x TW
// voxels x 64 ch, loaded once by TMA with zero-fill for the padding) feeds up to 9 MMAs: kh shifts are
// 1024 B-aligned row offsets into the slab (TW is a multiple of 8 rows of 128 B), kd shifts select the
// output plane the MMA targets. kw needs its own slab copy because a one-voxel shift along w is not a
// multiple of the 8-row swizzle atom.  1x1x1 convolutions (projector, ResBlock skip, attention
// qkv/proj) and stride-2 taps are phases with n_kh = n_kd = 1.
// The phase's 9 (kd,kh) weight tiles reach shared memory in UNITS of whole kd taps, unit u loaded
// just before slab u: voxel-major keeps all of them resident as one unit per phase, channel-major
// rings one kd tap (its n_kh tiles) per unit and releases it as soon as its last slab retires.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cstdint>
#include <vector>

namespace pixie {

constexpr int kConvMaxSrc = 8;
constexpr int kF8Shift = 6;        // power-of-two rebalancing between the E5M2 operands (see ConvDesc::Seg)
constexpr int kConvThreads = 288;    // voxel-major: warps 0-7: two MMA + epilogue warpgroups, warp 8: TMA producer
constexpr int kConvCmThreads = 384;  // channel-major: warps 0-7 as above, warps 8-11: producer warpgroup (warp 8 issues)

struct ConvPhase {        // 16 bytes, lives in global memory
    int8_t src;           // tensor-map index of the activation source
    int8_t dw;            // w offset of the slab origin relative to w0*stride
    int8_t dh0;           // h offset
    int8_t dd0;           // d offset
    int8_t n_kh;          // 1 or 3: kh taps served by row offsets inside one slab
    int8_t n_kd;          // 1 or 3: kd taps served by plane marching
    int16_t c0;           // first channel of the 64-channel chunk inside the source
    int32_t wtile_base;   // index of this phase's first weight tile (64 K-columns each)
    int32_t f8;           // 1: operands are E5M2 bytes (128 per row instead of 64 halfs), issued as wgmma .e5m2 (K = 32)
};
static_assert(sizeof(ConvPhase) == 16, "ConvPhase layout");

// Packed weight tile (64 K-columns) of tap (kh, kd) of a phase whose tiles start at wtile_base: kh major, then
// kd = n_kd - 1 .. 0, so that the kd taps a slab feeds are adjacent.
__host__ __device__ __forceinline__ int conv_wtile(int wtile_base, int n_kd, int kh, int kd) {
    return wtile_base + kh * n_kd + (n_kd - 1 - kd);
}

// Work items of a launch: one per (batch item, tile, channel tile, split-K range).
__host__ __device__ __forceinline__ int conv_work_items(int nb, int tiles_d, int tiles_h, int tiles_w, int n_tiles, int split_k) {
    return nb * tiles_d * tiles_h * tiles_w * n_tiles * split_k;
}

struct ConvKernelParams {
    CUtensorMap tmA[kConvMaxSrc];
    CUtensorMap tmB;
    const ConvPhase* phases;
    int n_phases;
    int split_k;          // phases are divided into split_k contiguous ranges
    // output geometry
    int NB, D, H, W;      // batch and OUTPUT spatial size
    int stride;           // 1 or 2
    int TW, TH, TD;       // tile: TH*TW == 128, TD in {1, 2, 4} (voxel-major); TH*TW == NV, TD == 2 (channel-major)
    int tiles_w, tiles_h, tiles_d;
    int Cout;             // real output channels
    int block_n;          // output channels per tile: 16 or 32 (voxel-major), 64 (channel-major)
    int n_tiles;          // ceil(Cout / block_n)
    // shared-memory plan
    int w_stage_bytes, w_stages;   // weight stages: all taps of one phase (voxel-major), one kd tap's n_kh tiles (channel-major)
    int s_stage_bytes, s_stages;   // slab stages
    int slab_rows[kConvMaxSrc];    // rows per slab for each source (TW * (TH + n_kh - 1))
    // epilogue
    const float* bias;       // [Cout] or nullptr
    const float* residual;   // same layout as out, or nullptr
    float* out;              // fp32
    int out_ld;              // channel stride of an NDHWC row (>= Cout)
    int out_c0;              // channel offset inside the row
    int out_planar;          // 1: write NCDHW (out[(n*Cout+c)*DHW + vox])
    int atomic_out;          // 1: red.add into out (split_k > 1); out must be pre-zeroed
    double* stats;           // optional [NB][Cout][2] = (sum, sum of squares) of the outputs over voxels,
                             // accumulated by the epilogue (fused LayerNorm/GroupNorm statistics); or nullptr
    int stats_ld;            // floats per statistics row in shared memory (Cout rounded up to 32)
    int smem_slack;          // bytes reserved for aligning the dynamic smem base to 1 KB (0: the base must already be aligned)
    int stats_scalar;        // 1: only the per-item totals are wanted; they land in channel 0's slot (LayerNorm consumers)
    int* err_flag;           // device int, set non-zero on pipeline timeout
};

typedef void (*ConvKernelFn)(ConvKernelParams);

// One activation source of a convolution.
struct ConvSrc {
    const __half* ptr;    // NDHWC fp16, [NB][Din][Hin][Win][C]
    int C;                // channels (multiple of 64)
    int Din, Hin, Win;
};

// Host description of one convolution launch.
struct ConvDesc {
    int NB = 1;
    int D = 0, H = 0, W = 0;   // output size
    int stride = 1;
    int Cout = 0;
    // K segments: each segment is (source, kernel size 1 or 3) over all of the source's channels.
    // wlo = 1 packs the fp16 rounding residual of the weights (w - fp16(w)) for split-precision mode.
    // f8 = 1: an E5M2 correction segment (tensor-core rate 2x fp16). Its source rows hold, per 64-channel chunk, 64 bytes
    // e5m2(a_lo * 2^kF8Shift) followed by 64 bytes e5m2(a * 2^-kF8Shift); its weight rows hold e5m2(w * 2^-kF8Shift) followed by
    // e5m2(w_lo * 2^kF8Shift), so one K = 128-byte chunk accumulates a_lo*w + a*w_lo — the two first-order terms a single
    // fp16 pass loses — into the same fp32 accumulator (`C` of such a source counts 2-byte units like the fp16 ones).
    // lo = 1 marks a segment over an activation rounding residual (a_lo * w in split-precision mode). Residual segments
    // (lo, wlo, f8) run before the others: see conv_build_phases.
    struct Seg { int src; int ks; int wlo = 0; int f8 = 0; int lo = 0; };
    std::vector<ConvSrc> srcs;
    std::vector<Seg> segs;
    const __half* weights = nullptr;   // packed by pack_conv_weights(), [Cout_pad][K_total]
    int Cout_pad = 0;                  // rows in the packed weight matrix (multiple of 16)
    const float* bias = nullptr;
    const float* residual = nullptr;
    float* out = nullptr;
    int out_ld = 0, out_c0 = 0, out_planar = 0;
    double* stats = nullptr;           // request fused output statistics (honoured iff plan.fused_stats)
    bool stats_scalar = false;         // totals only (see ConvKernelParams::stats_scalar)
    int split_k = 1;                   // >1 => atomics into pre-zeroed out
    int block_n = 0;                   // voxel-major: 0 = choose; else 16 or 32
    int td = 0;                        // voxel-major: 0 = choose
    int nv = 0;                        // channel-major voxels per plane tile: 0 = choose; else 64, 128 or 256
};

// K_total (in elements) of a ConvDesc: sum over segments of ks^3 * C.
int conv_k_total(const ConvDesc& d);

// Builds the phase table for `d` (host vector).
std::vector<ConvPhase> conv_build_phases(const ConvDesc& d);

// Packs torch-layout weights [Cout][Cin_seg][kd][kh][kw] (fp32, one tensor per segment) into the
// phase-ordered fp16 matrix [Cout_pad][K_total] expected by the kernel (host memory).
void conv_pack_weights(const ConvDesc& d, const std::vector<const float*>& seg_weights,
                       const std::vector<int>& seg_cin_real, std::vector<__half>& packed);

// A prepared launch: tensor maps encoded, phase table uploaded.
struct ConvPlan {
    ConvKernelParams p{};
    ConvPhase* d_phases = nullptr;
    ConvKernelFn kernel = nullptr;     // instance for (block_n, TD) or, channel-major, NV
    bool channel_major = false;
    int threads = 0;                   // kConvThreads or kConvCmThreads
    int grid = 0;
    int smem_bytes = 0;
    bool needs_zero = false;   // out must be zeroed before launch (atomic_out)
    bool fused_stats = false;  // the epilogue accumulates ConvDesc::stats (needs split_k == 1, Cout <= 256)
    size_t out_item_bytes = 0; // bytes of `out` per batch item; a split-K launch clears the launched items' share
};

// Returns 0 on success; on failure returns non-zero and fills `err`.
int conv_plan_create(const ConvDesc& d, int* d_err_flag, ConvPlan& plan, char* err, int errlen);
void conv_plan_destroy(ConvPlan& plan);
// Launches the plan for the first nb batch items (1 <= nb <= the planned batch; `out` need only hold those): fewer
// items only shrink the tile count. Returns 0 or a CUDA error code.
int conv_plan_launch(const ConvPlan& plan, int nb, cudaStream_t stream);
// Re-encode the activation tensor maps after the source pointers in `d` changed (same shapes).
int conv_plan_retarget(const ConvDesc& d, ConvPlan& plan, char* err, int errlen);
}  // namespace pixie
