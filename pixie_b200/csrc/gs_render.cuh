// Forward Gaussian-splatting rasterizer (the renderer gs_simulation.py:573-631 calls; see gs_render.cu).
#pragma once
#include <cuda_runtime.h>
#include "../../include/pixie_b200.h"

namespace pixie {

using GsRenderer = pixie_gs_renderer_s;    // the C ABI's handle is the renderer itself (gs_render.cu)

struct GsRenderArgs {
    const float* means;      // [n][3]
    const float* cov;        // [n][6] upper triangle: xx xy xz yy yz zz
    const float* opacity;    // [n]
    const float* shs;        // [n][sh_coeffs][3] or NULL (then colors)
    const float* colors;     // [n][3] or NULL (then shs)
    int n, sh_coeffs, sh_degree;
    float view[16], proj[16];  // world_view_transform / full_proj_transform as stored (row-vector convention)
    float campos[3], bg[3];
    float tan_fovx, tan_fovy;
    int width, height;
    float* image;            // [3][height][width]
    int* radii;              // [n]
};

GsRenderer* gs_renderer_create();    // nullptr, with the message of pixie_last_error() set, on failure
void gs_renderer_destroy(GsRenderer* r);
// One frame on `st`. Synchronises `st` once, for the number of (Gaussian, tile) pairs. *n_rendered receives it. With
// phase_ms non-NULL, also records events between the phases and writes their times (preprocess, scan + keys, sort,
// ranges, blend; a second synchronise). Returns 0, or 1 with the message of pixie_last_error() set. `st` first waits for
// the end of the renderer's previous frame, so frames on different streams run in call order. One host thread at a time
// per renderer.
int gs_render(GsRenderer* r, const GsRenderArgs& a, int* n_rendered, float* phase_ms, cudaStream_t st);

}  // namespace pixie
