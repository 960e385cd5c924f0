// Particle filling of hollow Gaussian objects (PG/particle_filling/filling.py:291-380); see particle_fill.cu.
#pragma once
#include <cuda_runtime.h>

namespace pixie {

// densify_grids (filling.py:26-87): count[grid_n^3] int32 = Gaussians per cell, density[grid_n^3] fp32 = sum over the
// Gaussians of opacity * (mean of exp(-1/2 d^T P d) over the cell's 8 corner nodes). Both grids are zeroed first.
// pos [n][3], opacity [n], cov [n][6] (upper triangle), positions already in the grid's frame.
int fill_density(const float* pos, const float* opacity, const float* cov, int n, int grid_n, float grid_dx, int* count,
                 float* density, cudaStream_t st);

// fill_dense_grids + internal_filling (filling.py:90-234) on the grids of fill_density. `count` is updated in place like
// the reference's `grid`. New particles (cell + U[0,1)^3) * grid_dx + origin go to out[max_samples][3], dense-fill ones
// first, each group in C order of cells. *n_dense_host / *n_total_host receive the counts (one stream sync). Returns 3 and
// writes nothing to `out` when the total exceeds max_samples.
int fill_grids(int* count, const float* density, int grid_n, float grid_dx, const float origin[3], float density_thres,
               float search_thres, int max_ppc, int exclude_dir, int ray_dir, unsigned long long seed, float* out, int max_samples,
               int* n_dense_host, int* n_total_host, cudaStream_t st);

}  // namespace pixie
