// Internal C++ interface of the MPM solver core (wrapped by the C ABI in capi.cu). Functions that return int return 0, or 1
// with the message of pixie_last_error() set.
#pragma once
#include <cuda_runtime.h>
#include "../../include/pixie_b200.h"

namespace pixie {
using Mpm = pixie_mpm_s;    // the C ABI's handle is the solver object itself (mpm.cu)
Mpm* mpm_create(int n_particles, int n_grid, float grid_lim);    // nullptr on failure
void mpm_destroy(Mpm* m);
int mpm_bind(Mpm* m, int field, void* ptr);
int mpm_set_params(Mpm* m, const pixie_mpm_params& p);
int mpm_add_bc(Mpm* m, const pixie_mpm_bc& b);
int mpm_clear_bcs(Mpm* m);
int mpm_set_time(Mpm* m, double t);
int mpm_get_time(Mpm* m, double* t);
int mpm_step(Mpm* m, int n_substeps, double dt, cudaStream_t st);
int mpm_compute_mu_lam(Mpm* m, cudaStream_t st);
int mpm_compute_bulk(Mpm* m, cudaStream_t st);
int mpm_compute_mass(Mpm* m, cudaStream_t st);
int mpm_compute_cov_from_F(Mpm* m, cudaStream_t st);
int mpm_compute_R_from_F(Mpm* m, cudaStream_t st);
int mpm_apply_additional_params(Mpm* m, const float* boxes_host, int n_boxes, cudaStream_t st);
int mpm_select_box(Mpm* m, const float* point, const float* size, int* mask, cudaStream_t st);
int mpm_select_cylinder(Mpm* m, const float* point, const float* normal, float hh, float radius, int* mask, cudaStream_t st);
int mpm_grid_ptrs(Mpm* m, float** mv4, float** v4);
int mpm_sync(Mpm* m, cudaStream_t st);
int mpm_set_active_count(Mpm* m, int n_active);
long long mpm_launch_count(Mpm* m);
int mpm_exchange_buffer(Mpm* m, void** base, size_t* bytes);
int mpm_slab_attach(Mpm* m, int x0, int x1, int slack, const void* left_xbuf, const void* right_xbuf);
int mpm_slab_phase(Mpm* m, int phase, double dt, cudaStream_t st);
int mpm_slab_error(Mpm* m, int* flag);
int mpm_slab_excursion(Mpm* m, int* d_out, cudaStream_t st);
}  // namespace pixie
