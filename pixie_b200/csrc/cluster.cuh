// Density-based clustering of particle subsets on the device (SURVEY.md 8f-1); see cluster.cu.
#pragma once
#include <cuda_runtime.h>

namespace pixie {

// DBSCAN (scikit-learn semantics) over the points i of pos [n][3] with ids[i] == select_id (all points when ids is null),
// taken in index order. index[t] = original index of the t-th selected point, labels[t] = its cluster label or -1; both
// need room for n entries. *n_selected_host / *n_clusters_host receive the counts (the call synchronises the stream).
cudaError_t dbscan(const float* pos, int n, const int* ids, int select_id, double eps, int min_samples, int* index, int* labels,
                   int* n_selected_host, int* n_clusters_host, cudaStream_t st);

// Per-cluster point count (core and border points) and float32 bounding box of the selected points labelled by dbscan.
// sizes [n_clusters], bbox_min / bbox_max [n_clusters][3].
cudaError_t cluster_stats(const float* pos, const int* index, const int* labels, int n_selected, int n_clusters, int* sizes,
                          float* bbox_min, float* bbox_max, cudaStream_t st);

}  // namespace pixie
