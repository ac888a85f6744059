// Host-side launch interface of simt.cu
#pragma once
#include "common.cuh"

namespace nphm {

struct SimtQuery {
    const float *xyz;         // n_queries * n_points * 3, or nullptr -> regular grid from `axes`
    const float *axes;        // 3 * res floats (grid mode)
    int res;
    long long first;          // global index of point 0 (grid mode), 0 otherwise
    long long total;          // index space size: the last point (total-1) always carries the eval quirk
    long long n_points;       // per query
    int n_queries;
    long long quirk_period;   // 0 = off
    const float *cvec;        // [n_queries][n_members][cvec_stride]
    const float *anchors;     // [n_queries][n_members-1][3] (ensemble) or nullptr (plain MLP)
    int blend;                // 1: Gaussian anchor blend of member outputs (ensemble); 0: write channels
    float *out;
    float *members_out;       // optional (tensor-core kernel only): un-blended member outputs [q][point][member]
    float *acts_out;          // optional (tensor-core kernel only): activation derivatives, see tc::Params::acts_out
    unsigned char *acts_packed_out;   // goes with acts_out, see tc::Params::acts_packed_out
    int acts_packed_tile_steps;
    int exact;                // 1: never use the opt-in pruned mode for this query (fitting needs every member)
    const int *live_rows;     // optional (plain MLP): query q computes only its points below live_rows[q] (device counts)
};

// description of the reference-layout parameters, used by the packing / cvec kernels
struct PackLayer {
    const float *W;     // [n_sets][N][in_total]
    const float *b;     // [n_sets][N]
    int N, Npad, in_total;
    int K;              // point-dependent leading columns kept in Wt
    int folded;         // 1: columns [K, in_total) multiply the per-query constant u
    float scale;        // 1/sqrt(2) on the skip layer (inputs are scaled before the affine map), else 1
    int coff;
};

struct PackSpec {
    int n_layers, n_members, n_symm;
    int lat_dim, lat_glob, lat_loc, cond_dim;
    int cvec_stride;
    PackLayer L[kMaxLayers];
};

int launch_folded_net(const FoldedNet &net, const SimtQuery &q, cudaStream_t stream);
// whether launch_folded_net can hold the network's activations in shared memory (hidden widths up to ~880)
bool folded_net_fits(const FoldedNet &net);
int launch_cvec(const PackSpec &spec, const float *latents, int n_queries, float *cvec, cudaStream_t stream);
int launch_anchors(const float *latents, int n_queries, int lat_dim, int lat_glob, int hid, int n_out,
                   const float *const *w, const float *const *b, const float *mean, float *anchors,
                   cudaStream_t stream);
int launch_grid_axes(const double mn[3], const double mx[3], int res, float *axes, cudaStream_t stream);
int launch_pack_wt(const float *W, int n_sets, int N, int in_total, int K, int Npad, float scale, float *Wt,
                   cudaStream_t stream);

}  // namespace nphm
