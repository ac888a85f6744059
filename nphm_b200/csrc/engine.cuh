// Handle types behind the C ABI.
#pragma once
#include "common.cuh"
#include "simt.cuh"
#include <algorithm>

namespace nphm {

struct DeviceBuffer {
    void *ptr = nullptr;
    size_t cap = 0;
    int reserve(size_t bytes);          // grows (never shrinks); contents are NOT preserved on growth
    template <class T> T *as() const { return reinterpret_cast<T *>(ptr); }
    DeviceBuffer() = default;
    DeviceBuffer(const DeviceBuffer &) = delete;
    DeviceBuffer &operator=(const DeviceBuffer &) = delete;
    ~DeviceBuffer();
};

struct StackDims {
    int n_lin, skip, cond_dim, cvec_stride, max_rows;
    int in_total[kMaxLayers], N[kMaxLayers], Npad[kMaxLayers], K[kMaxLayers], folded[kMaxLayers], coff[kMaxLayers];
    float scale[kMaxLayers];
};

struct NetWeights {
    DeviceBuffer W[kMaxLayers], b[kMaxLayers];   // copies in the reference layout (used for the per-query constants)
    DeviceBuffer Wt[kMaxLayers];                 // SIMT layout [set][k][Npad]
    int load(const StackDims &s, int n_sets, const float *const *w_dev, const float *const *b_dev, cudaStream_t stream);
};

int build_stack(StackDims &s, int cond_dim, int hidden, int n_layers, int out_dim);
void fill_descriptors(const StackDims &s, const NetWeights &w, int n_members, int n_symm, int lat_dim, int lat_glob,
                      int lat_loc, FoldedNet &net, PackSpec &spec);

}  // namespace nphm

namespace nphm { namespace fit { struct BackwardPacks; } struct PackedChain; }

struct nphm_ensemble {
    nphm_ensemble_config cfg;
    int n_members = 0, n_sets = 0, lat_dim = 0;
    bool loaded = false;
    nphm::StackDims dims;
    nphm::NetWeights weights;
    nphm::FoldedNet net;
    nphm::PackSpec spec;
    nphm::DeviceBuffer pos_w[3], pos_b[3], mean_anchors;
    // per-call scratch
    nphm::DeviceBuffer anchors, cvec, axes, host_latent, host_volume;
    // tensor-core path (tc_ensemble.cu)
    nphm::DeviceBuffer tc_weights, tc_consts, tc_coff, tc_l2slabs;
    nphm::DeviceBuffer tc_masks, tc_sched;     // member mask per tile (pre-pass), work counter of the tile schedule
    nphm::DeviceBuffer tc_absorb, tc_bounds;   // absorption: masks per tile, member bounds per query
    long long tc_mask_tiles = 0;               // tiles whose masks the last launch computed (0: it computed none)
    // debug view of the absorption decisions of the last launch (nphm_debug_ens_*): tiles with absorb masks (0: absorption
    // was off), bounds written, tiles with a skip log; the skip log (members skipped by vote, per tile) only when enabled
    long long tc_absorb_tiles = 0, tc_bound_count = 0, tc_skip_tiles = 0;
    nphm::DeviceBuffer tc_skip_log;
    bool tc_skip_log_on = false;
    // member-major dense grid queries: num, den and the row list of one chunk of tiles, and the rows listed per (chunk,
    // member) by the last launch (tc_mm_counts of them; 0 when it ran tile-major); the member bounds per 32^3-point sub-box
    // of that launch (tc_sub_bound_count of them, sub-boxes from x-slab tc_sub_x0, tc_sub_n per axis; 0 when tile-major)
    nphm::DeviceBuffer tc_mm_num, tc_mm_den, tc_mm_list, tc_mm_count, tc_sub_bounds;
    long long tc_mm_counts = 0, tc_sub_bound_count = 0;
    int tc_sub_x0 = 0, tc_sub_n = 0;
    double tc_bound_scale = 1.0;               // factor on every member bound (1; a debug entry sets it for a negative control)
    bool tc_ready = false;
    bool tc_prune = false;          // opt-in member pruning (NPHM_IMPL_TC_PRUNED)
    float tc_prune_tau = 1e-8f;
    // fitting (fit.cu)
    nphm::DeviceBuffer fit_scratch, fit_apply_scratch;
    nphm::fit::BackwardPacks *fit_packs = nullptr;      // adjoint weights of the backward GEMMs, built on first use
    // stage-1 training through grad_x sdf (mlp_chain.cu): the layer chain of all weight sets, packed on first use
    nphm::PackedChain *sdfgrad = nullptr;
};

namespace nphm { struct MlpChain; }

struct nphm_mlp {
    nphm_mlp_config cfg;
    bool loaded = false;
    nphm::StackDims dims;
    nphm::NetWeights weights;
    nphm::FoldedNet net;
    nphm::PackSpec spec;
    nphm::DeviceBuffer cvec;
    const int *live = nullptr;      // set around an evaluation by the Broyden loop: device counter, 0 = skip the evaluation
    const int *live_rows = nullptr; // set by the compacting Broyden loop: per-query device counts, rows beyond them are skipped
    // layer-by-layer tensor-core passes: any width, Jacobian, adjoint (mlp_chain.cu)
    nphm::MlpChain *chain = nullptr;
};

namespace nphm {
int ensemble_prepare(nphm_ensemble *h, const float *latents_dev, int n_queries, cudaStream_t stream);
// tensor-core ensemble kernel (tc_ensemble.cu)
bool tc_ensemble_supported(const nphm_ensemble *h);
int tc_ensemble_pack(nphm_ensemble *h, cudaStream_t stream);
int tc_ensemble_launch(nphm_ensemble *h, const SimtQuery &q, cudaStream_t stream);
// tensor-core MLP forward (mlp_chain.cu, layer by layer): the deformation backbone is the configuration AUTO sends there
bool tc_mlp_supported(const nphm_mlp *h);
bool chain_packed(const nphm_mlp *h);
int chain_forward(nphm_mlp *h, const float *xyz, int n_queries, long long n_points, float *out, cudaStream_t stream);
// fitting (fit.cu)
void fit_packs_destroy(nphm_ensemble *h);
void ensemble_chain_destroy(nphm_ensemble *h);
// layer chain (mlp_chain.cu)
int chain_pack(nphm_mlp *h, cudaStream_t stream);
void chain_destroy(nphm_mlp *h);
int mlp_prepare(nphm_mlp *h, const float *cond_dev, int n_queries, cudaStream_t stream);
}  // namespace nphm
