// Shared host/device helpers for libnphm_b200.so (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdarg>
#include "../../include/nphm_b200.h"

namespace nphm {

void set_error(const char *fmt, ...);

#define NPHM_CUDA_CHECK(expr)                                                              \
    do {                                                                                   \
        cudaError_t _e = (expr);                                                           \
        if (_e != cudaSuccess) {                                                           \
            nphm::set_error("%s failed at %s:%d: %s", #expr, __FILE__, __LINE__,           \
                            cudaGetErrorString(_e));                                       \
            return NPHM_ERR_CUDA;                                                          \
        }                                                                                  \
    } while (0)

#define NPHM_REQUIRE(cond, ...)                                                            \
    do {                                                                                   \
        if (!(cond)) {                                                                     \
            nphm::set_error(__VA_ARGS__);                                                  \
            return NPHM_ERR_INVALID;                                                       \
        }                                                                                  \
    } while (0)

inline int round_up(int x, int m) { return (x + m - 1) / m * m; }
inline long long ceil_div(long long a, long long b) { return (a + b - 1) / b; }

// Members and weight sets of an ensemble: members 2z and 2z + 1 of the first 2 n_symm are a mirrored pair sharing weight
// set z; every later member m has its own set m - n_symm.  A plain MLP is one member, n_symm = 0.
__host__ __device__ __forceinline__ int member_set(int m, int n_symm) { return m < 2 * n_symm ? m >> 1 : m - n_symm; }
struct SetMembers { int first, count; };
__host__ __device__ __forceinline__ SetMembers set_members(int z, int n_symm)
{
    return z < n_symm ? SetMembers{2 * z, 2} : SetMembers{z + n_symm, 1};
}

int sm_count();

// ---------------------------------------------------------------------------------------------
// Network description shared by the SIMT ensemble / MLP kernels.
// A "folded" network: the latent part of every layer input is constant over the points of a query, so it
// is pre-multiplied into a per-(query, member) constant vector `cvec`; the kernels only see the
// point-dependent columns (xyz, hidden activations).
//   layer l:  out[n] = act( sum_{k<K} Wt[set][k][n] * in[k]  +  cvec[q][member][coff + n] )
//   in of layer 0          = xyz (3)
//   in of the skip layer   = [h_{skip-1} (N_{skip-1}) , xyz (3)]     (1/sqrt(2) folded into Wt)
// ---------------------------------------------------------------------------------------------
constexpr int kMaxLayers = 12;

struct FoldedLayer {
    const float *Wt;      // [n_sets][K][Npad]
    int K;                // point-dependent input width
    int N;                // true output width
    int Npad;             // multiple of 8
    int coff;             // offset of this layer inside a cvec record
    int act;              // 1 = softplus(beta=100), 0 = identity
};

struct FoldedNet {
    int n_layers;                 // number of linear layers
    int skip;                     // index of the layer that re-reads xyz (or -1)
    int n_members;                // 1 for a plain MLP
    int n_symm;                   // weight sharing (0 for a plain MLP)
    int cvec_stride;              // floats per (query, member) record
    int max_rows;                 // rows of one activation buffer
    FoldedLayer L[kMaxLayers];
};

// softplus(beta=100, threshold=20) exactly as torch: x if 100x > 20 else log1p(exp(100x))/100
__device__ __forceinline__ float softplus100_exact(float x)
{
    float bx = x * 100.0f;
    return bx > 20.0f ? x : log1pf(expf(bx)) / 100.0f;
}
// derivative: sigmoid(100x) (1 beyond the threshold, as torch's backward)
__device__ __forceinline__ float softplus100_grad(float x)
{
    float bx = x * 100.0f;
    if (bx > 20.0f) return 1.0f;
    float e = expf(bx);
    return e / (e + 1.0f);
}

}  // namespace nphm
