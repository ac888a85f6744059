// Device-side layer routines shared by the SIMT forward kernel (simt.cu) and the fitting kernels (fit.cu).
// Activations of a tile of P = 32*TM points live in shared memory as [row][point]; every warp covers all points of
// the tile and a slice of the output columns with a TM x 8 register tile.
#pragma once
#include "common.cuh"

namespace nphm {

template <int TM>
__device__ __forceinline__ void load_act(const float *p, float (&a)[TM])
{
    if constexpr (TM == 4) {
        float4 v = *reinterpret_cast<const float4 *>(p);
        a[0] = v.x; a[1] = v.y; a[2] = v.z; a[3] = v.w;
    } else if constexpr (TM == 2) {
        float2 v = *reinterpret_cast<const float2 *>(p);
        a[0] = v.x; a[1] = v.y;
    } else {
        a[0] = *p;
    }
}
template <int TM>
__device__ __forceinline__ void store_act(float *p, const float (&a)[TM])
{
    if constexpr (TM == 4) {
        *reinterpret_cast<float4 *>(p) = make_float4(a[0], a[1], a[2], a[3]);
    } else if constexpr (TM == 2) {
        *reinterpret_cast<float2 *>(p) = make_float2(a[0], a[1]);
    } else {
        *p = a[0];
    }
}

// out[n][p] = act(sum_k Wt[k][n] in[k][p] + cvec[n]) for all n < N; warps split the columns.
template <int TM>
__device__ __forceinline__ void dense_layer(const FoldedLayer &L, const float *__restrict__ Wt,
                                            const float *__restrict__ cvec, const float *in_s, float *out_s,
                                            int warp, int lane, int nwarps)
{
    constexpr int P = 32 * TM;
    const int K = L.K, Npad = L.Npad;
    for (int n0 = warp * 8; n0 < L.N; n0 += nwarps * 8) {
        float acc[TM][8];
        {
            const float4 c0 = __ldg(reinterpret_cast<const float4 *>(cvec + n0));
            const float4 c1 = __ldg(reinterpret_cast<const float4 *>(cvec + n0 + 4));
#pragma unroll
            for (int i = 0; i < TM; ++i) {
                acc[i][0] = c0.x; acc[i][1] = c0.y; acc[i][2] = c0.z; acc[i][3] = c0.w;
                acc[i][4] = c1.x; acc[i][5] = c1.y; acc[i][6] = c1.z; acc[i][7] = c1.w;
            }
        }
        const float *w = Wt + n0;
        const float *a_ptr = in_s + lane * TM;
#pragma unroll 4
        for (int k = 0; k < K; ++k) {
            float a[TM];
            load_act<TM>(a_ptr + k * P, a);
            const float4 w0 = __ldg(reinterpret_cast<const float4 *>(w + (size_t)k * Npad));
            const float4 w1 = __ldg(reinterpret_cast<const float4 *>(w + (size_t)k * Npad + 4));
#pragma unroll
            for (int i = 0; i < TM; ++i) {
                acc[i][0] = fmaf(a[i], w0.x, acc[i][0]); acc[i][1] = fmaf(a[i], w0.y, acc[i][1]);
                acc[i][2] = fmaf(a[i], w0.z, acc[i][2]); acc[i][3] = fmaf(a[i], w0.w, acc[i][3]);
                acc[i][4] = fmaf(a[i], w1.x, acc[i][4]); acc[i][5] = fmaf(a[i], w1.y, acc[i][5]);
                acc[i][6] = fmaf(a[i], w1.z, acc[i][6]); acc[i][7] = fmaf(a[i], w1.w, acc[i][7]);
            }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            if (n0 + j < L.N) {
                float o[TM];
#pragma unroll
                for (int i = 0; i < TM; ++i) o[i] = L.act ? softplus100_exact(acc[i][j]) : acc[i][j];
                store_act<TM>(out_s + (size_t)(n0 + j) * P + lane * TM, o);
            }
        }
    }
}

// N <= 8: warps split K instead, partial sums go through rows [8, 8 + nwarps*8) of out_s.
template <int TM>
__device__ __forceinline__ void narrow_layer(const FoldedLayer &L, const float *__restrict__ Wt,
                                             const float *__restrict__ cvec, const float *in_s, float *out_s,
                                             int warp, int lane, int nwarps)
{
    constexpr int P = 32 * TM;
    const int K = L.K, Npad = L.Npad;      // Npad == 8
    float acc[TM][8];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
    const float *a_ptr = in_s + lane * TM;
    for (int k = warp; k < K; k += nwarps) {
        float a[TM];
        load_act<TM>(a_ptr + k * P, a);
        const float4 w0 = __ldg(reinterpret_cast<const float4 *>(Wt + (size_t)k * Npad));
        const float4 w1 = __ldg(reinterpret_cast<const float4 *>(Wt + (size_t)k * Npad + 4));
#pragma unroll
        for (int i = 0; i < TM; ++i) {
            acc[i][0] = fmaf(a[i], w0.x, acc[i][0]); acc[i][1] = fmaf(a[i], w0.y, acc[i][1]);
            acc[i][2] = fmaf(a[i], w0.z, acc[i][2]); acc[i][3] = fmaf(a[i], w0.w, acc[i][3]);
            acc[i][4] = fmaf(a[i], w1.x, acc[i][4]); acc[i][5] = fmaf(a[i], w1.y, acc[i][5]);
            acc[i][6] = fmaf(a[i], w1.z, acc[i][6]); acc[i][7] = fmaf(a[i], w1.w, acc[i][7]);
        }
    }
    float *scratch = out_s + (size_t)8 * P;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        if (j < L.N) {
            float o[TM];
#pragma unroll
            for (int i = 0; i < TM; ++i) o[i] = acc[i][j];
            store_act<TM>(scratch + (size_t)(warp * 8 + j) * P + lane * TM, o);
        }
    }
    __syncthreads();
    for (int t = threadIdx.x; t < L.N * P; t += blockDim.x) {
        const int n = t / P, p = t - n * P;
        float s = __ldg(cvec + n);
        for (int w = 0; w < nwarps; ++w) s += scratch[(size_t)(w * 8 + n) * P + p];
        out_s[(size_t)n * P + p] = L.act ? softplus100_exact(s) : s;
    }
}


// Backward of one dense layer, in place:  rows[j][p] <- scale * (sum_n W[n][j] * delta[n][p]) * sigma'(h[j][p])
//   W      reference layout [n_out][ldw] (row n of the forward weight), only columns j < J are used
//   delta  [n_out][P] rows of the upstream gradient
//   rows   on entry the forward activations h_prev (softplus outputs), on exit delta_prev
// sigma'(pre) = sigmoid(100 pre) = 1 - exp(-100 h) since h = softplus_100(pre); torch's threshold branch
// (100 pre > 20 -> derivative exactly 1) is reproduced through h > 0.2.
template <int TM>
__device__ __forceinline__ void dense_layer_bwd(const float *__restrict__ W, int ldw, int n_out, int J, float scale,
                                                const float *delta_s, float *rows_s, int warp, int lane, int nwarps)
{
    constexpr int P = 32 * TM;
    // the rows of W are 16-byte aligned only when W is and ldw is a multiple of 4 (a hidden width such as 77 is not)
    const bool vec = (reinterpret_cast<uintptr_t>(W) & 15) == 0 && (ldw & 3) == 0;
    for (int j0 = warp * 8; j0 < J; j0 += nwarps * 8) {
        float acc[TM][8];
#pragma unroll
        for (int i = 0; i < TM; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
        const float *w = W + j0;
        const float *d_ptr = delta_s + lane * TM;
        const bool full = vec && j0 + 8 <= J;
#pragma unroll 4
        for (int n = 0; n < n_out; ++n) {
            float a[TM];
            load_act<TM>(d_ptr + n * P, a);
            float wv[8];
            if (full) {
                const float4 w0 = __ldg(reinterpret_cast<const float4 *>(w + (size_t)n * ldw));
                const float4 w1 = __ldg(reinterpret_cast<const float4 *>(w + (size_t)n * ldw + 4));
                wv[0] = w0.x; wv[1] = w0.y; wv[2] = w0.z; wv[3] = w0.w; wv[4] = w1.x; wv[5] = w1.y; wv[6] = w1.z; wv[7] = w1.w;
            } else {
#pragma unroll
                for (int j = 0; j < 8; ++j) wv[j] = j0 + j < J ? __ldg(w + (size_t)n * ldw + j) : 0.f;
            }
#pragma unroll
            for (int i = 0; i < TM; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], wv[j], acc[i][j]);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            if (j0 + j < J) {
                float *ptr = rows_s + (size_t)(j0 + j) * P + lane * TM;
                float h[TM], o[TM];
                load_act<TM>(ptr, h);
#pragma unroll
                for (int i = 0; i < TM; ++i) {
                    const float sg = h[i] > 0.2f ? 1.0f : -expm1f(-100.0f * h[i]);
                    o[i] = acc[i][j] * scale * sg;
                }
                store_act<TM>(ptr, o);
            }
        }
    }
}

}  // namespace nphm
