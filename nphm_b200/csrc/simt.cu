// fp32 FFMA kernels for the folded networks (any configuration): the identity-SDF ensemble and the plain
// DeepSDF MLP.  One CTA owns a tile of P = 32*TM points and walks all members / layers with the activations
// of the tile resident in shared memory ([row][point], conflict free); every warp covers all points of the tile
// and a slice of the output columns with a TM x 8 register tile, weights come through the read-only path as
// warp-uniform 128-bit loads (L1/L2 resident: 11.6 MB for the whole ensemble).
//
// Reference semantics: FastEnsembleDeepSDFMirrored.forward  src/NPHM/models/EnsembledDeepSDF.py:203-267
//                      EnsembledDeepSDF.forward             src/NPHM/models/EnsembledDeepSDF.py:101-126
//                      sample_point_feature                 src/NPHM/models/EnsembledDeepSDF.py:129-150
//                      DeepSDF.forward                      src/NPHM/models/deepSDF.py:64-89
#include "common.cuh"
#include "simt.cuh"
#include "simt_layers.cuh"

namespace nphm {

// ------------------------------------------------------------------------------------------------
// the fused kernel
// ------------------------------------------------------------------------------------------------
template <int TM>
__global__ void __launch_bounds__(256) folded_net_kernel(const FoldedNet net, const SimtQuery q)
{
    constexpr int P = 32 * TM;
    extern __shared__ __align__(16) float smem[];
    float *buf[2] = {smem, smem + (size_t)net.max_rows * P};
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const long long tiles_per_query = (q.n_points + P - 1) / P;
    const long long n_tiles = tiles_per_query * q.n_queries;
    const int last = net.n_layers - 1;

    for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int qi = (int)(tile / tiles_per_query);
        const long long p0 = (tile - (long long)qi * tiles_per_query) * P;
        if (q.live_rows && p0 >= q.live_rows[qi]) continue;          // uniform over the CTA

        float x[TM], y[TM], z[TM];
        bool quirk[TM];
#pragma unroll
        for (int i = 0; i < TM; ++i) {
            const long long idx = p0 + lane * TM + i;
            const bool valid = idx < q.n_points;
            const long long g = q.first + (valid ? idx : 0);
            if (q.xyz) {
                const float *p = q.xyz + ((size_t)qi * q.n_points + (valid ? idx : 0)) * 3;
                x[i] = p[0]; y[i] = p[1]; z[i] = p[2];
            } else {
                const long long rr = (long long)q.res * q.res;
                const int ix = (int)(g / rr), iy = (int)((g - ix * rr) / q.res), iz = (int)(g % q.res);
                x[i] = q.axes[ix]; y[i] = q.axes[q.res + iy]; z[i] = q.axes[2 * q.res + iz];
            }
            quirk[i] = q.quirk_period > 0 && ((g % q.quirk_period) == q.quirk_period - 1 || g == q.total - 1);
        }

        float num[TM], den[TM];
#pragma unroll
        for (int i = 0; i < TM; ++i) { num[i] = 0.f; den[i] = 0.f; }

        for (int m = 0; m < net.n_members; ++m) {
            const int set = m < 2 * net.n_symm ? (m >> 1) : m - net.n_symm;
            const float *cv = q.cvec + ((size_t)qi * net.n_members + m) * net.cvec_stride;
            float cx[TM], cy[TM], cz[TM];
            float ax = 0.f, ay = 0.f, az = 0.f;
            const bool has_anchor = q.anchors != nullptr && m < net.n_members - 1;
            if (has_anchor) {
                const float *a = q.anchors + ((size_t)qi * (net.n_members - 1) + m) * 3;
                ax = __ldg(a); ay = __ldg(a + 1); az = __ldg(a + 2);
            }
            const bool mirror = (m & 1) && m < 2 * net.n_symm;
#pragma unroll
            for (int i = 0; i < TM; ++i) {
                cx[i] = x[i] - ax; cy[i] = y[i] - ay; cz[i] = z[i] - az;
                if (mirror) cx[i] = -cx[i];
            }
            __syncthreads();                 // previous member / tile finished with the buffers
            if (warp == 0) {
                store_act<TM>(buf[0] + 0 * P + lane * TM, cx);
                store_act<TM>(buf[0] + 1 * P + lane * TM, cy);
                store_act<TM>(buf[0] + 2 * P + lane * TM, cz);
            }
            __syncthreads();
            for (int l = 0; l <= last; ++l) {
                const FoldedLayer &L = net.L[l];
                const float *in_s = buf[l & 1];
                float *out_s = buf[(l + 1) & 1];
                if (l + 1 == net.skip && warp == 0) {
                    // rows [N_l, N_l+3) of this layer's output buffer carry xyz for the skip layer
                    store_act<TM>(out_s + (size_t)(L.N + 0) * P + lane * TM, cx);
                    store_act<TM>(out_s + (size_t)(L.N + 1) * P + lane * TM, cy);
                    store_act<TM>(out_s + (size_t)(L.N + 2) * P + lane * TM, cz);
                }
                const float *Wt = L.Wt + (size_t)set * L.K * L.Npad;
                if (L.N <= 8) narrow_layer<TM>(L, Wt, cv + L.coff, in_s, out_s, warp, lane, nwarps);
                else          dense_layer<TM>(L, Wt, cv + L.coff, in_s, out_s, warp, lane, nwarps);
                __syncthreads();
            }
            const float *res = buf[(last + 1) & 1];
            if (q.blend) {
                if (warp == 0) {
                    float s[TM];
                    load_act<TM>(res + lane * TM, s);
#pragma unroll
                    for (int i = 0; i < TM; ++i) {
                        float d;
                        if (has_anchor) {
                            // d = -(|a - x| + 1e-5)^2   (EnsembledDeepSDF.py:136-137; 10e-6 == 1e-5)
                            const float dx = ax - x[i], dy = ay - y[i], dz = az - z[i];
                            const float nrm = sqrtf(dx * dx + dy * dy + dz * dz) + 10e-6f;
                            d = -(nrm * nrm);
                        } else {
                            d = -0.2f;                                   // background member (:140-142)
                        }
                        const float w = expf(__fdiv_rn(d, 0.01f));          // var = 0.1**2  (:144)
                        const float sv = quirk[i] ? 1.0f : s[i];          // eval-mode quirk (:260-261)
                        num[i] = fmaf(w, sv, num[i]);
                        den[i] += w;
                    }
                }
            } else {
                // plain MLP: write the out_dim channels
                for (int t = threadIdx.x; t < net.L[last].N * P; t += blockDim.x) {
                    const int n = t / P, p = t - n * P;
                    const long long idx = p0 + p;
                    if (idx < q.n_points)
                        q.out[((size_t)qi * q.n_points + idx) * net.L[last].N + n] = res[(size_t)n * P + p];
                }
            }
        }
        if (q.blend && warp == 0) {
#pragma unroll
            for (int i = 0; i < TM; ++i) {
                const long long idx = p0 + lane * TM + i;
                if (idx < q.n_points)
                    q.out[(size_t)qi * q.n_points + idx] = __fdiv_rn(num[i], den[i] + 1e-6f);   // (:147-149)
            }
        }
    }
}

int simt_smem_bytes(const FoldedNet &net, int tm) { return 2 * net.max_rows * 32 * tm * (int)sizeof(float); }

bool folded_net_fits(const FoldedNet &net) { return simt_smem_bytes(net, 1) <= 227 * 1024; }

int launch_folded_net(const FoldedNet &net, const SimtQuery &q, cudaStream_t stream)
{
    // largest point tile whose two activation buffers fit in shared memory
    int tm = 4;
    while (tm > 1 && simt_smem_bytes(net, tm) > 220 * 1024) tm >>= 1;
    const int smem = simt_smem_bytes(net, tm);
    if (smem > 227 * 1024) {
        set_error("network too wide for the SIMT kernel: %d activation rows", net.max_rows);
        return NPHM_ERR_UNSUPPORTED;
    }
    const int P = 32 * tm;
    const long long n_tiles = ceil_div(q.n_points, P) * q.n_queries;
    if (n_tiles == 0) return NPHM_OK;
    const int ctas_per_sm = smem > 110 * 1024 ? 1 : 2;
    const int grid = (int)(n_tiles < (long long)sm_count() * ctas_per_sm ? n_tiles : (long long)sm_count() * ctas_per_sm);
    auto kern = tm == 4 ? folded_net_kernel<4> : (tm == 2 ? folded_net_kernel<2> : folded_net_kernel<1>);
    NPHM_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    kern<<<grid, 256, smem, stream>>>(net, q);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

// ------------------------------------------------------------------------------------------------
// per-query preparation: constant vectors, anchors, grid axes, weight packing
// ------------------------------------------------------------------------------------------------
// cvec[q][m][coff_l + n] = b_l[set][n] + scale_l * sum_j W_l[set][n][K_l + j] * u[j]   (folded layers)
//                        = b_l[set][n]                                               (other layers)
// u = [z_glob | z_m] for the ensemble, the condition vector for a plain MLP.
__global__ void cvec_kernel(const PackSpec spec, const float *__restrict__ latents, float *__restrict__ cvec)
{
    extern __shared__ float u[];
    const int m = blockIdx.x, qi = blockIdx.y;
    const float *lat = latents + (size_t)qi * spec.lat_dim;
    const int C = spec.cond_dim;
    for (int j = threadIdx.x; j < C; j += blockDim.x) {
        if (spec.n_members > 1) u[j] = j < spec.lat_glob ? lat[j] : lat[spec.lat_glob + m * spec.lat_loc + (j - spec.lat_glob)];
        else u[j] = lat[j];
    }
    __syncthreads();
    const int set = member_set(m, spec.n_symm);
    float *out = cvec + ((size_t)qi * spec.n_members + m) * spec.cvec_stride;
    // one warp per output row (coalesced reads of the weight row, shuffle reduction); blockIdx.z strides over the rows
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
    for (int l = 0; l < spec.n_layers; ++l) {
        const PackLayer &pl = spec.L[l];
        if (!pl.folded) {                    // plain bias copy: thread per element
            for (int n = blockIdx.z * blockDim.x + threadIdx.x; n < pl.Npad; n += gridDim.z * blockDim.x)
                out[pl.coff + n] = n < pl.N ? pl.b[(size_t)set * pl.N + n] : 0.f;
            continue;
        }
        for (int n = blockIdx.z * wpb + warp; n < pl.Npad; n += gridDim.z * wpb) {
            float v = 0.f;
            if (n < pl.N) {
                if (pl.folded) {
                    const float *w = pl.W + ((size_t)set * pl.N + n) * pl.in_total + pl.K;
                    float s = 0.f;
                    for (int j = lane; j < C; j += 32) s = fmaf(w[j], u[j], s);
#pragma unroll
                    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
                    v = fmaf(s, pl.scale, pl.b[(size_t)set * pl.N + n]);
                } else {
                    v = pl.b[(size_t)set * pl.N + n];
                }
            }
            if (lane == 0) out[pl.coff + n] = v;
        }
    }
}

// anchors[q] = mlp_pos(z_glob) + mean anchors       (EnsembledDeepSDF.py:228-229)
__global__ void anchors_kernel(const float *__restrict__ latents, int lat_dim, int lat_glob, int hid, int n_out,
                               const float *__restrict__ w0, const float *__restrict__ b0,
                               const float *__restrict__ w1, const float *__restrict__ b1,
                               const float *__restrict__ w2, const float *__restrict__ b2,
                               const float *__restrict__ mean, float *__restrict__ anchors)
{
    extern __shared__ float sh[];
    float *zin = sh, *h0 = sh + lat_glob, *h1 = h0 + hid;
    const int qi = blockIdx.x;
    for (int j = threadIdx.x; j < lat_glob; j += blockDim.x) zin[j] = latents[(size_t)qi * lat_dim + j];
    __syncthreads();
    // one warp per output row: coalesced reads of the weight row + shuffle reduction
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    auto dot = [&](const float *__restrict__ w, const float *x, int n) {
        float s = 0.f;
        for (int j = lane; j < n; j += 32) s = fmaf(w[j], x[j], s);
#pragma unroll
        for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        return s;
    };
    for (int n = warp; n < hid; n += nw) {
        const float s = dot(w0 + (size_t)n * lat_glob, zin, lat_glob) + b0[n];
        if (lane == 0) h0[n] = fmaxf(s, 0.f);
    }
    __syncthreads();
    for (int n = warp; n < hid; n += nw) {
        const float s = dot(w1 + (size_t)n * hid, h0, hid) + b1[n];
        if (lane == 0) h1[n] = fmaxf(s, 0.f);
    }
    __syncthreads();
    for (int n = warp; n < n_out; n += nw) {
        const float s = dot(w2 + (size_t)n * hid, h1, hid) + b2[n];
        if (lane == 0) anchors[(size_t)qi * n_out + n] = s + mean[n];
    }
}

// axes[a][i] = float32(np.linspace(min_a, max_a, res)[i]) : y_i = i*step + start in float64 (no FMA), y_last = stop
__global__ void grid_axes_kernel(double min0, double min1, double min2, double max0, double max1, double max2,
                                 int res, float *__restrict__ axes)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= res) return;
    const double mn[3] = {min0, min1, min2}, mx[3] = {max0, max1, max2};
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const double step = __ddiv_rn(__dsub_rn(mx[a], mn[a]), (double)(res - 1));
        double v = __dadd_rn(__dmul_rn((double)i, step), mn[a]);
        if (i == res - 1) v = mx[a];
        axes[a * res + i] = (float)v;
    }
}

// Wt[set][k][n] = scale * W[set][n][k]  (k < K point-dependent columns), zero padded to Npad
__global__ void pack_wt_kernel(const float *__restrict__ W, int n_sets, int N, int in_total, int K, int Npad,
                               float scale, float *__restrict__ Wt)
{
    const size_t total = (size_t)n_sets * K * Npad;
    for (size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
        const int n = (int)(t % Npad);
        const int k = (int)((t / Npad) % K);
        const int s = (int)(t / ((size_t)Npad * K));
        Wt[t] = n < N ? scale * W[((size_t)s * N + n) * in_total + k] : 0.f;
    }
}

int launch_cvec(const PackSpec &spec, const float *latents, int n_queries, float *cvec, cudaStream_t stream)
{
    // few (member, query) pairs (a plain MLP has one member): spread the rows of a pair over several CTAs
    const int pairs = spec.n_members * n_queries;
    dim3 grid(spec.n_members, n_queries, pairs >= 128 ? 1 : (pairs >= 16 ? 4 : 16));
    cvec_kernel<<<grid, 256, spec.cond_dim * sizeof(float), stream>>>(spec, latents, cvec);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

int launch_anchors(const float *latents, int n_queries, int lat_dim, int lat_glob, int hid, int n_out,
                   const float *const *w, const float *const *b, const float *mean, float *anchors,
                   cudaStream_t stream)
{
    const size_t smem = (lat_glob + 2 * hid) * sizeof(float);
    anchors_kernel<<<n_queries, 1024, smem, stream>>>(latents, lat_dim, lat_glob, hid, n_out,
                                                     w[0], b[0], w[1], b[1], w[2], b[2], mean, anchors);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

int launch_grid_axes(const double mn[3], const double mx[3], int res, float *axes, cudaStream_t stream)
{
    grid_axes_kernel<<<(res + 127) / 128, 128, 0, stream>>>(mn[0], mn[1], mn[2], mx[0], mx[1], mx[2], res, axes);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

int launch_pack_wt(const float *W, int n_sets, int N, int in_total, int K, int Npad, float scale, float *Wt,
                   cudaStream_t stream)
{
    pack_wt_kernel<<<256, 256, 0, stream>>>(W, n_sets, N, in_total, K, Npad, scale, Wt);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

}  // namespace nphm
