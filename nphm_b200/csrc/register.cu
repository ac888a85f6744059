// Global registration of observations against a head's SDF grid (DESIGN.md §4.25): a robust Gauss-Newton search over many
// similarity hypotheses per observation, all iterations of a stage in one launch.
//   prepare  the res^3 volume (get_logits' layout: x slowest, z fastest, end points included) to a float4 grid
//            (sdf, d/dx, d/dy, d/dz): central differences in world units, one-sided at the faces, with _rn intrinsics so that
//            models/registration.py:prepare_torch gives the same bits;
//   search   one warp per hypothesis (a row of the n_hyp x 13 float64 table, ObservationPoses' layout).  Per iteration the warp
//            moves its observation's points by q = exp(sigma) R p + t, samples the grid trilinearly (value and gradient), and
//            accumulates the truncated normal equations in float64, lane by lane in point order, then in a fixed butterfly.
//            Every lane then solves the same damped system (the same bits, so nothing is broadcast) and takes the step.  A last
//            pass scores the final pose.  A hypothesis' result depends on its row, its observation's points and the parameters
//            only, never on the other hypotheses of the launch, and the launch is bitwise repeatable.
// The residual is r = sdf(q) u_o / s: the distance in the scan's units, expressed in model units through the observation's fixed
// reference scale u_o.  Its Jacobian for the left perturbation R <- Exp(omega) R, t += dt, sigma += dsigma (the order of
// nphm_pose_grad) is (u_o / s) [a x n, n, n . a - sdf] with a = q - t and n the sampled gradient; the common factor
// (u_o / s)^2 of A = J^T W J and b = J^T W r cancels in the step and is left out.
#include <cmath>
#include "common.cuh"
#include "pose_math.cuh"

namespace nphm {
namespace reg {

using pose::add;
using pose::mul;
using pose::sub;

constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;
constexpr int kStride = 13;                       // R (9), t (3), sigma
constexpr int kMaxSmemBytes = 160 * 1024;         // larger point sets are read from global memory (L2) instead
constexpr double kSigmaBand = 0.086643397569993164;   // log 2 / 8: sigma stays within this of its seed

__global__ void __launch_bounds__(256) prepare_kernel(const float *__restrict__ vol, int res, float hx, float hy, float hz,
                                                      float4 *__restrict__ out)
{
    const long long n = (long long)res * res * res;
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const long long R = res;
    const int idx[3] = {(int)(i / (R * R)), (int)((i / R) % R), (int)(i % R)};
    const long long stride[3] = {R * R, R, 1};
    const float h[3] = {hx, hy, hz};
    float g[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        if (idx[a] == 0)
            g[a] = __fdiv_rn(__fsub_rn(vol[i + stride[a]], vol[i]), h[a]);
        else if (idx[a] == res - 1)
            g[a] = __fdiv_rn(__fsub_rn(vol[i], vol[i - stride[a]]), h[a]);
        else
            g[a] = __fdiv_rn(__fsub_rn(vol[i + stride[a]], vol[i - stride[a]]), __fmul_rn(2.0f, h[a]));
    }
    out[i] = make_float4(vol[i], g[0], g[1], g[2]);
}

__device__ __forceinline__ float4 lerp(const float4 &a, const float4 &b, float t)
{
    return make_float4(a.x + t * (b.x - a.x), a.y + t * (b.y - a.y), a.z + t * (b.z - a.z), a.w + t * (b.w - a.w));
}

// Trilinear value and gradient at q; false outside the grid's box (or for a non-finite q).
__device__ __forceinline__ bool sample(const float4 *__restrict__ field, const nphm_register_params &p, const float q[3],
                                       float4 &out)
{
    int i[3];
    float f[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float u = (q[a] - p.mini[a]) / p.h[a];
        if (!(u >= 0.0f && u <= (float)(p.res - 1))) return false;
        i[a] = min((int)u, p.res - 2);
        f[a] = u - (float)i[a];
    }
    const long long R = p.res;
    const float4 *c = field + ((long long)i[0] * R + i[1]) * R + i[2];
    const float4 v[8] = {__ldg(c), __ldg(c + 1), __ldg(c + R), __ldg(c + R + 1),
                         __ldg(c + R * R), __ldg(c + R * R + 1), __ldg(c + R * R + R), __ldg(c + R * R + R + 1)};
    const float4 z00 = lerp(v[0], v[1], f[2]), z01 = lerp(v[2], v[3], f[2]);
    const float4 z10 = lerp(v[4], v[5], f[2]), z11 = lerp(v[6], v[7], f[2]);
    out = lerp(lerp(z00, z01, f[1]), lerp(z10, z11, f[1]), f[0]);
    return true;
}

__device__ __forceinline__ double warp_sum(double x)
{
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) x = add(x, __shfl_xor_sync(0xffffffffu, x, m));
    return x;
}

// D = 7 (similarity) or 6 (rigid: sigma held).
template <int D>
__global__ void __launch_bounds__(kThreads) search_kernel(nphm_register_params p, const float4 *__restrict__ field,
                                                         const float *__restrict__ points, const long long *__restrict__ offsets,
                                                         const int *__restrict__ counts, const double *__restrict__ unit,
                                                         double *__restrict__ table, const double *__restrict__ sigma_seed,
                                                         const int *__restrict__ hyp_obs, int use_smem, double *__restrict__ score,
                                                         int *__restrict__ inliers)
{
    constexpr int kA = D * (D + 1) / 2;
    constexpr int kAcc = kA + D + 1;                        // A (packed lower), b, inlier count
    extern __shared__ float smem_pts[];
    const int first = blockIdx.x * kWarps;
    const int o_cta = hyp_obs[first];
    const bool cta_ok = use_smem && o_cta >= 0 && o_cta < p.n_obs;
    if (cta_ok) {
        const int m = min(counts[o_cta], p.n_use);
        const float *src = points + offsets[o_cta] * 3;
        for (int k = threadIdx.x; k < 3 * m; k += kThreads) smem_pts[k] = src[k];
    }
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int hyp = first + (threadIdx.x >> 5);
    if (hyp >= p.n_hyp) return;
    const int o = hyp_obs[hyp];
    if (o < 0 || o >= p.n_obs) return;
    const int m = min(counts[o], p.n_use);
    const float *P = (cta_ok && o == o_cta) ? smem_pts : points + offsets[o] * 3;
    double T[kStride];
#pragma unroll
    for (int k = 0; k < kStride; ++k) T[k] = table[(long long)hyp * kStride + k];
    const double sig0 = sigma_seed[hyp], u_o = unit[o];
    const double tau1_sq = p.tau1 * p.tau1;

    for (int it = 0; it <= p.n_iter; ++it) {
        const bool last = it == p.n_iter;
        double tau = p.tau1;
        if (!last && p.tau0 != p.tau1)
            tau = p.n_iter > 1 ? p.tau0 * pow(p.tau1 / p.tau0, (double)it / (double)(p.n_iter - 1)) : p.tau0;
        const double s = exp(T[12]);
        const double ws = u_o / s;
        float M[9], tt[3];
#pragma unroll
        for (int k = 0; k < 9; ++k) M[k] = (float)(s * T[k]);
#pragma unroll
        for (int k = 0; k < 3; ++k) tt[k] = (float)T[9 + k];

        double acc[kAcc];
#pragma unroll
        for (int k = 0; k < kAcc; ++k) acc[k] = 0.0;
        double sc = 0.0;
        int inl = 0;
        for (int j = lane; j < m; j += 32) {
            const float px = P[3 * j], py = P[3 * j + 1], pz = P[3 * j + 2];
            float a[3], q[3];
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                a[r] = M[3 * r] * px + M[3 * r + 1] * py + M[3 * r + 2] * pz;
                q[r] = a[r] + tt[r];
            }
            float4 g;
            if (!sample(field, p, q, g)) {
                sc += tau1_sq;
                continue;
            }
            const double f = g.x, r = f * ws;
            if (last) {
                sc += fmin(r * r, tau1_sq);
                inl += fabs(r) < p.tau1;
                continue;
            }
            if (!(fabs(r) < tau)) continue;
            const double a0 = a[0], a1 = a[1], a2 = a[2], n0 = g.y, n1 = g.z, n2 = g.w;
            double J[7];
            J[0] = sub(mul(a1, n2), mul(a2, n1));
            J[1] = sub(mul(a2, n0), mul(a0, n2));
            J[2] = sub(mul(a0, n1), mul(a1, n0));
            J[3] = n0; J[4] = n1; J[5] = n2;
            J[6] = sub(add(add(mul(n0, a0), mul(n1, a1)), mul(n2, a2)), f);
            int k = 0;
#pragma unroll
            for (int u = 0; u < D; ++u)
#pragma unroll
                for (int v = 0; v <= u; ++v, ++k) acc[k] = add(acc[k], mul(J[u], J[v]));
#pragma unroll
            for (int u = 0; u < D; ++u) acc[kA + u] = add(acc[kA + u], mul(J[u], f));
            acc[kA + D] = add(acc[kA + D], 1.0);
        }
        if (last) {
            sc = warp_sum(sc);
            double ni = warp_sum((double)inl);
            if (lane == 0) {
                score[hyp] = m > 0 ? sc / m : tau1_sq;
                inliers[hyp] = (int)ni;
            }
            break;
        }
#pragma unroll
        for (int k = 0; k < kAcc; ++k) acc[k] = warp_sum(acc[k]);
        if (acc[kA + D] < D) continue;                      // too few inliers to pin the pose: no step

        // Cholesky of A + damping diag(A) (packed lower, in place), then delta = -(A + damping diag(A))^-1 b
        bool ok = true;
#pragma unroll
        for (int u = 0; u < D; ++u) acc[u * (u + 1) / 2 + u] = mul(acc[u * (u + 1) / 2 + u], 1.0 + p.damping);
#pragma unroll
        for (int u = 0; u < D; ++u) {
#pragma unroll
            for (int v = 0; v <= u; ++v) {
                double x = acc[u * (u + 1) / 2 + v];
#pragma unroll
                for (int k = 0; k < v; ++k) x = sub(x, mul(acc[u * (u + 1) / 2 + k], acc[v * (v + 1) / 2 + k]));
                if (u == v) {
                    ok = ok && x > 0.0;
                    acc[u * (u + 1) / 2 + u] = sqrt(fmax(x, 1e-300));
                } else {
                    acc[u * (u + 1) / 2 + v] = x / acc[v * (v + 1) / 2 + v];
                }
            }
        }
        double y[D];
#pragma unroll
        for (int u = 0; u < D; ++u) {
            double x = acc[kA + u];
#pragma unroll
            for (int k = 0; k < u; ++k) x = sub(x, mul(acc[u * (u + 1) / 2 + k], y[k]));
            y[u] = x / acc[u * (u + 1) / 2 + u];
        }
#pragma unroll
        for (int u = D - 1; u >= 0; --u) {
            double x = y[u];
#pragma unroll
            for (int k = u + 1; k < D; ++k) x = sub(x, mul(acc[k * (k + 1) / 2 + u], y[k]));
            y[u] = x / acc[u * (u + 1) / 2 + u];
        }
        double d[7] = {0, 0, 0, 0, 0, 0, 0};
#pragma unroll
        for (int u = 0; u < D; ++u) {
            d[u] = -y[u];
            ok = ok && isfinite(d[u]);
        }
        if (!ok) continue;
        double E[9];
        pose::rodrigues(d, E);
        pose::rotate_left_orthonormal(E, T);
        T[9] = add(T[9], d[3]); T[10] = add(T[10], d[4]); T[11] = add(T[11], d[5]);
        if (D == 7) T[12] = fmin(fmax(add(T[12], d[6]), sub(sig0, kSigmaBand)), add(sig0, kSigmaBand));
    }
    if (lane == 0) {
#pragma unroll
        for (int k = 0; k < kStride; ++k) table[(long long)hyp * kStride + k] = T[k];
    }
}

}  // namespace reg
}  // namespace nphm

using namespace nphm;

extern "C" int nphm_register_prepare(const float *volume_dev, int res, float hx, float hy, float hz, void *field_dev, void *stream_)
{
    NPHM_REQUIRE(volume_dev && field_dev && res >= 2 && res <= 1024 && hx > 0 && hy > 0 && hz > 0 && std::isfinite(hx) &&
                 std::isfinite(hy) && std::isfinite(hz), "nphm_register_prepare: bad arguments");
    const long long n = (long long)res * res * res;
    reg::prepare_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, static_cast<cudaStream_t>(stream_)>>>(
        volume_dev, res, hx, hy, hz, static_cast<float4 *>(field_dev));
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

extern "C" int nphm_register_search(const nphm_register_params *p, const void *field_dev, const float *points_dev,
                                    const long long *offsets_dev, const int *counts_dev, const double *unit_dev,
                                    double *table_dev, const double *sigma_seed_dev, const int *hyp_obs_dev, int max_points,
                                    double *score_dev, int *inliers_dev, void *stream_)
{
    NPHM_REQUIRE(p && field_dev && points_dev && offsets_dev && counts_dev && unit_dev && table_dev && sigma_seed_dev &&
                 hyp_obs_dev && score_dev && inliers_dev, "nphm_register_search: null pointer");
    NPHM_REQUIRE(p->res >= 2 && p->n_obs >= 1 && p->n_use >= 1 && p->n_hyp >= 1 && p->n_iter >= 0 && max_points >= 0 &&
                 max_points <= p->n_use && (p->fit_scale == 0 || p->fit_scale == 1) && p->tau0 > 0 && p->tau1 > 0 &&
                 p->damping >= 0 && std::isfinite(p->damping) && p->h[0] > 0 && p->h[1] > 0 && p->h[2] > 0,
                 "nphm_register_search: bad parameters");
    const long long smem = 3LL * 4 * max_points;
    const int use_smem = smem <= reg::kMaxSmemBytes;
    const size_t bytes = use_smem ? (size_t)smem : 0;
    const unsigned grid = (unsigned)ceil_div(p->n_hyp, reg::kWarps);
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    const float4 *field = static_cast<const float4 *>(field_dev);
    if (p->fit_scale) {
        NPHM_CUDA_CHECK(cudaFuncSetAttribute(reg::search_kernel<7>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
        reg::search_kernel<7><<<grid, reg::kThreads, bytes, stream>>>(*p, field, points_dev, offsets_dev, counts_dev, unit_dev,
                                                                       table_dev, sigma_seed_dev, hyp_obs_dev, use_smem,
                                                                       score_dev, inliers_dev);
    } else {
        NPHM_CUDA_CHECK(cudaFuncSetAttribute(reg::search_kernel<6>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
        reg::search_kernel<6><<<grid, reg::kThreads, bytes, stream>>>(*p, field, points_dev, offsets_dev, counts_dev, unit_dev,
                                                                       table_dev, sigma_seed_dev, hyp_obs_dev, use_smem,
                                                                       score_dev, inliers_dev);
    }
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}
