// Per-observation similarity transforms of the fitters (DESIGN.md §4.24): observation o maps scan-frame points p to the model
// frame by q = exp(sigma_o) R_o p + t_o.  The state is one float64 table of all observations of a batch, row o =
// [R_o row-major (9) | t_o (3) | sigma_o], and every sampled row of points carries the int32 index of its observation.
//   apply  q of every point, in float64 from the table and rounded once to fp32;
//   grad   (g_omega, g_t, g_sigma) of every observation from the points and d loss / d q, summed in float64 in a fixed order
//          (within a row, then over the observation's rows in row order) - no atomics, so the result is bitwise repeatable;
//   adam   Adam on (omega, t, sigma) and the retraction R <- Exp(delta_omega) R, re-orthonormalised, for every observation.
// A row whose observation index lies outside [0, n_obs) is padding: apply passes its points through, grad leaves it out.
// The float64 products and sums are written with explicit _rn intrinsics so that no multiply-add contraction changes them: a
// float64 restatement in the same order gives the same bits, and the identity transform maps every point to itself.
#include <cmath>
#include "common.cuh"
#include "pose_math.cuh"

namespace nphm {
namespace pose {

constexpr int kThreads = 256;
constexpr int kStride = 13;     // R (9), t (3), sigma

__global__ void __launch_bounds__(kThreads) apply_kernel(const float *__restrict__ pts, const int *__restrict__ row_obs,
                                                         long long n_rows, long long n_point, const double *__restrict__ table,
                                                         int n_obs, float *__restrict__ out)
{
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n_rows * n_point) return;
    const int o = row_obs[i / n_point];
    const float x = pts[i * 3], y = pts[i * 3 + 1], z = pts[i * 3 + 2];
    if (o < 0 || o >= n_obs) {
        out[i * 3] = x; out[i * 3 + 1] = y; out[i * 3 + 2] = z;
        return;
    }
    const double *T = table + (long long)o * kStride;
    const double s = exp(T[12]);
    const double p[3] = {x, y, z};
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        double a = mul(T[3 * r], p[0]);
        a = add(a, mul(T[3 * r + 1], p[1]));
        a = add(a, mul(T[3 * r + 2], p[2]));
        out[i * 3 + r] = (float)add(mul(s, a), T[9 + r]);
    }
}

// One block per observation.  For every row of the observation, in row order: each thread sums its points (stride kThreads)
// in point order, the block reduces the thread sums in a fixed tree, and thread 0 adds the row's sum to the running total.
__global__ void __launch_bounds__(kThreads) grad_kernel(const float *__restrict__ q, const float *__restrict__ g,
                                                        const int *__restrict__ row_obs, long long n_rows, long long n_point,
                                                        const double *__restrict__ table, double lam, double *__restrict__ out)
{
    __shared__ double red[7][kThreads];
    const int o = blockIdx.x;
    const double *T = table + (long long)o * kStride;
    const double t0 = T[9], t1 = T[10], t2 = T[11];
    double total[7] = {0, 0, 0, 0, 0, 0, 0};
    for (long long r = 0; r < n_rows; ++r) {
        if (row_obs[r] != o) continue;                         // uniform over the block
        double acc[7] = {0, 0, 0, 0, 0, 0, 0};
        for (long long j = threadIdx.x; j < n_point; j += kThreads) {
            const long long k = (r * n_point + j) * 3;
            const double a0 = sub((double)q[k], t0), a1 = sub((double)q[k + 1], t1), a2 = sub((double)q[k + 2], t2);
            const double g0 = g[k], g1 = g[k + 1], g2 = g[k + 2];
            acc[0] = add(acc[0], sub(mul(a1, g2), mul(a2, g1)));    // (q - t) x g
            acc[1] = add(acc[1], sub(mul(a2, g0), mul(a0, g2)));
            acc[2] = add(acc[2], sub(mul(a0, g1), mul(a1, g0)));
            acc[3] = add(acc[3], g0);
            acc[4] = add(acc[4], g1);
            acc[5] = add(acc[5], g2);
            acc[6] = add(acc[6], add(add(mul(g0, a0), mul(g1, a1)), mul(g2, a2)));
        }
#pragma unroll
        for (int c = 0; c < 7; ++c) red[c][threadIdx.x] = acc[c];
        __syncthreads();
        for (int h = kThreads / 2; h > 0; h >>= 1) {
            if (threadIdx.x < h) {
#pragma unroll
                for (int c = 0; c < 7; ++c) red[c][threadIdx.x] = add(red[c][threadIdx.x], red[c][threadIdx.x + h]);
            }
            __syncthreads();
        }
        if (threadIdx.x == 0) {
#pragma unroll
            for (int c = 0; c < 7; ++c) total[c] = add(total[c], red[c][0]);
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
#pragma unroll
        for (int c = 0; c < 7; ++c) out[(long long)o * 7 + c] = mul(lam, total[c]);
    }
}

__global__ void adam_kernel(double *__restrict__ table, double *__restrict__ m, double *__restrict__ v,
                            const double *__restrict__ grad, int n_obs, double lr_rot, double lr_trans, double lr_scale,
                            int fit_scale, double bc1, double bc2_sqrt)
{
    const int o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= n_obs) return;
    double d[7];
#pragma unroll
    for (int c = 0; c < 7; ++c) {
        const long long k = (long long)o * 7 + c;
        const double gg = grad[k];
        const double mm = add(mul(0.9, m[k]), mul(0.1, gg));
        const double vv = add(mul(0.999, v[k]), mul(0.001, mul(gg, gg)));
        m[k] = mm; v[k] = vv;
        const double lr = c < 3 ? lr_rot : (c < 6 ? lr_trans : lr_scale);
        d[c] = -(mul(lr / bc1, mm / add(sqrt(vv) / bc2_sqrt, 1e-8)));
    }
    double *T = table + (long long)o * kStride;
    double E[9], R[9];
    rodrigues(d, E);
#pragma unroll
    for (int k = 0; k < 9; ++k) R[k] = T[k];
    rotate_left_orthonormal(E, R);
#pragma unroll
    for (int k = 0; k < 9; ++k) T[k] = R[k];
    T[9] = add(T[9], d[3]); T[10] = add(T[10], d[4]); T[11] = add(T[11], d[5]);
    if (fit_scale) T[12] = add(T[12], d[6]);
}

}  // namespace pose
}  // namespace nphm

using namespace nphm;

extern "C" int nphm_pose_apply(const float *points_dev, const int *row_obs_dev, long long n_rows, long long n_point,
                               const double *table_dev, int n_obs, float *out_dev, void *stream_)
{
    NPHM_REQUIRE(n_rows >= 0 && n_point >= 0 && n_obs >= 1 && table_dev && n_rows * n_point < (1LL << 40) &&
                 (n_rows * n_point == 0 || (points_dev && row_obs_dev && out_dev)), "nphm_pose_apply: bad arguments");
    const long long n = n_rows * n_point;
    if (n == 0) return NPHM_OK;
    pose::apply_kernel<<<(unsigned)ceil_div(n, pose::kThreads), pose::kThreads, 0, static_cast<cudaStream_t>(stream_)>>>(
        points_dev, row_obs_dev, n_rows, n_point, table_dev, n_obs, out_dev);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

extern "C" int nphm_pose_grad(const float *q_dev, const float *grad_q_dev, const int *row_obs_dev, long long n_rows,
                              long long n_point, const double *table_dev, int n_obs, double lam_surface, double *grad_dev,
                              void *stream_)
{
    NPHM_REQUIRE(n_rows >= 0 && n_point >= 0 && n_obs >= 1 && table_dev && grad_dev && std::isfinite(lam_surface) &&
                 (n_rows * n_point == 0 || (q_dev && grad_q_dev && row_obs_dev)), "nphm_pose_grad: bad arguments");
    pose::grad_kernel<<<(unsigned)n_obs, pose::kThreads, 0, static_cast<cudaStream_t>(stream_)>>>(
        q_dev, grad_q_dev, row_obs_dev, n_rows * n_point == 0 ? 0 : n_rows, n_point, table_dev, lam_surface, grad_dev);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

extern "C" int nphm_pose_adam(double *table_dev, double *adam_m_dev, double *adam_v_dev, const double *grad_dev, int n_obs,
                              double lr_rot, double lr_trans, double lr_scale, int fit_scale, int step, void *stream_)
{
    NPHM_REQUIRE(table_dev && adam_m_dev && adam_v_dev && grad_dev && n_obs >= 1 && step >= 1 && lr_rot >= 0 && lr_trans >= 0 &&
                 lr_scale >= 0 && std::isfinite(lr_rot) && std::isfinite(lr_trans) && std::isfinite(lr_scale),
                 "nphm_pose_adam: bad arguments");
    const double bc1 = 1.0 - std::pow(0.9, step), bc2 = 1.0 - std::pow(0.999, step);
    pose::adam_kernel<<<(unsigned)ceil_div(n_obs, 128), 128, 0, static_cast<cudaStream_t>(stream_)>>>(
        table_dev, adam_m_dev, adam_v_dev, grad_dev, n_obs, lr_rot, lr_trans, lr_scale, fit_scale, bc1, std::sqrt(bc2));
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}
