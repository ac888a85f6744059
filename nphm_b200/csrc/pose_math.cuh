// float64 rotation arithmetic shared by the pose fit (pose.cu) and the registration search (register.cu).  Products and sums
// are explicit _rn intrinsics, so no multiply-add contraction changes them and a float64 restatement in the same order
// (models/pose.py: rodrigues_f64, orthonormalise_f64) gives the same bits.
#pragma once

namespace nphm {
namespace pose {

__device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }

// Exp(w): I + A K + B K^2 (Rodrigues), K the cross-product matrix of w; the series near 0 so that Exp(0) is exactly I.
__device__ __forceinline__ void rodrigues(const double w[3], double E[9])
{
    const double th2 = add(add(mul(w[0], w[0]), mul(w[1], w[1])), mul(w[2], w[2]));
    double A, B;
    if (th2 < 1e-16) {
        A = sub(1.0, th2 / 6.0);
        B = sub(0.5, th2 / 24.0);
    } else {
        const double th = sqrt(th2);
        A = sin(th) / th;
        B = sub(1.0, cos(th)) / th2;
    }
    const double K[9] = {0.0, -w[2], w[1], w[2], 0.0, -w[0], -w[1], w[0], 0.0};
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const double k2 = add(add(mul(K[3 * r], K[c]), mul(K[3 * r + 1], K[3 + c])), mul(K[3 * r + 2], K[6 + c]));
            E[3 * r + c] = add(add(r == c ? 1.0 : 0.0, mul(A, K[3 * r + c])), mul(B, k2));
        }
}

// R <- Gram-Schmidt(E R): the left-multiplied rotation, its rows re-orthonormalised with the third row the cross product of
// the first two (det +1).  R is row-major.
__device__ __forceinline__ void rotate_left_orthonormal(const double E[9], double R[9])
{
    double P[9];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c)
            P[3 * r + c] = add(add(mul(E[3 * r], R[c]), mul(E[3 * r + 1], R[3 + c])), mul(E[3 * r + 2], R[6 + c]));
    const double n0 = sqrt(add(add(mul(P[0], P[0]), mul(P[1], P[1])), mul(P[2], P[2])));
    P[0] /= n0; P[1] /= n0; P[2] /= n0;
    const double dp = add(add(mul(P[0], P[3]), mul(P[1], P[4])), mul(P[2], P[5]));
    P[3] = sub(P[3], mul(dp, P[0])); P[4] = sub(P[4], mul(dp, P[1])); P[5] = sub(P[5], mul(dp, P[2]));
    const double n1 = sqrt(add(add(mul(P[3], P[3]), mul(P[4], P[4])), mul(P[5], P[5])));
    P[3] /= n1; P[4] /= n1; P[5] /= n1;
    P[6] = sub(mul(P[1], P[5]), mul(P[2], P[4]));
    P[7] = sub(mul(P[2], P[3]), mul(P[0], P[5]));
    P[8] = sub(mul(P[0], P[4]), mul(P[1], P[3]));
#pragma unroll
    for (int k = 0; k < 9; ++k) R[k] = P[k];
}

}  // namespace pose
}  // namespace nphm
