// Weight gradient of a linear layer from packed operands (tc_wgrad.cu):  dW[n][k] = scale * sum_rows D[row][n] H[row][k]
#pragma once
#include "engine.cuh"

namespace nphm {
namespace wgrad {

// D: packed pre-activation adjoints (d_ksteps k-steps), H: packed layer inputs (h_ksteps k-steps), both over M rows per member
// in the operand format of tc_linear.cuh.  `sets` weight sets in one launch (gridDim.z); set z writes dW + z dw_stride,
// dW[n * ldw + k] for n < N, k < K:  scale * inv_scale_dev[z inv_stride] * (D^T H)[n][k], summed over the rows of its members
// (set_members, common.cuh: w_pairs mirrored pairs), member by member; member m's operands start at D + m sD, H + m sH,
// D2 + m sD2, H2 + m sH2 (bytes).  One set, w_pairs = 0: a single stack.
// The rows are split over the CTAs; the partial sums go to `partials` and are added in a fixed order (no atomics), so equal
// inputs give bitwise-equal gradients.  `partials`: scratch, grown on demand.
// D2, H2 (optional, both or neither; same k-steps and rows as D, H): a second pair, dW = scale * inv_scale (D^T H + D2^T H2),
// accumulated in the same fixed order (each member's row tiles of the first pair, then those of the second).
int launch_sets(const uint8_t *D, int d_ksteps, const uint8_t *H, int h_ksteps, long long M, int N, int K, float scale,
                const float *inv_scale_dev, int inv_stride, float *dW, int ldw, long long dw_stride, int sets, int w_pairs,
                long long sD, long long sH, long long sD2, long long sH2, DeviceBuffer &partials, cudaStream_t stream,
                const uint8_t *D2 = nullptr, const uint8_t *H2 = nullptr);

}  // namespace wgrad
}  // namespace nphm
