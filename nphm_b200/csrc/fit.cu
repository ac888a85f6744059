// Fused identity-space fitting step (no autograd graph): one iteration of
//   inference_identity_space   reference src/NPHM/models/fitting.py:197-279
// = ensemble forward on the sampled observation points, mean clamped |sdf| + latent regularisers, analytic gradient
//   with respect to the latent code, torch.optim.Adam update (fitting.py:193, torch/optim/adam.py single-tensor path).
//
// Gradient routes (SURVEY.md 8a''):  (i) member inputs u_k = [z_glob | z_k];  (ii) anchors a = mlp_pos(z_glob) + mean,
// which enter the local coordinates c_k = x - a_k and the blend weights w_k;  (iii) the regularisers.
// Because u_k is constant over the points of a call, the input gradients of the two layers that see it reduce to
//     g_u = W0u^T (sum_p delta0_p) + W2u^T (sum_p delta2_p) / sqrt(2),      g_c likewise with the xyz columns,
// so the per-point backward only has to produce the per-member sums of the layer deltas.
//
// Kernels (fp32 FFMA; the step is latency bound: 5 x 1000 points):
//   fit_member_kernel<fwd>  one CTA per (64-point tile, member): forward, s_k -> global
//   fit_blend_kernel        per point: blend, |sdf| clamp, kept count / sum
//   fit_member_kernel<bwd>  (configurations without the tensor-core path) forward again with all activations resident in
//                           shared memory (199 KB), backward in place, per-member delta sums and blend-path anchor
//                           gradients -> atomics
//   tensor-core path        forward = tc::wg::ensemble_wgmma_kernel<.., ACTS> (member outputs + activation derivatives to global
//                           memory), backward = three batched wgmma GEMMs (tc_linear.cu) between fit_upstream_kernel and
//                           fit_reduce_kernel
//   fit_member_grad_kernel  per member: delta sums -> g_u, g_c -> latent / anchor gradients
//   fit_finalize_kernel     mlp_pos forward/backward, regularisers, loss terms, Adam
#include "engine.cuh"
#include "simt_layers.cuh"
#include "tc_ensemble.cuh"
#include "tc_linear.cuh"
#include <cmath>

namespace nphm {
namespace fit {

struct BackwardPacks { tcl::PackedLinear l3, l2, l1; };

constexpr int TM = 2;
constexpr int P = 32 * TM;
constexpr int kThreads = 512;

struct Dims {
    int n_members, n_symm, n_loc;
    int H, N1, C, G, Lc;            // hidden, layer-1 width, cond width, lat_glob, lat_loc
    int lat_dim, pos_hid;
    int cvec_stride, coff[5];
    // shared-memory rows
    int r_c, r_h0, r_h1, r_h2, r_h3, r_s, rows;
};

struct Weights {
    const float *W[5];              // reference layout [set][out][in]
    const float *Wt[5];             // forward layout [set][K][Npad]
    int Npad[5], K[5];
    const float *pos_w[3], *pos_b[3], *mean_anchors;
};

// Scan-batched calls (nphm_fit_*_batched) fit S independent scans of n points each in one launch sequence.  Point rows are
// [scan][n] (points, mask, member_s, out, S, gsign, grad_points); the tensor-core buffers (acts, the upstream gradients, the
// packed deltas) are [member][scan][tile][128]: every scan owns whole 128-row tiles.  The per-point kernels run on grids whose
// y index (or tile) is the scan, so no CTA straddles two scans.  Per-scan accumulators: acc [scan][member][2H], blend_acc and
// ganch [scan][n_loc * 3], stats [scan][8], grad [scan][lat_dim]; anchors / cvec come per scan from ensemble_prepare.
struct Buffers {
    const float *points;            // S x n x 3
    long long n;                    // points per scan
    long long tiles_per_scan;       // ceil(n / 128)
    const float *anchors;           // S x n_loc x 3
    const float *cvec;              // [members][cvec_stride]
    float *member_s;                // n x members
    const unsigned char *mask;      // optional n: 0 = the point is excluded from the loss (joint fitter: failed correspondences)
    float *grad_points;             // optional n x 3: d loss / d point (accumulated over members with atomics)
    float *acts;                    // optional: activation derivatives saved by the tensor-core forward, [member][tile][tc::kActLd][128];
                                    // the backward GEMMs overwrite them with the layer deltas
    float *out, *S, *gsign;         // n each
    float *acc;                     // members x 2H   (sum delta0 | sum delta2)
    float *blend_acc;               // n_loc x 3 (NULL: no latent gradient is wanted, the anchor part of the blend path is skipped)
    float *stats;                   // [count, sum |sdf| kept, -, -]
    float *sum_part;                // optional [scan][warp]: fit_blend_kernel's per-warp sums of |sdf| kept, which
                                    // fit_finalize_kernel adds in warp order (stats[1] then stays 0): a reproducible loss
    float *points_part;             // optional: the per-member point gradients of fit_reduce_kernel<true>, [member][tile][3][128]
                                    // (over the activation blocks, dead by then), added in member order by fit_points_kernel
    float *ganch;                   // n_loc x 3
    float *grad;                    // lat_dim
    const float *upstream;          // optional n: d L / d sdf_p given by the caller (nphm_ensemble_backward_inputs) instead of the
                                    // clamped-|sdf| loss of the fitters
    float *sdf_out;                 // optional n: copy of the blended forward output
    // eval-mode quirk of FastEnsembleDeepSDFMirrored (EnsembledDeepSDF.py:260-261: every member's output at the last point of
    // each decoder call is overwritten with 1): row i of a scan with period p > 0 is a quirk row when i % p == p - 1.  The
    // period is quirk_periods[scan] when that (device, one per scan) array is given, else quirk_period; 0 = training mode.
    long long quirk_period;
    const int *quirk_periods;
};

// whether row i_scan of scan `scan` carries the eval-mode quirk (s_k := 1, grad s_k := 0 for every member k)
__device__ __forceinline__ bool quirk_row(const Buffers &b, int scan, long long i_scan)
{
    const long long p = b.quirk_periods ? (long long)b.quirk_periods[scan] : b.quirk_period;
    return p > 0 && i_scan % p == p - 1;
}

template <bool BWD>
__global__ void __launch_bounds__(kThreads, 1) fit_member_kernel(const Dims d, const Weights w, const Buffers b,
                                                                 float lambda_surface)
{
    extern __shared__ __align__(16) float sm[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = kThreads / 32;
    const int m = blockIdx.y;
    const long long p0 = (long long)blockIdx.x * P;
    const int set = m < 2 * d.n_symm ? (m >> 1) : m - d.n_symm;
    const bool has_anchor = m < d.n_loc;
    const bool mirror = (m & 1) && m < 2 * d.n_symm;
    float ax = 0.f, ay = 0.f, az = 0.f;
    if (has_anchor) { ax = b.anchors[m * 3]; ay = b.anchors[m * 3 + 1]; az = b.anchors[m * 3 + 2]; }

    float x[TM], y[TM], z[TM];
    bool valid[TM];
#pragma unroll
    for (int i = 0; i < TM; ++i) {
        const long long idx = p0 + lane * TM + i;
        valid[i] = idx < b.n;
        const float *pp = b.points + (valid[i] ? idx : 0) * 3;
        x[i] = pp[0]; y[i] = pp[1]; z[i] = pp[2];
    }
    float *rc = sm + (size_t)d.r_c * P, *rh0 = sm + (size_t)d.r_h0 * P, *rh1 = sm + (size_t)d.r_h1 * P;
    float *rh2 = sm + (size_t)d.r_h2 * P, *rh3 = sm + (size_t)d.r_h3 * P, *rs = sm + (size_t)d.r_s * P;
    if (warp == 0) {
        float cx[TM], cy[TM], cz[TM];
#pragma unroll
        for (int i = 0; i < TM; ++i) {
            cx[i] = x[i] - ax; cy[i] = y[i] - ay; cz[i] = z[i] - az;
            if (mirror) cx[i] = -cx[i];
        }
        store_act<TM>(rc + 0 * P + lane * TM, cx); store_act<TM>(rc + 1 * P + lane * TM, cy); store_act<TM>(rc + 2 * P + lane * TM, cz);
        float *skip = rh1 + (size_t)d.N1 * P;       // rows N1..N1+2 of the skip layer input
        store_act<TM>(skip + 0 * P + lane * TM, cx); store_act<TM>(skip + 1 * P + lane * TM, cy); store_act<TM>(skip + 2 * P + lane * TM, cz);
    }
    __syncthreads();
    const float *cv = b.cvec + (size_t)m * d.cvec_stride;
    FoldedLayer L[5];
    const int Ns[5] = {d.H, d.N1, d.H, d.H, 1};
#pragma unroll
    for (int l = 0; l < 5; ++l)
        L[l] = FoldedLayer{w.Wt[l] + (size_t)set * w.K[l] * w.Npad[l], w.K[l], Ns[l], w.Npad[l], d.coff[l], l < 4 ? 1 : 0};
    dense_layer<TM>(L[0], L[0].Wt, cv + L[0].coff, rc, rh0, warp, lane, nwarps);
    __syncthreads();
    dense_layer<TM>(L[1], L[1].Wt, cv + L[1].coff, rh0, rh1, warp, lane, nwarps);
    __syncthreads();
    dense_layer<TM>(L[2], L[2].Wt, cv + L[2].coff, rh1, rh2, warp, lane, nwarps);
    __syncthreads();
    dense_layer<TM>(L[3], L[3].Wt, cv + L[3].coff, rh2, rh3, warp, lane, nwarps);
    __syncthreads();
    narrow_layer<TM>(L[4], L[4].Wt, cv + L[4].coff, rh3, rs, warp, lane, nwarps);
    __syncthreads();

    if (!BWD) {
        if (warp == 0) {
#pragma unroll
            for (int i = 0; i < TM; ++i) {
                const long long idx = p0 + lane * TM + i;
                if (valid[i]) b.member_s[idx * d.n_members + m] = rs[lane * TM + i];
            }
        }
        return;
    }

    // ------------------------------------------------------------------ backward
    // upstream: g_s = g_out * w_k / (S + 1e-6),   g_out = lambda_surface * sign(sdf) * kept / n_kept
    const float inv_count = b.stats[0] > 0.f ? 1.0f / b.stats[0] : 0.f;      // nothing kept: zero gradient (torch: mean of empty)
    float gs[TM];
    float ba[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int i = 0; i < TM; ++i) {
        const long long idx = p0 + lane * TM + i;
        gs[i] = 0.f;
        if (valid[i]) {
            const float g_out = lambda_surface * b.gsign[idx] * inv_count;
            const float Sp = b.S[idx] + 1e-6f;
            float dd, r = 0.f, dx = 0.f, dy = 0.f, dz = 0.f;
            if (has_anchor) {
                dx = ax - x[i]; dy = ay - y[i]; dz = az - z[i];
                r = sqrtf(dx * dx + dy * dy + dz * dz);
                const float nrm = r + 10e-6f;
                dd = -(nrm * nrm);
            } else {
                dd = -0.2f;
            }
            const float wk = expf(__fdiv_rn(dd, 0.01f));
            gs[i] = g_out * wk / Sp;
            if (has_anchor && warp == 0 && r > 0.f) {
                // blend path: d out / d w_k = (s_k - out) / (S + eps);  d w_k / d a_k = w_k/0.01 * (-2)(r + 1e-5) (a - x)/r
                const float s_k = rs[lane * TM + i];
                const float g_w = g_out * (s_k - b.out[idx]) / Sp;
                const float coef = g_w * wk * (1.0f / 0.01f) * (-2.0f) * (r + 10e-6f) / r;
                ba[0] += coef * dx; ba[1] += coef * dy; ba[2] += coef * dz;
            }
        }
    }
    if (has_anchor && warp == 0) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            float v = ba[a];
#pragma unroll
            for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            if (lane == 0 && v != 0.f) atomicAdd(b.blend_acc + m * 3 + a, v);
        }
    }
    // delta3 = g_s * w4 * sigma'(h3), in place over h3
    {
        const float *W4 = w.W[4] + (size_t)set * d.H;
        for (int n = warp; n < d.H; n += nwarps) {
            float *ptr = rh3 + (size_t)n * P + lane * TM;
            float h[TM], o[TM];
            load_act<TM>(ptr, h);
            const float w4 = __ldg(W4 + n);
#pragma unroll
            for (int i = 0; i < TM; ++i) o[i] = gs[i] * w4 * (h[i] > 0.2f ? 1.0f : -expm1f(-100.0f * h[i]));
            store_act<TM>(ptr, o);
        }
    }
    __syncthreads();
    dense_layer_bwd<TM>(w.W[3] + (size_t)set * d.H * d.H, d.H, d.H, d.H, 1.0f, rh3, rh2, warp, lane, nwarps);     // delta2
    __syncthreads();
    dense_layer_bwd<TM>(w.W[2] + (size_t)set * d.H * d.H, d.H, d.H, d.N1, 0.70710678118654752f, rh2, rh1, warp, lane, nwarps);   // delta1
    __syncthreads();
    dense_layer_bwd<TM>(w.W[1] + (size_t)set * d.N1 * d.H, d.H, d.N1, d.H, 1.0f, rh1, rh0, warp, lane, nwarps);    // delta0
    __syncthreads();
    // per-member sums over the points of the tile
    float *acc = b.acc + (size_t)m * 2 * d.H;
    for (int n = warp; n < 2 * d.H; n += nwarps) {
        const float *row = (n < d.H ? rh0 + (size_t)n * P : rh2 + (size_t)(n - d.H) * P) + lane * TM;
        float v[TM];
        load_act<TM>(row, v);
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < TM; ++i) s += v[i];
#pragma unroll
        for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0 && s != 0.f) atomicAdd(acc + n, s);
    }
}

// ---------------------------------------------------------------------------------------------------------------
// ---------------------------------------------------------------------------------------------------------------------
// Backward pass of the tensor-core path, layer by layer on wgmma (tc_linear.cu, batched over the members):
//   the forward (tc::wg::ensemble_wgmma_kernel<.., ACTS>) leaves sigma'_l = d softplus / d pre-activation of every hidden unit, a block
//   of tc::kActLd features x 128 points per (member, 128-point tile);
//   fit_upstream_kernel   g_s[m][p] = dL/d s_m(p) (blend + loss), blend-weight gradients w.r.t. anchors and points
//   3 batched GEMMs       delta2 = sigma'2 * (sigma'3 (diag(w4) W3));  delta1 = sigma'1 * (delta2 W2[:, :N1]) / sqrt2;
//                         delta0 = sigma'0 * (delta1 W1)      - per unit upstream gradient (times kDeltaScale), each written in
//                         place over the sigma' block it consumes
//   fit_reduce_kernel     per member: g_s-weighted column sums of delta0 / delta2 (-> acc), per point
//                         g_s (W0x^T delta0 + W2x^T delta2 / sqrt2) (-> grad_points)

// per point: upstream gradient of every member output, blend-weight path of the anchor / point gradients
__global__ void __launch_bounds__(256) fit_upstream_kernel(const Dims d, const Buffers b, float lambda_surface, float *__restrict__ gs,
                                                           long long gs_stride)
{
    __shared__ float s_anch[tc::kMaxMembers * 3], s_acc[tc::kMaxMembers * 3];     // n_loc < kMaxMembers (tc_ensemble_supported)
    const int lane = threadIdx.x & 31, scan = blockIdx.y;
    for (int i = threadIdx.x; i < d.n_loc * 3; i += blockDim.x) { s_anch[i] = b.anchors[(size_t)scan * d.n_loc * 3 + i]; s_acc[i] = 0.f; }
    __syncthreads();
    const long long i_scan = (long long)blockIdx.x * blockDim.x + threadIdx.x;     // point of the scan
    const long long idx = scan * b.n + i_scan;                                     // row of the point arrays
    const bool ok = i_scan < b.n;
    float x = 0.f, y = 0.f, z = 0.f, g_out = 0.f, Sp = 1.f, outv = 0.f;
    const bool quirk = ok && quirk_row(b, scan, i_scan);     // members' outputs are the constant 1: no member upstream
    if (ok) {
        const float *stats = b.stats + (size_t)scan * 8;
        const float inv_count = stats[0] > 0.f ? 1.0f / stats[0] : 0.f;
        x = b.points[idx * 3]; y = b.points[idx * 3 + 1]; z = b.points[idx * 3 + 2];
        g_out = lambda_surface * b.gsign[idx] * inv_count;
        Sp = b.S[idx] + 1e-6f;
        outv = b.out[idx];
    }
    float gx[3] = {0.f, 0.f, 0.f};
    for (int m = 0; m < d.n_members; ++m) {
        const bool has_anchor = m < d.n_loc;
        float c[3] = {0.f, 0.f, 0.f}, gsv = 0.f;
        if (ok) {
            float dd, r = 0.f, dx = 0.f, dy = 0.f, dz = 0.f;
            if (has_anchor) {
                dx = s_anch[m * 3] - x; dy = s_anch[m * 3 + 1] - y; dz = s_anch[m * 3 + 2] - z;
                r = sqrtf(dx * dx + dy * dy + dz * dz);
                const float nrm = r + 10e-6f;
                dd = -(nrm * nrm);
            } else {
                dd = -0.2f;
            }
            const float wk = expf(__fdiv_rn(dd, 0.01f));
            gsv = quirk ? 0.f : g_out * wk / Sp;
            if (has_anchor && r > 0.f) {
                const float s_k = quirk ? 1.0f : b.member_s[idx * d.n_members + m];
                const float g_w = g_out * (s_k - outv) / Sp;
                const float coef = g_w * wk * (1.0f / 0.01f) * (-2.0f) * (r + 10e-6f) / r;
                c[0] = coef * dx; c[1] = coef * dy; c[2] = coef * dz;
                gx[0] -= c[0]; gx[1] -= c[1]; gx[2] -= c[2];                  // d w_k / d x = - d w_k / d a_k
            }
            gs[(size_t)m * gs_stride + scan * b.tiles_per_scan * 128 + i_scan] = gsv;
        }
        if (has_anchor && b.blend_acc) {
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                float v = c[a];
#pragma unroll
                for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
                if (lane == 0 && v != 0.f) atomicAdd(&s_acc[m * 3 + a], v);
            }
        }
    }
    if (ok && b.grad_points) { b.grad_points[idx * 3] = gx[0]; b.grad_points[idx * 3 + 1] = gx[1]; b.grad_points[idx * 3 + 2] = gx[2]; }
    if (!b.blend_acc) return;
    __syncthreads();
    for (int i = threadIdx.x; i < d.n_loc * 3; i += blockDim.x)
        if (s_acc[i] != 0.f) atomicAdd(b.blend_acc + (size_t)scan * d.n_loc * 3 + i, s_acc[i]);
}

// one CTA per (128-point tile, member): (LATENT) g_s-weighted sums of delta0 / delta2 over the points (-> acc) and (POINTS) the
// gradient w.r.t. every point through the member's local coordinates (-> points_part).  The deltas come operand-ready from the
// GEMMs (packed: per k-step of 16 features [128 x 16 fp16 hi | 128 x 16 fp16 lo], value = hi + lo).
constexpr int kReduceThreads = 256;
constexpr float kDeltaScale = 64.0f;          // the GEMMs carry the deltas per unit upstream gradient, times this power of two: the
                                              // fp16 hi/lo operand split needs O(1) magnitudes (g_s itself is ~1e-4 / n_points)
constexpr int kStepsH = 13, kStepsN1 = 7;     // packed k-steps of a hidden-width (200) / layer-1-width (101) block
constexpr int kPackedPerTile = 2 * kStepsH + kStepsN1;      // [sigma'3 -> delta2 | delta1 | delta0]
template <bool POINTS, bool LATENT>
__global__ void __launch_bounds__(kReduceThreads) fit_reduce_kernel(const Dims d, const Weights w, const Buffers b,
                                                                   const uint8_t *__restrict__ packed, long long tiles,
                                                                   const float *__restrict__ gs)
{
    // A k-step of a packed tile is [row / 8][feature / 8][row % 8][feature % 8] fp16, hi then lo (4 KB each).  Warp (g, ch) reads,
    // per pass, the 128 contiguous bytes of row group 4 i + g, feature half ch: lane = (row % 8) * 4 + pair of features - every
    // load is one full line; a thread owns 2 features and, per k-step, 4 rows (one per pass).
    __shared__ float s_sum[2][kStepsH * 16];
    __shared__ float s_w[2][kStepsH * 16][3];
    __shared__ float s_up[128];
    __shared__ float s_g[2][128][3];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int g = warp & 3, ch = warp >> 2, r8 = lane >> 2, pr = lane & 3;
    const int m = blockIdx.y;
    const int set = m < 2 * d.n_symm ? (m >> 1) : m - d.n_symm;
    const int scan = (int)(blockIdx.x / b.tiles_per_scan);
    const long long row0 = ((long long)blockIdx.x - scan * b.tiles_per_scan) * 128;      // first point of the tile in its scan
    for (int i = threadIdx.x; i < 2 * kStepsH * 16; i += blockDim.x) (&s_sum[0][0])[i] = 0.f;
    // upstream gradient of s_m per point (zero beyond the scan's last point: the padding rows of a tile hold garbage)
    if (threadIdx.x < 128) {
        const long long row = row0 + threadIdx.x;
        s_up[threadIdx.x] = row < b.n ? gs[((size_t)m * tiles + blockIdx.x) * 128 + threadIdx.x] * (1.0f / kDeltaScale) : 0.f;
    }
    if (POINTS) {
        const int in0 = 3 + d.C;
        const float *W0 = w.W[0] + (size_t)set * d.H * in0;
        const float *W2 = w.W[2] + (size_t)set * d.H * d.H + d.N1;
        for (int i = threadIdx.x; i < kStepsH * 16 * 3; i += blockDim.x) {
            const int j = i / 3, a = i % 3;
            s_w[0][j][a] = j < d.H ? __ldg(W0 + (size_t)j * in0 + a) : 0.f;
            s_w[1][j][a] = j < d.H ? 0.70710678118654752f * __ldg(W2 + (size_t)j * d.H + a) : 0.f;
        }
    }
    __syncthreads();
    float up[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) up[i] = s_up[(4 * i + g) * 8 + r8];
    const uint8_t *tile = packed + ((size_t)m * tiles + blockIdx.x) * kPackedPerTile * 8192;
    float gp[4][3];
#pragma unroll
    for (int i = 0; i < 4; ++i) gp[i][0] = gp[i][1] = gp[i][2] = 0.f;
#pragma unroll 1
    for (int which = 0; which < 2; ++which) {
        const uint8_t *blk = tile + (size_t)(which ? 0 : kStepsH + kStepsN1) * 8192;       // delta2 first block, delta0 last
#pragma unroll 1
        for (int j = 0; j < kStepsH; ++j) {
            const int f = j * 16 + ch * 8 + pr * 2;
            float wa[3] = {0.f, 0.f, 0.f}, wb[3] = {0.f, 0.f, 0.f};
            if (POINTS) {
#pragma unroll
                for (int a = 0; a < 3; ++a) { wa[a] = s_w[which][f][a]; wb[a] = s_w[which][f + 1][a]; }
            }
            float c0 = 0.f, c1 = 0.f;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const uint8_t *src = blk + (size_t)j * 8192 + (size_t)(4 * i + g) * 256 + (size_t)ch * 128 + (size_t)lane * 4;
                const uint32_t hw = *reinterpret_cast<const uint32_t *>(src), lw = *reinterpret_cast<const uint32_t *>(src + 4096);
                const float2 hv = __half22float2(*reinterpret_cast<const __half2 *>(&hw));
                const float2 lv = __half22float2(*reinterpret_cast<const __half2 *>(&lw));
                // (an all-zero upstream row may hold NaN garbage in the padding rows of the last tile: select, do not multiply)
                const float v0 = up[i] != 0.f ? up[i] * (hv.x + lv.x) : 0.f, v1 = up[i] != 0.f ? up[i] * (hv.y + lv.y) : 0.f;
                c0 += v0; c1 += v1;
                if (POINTS) {
#pragma unroll
                    for (int a = 0; a < 3; ++a) gp[i][a] = fmaf(wa[a], v0, fmaf(wb[a], v1, gp[i][a]));
                }
            }
            if (LATENT) {
                // sum over the 8 rows of the group (lane bits 2..4), then over the row groups through shared memory
#pragma unroll
                for (int o = 4; o < 32; o <<= 1) { c0 += __shfl_xor_sync(0xffffffffu, c0, o); c1 += __shfl_xor_sync(0xffffffffu, c1, o); }
                if (lane < 4) {
                    if (c0 != 0.f) atomicAdd(&s_sum[which][f], c0);
                    if (c1 != 0.f) atomicAdd(&s_sum[which][f + 1], c1);
                }
            }
        }
    }
    if (POINTS) {
        // per row: sum over the feature pairs of the lane quad, then over the two feature halves (warps ch = 0, 1)
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                float v = gp[i][a];
                v += __shfl_xor_sync(0xffffffffu, v, 1);
                v += __shfl_xor_sync(0xffffffffu, v, 2);
                if (pr == 0) s_g[ch][(4 * i + g) * 8 + r8][a] = v;
            }
        __syncthreads();
        const bool mirror = (m & 1) && m < 2 * d.n_symm;
        float *part = b.points_part + ((size_t)m * tiles + blockIdx.x) * 3 * 128;
        for (int i = threadIdx.x; i < 128 * 3; i += blockDim.x) {
            const int pt = i % 128, a = i / 128;
            float v = s_g[0][pt][a] + s_g[1][pt][a];
            if (a == 0 && mirror) v = -v;
            part[i] = v;
        }
    }
    if (!LATENT) return;
    __syncthreads();
    float *acc = b.acc + ((size_t)scan * d.n_members + m) * 2 * d.H;
    for (int i = threadIdx.x; i < 2 * d.H; i += blockDim.x) {
        const float v = i < d.H ? s_sum[0][i] : s_sum[1][i - d.H];          // acc = [sum delta0 | sum delta2]
        if (v != 0.f) atomicAdd(acc + i, v);
    }
}

// grad_points += the members' point gradients in member order (one order the float atomics of a member-parallel sum could
// take, fixed, so that equal inputs give equal bits); zero terms are skipped like the atomics skip them
__global__ void __launch_bounds__(128) fit_points_kernel(const Dims d, const Buffers b, long long tiles)
{
    const int scan = blockIdx.y;
    const long long i_scan = (long long)blockIdx.x * 128 + threadIdx.x;
    if (i_scan >= b.n) return;
    const long long tile = scan * b.tiles_per_scan + blockIdx.x;
    float *g = b.grad_points + (scan * b.n + i_scan) * 3;
    for (int a = 0; a < 3; ++a) {
        float s = g[a];
        for (int m = 0; m < d.n_members; ++m) {
            const float v = b.points_part[(((size_t)m * tiles + tile) * 3 + a) * 128 + threadIdx.x];
            if (v != 0.f) s += v;
        }
        g[a] = s;
    }
}

// sdf = sum_k w_k s_k / (sum_k w_k + 1e-6); kept = |sdf| < clamp   (fitting.py:234-246); s_k = 1 at the eval-mode quirk rows
__global__ void fit_blend_kernel(const Dims d, const Buffers b, float clamp)
{
    const int scan = blockIdx.y;
    const long long i_scan = (long long)blockIdx.x * blockDim.x + threadIdx.x;     // point of the scan
    const long long idx = scan * b.n + i_scan;                                     // row of the point arrays
    const float *anchors = b.anchors + (size_t)scan * d.n_loc * 3;
    float cnt = 0.f, sum = 0.f;
    if (i_scan < b.n) {
        const float x = b.points[idx * 3], y = b.points[idx * 3 + 1], z = b.points[idx * 3 + 2];
        const bool quirk = quirk_row(b, scan, i_scan);
        float num = 0.f, den = 0.f;
        for (int k = 0; k < d.n_members; ++k) {
            float dd;
            if (k < d.n_loc) {
                const float dx = anchors[k * 3] - x, dy = anchors[k * 3 + 1] - y, dz = anchors[k * 3 + 2] - z;
                const float nrm = sqrtf(dx * dx + dy * dy + dz * dz) + 10e-6f;
                dd = -(nrm * nrm);
            } else {
                dd = -0.2f;
            }
            const float wk = expf(__fdiv_rn(dd, 0.01f));
            num = fmaf(wk, quirk ? 1.0f : b.member_s[idx * d.n_members + k], num);
            den += wk;
        }
        const float out = __fdiv_rn(num, den + 1e-6f);
        const float l = fabsf(out);
        b.out[idx] = out; b.S[idx] = den;
        if (b.sdf_out) b.sdf_out[idx] = out;
        if (b.upstream) {
            // plain vector-Jacobian product: the "loss" is sum_p upstream_p * sdf_p (count fixed to 1 so nothing is averaged)
            b.gsign[idx] = (!b.mask || b.mask[idx]) ? b.upstream[idx] : 0.f;
            if (i_scan == 0) cnt = 1.f;
            sum = b.gsign[idx] * out;
        } else {
            const bool kept = l < clamp && (!b.mask || b.mask[idx]);
            b.gsign[idx] = kept ? (out > 0.f ? 1.f : (out < 0.f ? -1.f : 0.f)) : 0.f;
            if (kept) { cnt = 1.f; sum = l; }
        }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
        sum += __shfl_xor_sync(0xffffffffu, sum, o);
    }
    float *stats = b.stats + (size_t)scan * 8;
    if ((threadIdx.x & 31) == 0) {
        // the count is a sum of small integers, exact in any order; the per-warp sums are added in warp order by the finalize
        if (cnt != 0.f) atomicAdd(stats + 0, cnt);
        b.sum_part[(size_t)scan * gridDim.x * (blockDim.x / 32) + (blockIdx.x * blockDim.x + threadIdx.x) / 32] = sum;
    }
}

// per member: g_u = W0u^T D0 + W2u^T D2 / sqrt2 ; g_c = W0x^T D0 + W2x^T D2 / sqrt2
// block = 128 columns x kGradSlices slices of the hidden index (partial sums through shared memory); grid (members, scans)
constexpr int kGradSlices = 4;
__global__ void __launch_bounds__(128 * kGradSlices) fit_member_grad_kernel(const Dims d, const Weights w, const Buffers b)
{
    const int m = blockIdx.x, scan = blockIdx.y;
    const int set = m < 2 * d.n_symm ? (m >> 1) : m - d.n_symm;
    const float *D0 = b.acc + ((size_t)scan * d.n_members + m) * 2 * d.H, *D2 = D0 + d.H;
    float *grad = b.grad + (size_t)scan * d.lat_dim;
    const int in0 = 3 + d.C, in2 = d.H;                 // row lengths of W0 / W2 in the reference layout
    const float *W0 = w.W[0] + (size_t)set * d.H * in0;
    const float *W2 = w.W[2] + (size_t)set * d.H * in2;
    const float r2 = 0.70710678118654752f;
    __shared__ float gc[3];
    __shared__ float part[kGradSlices][128];
    const int col = threadIdx.x & 127, slice = threadIdx.x >> 7;
    const int per = (d.H + kGradSlices - 1) / kGradSlices, n0 = slice * per, n1 = min(d.H, n0 + per);
    for (int j0 = 0; j0 < 3 + d.C; j0 += 128) {
        const int j = j0 + col;
        // j < 3: xyz columns; j >= 3: condition columns.  In W2 the order is [h1 (N1) | xyz (3) | cond (C)].
        float s0 = 0.f, s2 = 0.f;
        if (j < 3 + d.C) {
#pragma unroll 4
            for (int n = n0; n < n1; ++n) {
                s0 = fmaf(W0[(size_t)n * in0 + j], D0[n], s0);
                s2 = fmaf(W2[(size_t)n * in2 + d.N1 + j], D2[n], s2);
            }
        }
        part[slice][col] = s0 + r2 * s2;
        __syncthreads();
        if (slice == 0 && j < 3 + d.C) {
            float g = 0.f;
#pragma unroll
            for (int i = 0; i < kGradSlices; ++i) g += part[i][col];
            if (j < 3) gc[j] = g;
            else {
                const int u = j - 3;
                if (u < d.G) atomicAdd(grad + u, g);
                else grad[d.G + m * d.Lc + (u - d.G)] = g;
            }
        }
        __syncthreads();
    }
    if (threadIdx.x < 3 && m < d.n_loc) {
        const bool mirror = (m & 1) && m < 2 * d.n_symm;
        // c = x - a (x component negated for mirrored members)  =>  d c / d a = -1 (+1 for the mirrored x)
        const float sign = (threadIdx.x == 0 && mirror) ? 1.0f : -1.0f;
        const size_t a = (size_t)scan * d.n_loc * 3 + m * 3 + threadIdx.x;
        b.ganch[a] = b.blend_acc[a] + sign * gc[threadIdx.x];
    }
}

struct FinalizeArgs {
    float lambda_surface, lambda_reg_global, lambda_reg_loc, lambda_reg_unobserved, lambda_symm_dist;
    float step_size, bc2_sqrt, one_minus_beta1, beta2, one_minus_beta2, eps;
    int apply_update;
    int latent_grad;                // 0: only the loss terms are wanted (no mlp_pos backward)
};

// mlp_pos backward (anchor gradient -> z_glob), regularisers (fitting.py:252-268), loss terms, Adam; one CTA per scan (the
// latent, Adam moments, loss terms and gradient outputs are [scan][...])
__global__ void __launch_bounds__(1024) fit_finalize_kernel(const Dims d, const Weights w, const Buffers b, float *latent,
                                                           float *adam_m, float *adam_v, const FinalizeArgs a,
                                                           float *loss_terms, float *grad_out)
{
    extern __shared__ float sh[];
    const int scan = blockIdx.x;
    latent += (size_t)scan * d.lat_dim;
    if (adam_m) adam_m += (size_t)scan * d.lat_dim;
    if (adam_v) adam_v += (size_t)scan * d.lat_dim;
    if (loss_terms) loss_terms += (size_t)scan * 8;
    if (grad_out) grad_out += (size_t)scan * d.lat_dim;
    float *const grad = b.grad + (size_t)scan * d.lat_dim;
    const float *const ganch = b.ganch + (size_t)scan * d.n_loc * 3, *const stats = b.stats + (size_t)scan * 8;
    float *h0 = sh, *h1 = h0 + d.pos_hid, *g1 = h1 + d.pos_hid, *g0 = g1 + d.pos_hid, *red = g0 + d.pos_hid;
    const int tid = threadIdx.x, nt = blockDim.x;
    const int Hd = d.pos_hid, G = d.G, O = d.n_loc * 3;
    // forward of mlp_pos (ReLU masks): one warp per output row (coalesced weight rows + shuffle reduction)
    if (a.latent_grad) {
        const int lane = tid & 31, warp = tid >> 5, nw = nt >> 5;
        for (int n = warp; n < Hd; n += nw) {
            float s = 0.f;
            for (int j = lane; j < G; j += 32) s = fmaf(w.pos_w[0][(size_t)n * G + j], latent[j], s);
#pragma unroll
            for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (lane == 0) h0[n] = fmaxf(s + w.pos_b[0][n], 0.f);
        }
        __syncthreads();
        for (int n = warp; n < Hd; n += nw) {
            float s = 0.f;
            for (int j = lane; j < Hd; j += 32) s = fmaf(w.pos_w[1][(size_t)n * Hd + j], h0[j], s);
#pragma unroll
            for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (lane == 0) h1[n] = fmaxf(s + w.pos_b[1][n], 0.f);
        }
        __syncthreads();
    }
    // backward: out[j] = sum_n W[n][j] v[n] for j < cols - threads (j, slice of n), partial sums through shared memory
    float *scratch = red + 128;                                  // nt floats (red: 4 x 32 per-warp partials)
    auto matvec_t = [&](const float *W, int ld, int rows, int cols, const float *v, auto &&store) {
        const int cpad = cols <= 64 ? 64 : 256;                  // columns per pass (power of two <= nt)
        const int slices = nt / cpad, slice = tid / cpad, jj = tid % cpad;
        const int per = (rows + slices - 1) / slices, r0 = slice * per, r1 = min(rows, r0 + per);
        for (int j0 = 0; j0 < cols; j0 += cpad) {
            const int j = j0 + jj;
            float s = 0.f;
            if (j < cols) {
#pragma unroll 4
                for (int n = r0; n < r1; ++n) s = fmaf(W[(size_t)n * ld + j], v[n], s);
            }
            scratch[slice * cpad + jj] = s;
            __syncthreads();
            if (slice == 0 && j < cols) {
                float t = 0.f;
                for (int i = 0; i < slices; ++i) t += scratch[i * cpad + jj];
                store(j, t);
            }
            __syncthreads();
        }
    };
    if (a.latent_grad) {
        matvec_t(w.pos_w[2], Hd, O, Hd, ganch, [&](int j, float t) { g1[j] = h1[j] > 0.f ? t : 0.f; });
        matvec_t(w.pos_w[1], Hd, Hd, Hd, g1, [&](int j, float t) { g0[j] = h0[j] > 0.f ? t : 0.f; });
        matvec_t(w.pos_w[0], G, Hd, G, g0, [&](int j, float t) { grad[j] += t; });
    }
    // regularisers
    float part[4] = {0.f, 0.f, 0.f, 0.f};        // reg_global, reg_loc, reg_unobserved, (unused)
    const int unobs[3] = {30, 31, 39};
    for (int j = tid; j < d.lat_dim; j += nt) {
        const float zj = latent[j];
        float g = 0.f;
        if (j < G) { part[0] += zj * zj; g += a.lambda_reg_global * 2.f * zj; }
        else {
            part[1] += zj * zj; g += a.lambda_reg_loc * 2.f * zj;
            const int k = (j - G) / d.Lc;
            if (k == unobs[0] || k == unobs[1] || k == unobs[2]) { part[2] += zj * zj; g += a.lambda_reg_unobserved * 2.f * zj; }
        }
        grad[j] += g;
    }
    for (int i = 0; i < 3; ++i) {
        float v = part[i];
#pragma unroll
        for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if ((tid & 31) == 0) red[i * 32 + (tid >> 5)] = v;
    }
    __syncthreads();
    // symmetric-pair distance: mean_i ||z_2i - z_2i+1||  (one warp per pair)
    float symm_local = 0.f;
    for (int pair = tid >> 5; pair < d.n_symm; pair += nt >> 5) {
        const float *za = latent + G + (2 * pair) * d.Lc, *zb = za + d.Lc;
        float ss = 0.f;
        for (int j = tid & 31; j < d.Lc; j += 32) { const float df = za[j] - zb[j]; ss += df * df; }
#pragma unroll
        for (int o = 16; o; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
        const float nrm = sqrtf(ss);
        if (nrm > 0.f) {
            for (int j = tid & 31; j < d.Lc; j += 32) {
                const float g = a.lambda_symm_dist * (za[j] - zb[j]) / (nrm * d.n_symm);
                grad[G + (2 * pair) * d.Lc + j] += g;
                grad[G + (2 * pair + 1) * d.Lc + j] -= g;
            }
        }
        if ((tid & 31) == 0) symm_local += nrm;
    }
    if ((tid & 31) == 0) red[96 + (tid >> 5)] = symm_local;
    __syncthreads();
    if (tid == 0 && loss_terms) {
        float rg = 0.f, rl = 0.f, ru = 0.f, sy = 0.f;
        for (int wi = 0; wi < nt / 32; ++wi) { rg += red[wi]; rl += red[32 + wi]; ru += red[64 + wi]; sy += red[96 + wi]; }
        float sum = stats[1];
        if (b.sum_part) {
            const long long parts = (b.n + 127) / 128 * 4;
            const float *sp = b.sum_part + (size_t)scan * parts;
            for (long long i = 0; i < parts; ++i) if (sp[i] != 0.f) sum += sp[i];
        }
        loss_terms[0] = sum / stats[0];           // surface = mean |sdf| over kept points (NaN if none, like torch)
        loss_terms[1] = rg; loss_terms[2] = rl; loss_terms[3] = ru;
        loss_terms[4] = d.n_symm ? sy / d.n_symm : 0.f;
        loss_terms[5] = stats[0];
    }
    __syncthreads();
    // Adam (torch 2.x single-tensor update order)
    for (int j = tid; j < d.lat_dim; j += nt) {
        const float g = grad[j];
        if (grad_out) grad_out[j] = g;
        if (a.apply_update) {
            float mm = adam_m[j], vv = adam_v[j];
            mm = mm + (g - mm) * a.one_minus_beta1;                 // exp_avg.lerp_(grad, 1 - beta1)
            vv = vv * a.beta2 + a.one_minus_beta2 * g * g;          // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, 1 - beta2)
            const float denom = sqrtf(vv) / a.bc2_sqrt + a.eps;
            latent[j] = latent[j] - a.step_size * (mm / denom);     // param.addcdiv_(exp_avg, denom, value=-step_size)
            adam_m[j] = mm; adam_v[j] = vv;
        }
    }
}

}  // namespace fit
}  // namespace nphm

using namespace nphm;

namespace nphm { namespace fit {
// adjoint weights of the three hidden layers, one packed set per weight set of the ensemble (built on first use)
int backward_packs(nphm_ensemble *h, cudaStream_t stream)
{
    if (h->fit_packs) return NPHM_OK;
    const int H = h->cfg.hidden_dim, N1 = h->dims.N[1], sets = h->n_members - h->cfg.n_symm_pairs;
    BackwardPacks *bp = new BackwardPacks();
    int rc;
    // delta2_pre[p][j] = sum_f sigma'3[p][f] w4[f] W3[f][j]       (w4 folded into the rows of W3)
    if ((rc = bp->l3.pack(h->weights.W[3].as<float>(), H, H, H, 0, 0, true, kDeltaScale, stream, sets, (long long)H * H,
                          h->weights.W[4].as<float>(), H)) ||
        // delta1_pre[p][j] = sum_n delta2[p][n] W2[n][j] / sqrt2,  j < N1
        (rc = bp->l2.pack(h->weights.W[2].as<float>(), H, N1, H, 0, 0, true, 0.70710678118654752f, stream, sets, (long long)H * H)) ||
        // delta0_pre[p][j] = sum_n delta1[p][n] W1[n][j],           n < N1
        (rc = bp->l1.pack(h->weights.W[1].as<float>(), H, H, N1, 0, 0, true, 1.0f, stream, sets, (long long)N1 * H))) {
        delete bp;
        return rc;
    }
    h->fit_packs = bp;
    return NPHM_OK;
}
// fit_finalize_kernel over n_scans scans with the Adam constants of fp
int launch_finalize(const Dims &d, const Weights &w, const Buffers &b, int n_scans, float *latent_dev, float *adam_m_dev,
                    float *adam_v_dev, const nphm_fit_params *fp, int apply_update, float *loss_terms_dev, float *grad_out_dev,
                    cudaStream_t stream, bool latent_grad = true);
}}
namespace nphm {
void fit_packs_destroy(nphm_ensemble *h)
{
    delete h->fit_packs;
    h->fit_packs = nullptr;
}
}

extern "C" long long nphm_fit_batch_workspace_bytes(const nphm_ensemble *h, int n_scans, long long n_points)
{
    if (!h || n_scans < 1 || n_points < 0) return -1;
    const long long S = n_scans;
    long long floats = S * (n_points * (h->n_members + 3) + (long long)h->n_members * 2 * h->cfg.hidden_dim +
                            (long long)h->cfg.n_loc * 6 + 8 + h->lat_dim + (n_points + 127) / 128 * 4);
    // activation derivatives handed from the tensor-core forward to the backward GEMMs ([member][tile][kActLd][128], layers 0-2) and the upstream gradient of every member output ([member][rows]); every scan owns whole tiles
    const long long tiles = S * ((n_points + 127) / 128);
    floats += (long long)h->n_members * tiles * 128 * (nphm::tc::kActLd + 1);
    // operand-ready (packed) sigma'3 / deltas of the backward GEMMs
    return floats * 4 + (long long)h->n_members * tiles * nphm::fit::kPackedPerTile * 8192 + 1024;
}

extern "C" long long nphm_fit_workspace_bytes(const nphm_ensemble *h, long long n_points)
{
    return nphm_fit_batch_workspace_bytes(h, 1, n_points);
}

// One fitting step for n_scans scans of n_points each (layouts: fit::Buffers).  workspace_bytes < 0: the single-scan entry
// points, whose workspace is unsized (NULL = the handle's scratch).
static int fit_step_impl(nphm_ensemble *h, const float *points_dev, int n_scans, long long n_points, float *latent_dev,
                         float *adam_m_dev, float *adam_v_dev, const nphm_fit_params *fp, int apply_update,
                         float *loss_terms_dev, float *grad_out_dev, const unsigned char *mask_dev, float *grad_points_dev,
                         void *workspace_dev, long long workspace_bytes, void *stream_, const float *upstream_dev = nullptr,
                         float *sdf_out_dev = nullptr, long long quirk_period = 0, const int *quirk_periods_dev = nullptr,
                         bool latent_grad = true)
{
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    NPHM_REQUIRE(h && h->loaded, "nphm_fit_identity_step: weights not loaded");
    NPHM_REQUIRE(points_dev && latent_dev && fp && n_points > 0 && n_scans >= 1, "nphm_fit_identity_step: NULL argument or no points");
    NPHM_REQUIRE(!apply_update || (adam_m_dev && adam_v_dev), "nphm_fit_identity_step: Adam state is NULL");
    if (h->dims.n_lin != 5 || h->dims.skip != 2) {
        set_error("nphm_fit_identity_step: only ensembles with 4 hidden layers are supported");
        return NPHM_ERR_UNSUPPORTED;
    }
    const bool tc_path = tc_ensemble_supported(h) && h->tc_ready;
    NPHM_REQUIRE(quirk_period >= 0, "nphm_fit: quirk_period < 0");
    if ((quirk_period > 0 || quirk_periods_dev) && !tc_path) {
        set_error("the eval-mode quirk in fitting needs the tensor-core configuration (hidden 200, 4 layers, condition 96)");
        return NPHM_ERR_UNSUPPORTED;
    }
    if (n_scans > 1 && !tc_path) {
        set_error("scan-batched fitting needs the tensor-core configuration (hidden 200, 4 layers, condition 96)");
        return NPHM_ERR_UNSUPPORTED;
    }
    if (grad_points_dev && !tc_path) {
        set_error("gradient w.r.t. the points needs the tensor-core configuration (hidden 200, 4 layers, condition 96)");
        return NPHM_ERR_UNSUPPORTED;
    }
    fit::Dims d{};
    d.n_members = h->n_members; d.n_symm = h->cfg.n_symm_pairs; d.n_loc = h->cfg.n_loc;
    d.H = h->cfg.hidden_dim; d.N1 = h->dims.N[1]; d.C = h->dims.cond_dim; d.G = h->cfg.lat_dim_glob; d.Lc = h->cfg.lat_dim_loc;
    d.lat_dim = h->lat_dim; d.pos_hid = h->cfg.pos_mlp_dim; d.cvec_stride = h->dims.cvec_stride;
    for (int l = 0; l < 5; ++l) d.coff[l] = h->dims.coff[l];
    d.r_c = 0; d.r_h0 = 3; d.r_h1 = d.r_h0 + d.H; d.r_h2 = d.r_h1 + d.N1 + 3; d.r_h3 = d.r_h2 + d.H; d.r_s = d.r_h3 + d.H;
    d.rows = d.r_s + 8 + 8 * (fit::kThreads / 32);
    // nphm_b200/models/fitting.py restates this bound (ffma_fit_rows, FFMA_FIT_MAX_ROWS) to choose the autograd path for
    // the ensembles it rejects; keep the two in step (tests/test_gpu_ensemble_f64.py checks them against each other)
    const size_t smem = (size_t)d.rows * fit::P * sizeof(float);
    if (smem > 227 * 1024) {
        set_error("nphm_fit_identity_step: hidden width %d too large for the fitting kernel", d.H);
        return NPHM_ERR_UNSUPPORTED;
    }
    fit::Weights w{};
    for (int l = 0; l < 5; ++l) {
        w.W[l] = h->weights.W[l].as<float>(); w.Wt[l] = h->weights.Wt[l].as<float>();
        w.Npad[l] = h->dims.Npad[l]; w.K[l] = h->dims.K[l];
    }
    for (int i = 0; i < 3; ++i) { w.pos_w[i] = h->pos_w[i].as<float>(); w.pos_b[i] = h->pos_b[i].as<float>(); }
    w.mean_anchors = h->mean_anchors.as<float>();

    int rc;
    const long long need = nphm_fit_batch_workspace_bytes(h, n_scans, n_points);
    float *ws = static_cast<float *>(workspace_dev);
    if (workspace_bytes >= 0 && workspace_bytes < need) {
        set_error("fitting workspace too small: %lld bytes for %d scans of %lld points, %lld needed", workspace_bytes, n_scans,
                  n_points, need);
        return NPHM_ERR_CAPACITY;
    }
    if (!ws) {
        if ((rc = h->fit_scratch.reserve((size_t)need))) return rc;
        ws = h->fit_scratch.as<float>();
    }
    if ((rc = ensemble_prepare(h, latent_dev, n_scans, stream))) return rc;      // per-scan anchors + folded constants
    const long long S = n_scans, rows_total = S * ceil_div(n_points, 128) * 128;    // rows of all tiles of all scans
    fit::Buffers b{};
    b.points = points_dev; b.n = n_points; b.tiles_per_scan = ceil_div(n_points, 128);
    b.anchors = h->anchors.as<float>(); b.cvec = h->cvec.as<float>();
    float *p = ws;
    b.member_s = p; p += S * n_points * h->n_members;
    b.out = p; p += S * n_points; b.S = p; p += S * n_points; b.gsign = p; p += S * n_points;
    float *zero_begin = p;
    b.acc = p; p += S * h->n_members * 2 * d.H;
    b.blend_acc = p; p += S * d.n_loc * 3;
    b.stats = p; p += S * 8;
    b.ganch = p; p += S * d.n_loc * 3;
    b.grad = p; p += S * d.lat_dim;
    NPHM_CUDA_CHECK(cudaMemsetAsync(zero_begin, 0, (size_t)(p - zero_begin) * sizeof(float), stream));
    b.sum_part = p; p += S * b.tiles_per_scan * 4;                  // written whole by fit_blend_kernel
    p += (4 - ((p - ws) & 3)) & 3;                                  // 16-byte alignment of the activation block
    float *acts = p;
    b.acts = nullptr;
    b.mask = mask_dev;
    b.upstream = upstream_dev;
    b.sdf_out = sdf_out_dev;
    b.grad_points = grad_points_dev;
    // without a latent gradient the tensor-core backward keeps only what the point gradients need (the FFMA step computes
    // both in one kernel and drops the latent part)
    const bool skip_latent = !latent_grad && tc_path;
    if (skip_latent) b.blend_acc = nullptr;
    b.quirk_period = quirk_period;
    b.quirk_periods = quirk_periods_dev;

    const int tiles = (int)ceil_div(n_points, fit::P);
    dim3 grid(tiles, h->n_members);
    NPHM_CUDA_CHECK(cudaFuncSetAttribute(fit::fit_member_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    NPHM_CUDA_CHECK(cudaFuncSetAttribute(fit::fit_member_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    if (tc_path) {
        // forward pass on the tensor-core kernel, one query per scan: member outputs s_k -> member_s (the blended output is
        // recomputed by fit_blend_kernel together with the loss bookkeeping)
        SimtQuery q{};
        q.xyz = points_dev; q.first = 0; q.total = n_points; q.n_points = n_points; q.n_queries = n_scans; q.quirk_period = 0;
        q.cvec = h->cvec.as<float>(); q.anchors = h->anchors.as<float>(); q.blend = 1;
        q.out = b.out; q.members_out = b.member_s; q.exact = 1;
        q.acts_out = acts;
        q.acts_packed_out = reinterpret_cast<unsigned char *>(acts + (size_t)h->n_members * rows_total * (tc::kActLd + 1));
        // sigma'3 lands in the first kStepsH k-steps of every (member, tile) block of kPackedPerTile k-steps
        q.acts_packed_tile_steps = fit::kPackedPerTile;
        if ((rc = tc_ensemble_launch(h, q, stream))) return rc;
        b.acts = acts;
    } else {
        fit::fit_member_kernel<false><<<grid, fit::kThreads, smem, stream>>>(d, w, b, fp->lambda_surface);
        NPHM_CUDA_CHECK(cudaGetLastError());
    }
    fit::fit_blend_kernel<<<dim3((unsigned)ceil_div(n_points, 128), n_scans), 128, 0, stream>>>(d, b, fp->clamp);
    NPHM_CUDA_CHECK(cudaGetLastError());
    if (b.acts && !(skip_latent && !grad_points_dev)) {
        const long long n_tiles = rows_total / 128;
        float *gs = acts + (size_t)h->n_members * rows_total * tc::kActLd;
        uint8_t *packed = reinterpret_cast<uint8_t *>(gs + (size_t)h->n_members * rows_total);
        if ((rc = fit::backward_packs(h, stream))) return rc;
        const fit::BackwardPacks &bp = *h->fit_packs;
        fit::fit_upstream_kernel<<<dim3((unsigned)ceil_div(n_points, 256), n_scans), 256, 0, stream>>>(d, b, fp->lambda_surface, gs,
                                                                                                       rows_total);
        NPHM_CUDA_CHECK(cudaGetLastError());
        // per (member, tile): packed [sigma'3 -> delta2 (13 k-steps) | delta1 (7) | delta0 (13)], blocked fp32 sigma'0 | sigma'1 | sigma'2
        uint8_t *p32 = packed, *p1 = packed + (size_t)fit::kStepsH * 8192, *p0 = p1 + (size_t)fit::kStepsN1 * 8192;
        tcl::LinearParams lp{};
        // the GEMM rows are those of all tiles, up to the last point of the last scan (the rows are independent; the padding
        // rows between two scans carry finite activations of a clamped point and a zero upstream gradient)
        lp.M = rows_total - b.tiles_per_scan * 128 + n_points; lp.mode = tcl::kModeMult; lp.batch = h->n_members; lp.w_pairs = d.n_symm;
        lp.mul_blocked = 1; lp.ldmul = tc::kActLd; lp.sMul = rows_total * tc::kActLd;
        lp.sAp = lp.sCp = (long long)n_tiles * fit::kPackedPerTile * 8192;
        // strides between the tiles of one member: tc_linear indexes packed tiles with a_ksteps / c_ksteps, so a tile pitch of
        // kPackedPerTile k-steps is expressed through those counts
        lp.a_tile_steps = lp.c_tile_steps = fit::kPackedPerTile;
        // delta2 = sigma'2 * (sigma'3 (diag(w4) W3)), in place over sigma'3 (a CTA reads its tile before it writes it)
        lp.Ap = p32; lp.a_ksteps = fit::kStepsH; lp.Mul = acts + tc::kActOff2 * 128; lp.Cp = p32; lp.c_ksteps = fit::kStepsH;
        if ((rc = tcl::launch_linear(bp.l3, lp, stream))) return rc;
        // delta1 = sigma'1 * (delta2 W2[:, :N1]) / sqrt2
        lp.Ap = p32; lp.a_ksteps = fit::kStepsH; lp.Mul = acts + tc::kActOff1 * 128; lp.Cp = p1; lp.c_ksteps = fit::kStepsN1;
        if ((rc = tcl::launch_linear(bp.l2, lp, stream))) return rc;
        // delta0 = sigma'0 * (delta1 W1)
        lp.Ap = p1; lp.a_ksteps = fit::kStepsN1; lp.Mul = acts + tc::kActOff0 * 128; lp.Cp = p0; lp.c_ksteps = fit::kStepsH;
        if ((rc = tcl::launch_linear(bp.l1, lp, stream))) return rc;
        dim3 rgrid((unsigned)n_tiles, h->n_members);
        b.points_part = acts;           // the activation derivatives are dead once the three GEMMs have consumed them
        if (skip_latent) fit::fit_reduce_kernel<true, false><<<rgrid, fit::kReduceThreads, 0, stream>>>(d, w, b, packed, n_tiles, gs);
        else if (grad_points_dev) fit::fit_reduce_kernel<true, true><<<rgrid, fit::kReduceThreads, 0, stream>>>(d, w, b, packed, n_tiles, gs);
        else fit::fit_reduce_kernel<false, true><<<rgrid, fit::kReduceThreads, 0, stream>>>(d, w, b, packed, n_tiles, gs);
        NPHM_CUDA_CHECK(cudaGetLastError());
        if (grad_points_dev)
            fit::fit_points_kernel<<<dim3((unsigned)b.tiles_per_scan, n_scans), 128, 0, stream>>>(d, b, n_tiles);
    } else if (!b.acts) {
        fit::fit_member_kernel<true><<<grid, fit::kThreads, smem, stream>>>(d, w, b, fp->lambda_surface);
    }
    NPHM_CUDA_CHECK(cudaGetLastError());
    if (!skip_latent) {
        fit::fit_member_grad_kernel<<<dim3(h->n_members, n_scans), 128 * fit::kGradSlices, 0, stream>>>(d, w, b);
        NPHM_CUDA_CHECK(cudaGetLastError());
    }
    return fit::launch_finalize(d, w, b, n_scans, latent_dev, adam_m_dev, adam_v_dev, fp, apply_update, loss_terms_dev,
                                grad_out_dev, stream, !skip_latent);
}

extern "C" int nphm_fit_identity_step(nphm_ensemble *h, const float *points_dev, long long n_points, float *latent_dev,
                                      float *adam_m_dev, float *adam_v_dev, const nphm_fit_params *fp, int apply_update,
                                      float *loss_terms_dev, float *grad_out_dev, void *workspace_dev, void *stream)
{
    return fit_step_impl(h, points_dev, 1, n_points, latent_dev, adam_m_dev, adam_v_dev, fp, apply_update, loss_terms_dev,
                         grad_out_dev, nullptr, nullptr, workspace_dev, -1, stream);
}

extern "C" int nphm_fit_identity_step_quirk(nphm_ensemble *h, const float *points_dev, long long n_points, long long quirk_period,
                                            float *latent_dev, float *adam_m_dev, float *adam_v_dev, const nphm_fit_params *fp,
                                            int apply_update, float *loss_terms_dev, float *grad_out_dev, void *workspace_dev,
                                            void *stream)
{
    return fit_step_impl(h, points_dev, 1, n_points, latent_dev, adam_m_dev, adam_v_dev, fp, apply_update, loss_terms_dev,
                         grad_out_dev, nullptr, nullptr, workspace_dev, -1, stream, nullptr, nullptr, quirk_period);
}

static nphm_fit_params surface_params(float clamp)
{
    nphm_fit_params fp{};
    fp.lambda_surface = 1.0f;           // the regularisers of the latent code stay with the caller
    fp.clamp = clamp;
    fp.lr = 0.f;
    fp.step = 1;
    return fp;
}

extern "C" int nphm_fit_surface_grad(nphm_ensemble *h, const float *points_dev, long long n_points, const float *latent_dev,
                                     const unsigned char *mask_dev, float clamp, float *loss_terms_dev,
                                     float *grad_latent_dev, float *grad_points_dev, void *workspace_dev, void *stream)
{
    const nphm_fit_params fp = surface_params(clamp);
    return fit_step_impl(h, points_dev, 1, n_points, const_cast<float *>(latent_dev), nullptr, nullptr, &fp, 0, loss_terms_dev,
                         grad_latent_dev, mask_dev, grad_points_dev, workspace_dev, -1, stream, nullptr, nullptr, 0, nullptr,
                         grad_latent_dev != nullptr);
}

extern "C" int nphm_fit_surface_grad_quirk(nphm_ensemble *h, const float *points_dev, long long n_points, long long quirk_period,
                                           const float *latent_dev, const unsigned char *mask_dev, float clamp,
                                           float *loss_terms_dev, float *grad_latent_dev, float *grad_points_dev,
                                           void *workspace_dev, void *stream)
{
    const nphm_fit_params fp = surface_params(clamp);
    return fit_step_impl(h, points_dev, 1, n_points, const_cast<float *>(latent_dev), nullptr, nullptr, &fp, 0, loss_terms_dev,
                         grad_latent_dev, mask_dev, grad_points_dev, workspace_dev, -1, stream, nullptr, nullptr, quirk_period,
                         nullptr, grad_latent_dev != nullptr);
}

// the scan-batched entry points run only on the tensor-core path (no batched FFMA fallback)
static int require_batched(nphm_ensemble *h, const char *what, int n_scans, const void *workspace_dev)
{
    NPHM_REQUIRE(h && h->loaded, "%s: weights not loaded", what);
    NPHM_REQUIRE(n_scans >= 1 && workspace_dev, "%s: n_scans < 1 or NULL workspace", what);
    if (!(tc_ensemble_supported(h) && h->tc_ready)) {
        set_error("%s: needs the tensor-core configuration (hidden 200, 4 layers, condition 96)", what);
        return NPHM_ERR_UNSUPPORTED;
    }
    return NPHM_OK;
}

extern "C" int nphm_fit_identity_step_batched(nphm_ensemble *h, const float *points_dev, const unsigned char *mask_dev, int n_scans,
                                              long long n_points, float *latents_dev, float *adam_m_dev, float *adam_v_dev,
                                              const nphm_fit_params *fp, int apply_update, float *loss_terms_dev,
                                              float *grad_out_dev, void *workspace_dev, long long workspace_bytes, void *stream)
{
    int rc;
    if ((rc = require_batched(h, "nphm_fit_identity_step_batched", n_scans, workspace_dev))) return rc;
    return fit_step_impl(h, points_dev, n_scans, n_points, latents_dev, adam_m_dev, adam_v_dev, fp, apply_update, loss_terms_dev,
                         grad_out_dev, mask_dev, nullptr, workspace_dev, workspace_bytes, stream);
}

extern "C" int nphm_fit_identity_step_batched_quirk(nphm_ensemble *h, const float *points_dev, const unsigned char *mask_dev,
                                                    int n_scans, long long n_points, const int *quirk_periods_dev,
                                                    float *latents_dev, float *adam_m_dev, float *adam_v_dev,
                                                    const nphm_fit_params *fp, int apply_update, float *loss_terms_dev,
                                                    float *grad_out_dev, void *workspace_dev, long long workspace_bytes, void *stream)
{
    int rc;
    if ((rc = require_batched(h, "nphm_fit_identity_step_batched_quirk", n_scans, workspace_dev))) return rc;
    return fit_step_impl(h, points_dev, n_scans, n_points, latents_dev, adam_m_dev, adam_v_dev, fp, apply_update, loss_terms_dev,
                         grad_out_dev, mask_dev, nullptr, workspace_dev, workspace_bytes, stream, nullptr, nullptr, 0,
                         quirk_periods_dev);
}

extern "C" int nphm_fit_surface_grad_batched(nphm_ensemble *h, const float *points_dev, const unsigned char *mask_dev, int n_scans,
                                             long long n_points, const float *latents_dev, float clamp, float *loss_terms_dev,
                                             float *grad_latent_dev, float *grad_points_dev, void *workspace_dev,
                                             long long workspace_bytes, void *stream)
{
    int rc;
    if ((rc = require_batched(h, "nphm_fit_surface_grad_batched", n_scans, workspace_dev))) return rc;
    NPHM_REQUIRE(loss_terms_dev, "nphm_fit_surface_grad_batched: NULL loss terms");
    const nphm_fit_params fp = surface_params(clamp);
    return fit_step_impl(h, points_dev, n_scans, n_points, const_cast<float *>(latents_dev), nullptr, nullptr, &fp, 0,
                         loss_terms_dev, grad_latent_dev, mask_dev, grad_points_dev, workspace_dev, workspace_bytes, stream,
                         nullptr, nullptr, 0, nullptr, grad_latent_dev != nullptr);
}

extern "C" int nphm_fit_surface_grad_batched_quirk(nphm_ensemble *h, const float *points_dev, const unsigned char *mask_dev,
                                                   int n_scans, long long n_points, const int *quirk_periods_dev,
                                                   const float *latents_dev, float clamp, float *loss_terms_dev,
                                                   float *grad_latent_dev, float *grad_points_dev, void *workspace_dev,
                                                   long long workspace_bytes, void *stream)
{
    int rc;
    if ((rc = require_batched(h, "nphm_fit_surface_grad_batched_quirk", n_scans, workspace_dev))) return rc;
    NPHM_REQUIRE(loss_terms_dev, "nphm_fit_surface_grad_batched_quirk: NULL loss terms");
    const nphm_fit_params fp = surface_params(clamp);
    return fit_step_impl(h, points_dev, n_scans, n_points, const_cast<float *>(latents_dev), nullptr, nullptr, &fp, 0,
                         loss_terms_dev, grad_latent_dev, mask_dev, grad_points_dev, workspace_dev, workspace_bytes, stream,
                         nullptr, nullptr, 0, quirk_periods_dev, grad_latent_dev != nullptr);
}

// Vector-Jacobian product of the ensemble forward w.r.t. its inputs (SURVEY.md 8b: nphm_ensemble_backward_inputs):
//   grad_points[p]  = grad_sdf[p] * d sdf_p / d xyz_p           (local coordinates of every member + blend weights)
//   grad_latent     = sum_p grad_sdf[p] * d sdf_p / d latent     (member inputs + anchors/mlp_pos + blend weights)
// for the training-mode forward (no eval quirk) of FastEnsembleDeepSDFMirrored (EnsembledDeepSDF.py:203-267) - what
// torch.autograd computes for `decoder(xyz, lat)[0].backward(grad_sdf)`.  Same kernels as the fitting step.  The _quirk form
// takes the eval-mode forward: quirk_period = n_points is one decoder call.
extern "C" int nphm_ensemble_backward_inputs(nphm_ensemble *h, const float *points_dev, long long n_points, const float *latent_dev,
                                             const float *grad_sdf_dev, float *sdf_out_dev, float *grad_latent_dev,
                                             float *grad_points_dev, void *workspace_dev, void *stream)
{
    NPHM_REQUIRE(grad_sdf_dev && grad_latent_dev, "nphm_ensemble_backward_inputs: NULL gradient pointer");
    const nphm_fit_params fp = surface_params(0.f);
    return fit_step_impl(h, points_dev, 1, n_points, const_cast<float *>(latent_dev), nullptr, nullptr, &fp, 0, nullptr,
                         grad_latent_dev, nullptr, grad_points_dev, workspace_dev, -1, stream, grad_sdf_dev, sdf_out_dev);
}

extern "C" int nphm_ensemble_backward_inputs_quirk(nphm_ensemble *h, const float *points_dev, long long n_points,
                                                   long long quirk_period, const float *latent_dev, const float *grad_sdf_dev,
                                                   float *sdf_out_dev, float *grad_latent_dev, float *grad_points_dev,
                                                   void *workspace_dev, void *stream)
{
    NPHM_REQUIRE(grad_sdf_dev && grad_latent_dev, "nphm_ensemble_backward_inputs_quirk: NULL gradient pointer");
    const nphm_fit_params fp = surface_params(0.f);
    return fit_step_impl(h, points_dev, 1, n_points, const_cast<float *>(latent_dev), nullptr, nullptr, &fp, 0, nullptr,
                         grad_latent_dev, nullptr, grad_points_dev, workspace_dev, -1, stream, grad_sdf_dev, sdf_out_dev,
                         quirk_period);
}

// ------------------------------------------------------------------------------------------------ sharded fitting
namespace nphm { namespace fit {
// per scan: grad = lambda g, ganch = lambda ganch_in, stats[0..1] = stats_in[0..1]   (g [S][n], ganch_in [S][n_anch], stats_in [S][2])
__global__ void load_external_gradient_kernel(const float *__restrict__ g, const float *__restrict__ stats_in, float lambda,
                                              int n, int n_scans, float *__restrict__ grad, float *__restrict__ stats,
                                              const float *__restrict__ ganch_in, int n_anch, float *__restrict__ ganch)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < (long long)n_scans * n) grad[i] = lambda * g[i];
    if (ganch_in && i < (long long)n_scans * n_anch) ganch[i] = lambda * ganch_in[i];
    if (i < n_scans) { stats[i * 8] = stats_in[i * 2]; stats[i * 8 + 1] = stats_in[i * 2 + 1]; }
}

// torch.optim.Adam (betas 0.9 / 0.999, eps 1e-8, no weight decay; torch 2.x single-tensor update order) on a dense tensor
__global__ void adam_dense_kernel(float *__restrict__ param, const float *__restrict__ grad, float *__restrict__ m,
                                  float *__restrict__ v, long long n, float step_size, float bc2_sqrt)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float g = grad[i];
    float mm = m[i], vv = v[i];
    mm = mm + (g - mm) * 0.1f;
    vv = vv * 0.999f + 0.001f * g * g;
    const float denom = sqrtf(vv) / bc2_sqrt + 1e-8f;
    param[i] = param[i] - step_size * (mm / denom);
    m[i] = mm; v[i] = vv;
}

int launch_finalize(const Dims &d, const Weights &w, const Buffers &b, int n_scans, float *latent_dev, float *adam_m_dev,
                    float *adam_v_dev, const nphm_fit_params *fp, int apply_update, float *loss_terms_dev, float *grad_out_dev,
                    cudaStream_t stream, bool latent_grad)
{
    FinalizeArgs a{};
    a.lambda_surface = fp->lambda_surface; a.lambda_reg_global = fp->lambda_reg_global; a.lambda_reg_loc = fp->lambda_reg_loc;
    a.lambda_reg_unobserved = fp->lambda_reg_unobserved; a.lambda_symm_dist = fp->lambda_symm_dist;
    const double beta1 = 0.9, beta2 = 0.999;
    const int step = fp->step > 0 ? fp->step : 1;
    const double bc1 = 1.0 - std::pow(beta1, step), bc2 = 1.0 - std::pow(beta2, step);
    a.step_size = (float)((double)fp->lr / bc1);
    a.bc2_sqrt = (float)std::sqrt(bc2);
    a.one_minus_beta1 = (float)(1.0 - beta1); a.beta2 = (float)beta2; a.one_minus_beta2 = (float)(1.0 - beta2);
    a.eps = 1e-8f; a.apply_update = apply_update; a.latent_grad = latent_grad;
    const size_t fsm = (size_t)(4 * d.pos_hid + 128 + 1024) * sizeof(float);
    fit_finalize_kernel<<<n_scans, 1024, fsm, stream>>>(d, w, b, latent_dev, adam_m_dev, adam_v_dev, a, loss_terms_dev, grad_out_dev);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}
}}

static int apply_gradient_impl(nphm_ensemble *h, int n_scans, float *latent_dev, float *adam_m_dev, float *adam_v_dev,
                               const nphm_fit_params *fp, const float *surface_grad_dev, const float *surface_stats_dev,
                               const float *grad_anchors_dev, int apply_update, float *loss_terms_dev, float *grad_out_dev,
                               void *stream_)
{
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    NPHM_REQUIRE(h && h->loaded, "nphm_fit_apply_gradient: weights not loaded");
    NPHM_REQUIRE(n_scans >= 1 && latent_dev && adam_m_dev && adam_v_dev && fp && surface_grad_dev && surface_stats_dev,
                 "nphm_fit_apply_gradient: NULL argument or n_scans < 1");
    fit::Dims d{};
    d.n_members = h->n_members; d.n_symm = h->cfg.n_symm_pairs; d.n_loc = h->cfg.n_loc;
    d.H = h->cfg.hidden_dim; d.N1 = h->dims.N[1]; d.C = h->dims.cond_dim; d.G = h->cfg.lat_dim_glob; d.Lc = h->cfg.lat_dim_loc;
    d.lat_dim = h->lat_dim; d.pos_hid = h->cfg.pos_mlp_dim; d.cvec_stride = h->dims.cvec_stride;
    fit::Weights w{};
    for (int i = 0; i < 3; ++i) { w.pos_w[i] = h->pos_w[i].as<float>(); w.pos_b[i] = h->pos_b[i].as<float>(); }
    w.mean_anchors = h->mean_anchors.as<float>();
    int rc;
    const size_t floats = (size_t)n_scans * (d.n_loc * 3 + 8 + d.lat_dim);
    if ((rc = h->fit_apply_scratch.reserve(floats * sizeof(float)))) return rc;
    float *p = h->fit_apply_scratch.as<float>();
    fit::Buffers b{};
    b.ganch = p; p += (size_t)n_scans * d.n_loc * 3;     // zero unless the caller brings an anchor gradient of its own (joint fitter)
    b.stats = p; p += (size_t)n_scans * 8;
    b.grad = p;
    NPHM_CUDA_CHECK(cudaMemsetAsync(h->fit_apply_scratch.ptr, 0, floats * sizeof(float), stream));
    const long long n_threads = (long long)n_scans * (d.lat_dim > d.n_loc * 3 ? d.lat_dim : d.n_loc * 3);
    fit::load_external_gradient_kernel<<<(unsigned)((n_threads + 255) / 256), 256, 0, stream>>>(
        surface_grad_dev, surface_stats_dev, fp->lambda_surface, d.lat_dim, n_scans, b.grad, b.stats, grad_anchors_dev, d.n_loc * 3,
        b.ganch);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return fit::launch_finalize(d, w, b, n_scans, latent_dev, adam_m_dev, adam_v_dev, fp, apply_update, loss_terms_dev, grad_out_dev,
                                stream);
}

// Second half of a fitting iteration when the surface term was evaluated elsewhere - e.g. on the shards of a point-sharded
// fit (nphm_b200/distributed.py: every rank calls nphm_fit_surface_grad on its points, ONE all-reduce combines
// [n_r * grad_r, n_r * loss_r, n_r], then every rank calls this with the identical global mean gradient): adds the
// regularisers of fitting.py:252-268 and applies the Adam update exactly like nphm_fit_identity_step.
// surface_grad_dev: d(mean |sdf| over the kept points)/d latent (lat_dim, un-weighted); surface_stats_dev: [n_kept, sum |sdf|].
extern "C" int nphm_fit_apply_gradient(nphm_ensemble *h, float *latent_dev, float *adam_m_dev, float *adam_v_dev,
                                       const nphm_fit_params *fp, const float *surface_grad_dev, const float *surface_stats_dev,
                                       const float *grad_anchors_dev, int apply_update, float *loss_terms_dev,
                                       float *grad_out_dev, void *stream)
{
    return apply_gradient_impl(h, 1, latent_dev, adam_m_dev, adam_v_dev, fp, surface_grad_dev, surface_stats_dev, grad_anchors_dev,
                               apply_update, loss_terms_dev, grad_out_dev, stream);
}

// The same for n_scans independent scans sharing fp (schedule, lr, Adam step): every argument gains a leading scan axis.
extern "C" int nphm_fit_apply_gradient_batched(nphm_ensemble *h, int n_scans, float *latents_dev, float *adam_m_dev,
                                               float *adam_v_dev, const nphm_fit_params *fp, const float *surface_grad_dev,
                                               const float *surface_stats_dev, const float *grad_anchors_dev, int apply_update,
                                               float *loss_terms_dev, float *grad_out_dev, void *stream)
{
    return apply_gradient_impl(h, n_scans, latents_dev, adam_m_dev, adam_v_dev, fp, surface_grad_dev, surface_stats_dev,
                               grad_anchors_dev, apply_update, loss_terms_dev, grad_out_dev, stream);
}

// torch.optim.Adam.step() on a dense fp32 tensor (reference src/NPHM/models/fitting.py:36,169: the expression codes of the joint
// fitter - every row is updated every iteration, also the rows that were not sampled).  step = 1-based step count.
extern "C" int nphm_adam_step(float *param_dev, const float *grad_dev, float *adam_m_dev, float *adam_v_dev, long long n, float lr,
                              int step, void *stream_)
{
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    NPHM_REQUIRE(param_dev && grad_dev && adam_m_dev && adam_v_dev && n >= 0 && step >= 1, "nphm_adam_step: bad arguments");
    if (n == 0) return NPHM_OK;
    const double bc1 = 1.0 - std::pow(0.9, step), bc2 = 1.0 - std::pow(0.999, step);
    nphm::fit::adam_dense_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(param_dev, grad_dev, adam_m_dev, adam_v_dev, n,
                                                                                  (float)((double)lr / bc1), (float)std::sqrt(bc2));
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}
