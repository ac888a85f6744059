// Layer-by-layer passes of a DeepSDF-style stack on the generic wgmma linear layer (tc_linear.cu):
//
//   value pass     h_l = softplus(W_l in_l + c_l), s_l = softplus'(.)          (any width: the NPM baseline 515 -> 1024 x 8 ...)
//   tangent pass   forward-mode derivative w.r.t. xyz:  t_l = s_l * (W_l t_{l-1}),  3 rows per point  ->  Jacobian d out / d xyz
//   adjoint pass   d_l-1 = s_l-1 * (W_l^T d_l)  ->  gradient w.r.t. the per-query condition (and, optionally, w.r.t. xyz)
//
// Reference semantics: DeepSDF.forward src/NPHM/models/deepSDF.py:64-89 (skip connection `cat([x, inp]) / sqrt(2)` at layer
// nlayers // 2, Softplus(beta = 100)); `jac` src/NPHM/models/diff_operators.py:26-54 (three autograd passes there, one
// forward-mode pass here); the adjoint pass is what `loss.backward()` (src/NPHM/models/fitting.py:167) does to the deformation
// network in the joint fitter.  The condition is constant over the points of a query, so its part of layers 0 and `skip` is
// folded into per-query constants (simt.cu: cvec) and its gradient only needs the per-query column sums of d_0 and d_skip.
#include "tc_linear.cuh"
#include "tc_wgrad.cuh"
#include <algorithm>
#include <cmath>
#include <cuda_fp16.h>

namespace nphm {
namespace chain {

constexpr float kInvSqrt2 = 0.70710678118654752440f;
constexpr float kBeta = 100.0f;                       // Softplus(beta = 100): softplus'' = kBeta S (1 - S)

// out[q][c] += sum over the rows of query q of X[row][c], X a PACKED activation buffer (tc_linear.cuh: per 128-row tile and
// k-step [128 x 16 fp16 hi | 128 x 16 fp16 lo], core-matrix order; value = hi + lo), with float atomics.  grid (tiles, k-steps),
// 256 threads: thread = (row of the tile, 8 of the 16 columns).
__global__ void __launch_bounds__(256) column_sums_packed_kernel(const uint8_t *__restrict__ X, int ksteps, long long M,
                                                                 long long rows_per_query, int n_cols, float *__restrict__ out)
{
    __shared__ float s_sum[16];
    const int r = threadIdx.x >> 1, ch = threadIdx.x & 1, lane = threadIdx.x & 31;
    const int j = blockIdx.y;
    const long long row0 = (long long)blockIdx.x * 128, row = row0 + r;
    const bool ok = row < M;
    const long long q = (ok ? row : M - 1) / rows_per_query;
    const long long q_first = row0 / rows_per_query, q_last = (min(row0 + 127, M - 1)) / rows_per_query;
    const bool block_uniform = q_first == q_last;
    if (threadIdx.x < 16) s_sum[threadIdx.x] = 0.f;
    __syncthreads();
    float v[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = 0.f;
    if (ok) {
        const uint8_t *src = X + ((size_t)blockIdx.x * ksteps + j) * 8192 + (size_t)(r >> 3) * 256 + (size_t)ch * 128 + (size_t)(r & 7) * 16;
        const uint4 h = *reinterpret_cast<const uint4 *>(src), l = *reinterpret_cast<const uint4 *>(src + 4096);
        const uint32_t hw[4] = {h.x, h.y, h.z, h.w}, lw[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float2 a = __half22float2(*reinterpret_cast<const __half2 *>(&hw[i]));
            const float2 b = __half22float2(*reinterpret_cast<const __half2 *>(&lw[i]));
            v[2 * i] = a.x + b.x; v[2 * i + 1] = a.y + b.y;
        }
    }
    const int c0 = j * 16 + ch * 8;
    if (block_uniform) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            float x = v[i];
#pragma unroll
            for (int o = 2; o < 32; o <<= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
            if (lane < 2 && x != 0.f) atomicAdd(&s_sum[ch * 8 + i], x);
        }
        __syncthreads();
        if (threadIdx.x < 16 && j * 16 + threadIdx.x < n_cols && s_sum[threadIdx.x] != 0.f)
            atomicAdd(out + (size_t)q_first * n_cols + j * 16 + threadIdx.x, s_sum[threadIdx.x]);
    } else if (ok) {
#pragma unroll
        for (int i = 0; i < 8; ++i)
            if (c0 + i < n_cols && v[i] != 0.f) atomicAdd(out + (size_t)q * n_cols + c0 + i, v[i]);
    }
}

// grad_cond[m][q][j] = sum_n W0[n][3 + j] * S0[m][q][n]  +  sum_n Ws[n][c0s + j] * Ss[m][q][n] / sqrt(2), W0 and Ws those of
// member m's weight set.  grid (column blocks, queries, members x chunks of the n range): one chunk writes its sum in a fixed
// order; more add their partial sums with float atomics to an `out` the caller has zeroed.
__global__ void cond_grad_kernel(const float *__restrict__ W0, int ld0, int N0, const float *__restrict__ S0,
                                 const float *__restrict__ Ws, int lds, int Ns, int c0s, const float *__restrict__ Ss, int cond_dim,
                                 int n_queries, int n_symm, int chunks, float *__restrict__ out)
{
    const int j = blockIdx.x * blockDim.x + threadIdx.x, q = blockIdx.y;
    const int m = blockIdx.z / chunks, chunk = blockIdx.z % chunks, set = member_set(m, n_symm);
    if (j >= cond_dim) return;
    const size_t mq = (size_t)m * n_queries + q;
    const float *w0 = W0 + (size_t)set * N0 * ld0, *ws = Ws + (size_t)set * Ns * lds;
    const int c0 = (N0 + chunks - 1) / chunks, a0 = chunk * c0, b0 = min(N0, a0 + c0);
    float s = 0.f;
    for (int n = a0; n < b0; ++n) s = fmaf(w0[(size_t)n * ld0 + 3 + j], S0[mq * N0 + n], s);
    const int c1 = (Ns + chunks - 1) / chunks, a1 = chunk * c1, b1 = min(Ns, a1 + c1);
    float t = 0.f;
    for (int n = a1; n < b1; ++n) t = fmaf(ws[(size_t)n * lds + c0s + j], Ss[mq * Ns + n], t);
    s = fmaf(t, kInvSqrt2, s);
    if (chunks == 1) out[mq * cond_dim + j] = s;
    else atomicAdd(out + mq * cond_dim + j, s);
}

// out[(q, n)][i][j] = T[(q, n, j)][i]   (tangent rows -> Jacobian layout B x N x out x 3)
__global__ void jacobian_layout_kernel(const float *__restrict__ T, int ld, long long n_rows, int out_dim, float *__restrict__ J)
{
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n_rows * out_dim * 3) return;
    const int j = (int)(idx % 3);
    const int i = (int)((idx / 3) % out_dim);
    const long long n = idx / (3 * out_dim);
    J[idx] = T[(size_t)(n * 3 + j) * ld + i];
}

// in place: J (3 x 3 per point, row i = gradient of output i) -> (I + J)^-1  (adjugate / determinant)
__global__ void inverse_plus_identity_kernel(float *__restrict__ J, long long n)
{
    const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    float *m = J + p * 9;
    const float a = m[0] + 1.f, b = m[1], c = m[2], d = m[3], e = m[4] + 1.f, f = m[5], g = m[6], h = m[7], i = m[8] + 1.f;
    const float A = e * i - f * h, B = -(d * i - f * g), C = d * h - e * g;
    const float inv = 1.0f / (a * A + b * B + c * C);
    m[0] = A * inv; m[1] = -(b * i - c * h) * inv; m[2] = (b * f - c * e) * inv;
    m[3] = B * inv; m[4] = (a * i - c * g) * inv;  m[5] = -(a * f - c * d) * inv;
    m[6] = C * inv; m[7] = -(a * h - b * g) * inv; m[8] = (a * e - b * d) * inv;
}

// grad_xyz[m][r][i] = (a[m][r][i] + b[m][r][i]) * scale[sstride set(m) + 1]   (a, b: ld 4; scale == nullptr: 1)
__global__ void xyz_grad_kernel(const float *__restrict__ a, const float *__restrict__ b, long long M, int members,
                                const float *__restrict__ scale, int sstride, int n_symm, float *__restrict__ out)
{
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)members * M * 3) return;
    const long long r = idx / 3;
    const int i = (int)(idx % 3), m = (int)(r / M);
    out[idx] = (a[r * 4 + i] + b[r * 4 + i]) * (scale ? scale[sstride * member_set(m, n_symm) + 1] : 1.0f);
}

// dst[i] = src[i] * scale[2 q + which], q = i / per_query: one scale pair per query (grad_scale_kernel); in place is fine
__global__ void query_scale_kernel(const float *src, long long per_query, long long n, const float *__restrict__ scale, int which,
                                   float *dst)
{
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n) return;
    dst[idx] = src[idx] * scale[2 * (idx / per_query) + which];
}

}  // namespace chain

// ------------------------------------------------------------------------------------------------ members and packed stack
// The passes run over `count` members at once: tc_linear's batched launch over gridDim.z = member, tc_wgrad's over gridDim.z =
// weight set.  Member m uses weight set member_set(m, n_symm) of `sets` sets packed back to back, and its part of every per-row
// buffer starts at m times that buffer's member stride.  A DeepSDF handle is {1, 0, 1}, the NPHM ensemble {40, 16, 24}.
struct Members {
    int count = 1, n_symm = 0, sets = 1;
};

struct PackedChain {
    bool packed = false;
    tcl::PackedLinear fwd[kMaxLayers];        // B = W_l restricted to its point-dependent columns (1/sqrt2 folded at the skip)
    tcl::PackedLinear adj[kMaxLayers];        // B = W_l^T (input-activation columns only)
    tcl::PackedLinear adj_x0, adj_xs;         // W_0[:, 0:3]^T and W_skip[:, Nh:Nh+3]^T / sqrt2  (gradient w.r.t. xyz)
    int ld[kMaxLayers];
    // scratch of the backwards: GEMM partials, per-(member, query) column sums of d_0, d_skip and the other layers
    DeviceBuffer partials, sums0, sumss, sums;
};

// what only the DeepSDF handle has
struct MlpChain : PackedChain {
    // activations between the layers live in the packed operand format (Hp: values, Tp: tangents, Dp: adjoints), the
    // activation derivatives S in the blocked fp32 layout ([128-row tile][feature][128]) - every access of the passes is coalesced
    DeviceBuffer Hp[kMaxLayers], S[kMaxLayers], Tp[2], Dp[2], Tlast, out_tmp;
    DeviceBuffer Fp[2];                       // ping-pong activations of the forward-only pass (forward_pass)
    long long value_rows = 0;                 // rows of the last value pass that kept the activation derivatives
    bool have_deriv = false;
    // training (nphm_mlp_train_forward / _backward) with condition noise: layers 0, skip - 1 and skip take `train_nd` > 0
    // per-row condition columns more (layer 0: [xyz | noise], the skip layer: [h | xyz | noise] / sqrt2, the layer before it
    // appends them); packed on first use after every weight load.
    tcl::PackedLinear tfwd[kMaxLayers];
    int train_nd = -1;
    // scratch of the first-order backwards: the packed top adjoint, its scale pairs, the two [M][4] point-gradient parts (d_0
    // and d_skip times their layer's xyz columns), the scaled upstream of the adjoint pass
    DeviceBuffer Dl, gscale, xtmp, xs_tmp, gup;
};

// the stack a pass runs on
struct Stack {
    const StackDims &s;
    const NetWeights &w;
    PackedChain &c;
    Members m;
};

static Stack stack(nphm_mlp *h) { return Stack{h->dims, h->weights, *h->chain, Members{}}; }

static int pad4(int n) { return (n + 3) / 4 * 4; }
constexpr int kChainNt = 128;

// packs `sets` weight sets, set z of layer l at W_l + z N_l in_total_l
static int pack_chain(PackedChain &c, const StackDims &s, const NetWeights &wts, int sets, cudaStream_t stream)
{
    int rc;
    for (int l = 0; l < s.n_lin; ++l) {
        const float *W = wts.W[l].as<float>();
        const int ldw = s.in_total[l];
        const long long wst = (long long)s.N[l] * ldw;
        const float scale = l == s.skip ? chain::kInvSqrt2 : 1.0f;
        // forward: point-dependent leading columns (xyz | h_{l-1} | [h_{skip-1}, xyz])
        // (the layer in front of the skip layer reserves 3 output columns: its epilogue appends xyz / the tangent seeds)
        // tiles of <= 128 output columns: the passes run on a few thousand rows (fitting), where CTAs count more than tile width
        if ((rc = c.fwd[l].pack(W, ldw, s.N[l], s.K[l], 0, 0, false, scale, stream, sets, wst, nullptr, 0, l + 1 == s.skip ? 3 : 0,
                                kChainNt)))
            return rc;
        // adjoint w.r.t. the input activations of layer l (l >= 1): columns [0, N_{l-1})
        if (l >= 1 && (rc = c.adj[l].pack(W, ldw, s.N[l - 1], s.N[l], 0, 0, true, scale, stream, sets, wst, nullptr, 0, 0, kChainNt)))
            return rc;
        c.ld[l] = pad4(s.N[l]);
    }
    if ((rc = c.adj_x0.pack(wts.W[0].as<float>(), s.in_total[0], 3, s.N[0], 0, 0, true, 1.0f, stream, sets,
                            (long long)s.N[0] * s.in_total[0])))
        return rc;
    if (s.skip > 0 && s.skip < s.n_lin &&
        (rc = c.adj_xs.pack(wts.W[s.skip].as<float>(), s.in_total[s.skip], 3, s.N[s.skip], s.N[s.skip - 1], 0, true,
                            chain::kInvSqrt2, stream, sets, (long long)s.N[s.skip] * s.in_total[s.skip])))
        return rc;
    c.packed = true;
    return NPHM_OK;
}

int chain_pack(nphm_mlp *h, cudaStream_t stream)
{
    if (!h->chain) h->chain = new MlpChain();
    int rc = pack_chain(*h->chain, h->dims, h->weights, 1, stream);
    if (rc) return rc;
    h->chain->train_nd = -1;
    return NPHM_OK;
}

void chain_destroy(nphm_mlp *h)
{
    delete h->chain;
    h->chain = nullptr;
}

static size_t packed_bytes(long long rows, int ksteps) { return (size_t)ceil_div(rows, 128) * ksteps * 8192; }

// 256-byte aligned pieces of a workspace, from `off` on
struct Carver {
    size_t off = 0;
    size_t take(size_t bytes) { const size_t o = off; off += (bytes + 255) / 256 * 256; return o; }
};

// the layers that take the per-row condition noise as extra input columns (training, MlpChain::tfwd)
static bool noise_layer(const StackDims &s, int l) { return l == 0 || l + 1 == s.skip || l == s.skip; }

// the per-row buffers of a value pass over M rows per member; member m's part of each at m times its stride (floats; bytes
// for the packed Hp)
struct ValueRows {
    const float *X = nullptr; int ldx = 3; long long sX = 0;     // rows [xyz | nd noise columns]: the input of layer 0 and the
    int nd = 0;                                                 // columns appended behind layer skip - 1
    const tcl::PackedLinear *tfwd = nullptr;                    // nd > 0: the packs of the noise layers (MlpChain::tfwd)
    const float *bias = nullptr; long long rows_per_bias = 0, sBias = 0;     // the per-query constants of the first query
    uint8_t *Hp[kMaxLayers] = {}; long long sHp[kMaxLayers] = {};           // h_l, packed
    float *S[kMaxLayers] = {}; long long sS[kMaxLayers] = {};               // s_l, blocked (optional)
    float *out = nullptr; long long sOut = 0;                                // the output layer, row-major
    const int *live = nullptr;                                               // see forward_pass
    const int *live_rows = nullptr; long long live_off = 0;                  // see forward_pass
};

// value pass: softplus layers 0 .. n_lin - 2 and the linear output layer
static int value_layers(const Stack &k, long long M, const ValueRows &v, cudaStream_t stream)
{
    const StackDims &s = k.s;
    for (int l = 0; l < s.n_lin; ++l) {
        const tcl::PackedLinear &W = v.nd > 0 && noise_layer(s, l) ? v.tfwd[l] : k.c.fwd[l];
        tcl::LinearParams p;
        p.M = M; p.batch = k.m.count; p.w_pairs = k.m.n_symm;
        p.live = v.live;
        p.live_rows = v.live_rows; p.live_off = v.live_off;
        if (l == 0) { p.A1 = v.X; p.lda1 = v.ldx; p.K1 = 3 + v.nd; p.sA1 = v.sX; }
        else { p.Ap = v.Hp[l - 1]; p.a_ksteps = W.ksteps; p.sAp = v.sHp[l - 1]; }   // at the skip layer: [h | xyz | noise]
        p.bias = v.bias + s.coff[l]; p.ldb = s.cvec_stride; p.rows_per_bias = v.rows_per_bias; p.sBias = v.sBias;
        if (l == s.n_lin - 1) {
            p.mode = tcl::kModeLinear;
            p.C = v.out; p.ldc = s.N[l]; p.sC = v.sOut;
        } else {
            p.mode = tcl::kModeSoftplus;
            p.Cp = v.Hp[l]; p.c_ksteps = W.packed_ksteps_out(); p.sCp = v.sHp[l];
            if (l + 1 == s.skip) { p.app = v.X; p.app_ld = v.ldx; p.app_w = 3 + v.nd; p.sApp = v.sX; }
            if (v.S[l]) { p.Dv = v.S[l]; p.lddv = k.c.ld[l]; p.dv_blocked = 1; p.sDv = v.sS[l]; }
        }
        int rc = tcl::launch_linear(W, p, stream);
        if (rc) return rc;
    }
    return NPHM_OK;
}

// value pass over M = n_queries * n_points rows; keeps h_l (packed) and (want_deriv) s_l (blocked) of every hidden layer;
// `out` = last layer, row-major
static int value_pass(nphm_mlp *h, const float *xyz, int n_queries, long long n_points, bool want_deriv, float *out,
                      cudaStream_t stream)
{
    MlpChain &c = *h->chain;
    const StackDims &s = h->dims;
    const long long M = (long long)n_queries * n_points;
    ValueRows v;
    v.X = xyz;
    v.bias = h->cvec.as<float>(); v.rows_per_bias = n_points;
    v.out = out;
    int rc;
    for (int l = 0; l + 1 < s.n_lin; ++l) {
        if ((rc = c.Hp[l].reserve(packed_bytes(M, c.fwd[l].packed_ksteps_out())))) return rc;
        if (want_deriv && (rc = c.S[l].reserve((size_t)ceil_div(M, 128) * 128 * c.ld[l] * sizeof(float)))) return rc;
        v.Hp[l] = c.Hp[l].as<uint8_t>();
        if (want_deriv) v.S[l] = c.S[l].as<float>();
    }
    if ((rc = value_layers(stack(h), M, v, stream))) return rc;
    c.value_rows = M;
    c.have_deriv = want_deriv;
    return NPHM_OK;
}

// Forward only (no derivatives kept), in chunks of at most kForwardChunkRows rows through two ping-pong operand buffers: the
// memory it needs is bounded by the chunk (2 x 128 MB for the deformation backbone), not by the number of points, so a whole
// 256^3 grid can be queried in one call.  Chunks hold whole queries, or a run of rows of one query.  `live` (optional device
// counter): every launch returns at once when it reads 0.  `live_rows` (optional, per query): only the points below it are
// computed, the tiles beyond it return at once.
constexpr long long kForwardChunkRows = 1 << 16;
static int forward_pass(nphm_mlp *h, const float *xyz, int n_queries, long long n_points, float *out, const int *live,
                        const int *live_rows, cudaStream_t stream)
{
    if (n_points == 0) return NPHM_OK;
    MlpChain &c = *h->chain;
    const StackDims &s = h->dims;
    int ks_max = 1, rc;
    for (int l = 0; l + 1 < s.n_lin; ++l) ks_max = std::max(ks_max, c.fwd[l].packed_ksteps_out());
    const long long qpc = n_points <= kForwardChunkRows ? std::max(1LL, kForwardChunkRows / n_points) : 1;   // queries per chunk
    const long long ppc = std::min(n_points, kForwardChunkRows);                                             // points per chunk
    const long long max_rows = std::min((long long)n_queries, qpc) * ppc;
    for (int b = 0; b < 2; ++b)
        if ((rc = c.Fp[b].reserve(packed_bytes(max_rows, ks_max)))) return rc;
    ValueRows v;
    v.live = live;
    for (int l = 0; l + 1 < s.n_lin; ++l) v.Hp[l] = c.Fp[l & 1].as<uint8_t>();
    const int out_dim = s.N[s.n_lin - 1];
    for (long long q0 = 0; q0 < n_queries; q0 += qpc) {
        const long long nq = std::min(qpc, (long long)n_queries - q0);
        for (long long p0 = 0; p0 < n_points; p0 += ppc) {
            const long long np = std::min(ppc, n_points - p0);       // nq > 1 only with whole queries (np == n_points)
            const size_t row0 = (size_t)q0 * n_points + p0;
            v.X = xyz + row0 * 3;
            v.bias = h->cvec.as<float>() + (size_t)q0 * s.cvec_stride; v.rows_per_bias = np;
            v.out = out + row0 * out_dim;
            if (live_rows) { v.live_rows = live_rows + q0; v.live_off = p0; }
            if ((rc = value_layers(stack(h), nq * np, v, stream))) return rc;
        }
    }
    c.have_deriv = false;
    return NPHM_OK;
}

// the adjoint of a layer's pre-activations: row-major fp32 rows (the caller's output gradient) or packed (ks k-steps); member
// m's part at m times `stride` (floats or bytes)
struct Adjoint {
    const float *rows = nullptr; int ld = 0;
    const uint8_t *packed = nullptr; int ks = 0;
    long long stride = 0;
};

// what one adjoint walk reads and writes; per-layer entries for l < L = n_lin - 1, member strides in floats (S, cpl_z) or
// bytes (D, cpl_a)
struct AdjointWalk {
    Adjoint top;                                                      // d_L
    const float *S[kMaxLayers] = {}; long long sS[kMaxLayers] = {};   // s_l, blocked fp32
    uint8_t *D[kMaxLayers] = {}; long long sD[kMaxLayers] = {};       // where d_l goes, packed
    const float *cpl_z[kMaxLayers] = {};                              // optional coupling of the SDF-gradient backward:
    const uint8_t *cpl_a[kMaxLayers] = {}; long long sA[kMaxLayers] = {};   // d_l += kBeta (1 - s_l) * cpl_z[l] * cpl_a[l]
    float *xs = nullptr;                                              // optional [members][M][4]: d_skip W_skip[:, Nh:Nh+3]^T / sqrt2
};

// d_{l-1} = s_{l-1} * (d_l W_l) from d_L down to d_0 (left in w.D[0]) for every member.  hook(l, d_l) runs for l = L .. 1
// before the descent below layer l and for l = 0 at the bottom.
template <class Hook>
static int adjoint_walk(const Stack &k, long long M, const AdjointWalk &w, Hook &&hook, cudaStream_t stream)
{
    const StackDims &s = k.s;
    Adjoint d = w.top;
    int rc;
    for (int l = s.n_lin - 1; l >= 1; --l) {
        if ((rc = hook(l, d))) return rc;
        tcl::LinearParams p;
        p.M = M; p.batch = k.m.count; p.w_pairs = k.m.n_symm;
        if (d.packed) { p.Ap = d.packed; p.a_ksteps = d.ks; p.sAp = d.stride; }
        else { p.A1 = d.rows; p.lda1 = d.ld; p.K1 = s.N[l]; p.sA1 = d.stride; }
        if (l == s.skip && w.xs) {                 // d_skip is packed: chain_ready keeps the skip layer below the output layer
            tcl::LinearParams px = p;
            px.mode = tcl::kModeLinear; px.C = w.xs; px.ldc = 4; px.sC = M * 4;
            if ((rc = tcl::launch_linear(k.c.adj_xs, px, stream))) return rc;
        }
        const int ks = (s.N[l - 1] + 15) / 16;
        p.mode = tcl::kModeMult;
        p.Mul = w.S[l - 1]; p.ldmul = k.c.ld[l - 1]; p.mul_div = 1; p.mul_blocked = 1; p.sMul = w.sS[l - 1];
        if (w.cpl_a[l - 1]) {
            p.cpl_z = w.cpl_z[l - 1]; p.sCplZ = w.sS[l - 1];
            p.cpl_a = w.cpl_a[l - 1]; p.sCplA = w.sA[l - 1]; p.cpl_a_steps = ks; p.cpl_coef = chain::kBeta;
        }
        p.Cp = w.D[l - 1]; p.c_ksteps = ks; p.sCp = w.sD[l - 1];
        if ((rc = tcl::launch_linear(k.c.adj[l], p, stream))) return rc;
        d = Adjoint{nullptr, 0, w.D[l - 1], ks, w.sD[l - 1]};
    }
    return hook(0, d);
}

// grad_cond [members][q][cond_dim] from the per-(member, query) column sums of d_0 (sums0) and d_skip (sumss).  chunks: CTAs
// per output over the n range, added with float atomics; 1 keeps a fixed summation order.
static int cond_grad(const Stack &k, int n_queries, int chunks, float *grad_cond, cudaStream_t stream)
{
    const StackDims &s = k.s;
    if (chunks > 1) NPHM_CUDA_CHECK(cudaMemsetAsync(grad_cond, 0, (size_t)k.m.count * n_queries * s.cond_dim * sizeof(float), stream));
    dim3 grid((unsigned)ceil_div(s.cond_dim, 128), (unsigned)n_queries, (unsigned)(k.m.count * chunks));
    chain::cond_grad_kernel<<<grid, 128, 0, stream>>>(k.w.W[0].as<float>(), s.in_total[0], s.N[0], k.c.sums0.as<float>(),
                                                      k.w.W[s.skip].as<float>(), s.in_total[s.skip], s.N[s.skip],
                                                      s.N[s.skip - 1] + 3, k.c.sumss.as<float>(), s.cond_dim, n_queries,
                                                      k.m.n_symm, chunks, grad_cond);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

// grad_xyz = (d_0 W_0[:, 0:3]^T + xs) * scale[sstride set + 1] (scale == nullptr: 1): d_0 packed (w.D[0] of the walk, member
// stride d0_stride), x0 an [members][M][4] temporary, xs the walk's skip-layer part
static int xyz_grad(const Stack &k, long long M, const uint8_t *d0, long long d0_stride, float *x0, const float *xs,
                    const float *scale, int sstride, float *grad_xyz, cudaStream_t stream)
{
    tcl::LinearParams p;
    p.M = M; p.batch = k.m.count; p.w_pairs = k.m.n_symm;
    p.Ap = d0; p.a_ksteps = (k.s.N[0] + 15) / 16; p.sAp = d0_stride;
    p.mode = tcl::kModeLinear; p.C = x0; p.ldc = 4; p.sC = M * 4;
    int rc = tcl::launch_linear(k.c.adj_x0, p, stream);
    if (rc) return rc;
    chain::xyz_grad_kernel<<<(unsigned)ceil_div(k.m.count * M * 3, 256), 256, 0, stream>>>(x0, xs, M, k.m.count, scale, sstride,
                                                                                          k.m.n_symm, grad_xyz);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

}  // namespace nphm

using namespace nphm;

static int chain_ready(nphm_mlp *h, const char *who)
{
    NPHM_REQUIRE(h && h->loaded, "%s: weights not loaded", who);
    NPHM_REQUIRE(h->chain && h->chain->packed, "%s: layer chain not packed", who);
    NPHM_REQUIRE(h->dims.skip >= 1 && h->dims.skip < h->dims.n_lin - 1, "%s: unsupported skip position", who);
    return NPHM_OK;
}

namespace nphm {
// the forward-deformation backbone (DeepSDF MLP, hidden 512, 6 hidden layers, 3 outputs) with the condition of a
// DeformationNetwork mode whose condition is constant per query: 232 (`compress`, scripts/configs/nphm_def.yaml), 200
// (`expr_only`) or 264 (`glob_only`) - the shapes NPHM_IMPL_AUTO sends to the tensor cores (the Broyden search's evaluations
// included, which the FFMA kernel would otherwise run at a sixteenth of the rate)
bool tc_mlp_supported(const nphm_mlp *h)
{
    const int c = h->cfg.lat_dim;
    return h->cfg.hidden_dim == 512 && h->cfg.n_layers == 6 && (c == 232 || c == 200 || c == 264) && h->cfg.out_dim == 3 &&
           h->chain && h->chain->packed;
}

bool chain_packed(const nphm_mlp *h) { return h->chain && h->chain->packed; }

// forward with the constants of the last mlp_prepare
int chain_forward(nphm_mlp *h, const float *xyz, int n_queries, long long n_points, float *out, cudaStream_t stream)
{
    int rc = chain_ready(h, "chain_forward");
    if (rc) return rc;
    return forward_pass(h, xyz, n_queries, n_points, out, h->live, h->live_rows, stream);
}
}  // namespace nphm

// forward of an arbitrary-width stack, layer by layer (used when no fused kernel takes the shape)
extern "C" int nphm_mlp_query_layers(nphm_mlp *h, const float *xyz_dev, const float *cond_dev, int n_queries, long long n_points,
                                     float *out_dev, void *stream_)
{
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    int rc = chain_ready(h, "nphm_mlp_query_layers");
    if (rc) return rc;
    NPHM_REQUIRE(n_queries >= 1 && n_points >= 0 && cond_dev, "nphm_mlp_query_layers: bad arguments");
    if (n_points == 0) return NPHM_OK;
    NPHM_REQUIRE(xyz_dev && out_dev, "nphm_mlp_query_layers: NULL pointer");
    if ((rc = mlp_prepare(h, cond_dev, n_queries, stream))) return rc;
    return forward_pass(h, xyz_dev, n_queries, n_points, out_dev, nullptr, nullptr, stream);
}

// value + forward-mode tangents: out [q][n][out_dim] (optional), jac [q][n][out_dim][3] = d out / d xyz
extern "C" int nphm_mlp_jacobian(nphm_mlp *h, const float *xyz_dev, const float *cond_dev, int n_queries, long long n_points,
                                 float *out_dev, float *jac_dev, void *stream_)
{
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    int rc = chain_ready(h, "nphm_mlp_jacobian");
    if (rc) return rc;
    NPHM_REQUIRE(n_queries >= 1 && n_points >= 0 && cond_dev && jac_dev, "nphm_mlp_jacobian: bad arguments");
    if (n_points == 0) return NPHM_OK;
    MlpChain &c = *h->chain;
    const StackDims &s = h->dims;
    const long long M = (long long)n_queries * n_points;
    const int out_dim = s.N[s.n_lin - 1];
    if ((rc = mlp_prepare(h, cond_dev, n_queries, stream))) return rc;
    float *out = out_dev;
    if (!out) {
        if ((rc = c.out_tmp.reserve((size_t)M * out_dim * sizeof(float)))) return rc;
        out = c.out_tmp.as<float>();
    }
    if ((rc = value_pass(h, xyz_dev, n_queries, n_points, true, out, stream))) return rc;
    // tangent pass: rows (point, j), j = 0..2; tangents between the layers packed, the last layer row-major for the layout kernel
    int max_ks = 1;
    for (int l = 0; l + 1 < s.n_lin; ++l) max_ks = std::max(max_ks, c.fwd[l].packed_ksteps_out());
    for (int i = 0; i < 2; ++i)
        if ((rc = c.Tp[i].reserve(packed_bytes(3 * M, max_ks)))) return rc;
    const int ld_last = c.ld[s.n_lin - 1];
    if ((rc = c.Tlast.reserve((size_t)3 * M * ld_last * sizeof(float)))) return rc;
    for (int l = 0; l < s.n_lin; ++l) {
        const bool last = l == s.n_lin - 1;
        tcl::LinearParams p;
        p.M = 3 * M;
        if (l == 0) { p.K1 = 0; p.K2 = 3; p.a2_onehot = 1; }
        else { p.Ap = c.Tp[(l - 1) & 1].as<uint8_t>(); p.a_ksteps = c.fwd[l].ksteps; }
        if (last) {
            p.mode = tcl::kModeLinear;
            p.C = c.Tlast.as<float>(); p.ldc = ld_last;
        } else {
            p.mode = tcl::kModeMult; p.Mul = c.S[l].as<float>(); p.ldmul = c.ld[l]; p.mul_div = 3; p.mul_blocked = 1;
            p.Cp = c.Tp[l & 1].as<uint8_t>(); p.c_ksteps = c.fwd[l].packed_ksteps_out();
            if (l + 1 == s.skip) { p.app_onehot = 1; p.app_w = 3; }               // d xyz / d xyz_j = e_j
        }
        if ((rc = tcl::launch_linear(c.fwd[l], p, stream))) return rc;
    }
    const long long total = M * out_dim * 3;
    chain::jacobian_layout_kernel<<<(unsigned)ceil_div(total, 256), 256, 0, stream>>>(c.Tlast.as<float>(), ld_last, M, out_dim,
                                                                                      jac_dev);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

namespace nphm {
namespace train {
__global__ void grad_scale_kernel(const float *__restrict__ g, long long n, const float *__restrict__ g2, long long n2, int n_symm,
                                  float *__restrict__ scale);
}  // namespace train
}  // namespace nphm

// adjoint pass: grad_cond [q][cond_dim] = sum_n (d out_n / d cond)^T grad_out_n ; grad_xyz [q][n][3] optional
// fp16 range: every d_l is stored as an fp16 hi | lo pair, which keeps its bits only while |d_l| >= 2^-3 (see kGradExp), and
// the joint fitters' upstream u = -J^-T g_x is ~1e-4.  So the upstream is scaled on the device by one power of two per query,
// its largest magnitude to 2^kGradExp (grad_scale_kernel; an all-zero or non-finite query keeps scale 1), and the gradients
// are multiplied back in fp32 (exact).  Per query: a query's gradients do not depend on the other queries of the call.
extern "C" int nphm_mlp_backward_inputs(nphm_mlp *h, const float *xyz_dev, const float *cond_dev, int n_queries, long long n_points,
                                        const float *grad_out_dev, float *grad_cond_dev, float *grad_xyz_dev, void *stream_)
{
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    int rc = chain_ready(h, "nphm_mlp_backward_inputs");
    if (rc) return rc;
    NPHM_REQUIRE(n_queries >= 1 && n_points > 0 && cond_dev && grad_out_dev && (grad_cond_dev || grad_xyz_dev),
                 "nphm_mlp_backward_inputs: bad arguments");
    MlpChain &c = *h->chain;
    const StackDims &s = h->dims;
    const long long M = (long long)n_queries * n_points;
    const int L = s.n_lin - 1, out_dim = s.N[L];
    if (xyz_dev) {
        if ((rc = mlp_prepare(h, cond_dev, n_queries, stream))) return rc;
        if ((rc = c.out_tmp.reserve((size_t)M * out_dim * sizeof(float)))) return rc;
        if ((rc = value_pass(h, xyz_dev, n_queries, n_points, true, c.out_tmp.as<float>(), stream))) return rc;
        c.value_rows = M;
    } else {
        // xyz_dev == NULL: the activation derivatives of the previous nphm_mlp_jacobian / nphm_mlp_inverse_jacobian call on this
        // handle are reused (the joint fitter differentiates at the same points it just took the Jacobian at)
        NPHM_REQUIRE(c.value_rows == M && c.have_deriv, "nphm_mlp_backward_inputs: no matching value pass to reuse");
    }
    int max_ks = 1;
    for (int l = 1; l <= L; ++l) max_ks = std::max(max_ks, (s.N[l - 1] + 15) / 16);
    for (int i = 0; i < 2; ++i)
        if ((rc = c.Dp[i].reserve(packed_bytes(M, max_ks)))) return rc;
    if ((rc = c.sums0.reserve((size_t)n_queries * s.N[0] * sizeof(float))) ||
        (rc = c.sumss.reserve((size_t)n_queries * s.N[s.skip] * sizeof(float))))
        return rc;
    if (grad_xyz_dev && ((rc = c.xtmp.reserve((size_t)M * 4 * sizeof(float))) || (rc = c.xs_tmp.reserve((size_t)M * 4 * sizeof(float)))))
        return rc;
    NPHM_CUDA_CHECK(cudaMemsetAsync(c.sums0.ptr, 0, (size_t)n_queries * s.N[0] * sizeof(float), stream));
    NPHM_CUDA_CHECK(cudaMemsetAsync(c.sumss.ptr, 0, (size_t)n_queries * s.N[s.skip] * sizeof(float), stream));
    // the output layer's adjoint is the caller's grad_out times its query's scale; d_l lives in Dp[l & 1]
    if ((rc = c.gscale.reserve((size_t)2 * n_queries * sizeof(float))) || (rc = c.gup.reserve((size_t)M * out_dim * sizeof(float))))
        return rc;
    float *gs = c.gscale.as<float>(), *gup = c.gup.as<float>();
    train::grad_scale_kernel<<<n_queries, 1024, 0, stream>>>(grad_out_dev, n_points * out_dim, nullptr, 0, 0, gs);
    NPHM_CUDA_CHECK(cudaGetLastError());
    chain::query_scale_kernel<<<(unsigned)ceil_div(M * out_dim, 256), 256, 0, stream>>>(grad_out_dev, n_points * out_dim,
                                                                                       M * out_dim, gs, 0, gup);
    NPHM_CUDA_CHECK(cudaGetLastError());
    AdjointWalk w;
    w.top = Adjoint{gup, out_dim, nullptr, 0, 0};
    for (int l = 0; l < L; ++l) { w.S[l] = c.S[l].as<float>(); w.D[l] = c.Dp[l & 1].as<uint8_t>(); }
    w.xs = grad_xyz_dev ? c.xs_tmp.as<float>() : nullptr;
    // the column sums of d_0 and d_skip feed the condition gradient
    auto col_sums = [&](int l, const Adjoint &d) {
        if (l != 0 && l != s.skip) return NPHM_OK;
        chain::column_sums_packed_kernel<<<dim3((unsigned)ceil_div(M, 128), (unsigned)d.ks), 256, 0, stream>>>(
            d.packed, d.ks, M, n_points, s.N[l], l == 0 ? c.sums0.as<float>() : c.sumss.as<float>());
        NPHM_CUDA_CHECK(cudaGetLastError());
        return NPHM_OK;
    };
    const Stack k = stack(h);
    if ((rc = adjoint_walk(k, M, w, col_sums, stream))) return rc;
    // undo the scale: grad_cond rows per query, grad_xyz rows per query's points
    if (grad_cond_dev) {
        if ((rc = cond_grad(k, n_queries, 16, grad_cond_dev, stream))) return rc;
        chain::query_scale_kernel<<<(unsigned)ceil_div((long long)n_queries * s.cond_dim, 256), 256, 0, stream>>>(
            grad_cond_dev, s.cond_dim, (long long)n_queries * s.cond_dim, gs, 1, grad_cond_dev);
        NPHM_CUDA_CHECK(cudaGetLastError());
    }
    if (grad_xyz_dev) {
        if ((rc = xyz_grad(k, M, w.D[0], 0, c.xtmp.as<float>(), w.xs, nullptr, 0, grad_xyz_dev, stream))) return rc;
        chain::query_scale_kernel<<<(unsigned)ceil_div(M * 3, 256), 256, 0, stream>>>(grad_xyz_dev, n_points * 3, M * 3, gs, 1,
                                                                                     grad_xyz_dev);
        NPHM_CUDA_CHECK(cudaGetLastError());
    }
    return NPHM_OK;
}

extern "C" int nphm_mlp_inverse_jacobian(nphm_mlp *h, const float *xyz_dev, const float *cond_dev, int n_queries, long long n_points,
                                         float *out_dev, float *jinv_dev, void *stream_)
{
    NPHM_REQUIRE(h && h->loaded && h->dims.N[h->dims.n_lin - 1] == 3, "nphm_mlp_inverse_jacobian: needs a 3-output stack");
    int rc = nphm_mlp_jacobian(h, xyz_dev, cond_dev, n_queries, n_points, out_dev, jinv_dev, stream_);
    if (rc || n_points == 0) return rc;
    const long long M = (long long)n_queries * n_points;
    chain::inverse_plus_identity_kernel<<<(unsigned)ceil_div(M, 256), 256, 0, static_cast<cudaStream_t>(stream_)>>>(jinv_dev, M);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

// ================================================================================================ training
// One step of the stage-2 loss (reference scripts/training/train_corresp.py -> TrainerAutoDecoder.train_step,
// src/NPHM/models/training_corresp.py:154-176) needs, per decoder call, a value pass that keeps its activations, and later an
// adjoint pass with the weight gradient of every layer.  Everything the backward needs lives in the caller's workspace, so
// several forwards can be alive at once (the loss calls the decoder twice and autograd runs the backwards in reverse order).
//
// Per-row condition columns: in train mode the reference adds randn(B, N, 32) / 200 to the compressed columns of every point
// (deepSDF.py:220-221).  The noise enters layer 0 and the skip layer; both take it as extra point-dependent input columns:
// [xyz | noise] is staged once as a row array X0, read as A1 by layer 0 and appended (app) to the output of the layer in
// front of the skip.  Weight gradients of those columns fall out of the same GEMM; the per-query part of the condition is
// the outer product of the per-query column sums of d_0 / d_skip with the condition.
//
// fp16 range: the upstream gradient of the loss is of order 1e-5, where the hi part of the fp16 split is subnormal and the lo
// part is lost.  The backward scales it on the device by a power of two (its largest magnitude to 2^10) and undoes the scale in
// the fp32 epilogues of the gradients (grad_scale_kernel).
//
// The kernels below are member-indexed (Members): member m reads and writes its part of a per-row buffer at m times its member
// stride and uses the scale pair of its weight set, scale[2 set], scale[2 set + 1].
namespace nphm {
namespace train {

// workspace of one forward: 256-byte aligned pieces
struct Layout {
    size_t cond = 0, x0 = 0, x0p = 0, hp[kMaxLayers] = {}, s[kMaxLayers] = {}, total = 0;
    int ldx = 0, ks_x0 = 0, ks_h[kMaxLayers] = {};
};

static Layout layout(const StackDims &s, int n_queries, long long n_points, int nd)
{
    Layout L;
    const long long M = (long long)n_queries * n_points, tiles = ceil_div(M, 128);
    Carver w;
    L.cond = w.take((size_t)n_queries * s.cond_dim * sizeof(float));
    L.ldx = pad4(3 + nd);
    L.ks_x0 = (3 + nd + 15) / 16;
    L.x0 = w.take((size_t)M * L.ldx * sizeof(float));
    L.x0p = w.take((size_t)tiles * L.ks_x0 * 8192);
    for (int l = 0; l + 1 < s.n_lin; ++l) {
        L.ks_h[l] = (s.N[l] + (l + 1 == s.skip ? 3 + nd : 0) + 15) / 16;
        L.hp[l] = w.take((size_t)tiles * L.ks_h[l] * 8192);
        L.s[l] = w.take((size_t)tiles * 128 * pad4(s.N[l]) * sizeof(float));
    }
    L.total = w.off;
    return L;
}

// X0[row] = [xyz | noise | 0 ...]  (ldx columns)
__global__ void stage_x0_kernel(const float *__restrict__ xyz, const float *__restrict__ noise, int nd, long long M, int ldx,
                                float *__restrict__ X0)
{
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= M * ldx) return;
    const long long r = idx / ldx;
    const int c = (int)(idx % ldx);
    X0[idx] = c < 3 ? xyz[r * 3 + c] : (c < 3 + nd ? noise[r * nd + c - 3] : 0.f);
}

// fp32 rows [M][ld] (the first `width` columns, times scale[2 set] if given) -> packed operand tiles of `ks` k-steps
// (tc_linear.cuh); the rows of the last tile beyond M are zero.  Thread = (row, 8 columns); grid (row blocks, members):
// member m reads src + m src_stride (floats), writes dst + m dst_stride (bytes).
__global__ void pack_rows_kernel(const float *__restrict__ src, int ld, int width, long long M, int ks, long long src_stride,
                                 const float *__restrict__ scale, int n_symm, uint8_t *__restrict__ dst, long long dst_stride)
{
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int m = blockIdx.y;
    if (idx >= (M + 127) / 128 * 128 * 2 * ks) return;
    const long long row = idx / (2 * ks);
    const int g = (int)(idx % (2 * ks));
    const float sc = scale ? scale[2 * member_set(m, n_symm)] : 1.0f;
    const float *sr = src + (size_t)m * src_stride;
    float v[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int c = 8 * g + i;
        v[i] = (row < M && c < width) ? sr[(size_t)row * ld + c] * sc : 0.f;
    }
    uint32_t hi[4], lo[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) tc::split2(v[2 * i], v[2 * i + 1], hi[i], lo[i]);
    uint8_t *d = dst + (size_t)m * dst_stride + ((size_t)(row >> 7) * ks + (g >> 1)) * 8192 + (size_t)((row & 127) >> 3) * 256 +
                 (g & 1) * 128 + (row & 7) * 16;
    *reinterpret_cast<uint4 *>(d) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
    *reinterpret_cast<uint4 *>(d + 4096) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
}

// scale[2 z] = 2^(kGradExp - e) with 2^e <= max |.| < 2^(e+1) over the parts of weight set z's members of g (n values per
// member) and g2 (optional, n2 values per member); 1 for an all-zero or non-finite set; scale[2 z + 1] = 1 / scale[2 z].
// kGradExp: the adjoint shrinks layer by layer (~0.3x per 512-wide layer at initialisation), and an fp16 hi | lo pair only
// keeps its 22 bits while |x| >= 2^-3 (below that lo is subnormal): the top of the chain starts at 2^10 so that d_0 is still
// in that range, which leaves 2^5 of headroom below the fp16 maximum for an adjoint that grows instead.  One block per set.
constexpr int kGradExp = 10;
__global__ void grad_scale_kernel(const float *__restrict__ g, long long n, const float *__restrict__ g2, long long n2, int n_symm,
                                  float *__restrict__ scale)
{
    __shared__ float red[32];
    const int z = blockIdx.x;
    const SetMembers sm = set_members(z, n_symm);
    float m = 0.f;
    for (int k = 0; k < sm.count; ++k) {
        const float *a = g + (size_t)(sm.first + k) * n, *b = g2 + (size_t)(sm.first + k) * n2;
        for (long long i = threadIdx.x; i < n; i += blockDim.x) m = fmaxf(m, fabsf(a[i]));
        for (long long i = threadIdx.x; i < n2; i += blockDim.x) m = fmaxf(m, fabsf(b[i]));
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < (int)(blockDim.x >> 5); ++w) m = fmaxf(m, red[w]);
        const int e = (m > 0.f && isfinite(m)) ? max(-100, min(100, ilogbf(m))) - kGradExp : 0;
        scale[2 * z] = ldexpf(1.0f, -e);
        scale[2 * z + 1] = ldexpf(1.0f, e);
    }
}

// out[m][q][c] = scale[2 set(m) + 1] * (sum over the rows of (m, q) of the packed X[row][c]), in a fixed order.  grid (k-steps,
// queries, members), 256 threads = 16 columns x 16 row lanes.
__global__ void __launch_bounds__(256) query_sums_kernel(const uint8_t *__restrict__ X, int ks, long long stride, long long n_points,
                                                         int n_queries, int n_cols, const float *__restrict__ scale, int n_symm,
                                                         float *__restrict__ out)
{
    __shared__ float part[16][17];
    const int c = threadIdx.x & 15, rl = threadIdx.x >> 4, j = blockIdx.x, q = blockIdx.y, m = blockIdx.z;
    const uint8_t *Xm = X + (size_t)m * stride;
    const long long r1 = (long long)(q + 1) * n_points;
    float s = 0.f;
    for (long long r = (long long)q * n_points + rl; r < r1; r += 16) {
        const uint8_t *p = Xm + ((size_t)(r >> 7) * ks + j) * 8192 + (size_t)((r & 127) >> 3) * 256 + (c >> 3) * 128 + (r & 7) * 16 + (c & 7) * 2;
        s += __half2float(*reinterpret_cast<const __half *>(p)) + __half2float(*reinterpret_cast<const __half *>(p + 4096));
    }
    part[rl][c] = s;
    __syncthreads();
    if (rl == 0 && j * 16 + c < n_cols) {
        float t = 0.f;
        for (int i = 0; i < 16; ++i) t += part[i][c];
        out[((size_t)m * n_queries + q) * n_cols + j * 16 + c] = t * scale[2 * member_set(m, n_symm) + 1];
    }
}

// out[z][c] = sum over the members of weight set z (in order) and their queries of sums[m][q][c]  (bias gradient); grid
// (column blocks, sets)
__global__ void sum_queries_kernel(const float *__restrict__ sums, int n_queries, int n, int n_symm, float *__restrict__ out)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x, z = blockIdx.y;
    if (c >= n) return;
    const SetMembers sm = set_members(z, n_symm);
    float t = 0.f;
    for (int k = 0; k < sm.count; ++k)
        for (int q = 0; q < n_queries; ++q) t += sums[((size_t)(sm.first + k) * n_queries + q) * n + c];
    out[(size_t)z * n + c] = t;
}

// per-query condition columns of layer 0 / skip of weight set z:
//   dW[z][n][c0 + j] = (j < nd ? dW[z][n][c0 + j] : 0) + scale * sum over set z's members m and queries q of sums[m][q][n] cond[m][q][j]
// (the first nd columns already hold the noise part from the GEMM); grid (blocks of N x cond_dim, sets)
__global__ void cond_outer_kernel(const float *__restrict__ sums, const float *__restrict__ cond, int n_queries, int N, int cond_dim,
                                  int nd, int n_symm, float scale, float *__restrict__ dW, int ldw, long long w_stride, int c0)
{
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int z = blockIdx.y;
    if (idx >= (long long)N * cond_dim) return;
    const int n = (int)(idx / cond_dim), j = (int)(idx % cond_dim);
    const SetMembers sm = set_members(z, n_symm);
    float t = 0.f;
    for (int k = 0; k < sm.count; ++k)
        for (int q = 0; q < n_queries; ++q) {
            const size_t mq = (size_t)(sm.first + k) * n_queries + q;
            t = fmaf(sums[mq * N + n], cond[mq * cond_dim + j], t);
        }
    float *w = dW + (size_t)z * w_stride + (size_t)n * ldw + c0 + j;
    *w = (j < nd ? *w : 0.f) + scale * t;
}

// what the gradients of one layer read from the forward, and the caller's outputs; member strides in bytes
struct GradTargets {
    const float *cond = nullptr;                       // [members][queries][cond_dim]
    const uint8_t *in[kMaxLayers] = {};                // the input of layer l, packed (layer 0: [xyz | noise])
    int ks_in[kMaxLayers] = {};
    long long s_in[kMaxLayers] = {};
    const uint8_t *D2[kMaxLayers] = {}, *H2[kMaxLayers] = {};   // optional second operand pair of dW_l (H2: k-steps and
    long long sD2[kMaxLayers] = {};                             // member stride of `in`)
    int n_queries = 0, nd = 0;
    long long n_points = 0;
    const float *gs = nullptr;                         // [scale, 1 / scale] of the adjoints, per weight set
    float *const *grad_w = nullptr, *const *grad_b = nullptr;
    bool want_cond = false;
};

// the targets of a forward in the training layout L
static GradTargets targets(const StackDims &s, const Layout &L, const uint8_t *ws, int n_queries, long long n_points, int nd,
                           const float *gs)
{
    GradTargets g;
    g.cond = reinterpret_cast<const float *>(ws + L.cond);
    for (int l = 0; l < s.n_lin; ++l) {
        g.in[l] = l == 0 ? ws + L.x0p : ws + L.hp[l - 1];
        g.ks_in[l] = l == 0 ? L.ks_x0 : L.ks_h[l - 1];
    }
    g.n_queries = n_queries; g.nd = nd; g.n_points = n_points;
    g.gs = gs;
    return g;
}

// weight, bias and condition-column gradients of layer l of every weight set from its pre-activation adjoint d (packed,
// scaled by the set's gs[2 set]); with D2[l]: + D2^T H2 in the weight gradient (a second operand pair over the same rows)
static int layer_grads(const Stack &k, const GradTargets &g, int l, const Adjoint &d, cudaStream_t stream)
{
    PackedChain &c = k.c;
    const StackDims &s = k.s;
    const Members &mb = k.m;
    const long long M = (long long)g.n_queries * g.n_points;
    const int nd = g.nd;
    float *gw = g.grad_w ? g.grad_w[l] : nullptr, *gb = g.grad_b ? g.grad_b[l] : nullptr;
    const bool cond_layer = l == 0 || l == s.skip;
    const float sc = l == s.skip ? chain::kInvSqrt2 : 1.0f;
    const long long wstride = (long long)s.N[l] * s.in_total[l];
    if (gw) {
        const int K = l == 0 ? 3 + nd : l == s.skip ? s.N[l - 1] + 3 + nd : s.N[l - 1];
        int r = wgrad::launch_sets(d.packed, d.ks, g.in[l], g.ks_in[l], M, s.N[l], K, sc, g.gs + 1, 2, gw, s.in_total[l], wstride,
                                   mb.sets, mb.n_symm, d.stride, g.s_in[l], g.sD2[l], g.s_in[l], c.partials, stream, g.D2[l], g.H2[l]);
        if (r) return r;
    }
    float *sums = l == 0 ? c.sums0.as<float>() : l == s.skip ? c.sumss.as<float>() : c.sums.as<float>();
    if (gb || (cond_layer && (gw || g.want_cond))) {
        query_sums_kernel<<<dim3((unsigned)d.ks, (unsigned)g.n_queries, (unsigned)mb.count), 256, 0, stream>>>(
            d.packed, d.ks, d.stride, g.n_points, g.n_queries, s.N[l], g.gs, mb.n_symm, sums);
        NPHM_CUDA_CHECK(cudaGetLastError());
    }
    if (gb) {
        sum_queries_kernel<<<dim3((unsigned)ceil_div(s.N[l], 128), (unsigned)mb.sets), 128, 0, stream>>>(sums, g.n_queries, s.N[l],
                                                                                                          mb.n_symm, gb);
        NPHM_CUDA_CHECK(cudaGetLastError());
    }
    if (cond_layer && gw) {
        const long long total = (long long)s.N[l] * s.cond_dim;
        cond_outer_kernel<<<dim3((unsigned)ceil_div(total, 256), (unsigned)mb.sets), 256, 0, stream>>>(
            sums, g.cond, g.n_queries, s.N[l], s.cond_dim, nd, mb.n_symm, sc, gw, s.in_total[l], wstride,
            l == 0 ? 3 : s.N[l - 1] + 3);
        NPHM_CUDA_CHECK(cudaGetLastError());
    }
    return NPHM_OK;
}

// the per-(member, query) column sums the layer gradients and cond_grad use
static int reserve_sums(const Stack &k, int n_queries)
{
    const StackDims &s = k.s;
    int max_n = 1, rc;
    for (int l = 0; l < s.n_lin; ++l) max_n = std::max(max_n, s.N[l]);
    const size_t mq = (size_t)k.m.count * n_queries;
    if ((rc = k.c.sums.reserve(mq * max_n * sizeof(float))) || (rc = k.c.sums0.reserve(mq * s.N[0] * sizeof(float))) ||
        (rc = k.c.sumss.reserve(mq * s.N[s.skip] * sizeof(float))))
        return rc;
    return NPHM_OK;
}

// the training variants of layers 0, skip - 1 and skip for nd > 0 noise columns (without noise, fwd is used as it is)
static int pack(nphm_mlp *h, int nd, cudaStream_t stream)
{
    MlpChain &c = *h->chain;
    const StackDims &s = h->dims;
    if (nd == 0 || c.train_nd == nd) return NPHM_OK;
    for (int l = 0; l < s.n_lin; ++l) {
        if (!noise_layer(s, l)) continue;
        const int K = l == 0 ? 3 + nd : l == s.skip ? s.N[l - 1] + 3 + nd : s.K[l];
        int rc = c.tfwd[l].pack(h->weights.W[l].as<float>(), s.in_total[l], s.N[l], K, 0, 0, false,
                                l == s.skip ? chain::kInvSqrt2 : 1.0f, stream, 1, 0, nullptr, 0, l + 1 == s.skip ? 3 + nd : 0, kChainNt);
        if (rc) return rc;
    }
    c.train_nd = nd;
    return NPHM_OK;
}

}  // namespace train
}  // namespace nphm

extern "C" long long nphm_mlp_train_workspace_bytes(const nphm_mlp *h, int n_queries, long long n_points, int noise_dim)
{
    if (!h || !h->loaded || n_queries < 1 || n_points < 1 || noise_dim < 0 || noise_dim > h->dims.cond_dim) {
        set_error("nphm_mlp_train_workspace_bytes: bad arguments");
        return -1;
    }
    return (long long)train::layout(h->dims, n_queries, n_points, noise_dim).total;
}

extern "C" int nphm_mlp_train_forward(nphm_mlp *h, const float *xyz_dev, const float *cond_dev, const float *cond_noise_dev,
                                      int noise_dim, int n_queries, long long n_points, float *out_dev, void *workspace_dev,
                                      void *stream_)
{
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    int rc = chain_ready(h, "nphm_mlp_train_forward");
    if (rc) return rc;
    NPHM_REQUIRE(n_queries >= 1 && n_points >= 1 && xyz_dev && cond_dev && out_dev && workspace_dev,
                 "nphm_mlp_train_forward: bad arguments");
    NPHM_REQUIRE(noise_dim >= 0 && noise_dim <= h->dims.cond_dim && (noise_dim == 0 || cond_noise_dev),
                 "nphm_mlp_train_forward: noise_dim %d out of range [0, %d] or no noise given", noise_dim, h->dims.cond_dim);
    const StackDims &s = h->dims;
    const train::Layout L = train::layout(s, n_queries, n_points, noise_dim);
    uint8_t *ws = static_cast<uint8_t *>(workspace_dev);
    const long long M = (long long)n_queries * n_points;
    if ((rc = train::pack(h, noise_dim, stream))) return rc;
    if ((rc = mlp_prepare(h, cond_dev, n_queries, stream))) return rc;
    float *X0 = reinterpret_cast<float *>(ws + L.x0);
    train::stage_x0_kernel<<<(unsigned)ceil_div(M * L.ldx, 256), 256, 0, stream>>>(xyz_dev, cond_noise_dev, noise_dim, M, L.ldx, X0);
    NPHM_CUDA_CHECK(cudaGetLastError());
    train::pack_rows_kernel<<<(unsigned)ceil_div(ceil_div(M, 128) * 128 * 2 * L.ks_x0, 256), 256, 0, stream>>>(
        X0, L.ldx, 3 + noise_dim, M, L.ks_x0, 0, nullptr, 0, ws + L.x0p, 0);
    NPHM_CUDA_CHECK(cudaGetLastError());
    NPHM_CUDA_CHECK(cudaMemcpyAsync(ws + L.cond, cond_dev, (size_t)n_queries * s.cond_dim * sizeof(float), cudaMemcpyDeviceToDevice,
                                    stream));
    ValueRows v;
    v.X = X0; v.ldx = L.ldx; v.nd = noise_dim; v.tfwd = h->chain->tfwd;
    v.bias = h->cvec.as<float>(); v.rows_per_bias = n_points;
    for (int l = 0; l + 1 < s.n_lin; ++l) { v.Hp[l] = ws + L.hp[l]; v.S[l] = reinterpret_cast<float *>(ws + L.s[l]); }
    v.out = out_dev;
    return value_layers(stack(h), M, v, stream);
}

extern "C" int nphm_mlp_train_backward(nphm_mlp *h, const float *grad_out_dev, const void *workspace_dev,
                                       long long workspace_bytes, int nd, int n_queries, long long n_points, float *const *grad_w_dev, float *const *grad_b_dev, float *grad_cond_dev,
                                       float *grad_xyz_dev, void *stream_)
{
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    int rc = chain_ready(h, "nphm_mlp_train_backward");
    if (rc) return rc;
    NPHM_REQUIRE(n_queries >= 1 && n_points >= 1 && grad_out_dev && workspace_dev, "nphm_mlp_train_backward: bad arguments");
    MlpChain &c = *h->chain;
    const StackDims &s = h->dims;
    const uint8_t *ws = static_cast<const uint8_t *>(workspace_dev);
    // the caller states the shape the workspace was made for; checked against its size, without reading it back
    NPHM_REQUIRE(nd >= 0 && nd <= s.cond_dim && workspace_bytes == (long long)train::layout(s, n_queries, n_points, nd).total,
                 "nphm_mlp_train_backward: a workspace of %lld bytes does not hold a training forward of this network at %d x %lld "
                 "points with %d noise columns", workspace_bytes, n_queries, n_points, nd);
    const train::Layout L = train::layout(s, n_queries, n_points, nd);
    const Stack k = stack(h);
    const long long M = (long long)n_queries * n_points;
    const int last = s.n_lin - 1, out_dim = s.N[last];

    // upstream gradient scaled by 2^-e into the packed d_L
    if ((rc = c.gscale.reserve(2 * sizeof(float)))) return rc;
    const float *gs = c.gscale.as<float>();
    train::grad_scale_kernel<<<1, 1024, 0, stream>>>(grad_out_dev, M * out_dim, nullptr, 0, 0, c.gscale.as<float>());
    NPHM_CUDA_CHECK(cudaGetLastError());
    const int ks_out = (out_dim + 15) / 16;
    if ((rc = c.Dl.reserve(packed_bytes(M, ks_out)))) return rc;
    train::pack_rows_kernel<<<(unsigned)ceil_div(ceil_div(M, 128) * 128 * 2 * ks_out, 256), 256, 0, stream>>>(
        grad_out_dev, out_dim, out_dim, M, ks_out, 0, gs, 0, c.Dl.as<uint8_t>(), 0);
    NPHM_CUDA_CHECK(cudaGetLastError());

    int max_ks = 1;
    for (int l = 1; l <= last; ++l) max_ks = std::max(max_ks, (s.N[l - 1] + 15) / 16);
    for (int i = 0; i < 2; ++i)
        if ((rc = c.Dp[i].reserve(packed_bytes(M, max_ks)))) return rc;
    if ((rc = train::reserve_sums(k, n_queries))) return rc;
    if (grad_xyz_dev && ((rc = c.xtmp.reserve((size_t)M * 4 * sizeof(float))) || (rc = c.xs_tmp.reserve((size_t)M * 4 * sizeof(float)))))
        return rc;

    train::GradTargets tg = train::targets(s, L, ws, n_queries, n_points, nd, gs);
    tg.grad_w = grad_w_dev; tg.grad_b = grad_b_dev; tg.want_cond = grad_cond_dev != nullptr;
    auto layer_grads = [&](int l, const Adjoint &d) { return train::layer_grads(k, tg, l, d, stream); };

    // d_L in Dl, d_l in Dp[l & 1]
    AdjointWalk w;
    w.top = Adjoint{nullptr, 0, c.Dl.as<uint8_t>(), ks_out, 0};
    for (int l = 0; l < last; ++l) { w.S[l] = reinterpret_cast<const float *>(ws + L.s[l]); w.D[l] = c.Dp[l & 1].as<uint8_t>(); }
    w.xs = grad_xyz_dev ? c.xs_tmp.as<float>() : nullptr;
    if ((rc = adjoint_walk(k, M, w, layer_grads, stream))) return rc;
    // the noise does not change the gradient with respect to the condition; one chunk: a fixed summation order
    if (grad_cond_dev && (rc = cond_grad(k, n_queries, 1, grad_cond_dev, stream))) return rc;
    if (grad_xyz_dev && (rc = xyz_grad(k, M, w.D[0], 0, c.xtmp.as<float>(), w.xs, gs, 2, grad_xyz_dev, stream))) return rc;
    return NPHM_OK;
}

// ================================================================================================ training through grad_x sdf
// Stage 1 of the reference (scripts/training/train.py -> actual_compute_loss, src/NPHM/models/loss_functions.py:20-110)
// reaches a DeepSDF decoder through s = f(x) and g = grad_x s.  With upstream gradients s_bar, g_bar per row,
//   dL/dtheta = s_bar ds/dtheta + d/dtheta (g_bar . grad_x s),
// and the second term is the gradient of a forward-mode tangent in the direction v = g_bar.  With z_l = W_l h_{l-1} + b_l,
// h_l = softplus_100(z_l), S_l = sigmoid(100 z_l) (kept by the value pass) and softplus'' = 100 S (1 - S):
//   forward   value pass (keeps h_l packed, S_l blocked), then the adjoint with unit upstream  a_L = 1,
//             a_l = S_l * (W_{l+1}^T a_{l+1}) (kept packed): its bottom gives g through W_0[:, 0:3] and the skip's xyz columns
//   backward  tangent pass  zt_l = W_l ht_{l-1}, ht_l = S_l * zt_l  (ht_{-1} = v; v appended at the skip)
//             value adjoint zb_L = s_bar,  zb_l = S_l * (W_{l+1}^T zb_{l+1}) + 100 (1 - S_l) * zt_l * a_l
//             dW_l = zb_l^T h_{l-1} + a_l^T ht_{l-1} (one GEMM over both pairs), db_l = sum zb_l, condition and xyz as the
//             first-order backward does from zb
// fp16 range: a starts at 2^kGradExp (the unit column), so it spends the chain where an fp16 hi | lo pair keeps its bits;
// s_bar and g_bar (~1e-5 at the NPM batch) share one device-side power of two sigma per weight set that brings their largest
// magnitude to 2^kGradExp (grad_scale_kernel over both).  The direction is v' = sigma 2^-kGradExp g_bar, so zt' a' and a' ht'
// carry the same scale sigma as zb': the coupling keeps its plain coefficient 100 and the GEMM adds the two pairs as they are;
// the fp32 epilogues multiply by 1 / sigma.
// Members: the passes run for every member at once (Members), one launch per pass.  A DeepSDF handle is the one-member case;
// the NPHM ensemble (reference train.py -local) runs its 40 members, each on B queries of N points in its own frame.  A
// weight set gets its own sigma: through the blend weights, its members' s_bar and g_bar can differ by orders of magnitude
// from the other sets'; an all-zero set gets scale 1 and exactly zero gradients.
// Memory: everything per row lives in the caller's workspace, the backward's scratch included (its tail: the tangents, the
// adjoint ping-pong, the direction), so it is counted and released by the caller's allocator; the handle keeps only
// buffers of the layer widths (GEMM partials, per-query sums).
namespace nphm {
namespace sdfgrad {

// workspace of one forward and its backward: the per-(member, query) folded constants (cvec, when they do not live on the
// handle) and condition, one scale pair per weight set (gs) and the forward's (consts), the packed xyz rows (x0p), h_l
// packed, s_l blocked, the unit column and a_l; then the scratch of the backward: ht_l packed (tg) and zt_l blocked fp32
// (zg), the ping-pong of zb (dp), zb_L (dl), the direction as rows of 4 (v4) and packed (vp), and two [M][4] point-gradient
// temporaries (xa, xb).  Every per-row piece holds a whole number of 128-row tiles per member; m_* are the member strides
// (bytes).
struct Layout {
    size_t cvec = 0, cond = 0, gs = 0, consts = 0, x0p = 0, hp[kMaxLayers] = {}, s[kMaxLayers] = {}, unit = 0, a[kMaxLayers] = {};
    size_t tg[kMaxLayers] = {}, zg[kMaxLayers] = {}, dp[2] = {}, dl = 0, vp = 0, v4 = 0, xa = 0, xb = 0, total = 0;
    long long m_hp[kMaxLayers] = {}, m_s[kMaxLayers] = {}, m_a[kMaxLayers] = {}, m_dp = 0, m_one = 0, m_row4 = 0;
    int ks_h[kMaxLayers] = {}, ks_a[kMaxLayers] = {}, ks_dp = 1;
};

static Layout layout(const StackDims &s, const Members &mb, int n_queries, long long n_points, bool with_cvec)
{
    const int K = mb.count;
    const long long Mm = (long long)n_queries * n_points, T = ceil_div(Mm, 128);
    Layout G;
    Carver w;
    G.cvec = w.take(with_cvec ? (size_t)K * n_queries * s.cvec_stride * sizeof(float) : 0);
    G.cond = w.take((size_t)K * n_queries * s.cond_dim * sizeof(float));
    G.gs = w.take((size_t)mb.sets * 2 * sizeof(float));
    G.consts = w.take(2 * sizeof(float));
    G.m_one = T * 8192;
    G.m_row4 = Mm * 4 * sizeof(float);
    G.x0p = w.take((size_t)K * G.m_one);
    for (int l = 0; l + 1 < s.n_lin; ++l) {
        G.ks_h[l] = (s.N[l] + (l + 1 == s.skip ? 3 : 0) + 15) / 16;
        G.ks_a[l] = (s.N[l] + 15) / 16;
        G.ks_dp = std::max(G.ks_dp, G.ks_a[l]);
        G.m_hp[l] = T * G.ks_h[l] * 8192;
        G.m_s[l] = T * 128 * pad4(s.N[l]) * sizeof(float);
        G.m_a[l] = T * G.ks_a[l] * 8192;
        G.hp[l] = w.take((size_t)K * G.m_hp[l]);
        G.s[l] = w.take((size_t)K * G.m_s[l]);
        G.a[l] = w.take((size_t)K * G.m_a[l]);
        G.tg[l] = w.take((size_t)K * G.m_hp[l]);
        G.zg[l] = w.take((size_t)K * G.m_s[l]);
    }
    G.m_dp = T * G.ks_dp * 8192;
    G.unit = w.take((size_t)K * G.m_one);
    for (int i = 0; i < 2; ++i) G.dp[i] = w.take((size_t)K * G.m_dp);
    G.dl = w.take((size_t)K * G.m_one);
    G.vp = w.take((size_t)K * G.m_one);
    G.v4 = w.take((size_t)K * G.m_row4);
    G.xa = w.take((size_t)K * G.m_row4);
    G.xb = w.take((size_t)K * G.m_row4);
    G.total = w.off;
    return G;
}

// row r of a packed one-column operand (1 k-step): column 0 = v (the fp16 hi part; lo 0), columns 1 .. 15 = 0
__device__ __forceinline__ void store_column0(uint8_t *__restrict__ dst, long long r, float v)
{
    const uint32_t w0 = (uint32_t)__half_as_ushort(__float2half_rn(v));
    uint8_t *d = dst + (size_t)(r >> 7) * 8192 + (size_t)((r & 127) >> 3) * 256 + (r & 7) * 16;
    *reinterpret_cast<uint4 *>(d) = make_uint4(w0, 0, 0, 0);
    *reinterpret_cast<uint4 *>(d + 128) = make_uint4(0, 0, 0, 0);
    *reinterpret_cast<uint4 *>(d + 4096) = make_uint4(0, 0, 0, 0);
    *reinterpret_cast<uint4 *>(d + 4096 + 128) = make_uint4(0, 0, 0, 0);
}

// packed one-column operand of every member (member m at dst + m stride): column 0 = 2^kGradExp on the rows < M, everything
// else 0; consts = {2^E, 2^-E}.  grid (row blocks of the padded tiles, members), thread = row.
__global__ void unit_column_kernel(long long M, uint8_t *__restrict__ dst, long long stride, float *__restrict__ consts)
{
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r == 0 && blockIdx.y == 0) { consts[0] = ldexpf(1.0f, train::kGradExp); consts[1] = ldexpf(1.0f, -train::kGradExp); }
    if (r >= (M + 127) / 128 * 128) return;
    store_column0(dst + (size_t)blockIdx.y * stride, r, r < M ? ldexpf(1.0f, train::kGradExp) : 0.f);
}

// V[m][r] = (g_bar[m][r] * scale[2 set(m)] * 2^-kGradExp, 0): the tangent direction, ld 4
__global__ void direction_kernel(const float *__restrict__ gg, long long M, int members, const float *__restrict__ scale, int n_symm,
                                 float *__restrict__ V)
{
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)members * M * 4) return;
    const long long r = idx >> 2;
    const int c = (int)(idx & 3), m = (int)(r / M);
    V[idx] = c < 3 ? gg[r * 3 + c] * (scale[2 * member_set(m, n_symm)] * ldexpf(1.0f, -train::kGradExp)) : 0.f;
}

static int ready(nphm_mlp *h, const char *who)
{
    int rc = chain_ready(h, who);
    if (rc) return rc;
    if (h->dims.N[h->dims.n_lin - 1] != 1) {
        set_error("%s: needs a stack with one output (an SDF), this one has %d", who, h->dims.N[h->dims.n_lin - 1]);
        return NPHM_ERR_UNSUPPORTED;
    }
    return NPHM_OK;
}

// s and g = grad_x s of every member at xyz [members][B][N][3]; cond [members][B][cond_dim], cvec the folded constants
// [members][B][cvec_stride]
static int forward(const Stack &k, const Layout &G, const float *xyz, const float *cond, const float *cvec, int n_queries,
                   long long n_points, float *sdf_out, float *grad_out, uint8_t *ws, cudaStream_t stream)
{
    const StackDims &s = k.s;
    const int K = k.m.count;
    const long long M = (long long)n_queries * n_points, T = ceil_div(M, 128);
    NPHM_CUDA_CHECK(cudaMemcpyAsync(ws + G.cond, cond, (size_t)K * n_queries * s.cond_dim * sizeof(float), cudaMemcpyDeviceToDevice,
                                    stream));
    train::pack_rows_kernel<<<dim3((unsigned)ceil_div(T * 128 * 2, 256), (unsigned)K), 256, 0, stream>>>(
        xyz, 3, 3, M, 1, M * 3, nullptr, k.m.n_symm, ws + G.x0p, G.m_one);
    NPHM_CUDA_CHECK(cudaGetLastError());
    // value pass: h_l packed, S_l blocked; the output layer writes s row-major
    ValueRows v;
    v.X = xyz; v.sX = M * 3;
    v.bias = cvec; v.rows_per_bias = n_points; v.sBias = (long long)n_queries * s.cvec_stride;
    for (int l = 0; l + 1 < s.n_lin; ++l) {
        v.Hp[l] = ws + G.hp[l]; v.sHp[l] = G.m_hp[l];
        v.S[l] = reinterpret_cast<float *>(ws + G.s[l]); v.sS[l] = G.m_s[l] / 4;
    }
    v.out = sdf_out; v.sOut = M;
    int rc;
    if ((rc = value_layers(k, M, v, stream))) return rc;
    float *consts = reinterpret_cast<float *>(ws + G.consts);
    unit_column_kernel<<<dim3((unsigned)ceil_div(T * 128, 256), (unsigned)K), 256, 0, stream>>>(M, ws + G.unit, G.m_one, consts);
    NPHM_CUDA_CHECK(cudaGetLastError());
    // a_{l-1} = S_{l-1} * (a_l W_l) from the unit column down to a_0, kept in the workspace
    AdjointWalk w;
    w.top = Adjoint{nullptr, 0, ws + G.unit, 1, G.m_one};
    for (int l = 0; l + 1 < s.n_lin; ++l) { w.S[l] = v.S[l]; w.sS[l] = v.sS[l]; w.D[l] = ws + G.a[l]; w.sD[l] = G.m_a[l]; }
    w.xs = reinterpret_cast<float *>(ws + G.xb);
    if ((rc = adjoint_walk(k, M, w, [](int, const Adjoint &) { return NPHM_OK; }, stream))) return rc;
    return xyz_grad(k, M, w.D[0], w.sD[0], reinterpret_cast<float *>(ws + G.xa), w.xs, consts, 0, grad_out, stream);
}

// weight, bias, condition and point gradients of every member from s_bar [members][B][N] and g_bar [members][B][N][3]
static int backward(const Stack &k, const Layout &G, const float *grad_sdf, const float *grad_grad, uint8_t *ws, int n_queries,
                    long long n_points, float *const *grad_w, float *const *grad_b, float *grad_cond, float *grad_xyz,
                    cudaStream_t stream)
{
    const StackDims &s = k.s;
    const Members &mb = k.m;
    const int K = mb.count, last = s.n_lin - 1;
    const long long M = (long long)n_queries * n_points, T = ceil_div(M, 128);
    float *const gs = reinterpret_cast<float *>(ws + G.gs), *const v4 = reinterpret_cast<float *>(ws + G.v4);
    float *const xa = reinterpret_cast<float *>(ws + G.xa), *const xb = reinterpret_cast<float *>(ws + G.xb);

    // one power of two per weight set for both upstream gradients; zb_L = s_bar packed, the direction as rows and packed
    train::grad_scale_kernel<<<mb.sets, 1024, 0, stream>>>(grad_sdf, M, grad_grad, M * 3, mb.n_symm, gs);
    NPHM_CUDA_CHECK(cudaGetLastError());
    const dim3 pack_grid((unsigned)ceil_div(T * 128 * 2, 256), (unsigned)K);
    train::pack_rows_kernel<<<pack_grid, 256, 0, stream>>>(grad_sdf, 1, 1, M, 1, M, gs, mb.n_symm, ws + G.dl, G.m_one);
    NPHM_CUDA_CHECK(cudaGetLastError());
    direction_kernel<<<(unsigned)ceil_div(K * M * 4, 256), 256, 0, stream>>>(grad_grad, M, K, gs, mb.n_symm, v4);
    NPHM_CUDA_CHECK(cudaGetLastError());
    train::pack_rows_kernel<<<pack_grid, 256, 0, stream>>>(v4, 4, 3, M, 1, M * 4, nullptr, mb.n_symm, ws + G.vp, G.m_one);
    NPHM_CUDA_CHECK(cudaGetLastError());

    // tangent pass: ht_l packed (tg, the next layer's input and the GEMM's second H), zt_l blocked fp32 (zg)
    int rc;
    for (int l = 0; l < last; ++l) {
        const tcl::PackedLinear &W = k.c.fwd[l];
        tcl::LinearParams p;
        p.M = M; p.batch = K; p.w_pairs = mb.n_symm;
        if (l == 0) { p.A1 = v4; p.lda1 = 4; p.K1 = 3; p.sA1 = M * 4; }
        else { p.Ap = ws + G.tg[l - 1]; p.a_ksteps = W.ksteps; p.sAp = G.m_hp[l - 1]; }
        p.mode = tcl::kModeMult;
        p.Mul = reinterpret_cast<const float *>(ws + G.s[l]); p.ldmul = k.c.ld[l]; p.mul_div = 1; p.mul_blocked = 1; p.sMul = G.m_s[l] / 4;
        p.Cp = ws + G.tg[l]; p.c_ksteps = G.ks_h[l]; p.sCp = G.m_hp[l];
        if (l + 1 == s.skip) { p.app = v4; p.app_ld = 4; p.app_w = 3; p.sApp = M * 4; }
        p.Dv = reinterpret_cast<float *>(ws + G.zg[l]); p.lddv = k.c.ld[l]; p.dv_blocked = 1; p.sDv = G.m_s[l] / 4;
        if ((rc = tcl::launch_linear(W, p, stream))) return rc;
    }

    if ((rc = train::reserve_sums(k, n_queries))) return rc;
    // dW_l = zb_l^T h_{l-1} + a_l^T ht_{l-1}  (a_L: the unit column, ht_{-1}: the direction)
    train::GradTargets g;
    g.cond = reinterpret_cast<const float *>(ws + G.cond);
    for (int l = 0; l <= last; ++l) {
        g.in[l] = l == 0 ? ws + G.x0p : ws + G.hp[l - 1];
        g.ks_in[l] = l == 0 ? 1 : G.ks_h[l - 1];
        g.s_in[l] = l == 0 ? G.m_one : G.m_hp[l - 1];
        g.D2[l] = l == last ? ws + G.unit : ws + G.a[l];
        g.sD2[l] = l == last ? G.m_one : G.m_a[l];
        g.H2[l] = l == 0 ? ws + G.vp : ws + G.tg[l - 1];
    }
    g.n_queries = n_queries; g.n_points = n_points;
    g.gs = gs;
    g.grad_w = grad_w; g.grad_b = grad_b; g.want_cond = grad_cond != nullptr;
    auto layer_grads = [&](int l, const Adjoint &d) { return train::layer_grads(k, g, l, d, stream); };

    // value adjoint with the coupling, from zb_L = s_bar (in dl) down to zb_0; zb_l lives in dp[l & 1]
    AdjointWalk w;
    w.top = Adjoint{nullptr, 0, ws + G.dl, 1, G.m_one};
    for (int l = 0; l < last; ++l) {
        w.S[l] = reinterpret_cast<const float *>(ws + G.s[l]); w.sS[l] = G.m_s[l] / 4;
        w.D[l] = ws + G.dp[l & 1]; w.sD[l] = G.m_dp;
        w.cpl_z[l] = reinterpret_cast<const float *>(ws + G.zg[l]);
        w.cpl_a[l] = ws + G.a[l]; w.sA[l] = G.m_a[l];
    }
    w.xs = grad_xyz ? xb : nullptr;
    if ((rc = adjoint_walk(k, M, w, layer_grads, stream))) return rc;
    if (grad_cond && (rc = cond_grad(k, n_queries, 1, grad_cond, stream))) return rc;
    // s_bar g + H v: the point gradient of zb, as in the first-order backward
    if (grad_xyz && (rc = xyz_grad(k, M, w.D[0], w.sD[0], xa, xb, gs, 2, grad_xyz, stream))) return rc;
    return NPHM_OK;
}

}  // namespace sdfgrad
}  // namespace nphm

extern "C" long long nphm_mlp_sdfgrad_workspace_bytes(const nphm_mlp *h, int n_queries, long long n_points)
{
    if (!h || !h->loaded || n_queries < 1 || n_points < 1) {
        set_error("nphm_mlp_sdfgrad_workspace_bytes: bad arguments");
        return -1;
    }
    return (long long)sdfgrad::layout(h->dims, Members{}, n_queries, n_points, false).total;
}

extern "C" int nphm_mlp_sdfgrad_forward(nphm_mlp *h, const float *xyz_dev, const float *cond_dev, int n_queries, long long n_points,
                                        float *sdf_out_dev, float *grad_out_dev, void *workspace_dev, void *stream_)
{
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    int rc = sdfgrad::ready(h, "nphm_mlp_sdfgrad_forward");
    if (rc) return rc;
    NPHM_REQUIRE(n_queries >= 1 && n_points >= 1 && xyz_dev && cond_dev && sdf_out_dev && grad_out_dev && workspace_dev,
                 "nphm_mlp_sdfgrad_forward: bad arguments");
    const sdfgrad::Layout G = sdfgrad::layout(h->dims, Members{}, n_queries, n_points, false);
    if ((rc = mlp_prepare(h, cond_dev, n_queries, stream))) return rc;
    return sdfgrad::forward(stack(h), G, xyz_dev, cond_dev, h->cvec.as<float>(), n_queries, n_points, sdf_out_dev, grad_out_dev,
                            static_cast<uint8_t *>(workspace_dev), stream);
}

extern "C" int nphm_mlp_sdfgrad_backward(nphm_mlp *h, const float *grad_sdf_dev, const float *grad_grad_dev, void *workspace_dev,
                                         long long workspace_bytes, int n_queries, long long n_points, float *const *grad_w_dev,
                                         float *const *grad_b_dev, float *grad_cond_dev, float *grad_xyz_dev, void *stream_)
{
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    int rc = sdfgrad::ready(h, "nphm_mlp_sdfgrad_backward");
    if (rc) return rc;
    NPHM_REQUIRE(n_queries >= 1 && n_points >= 1 && grad_sdf_dev && grad_grad_dev && workspace_dev,
                 "nphm_mlp_sdfgrad_backward: bad arguments");
    const sdfgrad::Layout G = sdfgrad::layout(h->dims, Members{}, n_queries, n_points, false);
    // the caller states the shape the workspace was made for; checked against its size, without reading it back
    NPHM_REQUIRE(workspace_bytes == (long long)G.total,
                 "nphm_mlp_sdfgrad_backward: a workspace of %lld bytes does not hold an SDF-gradient forward of this network at "
                 "%d x %lld points", workspace_bytes, n_queries, n_points);
    return sdfgrad::backward(stack(h), G, grad_sdf_dev, grad_grad_dev, static_cast<uint8_t *>(workspace_dev), n_queries, n_points,
                             grad_w_dev, grad_b_dev, grad_cond_dev, grad_xyz_dev, stream);
}

// ================================================================================================ fitting a one-output stack
// The surface term of both fitters with a DeepSDF decoder (reference src/NPHM/models/fitting.py:114-125 and :229-247):
//   loss = mean over the kept points of |s|,  kept = mask != 0 and |s| < clamp
// with its gradients w.r.t. the per-query condition (the identity code) and the points.  One value pass (the first-order
// training forward, no noise), one kernel that forms the kept set, counts it, sums |s| in a fixed order and writes the upstream
// sign(s) * kept as the packed output-layer adjoint, then the adjoint chain with the per-query condition sums.
// fp16 range: the true upstream is 1 / n_kept (~2e-4 at 5 x 1000 points) and the adjoint shrinks through eight 1024-wide
// layers; the adjoint starts at +-2^kGradExp like the unit column of the SDF-gradient forward, and the fp32 epilogues multiply
// by 2^-kGradExp / n_kept (0 when nothing is kept, so both gradients are exactly zero then).
// Memory: everything per point lives in the caller's workspace (the training layout, s, the adjoint ping-pong, the point-
// gradient temporaries); the handle keeps only the per-query sums of the layer widths.
namespace nphm {
namespace fitsurf {

constexpr int kThreads = 1024;

struct Layout {
    train::Layout base;
    size_t sdf = 0, dl = 0, consts = 0, dp[2] = {}, xa = 0, xb = 0, total = 0;
    int ks_dp = 1;
};

static Layout layout(const StackDims &s, int n_queries, long long n_points)
{
    Layout F;
    F.base = train::layout(s, n_queries, n_points, 0);
    const size_t M = (size_t)n_queries * n_points, tiles = (size_t)ceil_div((long long)M, 128);
    Carver w{F.base.total};
    F.sdf = w.take(M * sizeof(float));
    F.dl = w.take(tiles * 8192);
    F.consts = w.take(2 * sizeof(float));
    for (int l = 0; l + 1 < s.n_lin; ++l) F.ks_dp = std::max(F.ks_dp, (s.N[l] + 15) / 16);
    for (int i = 0; i < 2; ++i) F.dp[i] = w.take(tiles * F.ks_dp * 8192);
    F.xa = w.take(M * 4 * sizeof(float));
    F.xb = w.take(M * 4 * sizeof(float));
    F.total = w.off;
    return F;
}

// One block per group of `n` consecutive rows (the single call: one group of all rows; the batched call: one group per scan).
// Row r of the padded tiles: column 0 of the packed adjoint = 2^kGradExp sign(s_r) if r is kept, else 0 (sign(0) = 0, as torch's
// abs backward); the last group's block also zeroes the padding rows of the last tile.  A group's n_kept and sum |s| are reduced
// in a fixed order (strided per thread, then a fixed tree), so the call is bitwise deterministic.  Group g writes loss_terms
// [g][8] = [loss, 0, 0, 0, 0, n_kept].  gs = {2^kGradExp, 2^-kGradExp / n_kept} with one group; with per_group the factor is
// the uniform 2^-kGradExp and scan_factor_kernel applies each group's 1 / n_kept after the chain.
__global__ void __launch_bounds__(kThreads) surface_upstream_kernel(const float *__restrict__ sdf, const unsigned char *__restrict__ mask,
                                                                     long long n, float clamp, bool per_group, uint8_t *__restrict__ dst,
                                                                     float *__restrict__ gs, float *__restrict__ loss_terms)
{
    __shared__ float w_sum[kThreads / 32];
    __shared__ int w_cnt[kThreads / 32];
    const float top = ldexpf(1.0f, train::kGradExp);
    float sum = 0.f;
    int cnt = 0;
    const long long r0 = (long long)blockIdx.x * n, r1 = r0 + n;
    const long long rows = blockIdx.x + 1 == gridDim.x ? (r1 + 127) / 128 * 128 : r1;
    for (long long r = r0 + threadIdx.x; r < rows; r += kThreads) {
        float v = 0.f;
        if (r < r1) {
            const float s = sdf[r], a = fabsf(s);
            if ((!mask || mask[r]) && a < clamp) {
                sum += a;
                ++cnt;
                v = s > 0.f ? top : (s < 0.f ? -top : 0.f);
            }
        }
        sdfgrad::store_column0(dst, r, v);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        sum += __shfl_xor_sync(0xffffffffu, sum, o);
        cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    }
    if ((threadIdx.x & 31) == 0) { w_sum[threadIdx.x >> 5] = sum; w_cnt[threadIdx.x >> 5] = cnt; }
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        int k = 0;
        for (int w = 0; w < kThreads / 32; ++w) { t += w_sum[w]; k += w_cnt[w]; }
        if (blockIdx.x == 0) {
            gs[0] = top;
            gs[1] = per_group ? ldexpf(1.0f, -train::kGradExp) : k > 0 ? ldexpf(1.0f, -train::kGradExp) / (float)k : 0.f;
        }
        float *lt = loss_terms + (size_t)blockIdx.x * 8;
        lt[0] = t / (float)k;                           // NaN when nothing is kept, like torch's mean of an empty tensor
        lt[1] = lt[2] = lt[3] = lt[4] = 0.f;
        lt[5] = (float)k;
    }
}

// grad_cond[q] and the rows of query q of grad_xyz (may be NULL) times 1 / n_kept of group q (loss_terms[q][5]; 0 when nothing is
// kept).  grid (blocks over max(cond_dim, 3 n), queries)
__global__ void scan_factor_kernel(const float *__restrict__ loss_terms, int cond_dim, long long n3, float *__restrict__ grad_cond,
                                   float *__restrict__ grad_xyz)
{
    const int q = blockIdx.y;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const float k = loss_terms[(size_t)q * 8 + 5], f = k > 0.f ? 1.0f / k : 0.f;
    if (i < cond_dim) grad_cond[(size_t)q * cond_dim + i] *= f;
    if (grad_xyz && i < n3) grad_xyz[(size_t)q * n3 + i] *= f;
}

// The surface term of one loss over all queries (per_query false) or of one loss per query (per_query: query q = scan q).
static int surface_grad(nphm_mlp *h, const float *xyz_dev, const float *cond_dev, int n_queries, long long n_points,
                        const unsigned char *mask_dev, float clamp, bool per_query, float *loss_terms_dev, float *grad_cond_dev,
                        float *grad_xyz_dev, void *workspace_dev, long long workspace_bytes, void *stream_, const char *who)
{
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    int rc = sdfgrad::ready(h, who);
    if (rc) return rc;
    NPHM_REQUIRE(n_queries >= 1 && n_points >= 1 && xyz_dev && cond_dev && loss_terms_dev && grad_cond_dev && workspace_dev,
                 "%s: bad arguments", who);
    const StackDims &s = h->dims;
    const Layout F = layout(s, n_queries, n_points);
    NPHM_REQUIRE(workspace_bytes == (long long)F.total,
                 "%s: a workspace of %lld bytes does not fit this network at %d x %lld points (needs %lld)",
                 who, workspace_bytes, n_queries, n_points, (long long)F.total);
    uint8_t *ws = static_cast<uint8_t *>(workspace_dev);
    const Stack k = stack(h);
    const long long M = (long long)n_queries * n_points;
    const int last = s.n_lin - 1;
    float *const sdf = reinterpret_cast<float *>(ws + F.sdf), *const gs = reinterpret_cast<float *>(ws + F.consts);
    float *const xa = reinterpret_cast<float *>(ws + F.xa), *const xb = reinterpret_cast<float *>(ws + F.xb);
    if ((rc = nphm_mlp_train_forward(h, xyz_dev, cond_dev, nullptr, 0, n_queries, n_points, sdf, ws, stream_))) return rc;
    surface_upstream_kernel<<<per_query ? (unsigned)n_queries : 1u, kThreads, 0, stream>>>(sdf, mask_dev, per_query ? n_points : M,
                                                                                         clamp, per_query, ws + F.dl, gs,
                                                                                         loss_terms_dev);
    NPHM_CUDA_CHECK(cudaGetLastError());
    if ((rc = train::reserve_sums(k, n_queries))) return rc;
    train::GradTargets tg = train::targets(s, F.base, ws, n_queries, n_points, 0, gs);
    tg.want_cond = true;
    // no weights or biases: the condition sums at layers 0 and skip
    auto cond_sums = [&](int l, const Adjoint &d) { return train::layer_grads(k, tg, l, d, stream); };

    // d_{l-1} = s_{l-1} * (d_l W_l) from the packed upstream down to d_0; d_l lives in dp[l & 1]
    AdjointWalk w;
    w.top = Adjoint{nullptr, 0, ws + F.dl, 1, 0};
    for (int l = 0; l < last; ++l) { w.S[l] = reinterpret_cast<const float *>(ws + F.base.s[l]); w.D[l] = ws + F.dp[l & 1]; }
    w.xs = grad_xyz_dev ? xb : nullptr;
    if ((rc = adjoint_walk(k, M, w, cond_sums, stream))) return rc;
    if ((rc = cond_grad(k, n_queries, 1, grad_cond_dev, stream))) return rc;           // one chunk: a fixed summation order
    if (grad_xyz_dev && (rc = xyz_grad(k, M, w.D[0], 0, xa, xb, gs, 2, grad_xyz_dev, stream))) return rc;
    if (per_query) {
        const long long n3 = grad_xyz_dev ? 3 * n_points : 0;
        const dim3 grid((unsigned)ceil_div(std::max((long long)s.cond_dim, n3), 256), (unsigned)n_queries);
        scan_factor_kernel<<<grid, 256, 0, stream>>>(loss_terms_dev, s.cond_dim, n3, grad_cond_dev, grad_xyz_dev);
        NPHM_CUDA_CHECK(cudaGetLastError());
    }
    return NPHM_OK;
}

}  // namespace fitsurf
}  // namespace nphm

extern "C" long long nphm_mlp_fit_workspace_bytes(const nphm_mlp *h, int n_queries, long long n_points)
{
    if (!h || !h->loaded || n_queries < 1 || n_points < 1) {
        set_error("nphm_mlp_fit_workspace_bytes: bad arguments");
        return -1;
    }
    return (long long)fitsurf::layout(h->dims, n_queries, n_points).total;
}

extern "C" int nphm_mlp_fit_surface_grad(nphm_mlp *h, const float *xyz_dev, const float *cond_dev, int n_queries, long long n_points,
                                         const unsigned char *mask_dev, float clamp, float *loss_terms_dev, float *grad_cond_dev,
                                         float *grad_xyz_dev, void *workspace_dev, long long workspace_bytes, void *stream_)
{
    return fitsurf::surface_grad(h, xyz_dev, cond_dev, n_queries, n_points, mask_dev, clamp, false, loss_terms_dev, grad_cond_dev,
                                 grad_xyz_dev, workspace_dev, workspace_bytes, stream_, "nphm_mlp_fit_surface_grad");
}

extern "C" int nphm_mlp_fit_surface_grad_batched(nphm_mlp *h, const float *xyz_dev, const float *cond_dev, const unsigned char *mask_dev,
                                                 int n_scans, long long n_points, float clamp, float *loss_terms_dev,
                                                 float *grad_cond_dev, float *grad_xyz_dev, void *workspace_dev,
                                                 long long workspace_bytes, void *stream_)
{
    return fitsurf::surface_grad(h, xyz_dev, cond_dev, n_scans, n_points, mask_dev, clamp, true, loss_terms_dev, grad_cond_dev,
                                 grad_xyz_dev, workspace_dev, workspace_bytes, stream_, "nphm_mlp_fit_surface_grad_batched");
}

// ================================================================================================ the NPHM ensemble through grad_x sdf
// Stage 1 of the ensemble (reference train.py -local): the SDF-gradient passes above with the ensemble's members.  Member k
// sees B queries of N points in its own frame; its per-(member, query) bias rows carry the folded condition constants.
namespace nphm {

void ensemble_chain_destroy(nphm_ensemble *h)
{
    delete h->sdfgrad;
    h->sdfgrad = nullptr;
}

namespace esdf {

static Members members(const nphm_ensemble *h) { return Members{h->n_members, h->cfg.n_symm_pairs, h->n_sets}; }
static Stack stack(nphm_ensemble *h) { return Stack{h->dims, h->weights, *h->sdfgrad, members(h)}; }

// the packed chain of all weight sets, built on the first call after a weight load
static int pack(nphm_ensemble *h, cudaStream_t stream)
{
    if (!h->sdfgrad) h->sdfgrad = new PackedChain();
    if (h->sdfgrad->packed) return NPHM_OK;
    return pack_chain(*h->sdfgrad, h->dims, h->weights, h->n_sets, stream);
}

// cvec[k][q][coff_l + n]: b_l[sigma][n], plus at the folded layers scale_l * W_l[sigma][n][K_l:] . cond[k][q], summed in the
// order of simt.cu's cvec_kernel (so a member's constants equal those of its weight set as a single stack).  grid (members,
// queries), one warp per output row
__global__ void cvec_kernel(const PackSpec spec, const float *__restrict__ cond, int n_batch, float *__restrict__ cvec)
{
    const int m = blockIdx.x, q = blockIdx.y, C = spec.cond_dim, set = member_set(m, spec.n_symm);
    const float *u = cond + ((size_t)m * n_batch + q) * C;
    float *out = cvec + ((size_t)m * n_batch + q) * spec.cvec_stride;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
    for (int l = 0; l < spec.n_layers; ++l) {
        const PackLayer &pl = spec.L[l];
        for (int n = warp; n < pl.Npad; n += wpb) {
            float v = 0.f;
            if (n < pl.N) {
                v = pl.b[(size_t)set * pl.N + n];
                if (pl.folded) {
                    const float *w = pl.W + ((size_t)set * pl.N + n) * pl.in_total + pl.K;
                    float s = 0.f;
                    for (int j = lane; j < C; j += 32) s = fmaf(w[j], u[j], s);
#pragma unroll
                    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
                    v = fmaf(s, pl.scale, v);
                }
            }
            if (lane == 0) out[pl.coff + n] = v;
        }
    }
}

static int ready(nphm_ensemble *h, const char *who)
{
    NPHM_REQUIRE(h && h->loaded, "%s: weights not loaded", who);
    const StackDims &s = h->dims;
    if (s.N[s.n_lin - 1] != 1 || s.skip < 1 || s.skip >= s.n_lin - 1) {
        set_error("%s: needs a one-output stack with its skip below the output layer", who);
        return NPHM_ERR_UNSUPPORTED;
    }
    return NPHM_OK;
}

}  // namespace esdf
}  // namespace nphm

extern "C" long long nphm_ensemble_sdfgrad_workspace_bytes(const nphm_ensemble *h, int n_batch, long long n_points)
{
    if (!h || !h->loaded || n_batch < 1 || n_points < 1) {
        set_error("nphm_ensemble_sdfgrad_workspace_bytes: bad arguments");
        return -1;
    }
    return (long long)sdfgrad::layout(h->dims, esdf::members(h), n_batch, n_points, true).total;
}

extern "C" int nphm_ensemble_sdfgrad_forward(nphm_ensemble *h, const float *xyz_local_dev, const float *cond_dev, int n_batch,
                                             long long n_points, float *sdf_out_dev, float *grad_out_dev, void *workspace_dev,
                                             void *stream_)
{
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    int rc = esdf::ready(h, "nphm_ensemble_sdfgrad_forward");
    if (rc) return rc;
    NPHM_REQUIRE(n_batch >= 1 && n_points >= 1 && xyz_local_dev && cond_dev && sdf_out_dev && grad_out_dev && workspace_dev,
                 "nphm_ensemble_sdfgrad_forward: bad arguments");
    if ((rc = esdf::pack(h, stream))) return rc;
    const sdfgrad::Layout G = sdfgrad::layout(h->dims, esdf::members(h), n_batch, n_points, true);
    uint8_t *ws = static_cast<uint8_t *>(workspace_dev);
    float *cvec = reinterpret_cast<float *>(ws + G.cvec);
    esdf::cvec_kernel<<<dim3((unsigned)h->n_members, (unsigned)n_batch), 256, 0, stream>>>(h->spec, cond_dev, n_batch, cvec);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return sdfgrad::forward(esdf::stack(h), G, xyz_local_dev, cond_dev, cvec, n_batch, n_points, sdf_out_dev, grad_out_dev, ws,
                            stream);
}

extern "C" int nphm_ensemble_sdfgrad_backward(nphm_ensemble *h, const float *grad_sdf_dev, const float *grad_grad_dev, void *workspace_dev,
                                              long long workspace_bytes, int n_batch, long long n_points, float *const *grad_w_dev,
                                              float *const *grad_b_dev, float *grad_cond_dev, float *grad_xyz_dev, void *stream_)
{
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    int rc = esdf::ready(h, "nphm_ensemble_sdfgrad_backward");
    if (rc) return rc;
    NPHM_REQUIRE(n_batch >= 1 && n_points >= 1 && grad_sdf_dev && grad_grad_dev && workspace_dev,
                 "nphm_ensemble_sdfgrad_backward: bad arguments");
    NPHM_REQUIRE(h->sdfgrad && h->sdfgrad->packed, "nphm_ensemble_sdfgrad_backward: no forward since the last weight load");
    const sdfgrad::Layout G = sdfgrad::layout(h->dims, esdf::members(h), n_batch, n_points, true);
    // the caller states the shape the workspace was made for; checked against its size, without reading it back
    NPHM_REQUIRE(workspace_bytes == (long long)G.total,
                 "nphm_ensemble_sdfgrad_backward: a workspace of %lld bytes does not hold an SDF-gradient forward of this ensemble "
                 "at %d x %lld points", workspace_bytes, n_batch, n_points);
    return sdfgrad::backward(esdf::stack(h), G, grad_sdf_dev, grad_grad_dev, static_cast<uint8_t *>(workspace_dev), n_batch, n_points,
                             grad_w_dev, grad_b_dev, grad_cond_dev, grad_xyz_dev, stream);
}
