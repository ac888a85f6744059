// Weight-gradient GEMM of the training backward:  dW_l = D_l^T H_l, reduced over the rows (points), not over the features.
//
// Both operands are the packed activations the value and adjoint passes already write (tc_linear.cuh: per 128-row tile and
// k-step [128 x 16 fp16 hi | 128 x 16 fp16 lo], core matrices of 8 rows x 8 features, one 16-byte line = 8 features of one
// row).  For this product the rows are the reduction dimension, so every 8 x 8 core matrix is stored MN-major; ldmatrix.trans
// turns it into the K-major fragments of mma.sync m16n8k16 without any re-layout in memory.  Same 3-pass fp16 split as the
// forward (hi*hi + hi*lo + lo*hi, fp32 accumulators), i.e. fp32-level accuracy.
//
// CTA: 64 output rows (features of D) x 64 output columns (features of H), 4 warps of 32 x 32; the rows of the problem
// (M = 3 200 .. 35 200 per call) are split over gridDim.y so that the few output tiles of a layer still fill the GPU.  Each
// CTA streams its 128-row tiles through a two-stage cp.async ring (32 KB of D | 32 KB of H per stage; rows beyond M are
// zero-filled) and writes its partial sums; a second kernel adds the partials in split order.
//
// Two operand pairs (dW = D^T H + D2^T H2, the SDF-gradient training backward): the row tiles of the second pair follow
// those of the first in one sequence of 2 x row_tiles tiles, so the sum is taken in one fixed order.
#include "tc_wgrad.cuh"
#include "tc_common.cuh"

namespace nphm {
namespace wgrad {
using tc::smem_u32;

constexpr int kTile = 64;                    // output tile edge = 4 k-steps of a packed operand
constexpr int kThreads = 128;
constexpr int kOpBytes = 4 * 8192;           // 4 k-steps of one 128-row tile
constexpr int kStageBytes = 2 * kOpBytes;    // D block | H block
constexpr int kSmem = 2 * kStageBytes;

__device__ __forceinline__ void cp_async16(uint32_t dst, const void *src, bool ok)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(ok ? 16 : 0) : "memory");
}

__device__ __forceinline__ void ldsm_x4_trans(uint32_t addr, uint32_t (&r)[4])
{
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}

__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1)
{
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
                 "{%0, %1, %2, %3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// partial[split][n][k] (ld kb_count * 64) of output tile (blockIdx.x / kb_count, blockIdx.x % kb_count) over row tiles
// [split * tiles_per_split, ...) of the row_tiles tiles of (D, H) followed, with D2 given, by the row_tiles tiles of (D2, H2)
// Set-batched (gridDim.z = weight set, Members): set z reduces over the row tiles of its members m0 (and m0 + 1 for the
// w_pairs mirrored pairs), member after member, each with its pairs in the order above; member m's operands start at
// D + m sD (bytes), and so on.  One set (gridDim.z = 1, w_pairs = 0): member 0, the plain launch.
struct Members { int w_pairs; long long sD, sH, sD2, sH2; };

__global__ void __launch_bounds__(kThreads) wgrad_kernel(const uint8_t *__restrict__ D, int ks_d, const uint8_t *__restrict__ H,
                                                         int ks_h, const uint8_t *__restrict__ D2, const uint8_t *__restrict__ H2,
                                                         long long M, int row_tiles, int tiles_per_split, int nb_count,
                                                         int kb_count, const Members mem, float *__restrict__ partial)
{
    extern __shared__ __align__(128) uint8_t smem[];
    const int nb = blockIdx.x / kb_count, kb = blockIdx.x % kb_count, split = blockIdx.y, set = blockIdx.z;
    const SetMembers sm = set_members(set, mem.w_pairs);
    const int m0 = sm.first, n_mem = sm.count;
    const int per_mem = D2 ? 2 * row_tiles : row_tiles;
    const int t0 = split * tiles_per_split, t1 = min(n_mem * per_mem, t0 + tiles_per_split);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wn = warp >> 1, wk = warp & 1;

    // one stage: 2 operands x 4 k-steps x 512 lines of 16 bytes; line -> row of the tile: ((line & 255) >> 4) * 8 + (line & 7)
    auto load = [&](int t, int s) {
        const uint32_t dst0 = smem_u32(smem + (size_t)s * kStageBytes);
        const int m = m0 + t / per_mem;
        t %= per_mem;
        const bool second = t >= row_tiles;
        if (second) t -= row_tiles;
        const uint8_t *bd = second ? D2 + m * mem.sD2 : D + m * mem.sD, *bh = second ? H2 + m * mem.sH2 : H + m * mem.sH;
        for (int i = threadIdx.x; i < 2 * 4 * 512; i += kThreads) {
            const int op = i >> 11, u = (i >> 9) & 3, line = i & 511;
            const uint8_t *base = op ? bh : bd;
            const int ks = op ? ks_h : ks_d, j = (op ? kb : nb) * 4 + u;
            const int r = ((line & 255) >> 4) * 8 + (line & 7);
            const bool ok = j < ks && (long long)t * 128 + r < M;
            const uint8_t *src = ok ? base + ((size_t)t * ks + j) * 8192 + (size_t)line * 16 : base;
            cp_async16(dst0 + op * kOpBytes + u * 8192 + line * 16, src, ok);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };

    float acc[2][4][4];
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[a][b][e] = 0.f;

    const int mtx = lane >> 3, li = lane & 7;
    if (t0 < t1) load(t0, 0);
    for (int t = t0, s = 0; t < t1; ++t, s ^= 1) {
        if (t + 1 < t1) {
            load(t + 1, s ^ 1);
            asm volatile("cp.async.wait_group 1;" ::: "memory");
        } else {
            asm volatile("cp.async.wait_group 0;" ::: "memory");
        }
        __syncthreads();
        const uint32_t sd = smem_u32(smem + (size_t)s * kStageBytes), sh = sd + kOpBytes;
#pragma unroll 2
        for (int kk = 0; kk < 8; ++kk) {           // 16 rows per MMA k-step
            uint32_t ahi[2][4], alo[2][4], bhi[2][4], blo[2][4];
#pragma unroll
            for (int mi = 0; mi < 2; ++mi) {
                // A = D^T (16 features x 16 rows): matrices (rows 0-7 | feat 0-7), (rows 0-7 | feat 8-15), (rows 8-15 | ...) ...
                const uint32_t addr = sd + (wn * 2 + mi) * 8192 + (2 * kk + (mtx >> 1)) * 256 + (mtx & 1) * 128 + li * 16;
                ldsm_x4_trans(addr, ahi[mi]);
                ldsm_x4_trans(addr + 4096, alo[mi]);
            }
#pragma unroll
            for (int pr = 0; pr < 2; ++pr) {
                // B = H (16 rows x 8 features), two n8 tiles per ldmatrix: (feat 0-7: rows 0-7, rows 8-15), (feat 8-15: ...)
                const uint32_t addr = sh + (wk * 2 + pr) * 8192 + (2 * kk + (mtx & 1)) * 256 + (mtx >> 1) * 128 + li * 16;
                ldsm_x4_trans(addr, bhi[pr]);
                ldsm_x4_trans(addr + 4096, blo[pr]);
            }
#pragma unroll
            for (int mi = 0; mi < 2; ++mi)
#pragma unroll
                for (int ni = 0; ni < 4; ++ni) {
                    const int pr = ni >> 1, q = (ni & 1) * 2;
                    mma16816(acc[mi][ni], ahi[mi], bhi[pr][q], bhi[pr][q + 1]);
                    mma16816(acc[mi][ni], ahi[mi], blo[pr][q], blo[pr][q + 1]);
                    mma16816(acc[mi][ni], alo[mi], bhi[pr][q], bhi[pr][q + 1]);
                }
        }
        __syncthreads();                           // stage s is refilled at the next iteration
    }
    const int ldk = kb_count * kTile;
    float *out = partial + ((size_t)set * gridDim.y + split) * nb_count * kTile * ldk;
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int ni = 0; ni < 4; ++ni) {
            const int n = nb * kTile + wn * 32 + mi * 16 + (lane >> 2);
            const int k = kb * kTile + wk * 32 + ni * 8 + 2 * (lane & 3);
            *reinterpret_cast<float2 *>(out + (size_t)n * ldk + k) = make_float2(acc[mi][ni][0], acc[mi][ni][1]);
            *reinterpret_cast<float2 *>(out + (size_t)(n + 8) * ldk + k) = make_float2(acc[mi][ni][2], acc[mi][ni][3]);
        }
}

// dW[n][k] = scale * inv_scale * sum over the splits, in split order; set z = blockIdx.y: partials, dW + z dw_stride,
// inv_scale + z inv_stride
__global__ void wgrad_finish_kernel(const float *__restrict__ partial, int splits, int ldn, int ldk, int N, int K, float scale,
                                    const float *__restrict__ inv_scale, int inv_stride, float *__restrict__ dW, int ldw,
                                    long long dw_stride)
{
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)N * K) return;
    const int n = (int)(idx / K), k = (int)(idx % K), set = blockIdx.y;
    const float *part = partial + (size_t)set * splits * ldn * ldk;
    float s = 0.f;
    for (int i = 0; i < splits; ++i) s += part[((size_t)i * ldn + n) * ldk + k];
    dW[(size_t)set * dw_stride + (size_t)n * ldw + k] = s * (scale * inv_scale[(size_t)set * inv_stride]);
}

int launch_sets(const uint8_t *D, int d_ksteps, const uint8_t *H, int h_ksteps, long long M, int N, int K, float scale,
                const float *inv_scale_dev, int inv_stride, float *dW, int ldw, long long dw_stride, int sets, int w_pairs,
                long long sD, long long sH, long long sD2, long long sH2, DeviceBuffer &partials, cudaStream_t stream,
                const uint8_t *D2, const uint8_t *H2)
{
    NPHM_REQUIRE(M > 0 && N <= d_ksteps * 16 && K <= h_ksteps * 16 && !D2 == !H2 && sets >= 1 && w_pairs >= 0 && w_pairs <= sets,
                 "wgrad: bad operand shapes");
    const int nb_count = (d_ksteps + 3) / 4, kb_count = (h_ksteps + 3) / 4;
    const int row_tiles = (int)ceil_div(M, 128), all_tiles = (w_pairs ? 2 : 1) * (D2 ? 2 * row_tiles : row_tiles);
    const int tiles = nb_count * kb_count;
    int splits = std::max(1, std::min(all_tiles, (int)ceil_div(2LL * sm_count(), (long long)tiles * sets)));
    const int tiles_per_split = (int)ceil_div(all_tiles, splits);
    splits = (int)ceil_div(all_tiles, tiles_per_split);
    const int ldn = nb_count * kTile, ldk = kb_count * kTile;
    int rc;
    if ((rc = partials.reserve((size_t)sets * splits * ldn * ldk * sizeof(float)))) return rc;
    static bool smem_set[64] = {};                 // the attribute is per device: set once on each
    int dev = 0;
    NPHM_CUDA_CHECK(cudaGetDevice(&dev));
    if (dev >= 64 || !smem_set[dev]) {
        NPHM_CUDA_CHECK(cudaFuncSetAttribute(wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
        if (dev < 64) smem_set[dev] = true;
    }
    const Members mem{w_pairs, sD, sH, sD2, sH2};
    wgrad_kernel<<<dim3(tiles, splits, sets), kThreads, kSmem, stream>>>(D, d_ksteps, H, h_ksteps, D2, H2, M, row_tiles,
                                                                         tiles_per_split, nb_count, kb_count, mem,
                                                                         partials.as<float>());
    NPHM_CUDA_CHECK(cudaGetLastError());
    const long long total = (long long)N * K;
    wgrad_finish_kernel<<<dim3((unsigned)ceil_div(total, 256), sets), 256, 0, stream>>>(
        partials.as<float>(), splits, ldn, ldk, N, K, scale, inv_scale_dev, inv_stride, dW, ldw, dw_stride);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

}  // namespace wgrad
}  // namespace nphm
