// Tensor-core path of the identity-SDF ensemble (NPHM configuration: 40 members, hidden 200, 4 hidden layers, condition
// 64+32) - the dominant kernel of the hot path: weight packing, per-(query, member) records, launch (kernel: tc_ensemble_wgmma.cu).
//
// Reference semantics: FastEnsembleDeepSDFMirrored.forward  src/NPHM/models/EnsembledDeepSDF.py:203-267
//
// Math (SURVEY.md 8a'): per member, per point
//   h0 = sp(W0x c + v0)            K=3   -> CUDA cores (v0 = latent part + bias, per query/member)
//   h1 = sp(W1 h0 + b1)            64x104x208 wgmma per warpgroup   (N 101 -> 104, K 200 -> 208)
//   h2 = sp(W2a h1/r2 + W2x c/r2 + v2)   64x200x112 wgmma   (K = 101 + 3 -> 112)
//   h3 = sp(W3 h2 + b3)            64x200x208 wgmma
//   s  = w4 . h3 + b4              CUDA cores, on the layer-3 accumulators; Gaussian anchor blend in registers.
// Precision: tensor cores run fp16 MMAs with fp32 accumulation; every operand is split in two fp16 terms
// (x = hi + lo, 22 significant bits) and each product is evaluated as hi*hi + hi*lo + lo*hi (3 MMAs), which
// keeps the result at fp32 round-off level (tolerance 1e-5 against the fp32 reference).
// Activations are kept in "log2 units": t = a * 100*log2(e), sp'(t) = max(t,0) + lg2(1 + 2^-|t|) = 100*log2(e) *
// softplus_100(a), so the softplus costs 2 MUFU + 3 ALU and the unit change is folded into biases / w4.
#include "tc_ensemble.cuh"
#include <cstdlib>

namespace nphm {
namespace tc {

// ------------------------------------------------------------------------------------------------ packing
// Weight units (tc_ensemble.cuh): for weight set s, unit u, k-step j of the unit: nw x 16 fp16 hi then nw x 16 fp16 lo, each in
// no-swizzle K-major core-matrix order: byte offset of (n, kk) = (n/8)*256 + (kk/8)*128 + (n%8)*16 + (kk%8)*2, n counted from
// the unit's first column.
// Bias rows: the K padding of layers 1 and 3 (k = 200) carries S * b_l (per weight set, no latent part); the A operand has
// the constant 1.0 at that k, so the MMAs add the bias and the epilogues do not (layer 2's constant depends on the latent:
// its k-step-6 slabs are re-built per (query, member), see l2_slab_kernel).
__global__ void pack_slabs_kernel(const float *__restrict__ W1, const float *__restrict__ W2, const float *__restrict__ W3,
                                  const float *__restrict__ b1, const float *__restrict__ b3,
                                  int n_sets, uint8_t *__restrict__ out)
{
    const int total_per_set = kSetBytes / 4;       // (unit, k-step, n, kk) quadruples: 4 bytes (hi + lo) each
    const float inv_sqrt2 = 0.70710678118654752440f;
    for (size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x; t < (size_t)n_sets * total_per_set;
         t += (size_t)gridDim.x * blockDim.x) {
        const int s = (int)(t / total_per_set);
        int r = (int)(t % total_per_set), u = 0;
        while (r >= unit_bytes(u) / 4) { r -= unit_bytes(u) / 4; ++u; }
        const int layer = unit_layer(u), nw = unit_nw(u);
        const int j = r / (nw * 16), nl = (r / 16) % nw, kk = r % 16;
        const int n = unit_n0(u) + nl, k = (unit_k0(u) + j) * 16 + kk;
        float v = 0.f;
        if (layer == 1) {
            if (n < kN1 && k < kH) v = W1[((size_t)s * kN1 + n) * kH + k];
            else if (n < kN1 && k == kH) v = kS * b1[(size_t)s * kN1 + n];
        } else if (layer == 2) {
            // reference input order of the skip layer: [h1 (101), xyz (3), cond (96)] / sqrt(2); the cond part is folded
            if (n < kH && k < kN1 + 3) v = W2[((size_t)s * kH + n) * kH + k] * inv_sqrt2;
        } else {
            if (n < kH && k < kH) v = W3[((size_t)s * kH + n) * kH + k];
            else if (n < kH && k == kH) v = kS * b3[(size_t)s * kH + n];
        }
        const __half hi = __float2half_rn(v);
        const __half lo = __float2half_rn(v - __half2float(hi));
        const size_t off = (size_t)(nl >> 3) * 256 + (size_t)(kk >> 3) * 128 + (size_t)(nl & 7) * 16 + (size_t)(kk & 7) * 2;
        uint8_t *base = out + (size_t)s * kSetBytes + unit_off(u) + (size_t)j * nw * 64;
        *reinterpret_cast<__half *>(base + off) = hi;
        *reinterpret_cast<__half *>(base + (size_t)nw * 32 + off) = lo;
    }
}

// record of (query, member): see kRec* offsets.  cvec holds b_l + latent-folded parts (simt.cu:cvec_kernel).
__global__ void records_kernel(const float *__restrict__ cvec, int cvec_stride, const int *__restrict__ coff,
                               const float *__restrict__ W0, const float *__restrict__ W4,
                               const float *__restrict__ anchors, int n_members, int n_symm, float *__restrict__ recs)
{
    const int m = blockIdx.x, qi = blockIdx.y;
    const int set = member_set(m, n_symm);
    const float *cv = cvec + ((size_t)qi * n_members + m) * cvec_stride;
    float *rec = recs + ((size_t)qi * n_members + m) * kRecFloats;
    const int d_in = 3 + kCond;
    for (int n = threadIdx.x; n < 208; n += blockDim.x) {
        const float *w = W0 + ((size_t)set * kH + (n < kH ? n : 0)) * d_in;
        const bool real = n < kH;
        rec[kRecL0 + 4 * n + 0] = real ? w[0] : 0.f;
        rec[kRecL0 + 4 * n + 1] = real ? w[1] : 0.f;
        rec[kRecL0 + 4 * n + 2] = real ? w[2] : 0.f;
        rec[kRecL0 + 4 * n + 3] = real ? kS * cv[coff[0] + n] : 0.f;
    }
    for (int n = threadIdx.x; n < 112; n += blockDim.x) rec[kRecB1 + n] = n < kN1 ? kS * cv[coff[1] + n] : 0.f;
    for (int n = threadIdx.x; n < 208; n += blockDim.x) {
        rec[kRecB2 + n] = n < kH ? kS * cv[coff[2] + n] : 0.f;
        rec[kRecB3 + n] = n < kH ? kS * cv[coff[3] + n] : 0.f;
        rec[kRecW4 + n] = n < kH ? W4[(size_t)set * kH + n] / kS : 0.f;
    }
    if (threadIdx.x == 0) {
        const bool has_anchor = m < n_members - 1;
        rec[kRecMisc + 0] = cv[coff[4]];
        rec[kRecMisc + 1] = has_anchor ? anchors[((size_t)qi * (n_members - 1) + m) * 3 + 0] : 0.f;
        rec[kRecMisc + 2] = has_anchor ? anchors[((size_t)qi * (n_members - 1) + m) * 3 + 1] : 0.f;
        rec[kRecMisc + 3] = has_anchor ? anchors[((size_t)qi * (n_members - 1) + m) * 3 + 2] : 0.f;
        rec[kRecMisc + 4] = has_anchor ? 1.f : 0.f;
        rec[kRecMisc + 5] = ((m & 1) && m < 2 * n_symm) ? 1.f : 0.f;
        rec[kRecMisc + 6] = 0.f;
        rec[kRecMisc + 7] = 0.f;
    }
}

// Layer 2's per-column constant v2 = S * (b2 + W2u u / sqrt(2)) depends on the latent, i.e. on (query, member): the last
// k-step slabs of layer 2 (k 96..111, of which 96..103 are real inputs; column half a then half b) are copied per (query,
// member) and their K-padding row k = 104 filled with v2 (fp16 hi | lo); the A operand carries 1.0 there.  12.5 KB per
// (query, member).
__global__ void l2_slab_kernel(const uint8_t *__restrict__ weights, const float *__restrict__ cvec, int cvec_stride,
                               const int *__restrict__ coff, int n_members, int n_symm, uint8_t *__restrict__ out)
{
    const int m = blockIdx.x, qi = blockIdx.y;
    const int set = member_set(m, n_symm);
    const uint8_t *w = weights + (size_t)set * kSetBytes;
    uint8_t *dst = out + ((size_t)qi * n_members + m) * kL2SlabBytes;
    for (int i = threadIdx.x; i < kL2SlabBytes / 16; i += blockDim.x) {
        const bool half_b = i >= kL2SlabABytes / 16;
        const uint8_t *src = half_b ? w + unit_off(3) + (kKS2 - 1) * kNB * 64 - kL2SlabABytes : w + unit_off(2) + (kKS2 - 1) * kNA * 64;
        reinterpret_cast<uint4 *>(dst)[i] = reinterpret_cast<const uint4 *>(src)[i];
    }
    __syncthreads();
    const float *cv = cvec + ((size_t)qi * n_members + m) * cvec_stride;
    const int kk = (kN1 + 3) - (kKS2 - 1) * 16;          // 104 - 96 = 8
    for (int n = threadIdx.x; n < kNA + kNB; n += blockDim.x) {
        const float v = n < kH ? kS * cv[coff[2] + n] : 0.f;
        const __half hi = __float2half_rn(v);
        const __half lo = __float2half_rn(v - __half2float(hi));
        const int nw = n < kNA ? kNA : kNB, nl = n < kNA ? n : n - kNA;
        uint8_t *slab = dst + (n < kNA ? 0 : kL2SlabABytes);
        const size_t off = (size_t)(nl >> 3) * 256 + (size_t)(kk >> 3) * 128 + (size_t)(nl & 7) * 16 + (size_t)(kk & 7) * 2;
        *reinterpret_cast<__half *>(slab + off) = hi;
        *reinterpret_cast<__half *>(slab + (size_t)nw * 32 + off) = lo;
    }
}

// ------------------------------------------------------------------------------------------------ MMA self test
// One warpgroup: D[64 x n] = A[64 x 16*ks] * B[n x 16*ks]^T with the operand plumbing of the ensemble kernel (fp16 hi/lo split,
// A in registers, B slabs in shared memory, 16-column wgmmas).  Rows 64 .. 127 of a 128-row test run in a second CTA.
// `variant` bit0: swap LBO/SBO, bit1: swap the fp16 pair order (layout probes: only variant 0 is right).
__global__ void __launch_bounds__(128, 1) mma_selftest_kernel(const float *__restrict__ A, const uint8_t *__restrict__ slabs,
                                                              int n, int ks, int variant, float *__restrict__ D)
{
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, q4 = lane & 3;
    const int slab_bytes = n * 64;
    for (int i = threadIdx.x; i < ks * slab_bytes / 16; i += blockDim.x)
        reinterpret_cast<uint4 *>(smem_raw)[i] = reinterpret_cast<const uint4 *>(slabs)[i];
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    const int r0 = 64 * blockIdx.x + 16 * warp + (lane >> 2);
    const uint32_t lbo = (variant & 1) ? 256 : 128, sbo = (variant & 1) ? 128 : 256;
    for (int c = 0; c < n; c += 16) {
        float d[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        for (int j = 0; j < ks; ++j) {
            uint32_t ah[4], al[4];
            for (int f = 0; f < 4; ++f) {                    // register A: (row r0 | r0 + 8, k 2 q4 | 8 + 2 q4)
                const int r = r0 + 8 * (f & 1), k = 16 * j + 8 * (f >> 1) + 2 * q4;
                float v0 = A[(size_t)r * ks * 16 + k], v1 = A[(size_t)r * ks * 16 + k + 1];
                if (variant & 2) { const float t = v0; v0 = v1; v1 = t; }
                split2(v0, v1, ah[f], al[f]);
            }
            const uint32_t b = smem_u32(smem_raw + (size_t)j * slab_bytes) + 2 * c * 16;
            const uint64_t bh = make_desc(b, lbo, sbo), bl = make_desc(b + n * 32, lbo, sbo);
            wg_fence();
            wgmma_rs_n16(d, ah, bh, 1);
            wgmma_rs_n16(d, ah, bl, 1);
            wgmma_rs_n16(d, al, bh, 1);
            wg_commit();
            wg_wait<0>();
            wg_reg_fence(d);
        }
        for (int i = 0; i < 8; ++i) {
            const int r = r0 + 8 * ((i >> 1) & 1), col = c + 8 * (i >> 2) + 2 * q4 + (i & 1);
            D[(size_t)r * n + col] = d[i];
        }
    }
}

__global__ void pack_test_slabs_kernel(const float *__restrict__ B, int n, int ks, uint8_t *__restrict__ out)
{
    // B: [n][16*ks] fp32 row-major -> ks slabs (hi | lo) in core-matrix order
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n * ks * 16; t += gridDim.x * blockDim.x) {
        const int row = t / (ks * 16), k = t % (ks * 16), j = k / 16, kk = k % 16;
        const float v = B[t];
        const __half hi = __float2half_rn(v);
        const __half lo = __float2half_rn(v - __half2float(hi));
        const size_t off = (size_t)(row >> 3) * 256 + (size_t)(kk >> 3) * 128 + (size_t)(row & 7) * 16 + (size_t)(kk & 7) * 2;
        uint8_t *base = out + (size_t)j * n * 64;
        *reinterpret_cast<__half *>(base + off) = hi;
        *reinterpret_cast<__half *>(base + (size_t)n * 32 + off) = lo;
    }
}

}  // namespace tc

// ------------------------------------------------------------------------------------------------ host side
bool tc_ensemble_supported(const nphm_ensemble *h)
{
    return h->cfg.hidden_dim == tc::kH && h->cfg.n_layers == 4 && h->cfg.lat_dim_glob + h->cfg.lat_dim_loc == tc::kCond &&
           h->dims.N[1] == tc::kN1 && h->n_members <= tc::kMaxMembers;
}

int tc_ensemble_pack(nphm_ensemble *h, cudaStream_t stream)
{
    h->tc_ready = false;
    if (!tc_ensemble_supported(h)) return NPHM_OK;
    int rc;
    if ((rc = h->tc_weights.reserve((size_t)h->n_sets * tc::kSetBytes))) return rc;
    tc::pack_slabs_kernel<<<512, 256, 0, stream>>>(h->weights.W[1].as<float>(), h->weights.W[2].as<float>(),
                                                   h->weights.W[3].as<float>(), h->weights.b[1].as<float>(),
                                                   h->weights.b[3].as<float>(), h->n_sets, h->tc_weights.as<uint8_t>());
    NPHM_CUDA_CHECK(cudaGetLastError());
    if ((rc = h->tc_coff.reserve(kMaxLayers * sizeof(int)))) return rc;
    NPHM_CUDA_CHECK(cudaMemcpyAsync(h->tc_coff.ptr, h->dims.coff, kMaxLayers * sizeof(int), cudaMemcpyHostToDevice, stream));
    NPHM_CUDA_CHECK(cudaStreamSynchronize(stream));      // dims.coff is host memory of the handle; keep it simple
    h->tc_ready = true;
    return NPHM_OK;
}

int tc_ensemble_launch(nphm_ensemble *h, const SimtQuery &q, cudaStream_t stream)
{
    NPHM_REQUIRE(h->tc_ready, "tensor-core ensemble kernel: weights not packed");
    int rc;
    if ((rc = h->tc_consts.reserve((size_t)q.n_queries * h->n_members * tc::kRecFloats * sizeof(float)))) return rc;
    dim3 grid(h->n_members, q.n_queries);
    tc::records_kernel<<<grid, 256, 0, stream>>>(q.cvec, h->dims.cvec_stride, h->tc_coff.as<int>(), h->weights.W[0].as<float>(),
                                                 h->weights.W[4].as<float>(), q.anchors, h->n_members, h->cfg.n_symm_pairs,
                                                 h->tc_consts.as<float>());
    NPHM_CUDA_CHECK(cudaGetLastError());
    if ((rc = h->tc_l2slabs.reserve((size_t)q.n_queries * h->n_members * tc::kL2SlabBytes))) return rc;
    tc::l2_slab_kernel<<<grid, 256, 0, stream>>>(h->tc_weights.as<uint8_t>(), q.cvec, h->dims.cvec_stride, h->tc_coff.as<int>(),
                                                 h->n_members, h->cfg.n_symm_pairs, h->tc_l2slabs.as<uint8_t>());
    NPHM_CUDA_CHECK(cudaGetLastError());
    tc::Params p{};
    p.weights = h->tc_weights.as<uint8_t>();
    p.l2_slabs = h->tc_l2slabs.as<uint8_t>();
    p.recs = h->tc_consts.as<float>();
    p.xyz = q.xyz; p.axes = q.axes; p.res = q.res; p.first = q.first; p.total = q.total; p.n_points = q.n_points;
    p.n_queries = q.n_queries; p.quirk_period = q.quirk_period; p.out = q.out; p.members_out = q.members_out; p.acts_out = q.acts_out; p.acts_packed_out = q.acts_packed_out; p.acts_packed_tile_steps = q.acts_packed_tile_steps;
    p.n_members = h->n_members; p.n_symm = h->cfg.n_symm_pairs;
    const bool prune = h->tc_prune && !q.exact;
    NPHM_REQUIRE(!q.acts_out || (q.exact && q.acts_packed_out && q.acts_packed_tile_steps >= tc::kActPackedSteps),
                 "activation dump needs an exact query");
    p.anchors = q.anchors; p.prune_tau = h->tc_prune_tau;
    // dense queries skip the members whose blend weight is exactly zero on a whole tile; fitting needs every member's output
    p.zero_skip = !prune && !q.members_out && !q.acts_out;
    p.blocked = 0; p.px0 = p.px1 = 0; p.by = p.bz = 1; p.tbx = p.tby = p.tbz = 1;
    long long n_tiles = ceil_div(q.n_points, 128) * q.n_queries;
    if ((prune || p.zero_skip) && !q.xyz && q.n_points > 0) {
        // compact blocks over the x-plane range that contains [first, first + n_points), so that a tile is near few anchors:
        // 8 x 4 x 4 for the pruned rule (its mask depends on the composition of a tile), 1 x 16 x 8 for the dense rule - it
        // never crosses an x-plane, so plane-aligned ranges (the whole grid, x-slabs) tile without wasted rows
        const long long rr = (long long)q.res * q.res;
        const int tbx = prune ? 8 : 1, tby = prune ? 4 : 16, tbz = prune ? 4 : 8;
        const int px0 = (int)(q.first / rr), px1 = (int)((q.first + q.n_points - 1) / rr);
        const int by = (q.res + tby - 1) / tby, bz = (q.res + tbz - 1) / tbz;
        const long long blocked_tiles = (long long)((px1 - px0 + tbx) / tbx) * by * bz;
        // dense rule: keep linear tiles where blocks would add more than 3 % tiles (partial planes, small or odd grids)
        if (prune || blocked_tiles * 100 <= n_tiles * 103) {
            p.blocked = 1;
            p.px0 = px0; p.px1 = px1; p.by = by; p.bz = bz; p.tbx = tbx; p.tby = tby; p.tbz = tbz;
            n_tiles = blocked_tiles;
        }
    }
    p.n_tiles = n_tiles;
    p.member_groups = 1;
    if (q.acts_out) {
        // fitting: a few dozen tiles per scan - split the members of a tile over several CTAs so that every SM has work.  Cost
        // model: waves * (members per group + pipeline fill of a work item); groups must all be non-empty.  With many scans in
        // one launch (hundreds of tiles) it keeps whole tiles (one group): the waves are already full.
        double best = 1e30;
        for (int g = 1; g <= h->n_members; ++g) {
            const int per = (h->n_members + g - 1) / g;
            if (per * (g - 1) >= h->n_members) continue;
            const double cost = (double)ceil_div(n_tiles * g, (long long)sm_count()) * (per + 0.7);
            if (cost < best - 1e-9) { best = cost; p.member_groups = g; }
        }
    }
    h->tc_mask_tiles = 0;
    if (prune || p.zero_skip) {
        if ((rc = h->tc_masks.reserve((size_t)n_tiles * sizeof(unsigned long long)))) return rc;
        p.tile_masks = h->tc_masks.as<unsigned long long>();
        h->tc_mask_tiles = n_tiles;
    }
    // the kernel leaves the counter at zero when it ends; it starts at zero when allocated
    if (!h->tc_sched.ptr) {
        if ((rc = h->tc_sched.reserve(2 * sizeof(unsigned int)))) return rc;
        NPHM_CUDA_CHECK(cudaMemsetAsync(h->tc_sched.ptr, 0, 2 * sizeof(unsigned int), stream));
    }
    p.sched = h->tc_sched.as<unsigned int>();
    const long long n_items = n_tiles * p.member_groups;
    // 32-bit counter: the counter passes n_items by at most one per CTA
    NPHM_REQUIRE(n_items + sm_count() < (1ll << 32), "tensor-core ensemble kernel: %lld work items", n_items);
    const int grid_x = (int)(n_items < sm_count() ? n_items : sm_count());
    if ((rc = tc::launch_ensemble_wgmma(p, prune, q.acts_out != nullptr, grid_x, stream))) return rc;
    return NPHM_OK;
}

}  // namespace nphm

// Debug entry (not part of the public ABI): the member masks the pre-pass computed for the tiles of the handle's last
// tensor-core launch.  *n_tiles receives their number (0 when that launch evaluated every member); up to `cap` masks are
// copied to `host`.
extern "C" int nphm_debug_ens_tile_masks(nphm_ensemble *h, unsigned long long *host, long long cap, long long *n_tiles)
{
    using namespace nphm;
    NPHM_REQUIRE(h && n_tiles, "nphm_debug_ens_tile_masks: null argument");
    *n_tiles = h->tc_mask_tiles;
    const long long n = std::min(cap, h->tc_mask_tiles);
    NPHM_CUDA_CHECK(cudaDeviceSynchronize());
    if (n > 0) NPHM_CUDA_CHECK(cudaMemcpy(host, h->tc_masks.ptr, (size_t)n * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    return NPHM_OK;
}

// Debug entry (not part of the public ABI): D = A * B^T through the tensor-core operand path.
extern "C" int nphm_debug_tc_mma(const float *a_dev, const float *b_dev, int n, int ks, int variant, float *d_dev,
                                 void *stream_)
{
    using namespace nphm;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    NPHM_REQUIRE(n % 16 == 0 && n >= 16 && n <= 208 && ks >= 1 && ks <= 13, "nphm_debug_tc_mma: bad shape");
    uint8_t *slabs = nullptr;
    NPHM_CUDA_CHECK(cudaMalloc(&slabs, (size_t)ks * n * 64));
    tc::pack_test_slabs_kernel<<<64, 256, 0, stream>>>(b_dev, n, ks, slabs);
    const int smem = ks * n * 64;
    NPHM_CUDA_CHECK(cudaFuncSetAttribute(tc::mma_selftest_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    tc::mma_selftest_kernel<<<2, 128, smem, stream>>>(a_dev, slabs, n, ks, variant, d_dev);
    cudaError_t e = cudaStreamSynchronize(stream);
    cudaFree(slabs);
    if (e != cudaSuccess) { set_error("nphm_debug_tc_mma: %s", cudaGetErrorString(e)); return NPHM_ERR_CUDA; }
    return NPHM_OK;
}

