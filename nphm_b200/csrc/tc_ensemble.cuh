// Shared definitions of the tensor-core ensemble kernel (tc_ensemble.cu: packing and launch, tc_ensemble_wgmma.cu: the
// kernel): shapes, weight-slab / record layout, kernel parameters.
#pragma once
#include "engine.cuh"
#include "tc_common.cuh"

namespace nphm {
namespace tc {

constexpr int kH = 200;            // hidden width
constexpr int kN1 = 101;           // layer-1 width (hidden - d_in)
constexpr int kCond = 96;
// members of one ensemble: the dense kernel keeps member sets in 64-bit masks and fit_upstream_kernel stages the anchors of
// at most 64 members in shared memory; a larger ensemble runs on the FFMA kernels
constexpr int kMaxMembers = 64;
constexpr int kNP1 = 104;                            // layer-1 MMA width (101 -> 104)
constexpr int kNA = 112, kNB = 88;                   // column halves of the 200-wide layers 2 and 3 (200 = 112 + 88)
constexpr int kKS1 = 13, kKS2 = 7, kKS3 = 13;       // k-steps of 16
// Weight units: each weight set is packed in the order the kernel consumes it, as 8 units of at most kUnitMaxBytes that one
// bulk copy each fills: L1 k-steps 0-6 | 7-12, L2 half a | half b, L3 half a k-steps 0-6 | 7-12, L3 half b k-steps 0-6 | 7-12.
// A unit holds consecutive k-step slabs of one column range: per k-step nw x 16 fp16 hi then nw x 16 fp16 lo (nw x 64 bytes).
constexpr int kUnits = 8;
__host__ __device__ constexpr int unit_layer(int u) { return u < 2 ? 1 : (u < 4 ? 2 : 3); }
__host__ __device__ constexpr int unit_n0(int u) { return (u == 3 || u >= 6) ? kNA : 0; }            // first column
__host__ __device__ constexpr int unit_nw(int u) { return u < 2 ? kNP1 : ((u == 3 || u >= 6) ? kNB : kNA); }
__host__ __device__ constexpr int unit_k0(int u) { return (u == 1 || u == 5 || u == 7) ? 7 : 0; }    // first k-step
__host__ __device__ constexpr int unit_nk(int u) { return (u == 1 || u == 5 || u == 7) ? 6 : 7; }
__host__ __device__ constexpr int unit_bytes(int u) { return unit_nk(u) * unit_nw(u) * 64; }
__host__ __device__ constexpr int unit_off(int u)
{
    int off = 0;
    for (int i = 0; i < u; ++i) off += unit_bytes(i);
    return off;
}
constexpr int kUnitMaxBytes = 7 * kNA * 64;                 // 50176
constexpr int kSetBytes = unit_off(kUnits);                // 342528 per weight set
// the last k-step slab of layer 2 of both column halves, re-built per (query, member) with the latent-dependent bias row
constexpr int kL2SlabABytes = kNA * 64, kL2SlabBytes = (kNA + kNB) * 64;
constexpr int kRecSlots = 3;
// activation derivatives saved per (member, point) for the fitting backward: sigma'0 [208] | sigma'1 [112] | sigma'2 [208] | sigma'3 [208]
constexpr int kActOff0 = 0, kActOff1 = 208, kActOff2 = 320, kActLd = 528;
constexpr int kActPackedSteps = 13;               // sigma'3 goes out operand-ready: 13 k-steps of 8 KB per (member, tile)
// per-(query, member) record, in floats
constexpr int kRecL0 = 0;          // 208 x float4 (W0x row, S*v0), rows >= 200 are zero
constexpr int kRecB1 = 832;        // 112
constexpr int kRecB2 = 944;        // 208
constexpr int kRecB3 = 1152;       // 208
constexpr int kRecW4 = 1360;       // 208
constexpr int kRecMisc = 1568;     // b4, ax, ay, az, has_anchor, mirror, -, -
constexpr int kRecFloats = 1576;

struct Params {
    const uint8_t *weights;     // [n_sets][kSetBytes]
    const float *recs;          // [n_queries][n_members][kRecFloats]
    const uint8_t *l2_slabs;    // [n_queries][n_members][kL2SlabBytes]: last k-step slabs of layer 2 (half a | half b) with the latent-dependent bias row
    const float *xyz;
    const float *axes;
    int res;
    long long first, total, n_points;
    int n_queries;
    long long quirk_period;
    float *out;
    float *members_out;         // optional [n_queries][n_points][n_members]: un-blended member outputs s_k (fitting)
    float *acts_out;            // optional [n_members][tiles][kActLd][128]: activation derivatives of layers 0-2 (fitting backward)
    uint8_t *acts_packed_out;   // with acts_out: [n_members][tiles][acts_packed_tile_steps >= kActPackedSteps][8 KB]: sigma'3 as
    int acts_packed_tile_steps; // packed GEMM operand in the first kActPackedSteps k-steps of every (member, tile) block
    int n_members, n_symm;
    // pruned mode (opt-in): members whose normalised blend weight is < prune_tau for every point of a tile are skipped
    const float *anchors;       // [n_queries][n_members-1][3] (bit for bit the anchors of the records)
    float prune_tau;
    int member_groups;          // activation-dump variant: CTAs per tile (each evaluates a range of members), >= 1
    // dense variant: a tile skips the members whose blend weight is exactly +0 at all of its points (bit-identical result)
    int zero_skip;
    long long n_tiles;          // tiles to process
    // grid mode with compact tiles: blocks of tbx x tby x tbz grid points (tbx tby tbz = 128) over the x-planes px0..px1,
    // by x bz blocks per plane
    int blocked, px0, px1, by, bz, tbx, tby, tbz;
    // pruned and zero-skipping queries: the member mask of every tile, written by the mask pre-pass (tile_mask_kernel)
    unsigned long long *tile_masks;
    // work counter of the on-demand tile schedule: [0] next work item, [1] CTAs finished; zero between launches
    unsigned int *sched;
    // dense grid queries: also skip the members whose blend terms fp32 rounding absorbs (tc_ensemble_wgmma.cu).  The pre-pass
    // writes per tile the members with den + w == den at every valid point (absorb_masks); member_bound_kernel writes
    // B >= |s_k| per (query, member) (bounds, +inf: never skipped)
    int absorb;
    unsigned long long *absorb_masks;
    const float *bounds;
    // debug (nphm_debug_ens_skip_log): per tile, bit m set when the producer skipped member m by vote; nullptr unless enabled
    unsigned long long *skip_log;
    // member-major dense grid queries (tc_ensemble_wgmma.cu, member_pass_kernel): a chunk of whole tiles mm_t0 ..
    // mm_t0 + mm_tiles - 1 keeps num and den per row (index (tile - mm_t0) * 128 + row); the pass of member mm_member lists
    // the rows that still need it in mm_list and counts them in mm_count[mm_member]
    int mm_member;
    long long mm_t0, mm_tiles;
    float *mm_num, *mm_den;
    int *mm_list;
    unsigned int *mm_count;
    // member bounds per 32^3-point sub-box of the grid (member_bound_kernel over the sub-box): [sub-box][member], sub-boxes
    // (sx - sub_x0, sy, sz) in x-major order, sub_n per axis; nullptr: the whole-box bounds
    const float *sub_bounds;
    int sub_x0, sub_n;
};

// One row (point) of a tile: its index in the query, its global point index, whether the tile covers a real point with
// this row, and its coordinates.  The ensemble kernel and the mask pre-pass both call this function, so that they cannot
// disagree about a point.  `blocked`: compact grid blocks (Params::tbx, tby, tbz); otherwise 128 consecutive points of
// query qi (from p.xyz, or grid points from p.axes).
struct TilePoint {
    long long idx, g;
    bool valid;
    float x, y, z;
    int ix, iy, iz;            // grid coordinates (grid queries), clamped to the grid
};
__device__ __forceinline__ TilePoint tile_point(const Params &p, bool blocked, long long tile, int qi,
                                                long long tiles_per_query, int row)
{
    TilePoint t;
    if (blocked) {
        // compact tbx x tby x tbz block of grid points (z fastest inside the block)
        const long long tz = tile % p.bz, txy = tile / p.bz;
        const int ty = (int)(txy % p.by), tx = (int)(txy / p.by);
        const int ix = p.px0 + tx * p.tbx + row / (p.tby * p.tbz), iy = ty * p.tby + (row / p.tbz) % p.tby,
                  iz = (int)tz * p.tbz + row % p.tbz;
        t.g = ((long long)ix * p.res + iy) * p.res + iz;
        t.valid = ix <= p.px1 && iy < p.res && iz < p.res && t.g >= p.first && t.g < p.first + p.n_points;
        t.idx = t.g - p.first;
        const int cx_ = min(ix, p.res - 1), cy_ = min(iy, p.res - 1), cz_ = min(iz, p.res - 1);
        t.x = __ldg(p.axes + cx_); t.y = __ldg(p.axes + p.res + cy_); t.z = __ldg(p.axes + 2 * p.res + cz_);
        t.ix = cx_; t.iy = cy_; t.iz = cz_;
        if (!t.valid) t.g = p.first;
    } else {
        t.idx = (tile - (long long)qi * tiles_per_query) * 128 + row;
        t.valid = t.idx < p.n_points;
        t.g = p.first + (t.valid ? t.idx : 0);
        if (p.xyz) {
            const float *pp = p.xyz + ((size_t)qi * p.n_points + (t.valid ? t.idx : 0)) * 3;
            t.x = pp[0]; t.y = pp[1]; t.z = pp[2];
            t.ix = t.iy = t.iz = 0;
        } else {
            const long long rr = (long long)p.res * p.res;
            const int ix = (int)(t.g / rr), iy = (int)((t.g - ix * rr) / p.res), iz = (int)(t.g % p.res);
            t.x = __ldg(p.axes + ix); t.y = __ldg(p.axes + p.res + iy); t.z = __ldg(p.axes + 2 * p.res + iz);
            t.ix = ix; t.iy = iy; t.iz = iz;
        }
    }
    return t;
}

// Blend weight of a member at (x, y, z): exp(-(|a - x| + 1e-5)^2 / 0.01) for a member with anchor a, exp(-20) for the
// global member.  The tile masks and the blend call this one function with the same inputs, so that a member skipped for
// an exactly zero weight is one whose blend term would have been exactly zero.  The squared distance is spelled out as
// fma(dz, dz, fma(dx, dx, dy * dy)), the contraction the compiler chose for dx * dx + dy * dy + dz * dz in the kernel before
// this function existed, so that no inlining context can contract it another way.
__device__ __forceinline__ float blend_weight(bool has_anchor, float ax, float ay, float az, float x, float y, float z)
{
    float d = -0.2f;
    if (has_anchor) {
        const float dx = ax - x, dy = ay - y, dz = az - z;
        const float nrm = sqrtf(__fmaf_rn(dz, dz, __fmaf_rn(dx, dx, __fmul_rn(dy, dy)))) + 10e-6f;
        d = -(nrm * nrm);
    }
    return expf(__fdiv_rn(d, 0.01f));
}

// Blend weight of member k of query qi (anchors `anc` = p.anchors of that query; the last member is the global one)
__device__ __forceinline__ float member_weight(const float *anc, int k, int n_members, float x, float y, float z)
{
    if (k == n_members - 1) return blend_weight(false, 0.f, 0.f, 0.f, x, y, z);
    return blend_weight(true, __ldg(anc + 3 * k), __ldg(anc + 3 * k + 1), __ldg(anc + 3 * k + 2), x, y, z);
}

// The pruned rule's normaliser at a point: S = sum_k w_k, summed in member order
__device__ __forceinline__ float weight_sum(const float *anc, int n_members, float x, float y, float z)
{
    float S = 0.f;
    for (int k = 0; k < n_members; ++k) S += member_weight(anc, k, n_members, x, y, z);
    return S;
}

int launch_ensemble_wgmma(const Params &p, bool prune, bool acts, int grid_x, cudaStream_t stream);
// member-major order of a dense grid query with absorption (p.mm_* set, chunk of at most kMmChunkTiles tiles): per member,
// the pass that blends quirk rows, skips absorbed rows and lists the rest, then the ensemble kernel on that list
constexpr long long kMmChunkTiles = 1ll << 17;     // 2^24 rows: 12 B of state per row
int launch_member_major_chunk(const Params &p, int grid_x, cudaStream_t stream);
int launch_ensemble_mask(const Params &p, bool prune, cudaStream_t stream);

}  // namespace tc
}  // namespace nphm
