// Warpgroup-MMA (wgmma, sm_90a) kernel for the identity-SDF ensemble.
//
// Reference semantics: FastEnsembleDeepSDFMirrored.forward  src/NPHM/models/EnsembledDeepSDF.py:203-267
// Math, weight slabs and per-(query, member) records are those of tc_ensemble.cu (see the header there).
//
// A CTA is persistent over 128-point tiles: two consumer warpgroups of 64 points each and one producer warpgroup, which
// hands most of its registers to the consumers (setmaxnreg: 24 / 240 per thread).
//   producer (warp 8, one lane): bulk async copies of the record of every member and of its 8 weight units (tc_ensemble.cuh)
//       into a ring of 4 shared-memory slots (one mbarrier pair each), up to 4 units ahead of the consumers.  A slot is
//       released when the MMAs of both warpgroups on it have retired.
//   consumers (warps 0-7): per member, layer 0 on CUDA cores straight into registers; layers 1-3 as 64 x N x 16 wgmmas with
//       A in REGISTERS and B (weights) in shared memory.  The accumulator layout of a 64 x N wgmma is the register layout of
//       its A operand (tc_common.cuh), so the epilogue of a layer (softplus, fp16 hi/lo split) produces the next layer's A
//       operand in place, without a round trip through memory.  The output layer (dot with w4) and the anchor blend run on
//       the accumulator registers of layer 3.
// Wide layers are issued in two column halves (112 + 88) so that the accumulators and the A operand of a layer fit the
// register file together: the first half of layer 2 is converted while the MMAs of the second half run.  MMA issue
// alternates between the two warpgroups phase by phase (layer 1, layer 2, layer 3 half a, layer 3 half b), so that one
// warpgroup's epilogue (and its next member's layer 0) runs while the other one's MMAs occupy the tensor cores.  The
// accumulation order of every output is that of a single warpgroup running alone: the results do not depend on the offset.
// Tiles are handed out on demand: the producer lane takes the next work item from a device counter, reads the item's member
// mask and passes (item, mask) to the consumers through a two-deep queue in shared memory, so that no SM idles while others
// still have tiles, and the producer streams the next tile's weights while the consumers finish the current one.  A mask
// pre-pass (tile_mask_kernel) computes which members each tile needs (dense: a blend weight that is not exactly zero at
// some valid point; pruned: the tau rule) and the producer streams only those; grid queries use compact tiles
// (Params::tbx, tby, tbz) so that a tile lies far from many anchors.
#include "tc_ensemble.cuh"

namespace nphm {
namespace tc {
namespace wg {

#ifdef NPHM_ENS_TRACE
// Timeline of CTA 0 (tools/ens_trace.py): clock64 stamps of kTraceMembers consecutive members, from the kTraceFirst-th member
// the CTA evaluates.  [0] = CTA start, then per member kTraceStride stamps: consumer warpgroup 0 | warpgroup 1 (kTraceWg each:
// phase p (L1, L2, L3 half a, L3 half b) event e at 6 p + e, e = weight wait start, weights ready, MMA issue start, MMAs
// issued, MMAs retired, epilogue done; member start at 24, layer 0 done at 25) | producer (unit u issued at u, slot wait
// start at 8 + u).
constexpr int kTraceFirst = 4, kTraceMembers = 4, kTraceWg = 32, kTraceStride = 2 * kTraceWg + 16;
__device__ long long g_ens_trace[1 + kTraceMembers * kTraceStride];
// Tile boundaries of CTA 0, for its first kTraceTiles tiles: warpgroup 0 takes the tile (and its member mask) from the queue,
// the producer knows the tile's mask, warpgroup 0 has the layer-1 weights of the tile's first member.
constexpr int kTraceTiles = 4;
__device__ long long g_ens_tiles[3 * kTraceTiles];
// Work of every CTA: [0] = CTAs of the last launch, then per CTA the member-tiles it evaluated and its cycles.
constexpr int kTraceMaxCtas = 1024;
__device__ long long g_ens_ctas[1 + 2 * kTraceMaxCtas];
#define ENS_STAMP(member, off) do { const int mi_ = (int)(member) - kTraceFirst;                                           \
        if (blockIdx.x == 0 && mi_ >= 0 && mi_ < kTraceMembers) g_ens_trace[1 + mi_ * kTraceStride + (off)] = clock64(); } while (0)
#define ENS_CEVT(member, phase, e) do { if ((threadIdx.x & 127) == 0)                                                       \
        ENS_STAMP(member, (threadIdx.x >> 7) * kTraceWg + 6 * (phase) + (e)); } while (0)
#define ENS_CMARK(member, off) do { if ((threadIdx.x & 127) == 0) ENS_STAMP(member, (threadIdx.x >> 7) * kTraceWg + (off)); } while (0)
#define ENS_PEVT(member, off) ENS_STAMP(member, 2 * kTraceWg + (off))
#define ENS_TILE(t, e) do { if (blockIdx.x == 0 && (t) < kTraceTiles) g_ens_tiles[3 * (t) + (e)] = clock64(); } while (0)
#else
#define ENS_CEVT(member, phase, e) do { } while (0)
#define ENS_CMARK(member, off) do { } while (0)
#define ENS_PEVT(member, off) do { } while (0)
#define ENS_TILE(t, e) do { } while (0)
#endif

constexpr int kConsumerWarps = 8;
constexpr int kThreads = 32 * (kConsumerWarps + 4);
constexpr int kUnits208 = 13, kUnits112 = 7;
constexpr int kSlots = 4;                      // weight ring: unit u of every member lands in slot u % 4
constexpr int kTurnBar = 1;                    // named barriers kTurnBar + w: "warpgroup w may issue its MMAs"
static_assert(kUnits == 2 * kSlots, "unit u uses slot u % 4 on its (u / 4)-th use per member");

struct __align__(128) Smem {
    uint8_t wbuf[kSlots][kUnitMaxBytes];     // weight units (one bulk copy + one barrier each)
    float rec[kRecSlots][kRecFloats];
    uint64_t w_full[kSlots], w_empty[kSlots];
    uint64_t rec_full[kRecSlots], rec_empty[kRecSlots];
    // tile queue (producer -> consumers): work item (-1 = no more work) and member mask of the next two tiles
    uint64_t q_full[2], q_empty[2];
    long long q_item[2];
    unsigned long long q_mask[2];
};
static_assert(sizeof(Smem) <= 227 * 1024, "shared memory of the ensemble kernel exceeds the 227 KB of an H100 block");

// 3 MMAs of one k-step (hi*hi + hi*lo + lo*hi): `b` = shared address of the slab's hi half, its lo half lies lo_off further
template <int N, typename F>
__device__ __forceinline__ void kstep(F &&mma, float (&d)[N / 2], const uint32_t (&ah)[4], const uint32_t (&al)[4], uint32_t b,
                                      uint32_t lo_off)
{
    const uint64_t bh = make_desc(b, 128, 256), bl = make_desc(b + lo_off, 128, 256);
    mma(d, ah, bh, 1);
    mma(d, ah, bl, 1);
    mma(d, al, bh, 1);
}

// k-step j of an accumulator -> A registers of the next layer.  f(value, column, row 0/1, element) returns the activation;
// columns beyond the accumulator (the constant columns of the next layer's operand) pass 0 as the value.
template <int N, typename F>
__device__ __forceinline__ void to_operand(const float (&d)[N], int j, int col0, int q4, uint32_t (&ah)[4], uint32_t (&al)[4], F &&f)
{
    float v[2][4];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh)
#pragma unroll
        for (int r = 0; r < 2; ++r)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int col = col0 + 16 * j + 8 * hh + 2 * q4 + e;
                v[r][2 * hh + e] = f(4 * (2 * j + hh) < N ? d[4 * (2 * j + hh) + 2 * r + e] : 0.f, col, r, 2 * hh + e);
            }
    split2(v[0][0], v[0][1], ah[0], al[0]);
    split2(v[1][0], v[1][1], ah[1], al[1]);
    split2(v[0][2], v[0][3], ah[2], al[2]);
    split2(v[1][2], v[1][3], ah[3], al[3]);
}

// Mask pre-pass: one warp per tile, 4 rows per lane; bit k of p.tile_masks[tile] is set when the tile needs member k.  The
// last, global member is always needed: every tile evaluates >= 1 member.  Dense rule: a member is needed if w_k != 0 at some
// valid point - a member with w_k = +0 everywhere adds exactly nothing to num and den (denormal weights count as nonzero).
// Pruned rule: S = sum_k w_k; a member is needed if w_k >= tau * (S + 1e-6) at some valid point (dropped mass per point
// < n_members * tau).  Points and weights come from tile_point and member_weight, as in the ensemble kernel.
constexpr int kMaskWarps = 8;
template <bool PRUNE>
__global__ void __launch_bounds__(32 * kMaskWarps) tile_mask_kernel(const Params p)
{
    const long long tile = (long long)blockIdx.x * kMaskWarps + (threadIdx.x >> 5);
    if (tile >= p.n_tiles) return;
    const int lane = threadIdx.x & 31;
    const long long tiles_per_query = p.blocked ? p.n_tiles : (p.n_points + 127) / 128;
    const int qi = p.blocked ? 0 : (int)(tile / tiles_per_query);
    const float *anc = p.anchors + (size_t)qi * (p.n_members - 1) * 3;
    TilePoint pt[4];
    float thr[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        pt[i] = tile_point(p, p.blocked, tile, qi, tiles_per_query, lane + 32 * i);
        thr[i] = PRUNE ? p.prune_tau * (weight_sum(anc, p.n_members, pt[i].x, pt[i].y, pt[i].z) + 1e-6f) : 0.f;
    }
    unsigned long long mask = 1ull << (p.n_members - 1);
    for (int k = 0; k < p.n_members - 1; ++k) {
        bool need = false;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            if (!pt[i].valid) continue;
            const float w = member_weight(anc, k, p.n_members, pt[i].x, pt[i].y, pt[i].z);
            need |= PRUNE ? w >= thr[i] : w != 0.f;
        }
        if (__any_sync(0xffffffffu, need)) mask |= 1ull << k;
    }
    if (lane == 0) p.tile_masks[tile] = mask;
}

template <bool PRUNE, bool ACTS>
__global__ void __launch_bounds__(kThreads, 1) ensemble_wgmma_kernel(const Params p)
{
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    Smem &sm = *reinterpret_cast<Smem *>(smem_raw);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long tiles_per_query = p.blocked ? p.n_tiles : (p.n_points + 127) / 128;
    const long long n_tiles = p.n_tiles;
    // ACTS (fitting: few points, so few tiles): the members of a tile are split over `member_groups` CTAs - a work item is
    // (tile, group of consecutive members), the in-kernel blend is meaningless then and `out` is not written
    const int n_groups = ACTS ? p.member_groups : 1;
    const long long n_items = n_tiles * n_groups;
    auto group_mask = [&](long long item) -> unsigned long long {
        const unsigned long long all = p.n_members >= 64 ? ~0ull : (1ull << p.n_members) - 1;
        if (!ACTS || n_groups == 1) return all;
        const int per = (p.n_members + n_groups - 1) / n_groups, lo = (int)(item % n_groups) * per;
        const int hi = min(p.n_members, lo + per);
        return ((1ull << hi) - 1) & ~((1ull << lo) - 1);
    };

    if (threadIdx.x == 0) {
        for (int i = 0; i < kSlots; ++i) { mbar_init(&sm.w_full[i], 1); mbar_init(&sm.w_empty[i], kConsumerWarps); }
        for (int i = 0; i < kRecSlots; ++i) { mbar_init(&sm.rec_full[i], 1); mbar_init(&sm.rec_empty[i], kConsumerWarps); }
        for (int i = 0; i < 2; ++i) { mbar_init(&sm.q_full[i], 1); mbar_init(&sm.q_empty[i], kConsumerWarps); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
#ifdef NPHM_ENS_TRACE
    const long long cta_start = clock64();
    if (blockIdx.x == 0 && threadIdx.x == 0) { g_ens_trace[0] = cta_start; g_ens_ctas[0] = gridDim.x; }
#endif
    // tile masks from the pre-pass: the pruned rule, or (dense variant) exactly zero blend weights
    const bool premask = PRUNE || (!ACTS && p.zero_skip);

    if (warp >= kConsumerWarps) {
        // =========================================================================== producer (tiles, bulk async copies)
        asm volatile("setmaxnreg.dec.sync.aligned.u32 24;" ::: "memory");
        if (warp == kConsumerWarps && lane == 0) {
            uint32_t rcount = 0;
            for (uint32_t tcount = 0;; ++tcount) {
                // take the next work item and pass it on with its member mask (the end of the work as item -1)
                const unsigned int item = atomicAdd(p.sched, 1u);
                const bool more = item < n_items;
                const unsigned int tile = ACTS ? item / n_groups : item;
                const int qi = p.blocked ? 0 : (int)(tile / (unsigned int)tiles_per_query);
                unsigned long long mask = !more ? 0ull : (premask ? p.tile_masks[tile] : group_mask(item));
                ENS_TILE(tcount, 1);
                const int qs = tcount & 1;
                mbar_wait(&sm.q_empty[qs], ((tcount >> 1) & 1) ^ 1);
                sm.q_item[qs] = more ? (long long)item : -1;
                sm.q_mask[qs] = mask;
                mbar_arrive(&sm.q_full[qs]);
                if (!more) break;
                for (; mask; mask &= mask - 1) {         // the tile's members in ascending order
                    const int m = __ffsll((long long)mask) - 1;
                    const int rslot = rcount % kRecSlots;
                    mbar_wait(&sm.rec_empty[rslot], ((rcount / kRecSlots) & 1) ^ 1);
                    mbar_expect_tx(&sm.rec_full[rslot], kRecFloats * 4);
                    bulk_g2s(sm.rec[rslot], p.recs + ((size_t)qi * p.n_members + m) * kRecFloats, kRecFloats * 4, &sm.rec_full[rslot]);
                    ++rcount;
                    const int set = m < 2 * p.n_symm ? (m >> 1) : m - p.n_symm;
                    const uint8_t *w = p.weights + (size_t)set * kSetBytes;
                    const uint8_t *l2 = p.l2_slabs + ((size_t)qi * p.n_members + m) * kL2SlabBytes;
#pragma unroll 1
                    for (int u = 0; u < kUnits; ++u) {
                        // every member has 8 units, so unit u always goes to slot u % 4, on its (u / 4)-th use per member
                        const int slot = u & 3;
                        const uint32_t bytes = unit_bytes(u);
                        ENS_PEVT(rcount - 1, 8 + u);
                        mbar_wait(&sm.w_empty[slot], ((u >> 2) & 1) ^ 1);
                        ENS_PEVT(rcount - 1, u);
                        mbar_expect_tx(&sm.w_full[slot], bytes);
                        if (u == 2 || u == 3) {
                            // layer 2: the last k-step slab carries this (query, member)'s bias row (l2_slab_kernel)
                            const uint32_t last = unit_nw(u) * 64;
                            bulk_g2s(sm.wbuf[slot], w + unit_off(u), bytes - last, &sm.w_full[slot]);
                            bulk_g2s(sm.wbuf[slot] + (bytes - last), l2 + (u == 3 ? kL2SlabABytes : 0), last, &sm.w_full[slot]);
                        } else {
                            bulk_g2s(sm.wbuf[slot], w + unit_off(u), bytes, &sm.w_full[slot]);
                        }
                    }
                }
            }
            // every CTA has taken its last item once all have counted themselves finished: the last one resets the counter
            // for the next launch on the stream
            __threadfence();
            if (atomicAdd(p.sched + 1, 1u) == gridDim.x - 1) {
                atomicExch(p.sched, 0u);
                atomicExch(p.sched + 1, 0u);
            }
        }
        return;
    }

    // =========================================================================== consumer warpgroups
    asm volatile("setmaxnreg.inc.sync.aligned.u32 240;" ::: "memory");
    const int q4 = lane & 3, wgi = warp >> 2;
    int rl[2];                                   // tile rows (points) of this thread's accumulator rows
    rl[0] = 64 * wgi + 16 * (warp & 3) + (lane >> 2);
    rl[1] = rl[0] + 8;
    uint32_t rcount = 0;
    auto release = [&](int u) { __syncwarp(); if (lane == 0) mbar_arrive(&sm.w_empty[u & 3]); };
    auto release_rec = [&](uint64_t *bar) { __syncwarp(); if (lane == 0) mbar_arrive(bar); };
    auto wait_unit = [&](int u) { mbar_wait(&sm.w_full[u & 3], (u >> 2) & 1); };
    auto unit_addr = [&](int u) { return smem_u32(sm.wbuf[u & 3]); };
    // MMA issue alternates between the warpgroups, phase by phase (named barriers kTurnBar + warpgroup): a warpgroup
    // issues, hands the turn to the other one and runs its epilogue while the other warpgroup's MMAs occupy the tensor cores.
    auto take_turn = [&]() {
        if (wgi == 0) asm volatile("bar.sync %0, 256;" ::"n"(kTurnBar) : "memory");
        else asm volatile("bar.sync %0, 256;" ::"n"(kTurnBar + 1) : "memory");
    };
    auto pass_turn = [&]() {
        if (wgi == 0) asm volatile("bar.arrive %0, 256;" ::"n"(kTurnBar + 1) : "memory");
        else asm volatile("bar.arrive %0, 256;" ::"n"(kTurnBar) : "memory");
    };
    if (wgi == 1) pass_turn();                   // warpgroup 0 issues first

    for (uint32_t tcount = 0;; ++tcount) {
        // the next tile and its member mask from the producer's queue: no vote and no wait for the other warpgroup, so the
        // phase offset of the warpgroups carries over from one tile to the next
        const int qs = tcount & 1;
        mbar_wait(&sm.q_full[qs], (tcount >> 1) & 1);
        const long long item = sm.q_item[qs];
        const unsigned long long mask = sm.q_mask[qs];
        __syncwarp();
        if (lane == 0) mbar_arrive(&sm.q_empty[qs]);
        if (item < 0) break;
        if (threadIdx.x == 0) ENS_TILE(tcount, 0);
        const long long tile = ACTS ? item / n_groups : item;
        const int qi = p.blocked ? 0 : (int)(tile / tiles_per_query);
        long long idx[2], g[2];
        bool valid[2], quirk[2];
        float x[2], y[2], z[2];
        float num[2] = {0.f, 0.f}, den[2] = {0.f, 0.f};
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            // (the fitting variant only runs linear tiles)
            const TilePoint t = tile_point(p, !ACTS && p.blocked, tile, qi, tiles_per_query, rl[i]);
            idx[i] = t.idx; g[i] = t.g; valid[i] = t.valid; x[i] = t.x; y[i] = t.y; z[i] = t.z;
            quirk[i] = p.quirk_period > 0 && ((g[i] % p.quirk_period) == p.quirk_period - 1 || g[i] == p.total - 1);
            // pruned rule: the blend divides by S = sum_k w_k over all members, evaluated or not
            if (PRUNE) den[i] = weight_sum(p.anchors + (size_t)qi * (p.n_members - 1) * 3, p.n_members, x[i], y[i], z[i]);
        }
        const uint32_t tile_rc0 = rcount;        // the tile's first member (timeline build)

        for (int m = 0; m < p.n_members; ++m) {
            if (!((mask >> m) & 1)) continue;
            const uint32_t rslot = rcount % kRecSlots;
            ENS_CMARK(rcount, 24);
            mbar_wait(&sm.rec_full[rslot], (rcount / kRecSlots) & 1);
            const float *rec = sm.rec[rslot];
            float cx[2], cy[2], cz[2];
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                cx[i] = x[i] - rec[kRecMisc + 1]; cy[i] = y[i] - rec[kRecMisc + 2]; cz[i] = z[i] - rec[kRecMisc + 3];
                if (rec[kRecMisc + 5] != 0.f) cx[i] = -cx[i];          // mirrored member
                cx[i] *= kS; cy[i] *= kS; cz[i] *= kS;                 // coordinates in log2 units
            }
            // activation derivatives for the fitting backward, sigma'(pre) = 1 - 2^(-softplus) (log2 units): per (member, tile) a
            // block of kActLd features x 128 points, feature-major, tiles numbered over all queries (the tiles of query qi follow
            // those of query qi - 1).  Columns beyond a layer's width receive don't-care values.
            float *const ab = ACTS ? p.acts_out + ((size_t)m * n_tiles + tile) * kActLd * 128 : nullptr;
            auto save_act = [&](int off, int col, int r, float v) {
                if (ACTS) {
                    float ex;
                    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(ex) : "f"(-v));
                    ab[(size_t)(off + col) * 128 + rl[r]] = 1.0f - ex;
                }
            };

            // ---------------- layer 0 on CUDA cores -> A operand of layer 1 (K 208: h0 (200) | 1.0 (bias row) | zeros)
            uint32_t a0h[kUnits208][4], a0l[kUnits208][4];
#pragma unroll
            for (int j = 0; j < kUnits208; ++j) {
                float v[2][4];
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const int col = 16 * j + 8 * (c >> 1) + 2 * q4 + (c & 1);
                    const float4 w = reinterpret_cast<const float4 *>(rec + kRecL0)[col];
#pragma unroll
                    for (int r = 0; r < 2; ++r) {
                        float a;
                        if (col < kH) a = sp_sel(fmaf(w.x, cx[r], fmaf(w.y, cy[r], fmaf(w.z, cz[r], w.w))), c);
                        else a = col == kH ? 1.0f : 0.0f;
                        save_act(kActOff0, col, r, a);
                        v[r][c] = a;
                    }
                }
                split2(v[0][0], v[0][1], a0h[j][0], a0l[j][0]);
                split2(v[1][0], v[1][1], a0h[j][1], a0l[j][1]);
                split2(v[0][2], v[0][3], a0h[j][2], a0l[j][2]);
                split2(v[1][2], v[1][3], a0h[j][3], a0l[j][3]);
            }
            ENS_CMARK(rcount, 25);

            // ---------------- layer 1 (N 104, K 208: units 0 | 1)
            float acc1[kNP1 / 2];
#pragma unroll
            for (int i = 0; i < kNP1 / 2; ++i) acc1[i] = 0.f;
            ENS_CEVT(rcount, 0, 0);
            wait_unit(0);
            wait_unit(1);
            ENS_CEVT(rcount, 0, 1);
            if (threadIdx.x == 0 && rcount == tile_rc0) ENS_TILE(tcount, 2);
            take_turn();
            ENS_CEVT(rcount, 0, 2);
            {
                wg_fence();
#pragma unroll
                for (int j = 0; j < kUnits208; ++j) {
                    kstep<kNP1>(wgmma_rs_n104, acc1, a0h[j], a0l[j], unit_addr(j < 7 ? 0 : 1) + (j % 7) * kNP1 * 64, kNP1 * 32);
                }
                wg_commit();
                pass_turn();
                ENS_CEVT(rcount, 0, 3);
                wg_wait<0>();
                wg_reg_fence(acc1);
                ENS_CEVT(rcount, 0, 4);
            }
            release(0);
            release(1);

            // ---------------- epilogue of layer 1 -> A operand of layer 2 (K 112: h1 (101) | c (3) | 1.0 (bias row) | zeros)
            uint32_t a1h[kUnits112][4], a1l[kUnits112][4];
#pragma unroll
            for (int j = 0; j < kUnits112; ++j)
                to_operand(acc1, j, 0, q4, a1h[j], a1l[j], [&](float t, int col, int r, int e) {
                    float a;
                    if (col < kN1) a = sp_sel(t, e);
                    else if (col < kN1 + 3) a = col == kN1 ? cx[r] : (col == kN1 + 1 ? cy[r] : cz[r]);
                    else a = col == kN1 + 3 ? 1.0f : 0.0f;
                    save_act(kActOff1, col, r, a);
                    return a;
                });
            ENS_CEVT(rcount, 0, 5);

            // ---------------- layer 2 (N 200 = 112 (unit 2) + 88 (unit 3), K 112): the first half is converted while the
            // second one runs
            float acc2a[kNA / 2], acc2b[kNB / 2];
#pragma unroll
            for (int i = 0; i < kNA / 2; ++i) acc2a[i] = 0.f;
#pragma unroll
            for (int i = 0; i < kNB / 2; ++i) acc2b[i] = 0.f;
            ENS_CEVT(rcount, 1, 0);
            wait_unit(2);
            wait_unit(3);
            ENS_CEVT(rcount, 1, 1);
            take_turn();
            ENS_CEVT(rcount, 1, 2);
            uint32_t a2h[kUnits208][4], a2l[kUnits208][4];
            auto e2 = [&](float t, int col, int r, int e) {
                const float a = col < kH ? sp_sel(t, e) : (col == kH ? 1.0f : 0.0f);     // k = 200: bias row of layer 3
                save_act(kActOff2, col, r, a);
                return a;
            };
            {
                wg_fence();
#pragma unroll
                for (int j = 0; j < kUnits112; ++j)
                    kstep<kNA>(wgmma_rs_n112, acc2a, a1h[j], a1l[j], unit_addr(2) + j * kNA * 64, kNA * 32);
                wg_commit();
#pragma unroll
                for (int j = 0; j < kUnits112; ++j)
                    kstep<kNB>(wgmma_rs_n88, acc2b, a1h[j], a1l[j], unit_addr(3) + j * kNB * 64, kNB * 32);
                wg_commit();
                pass_turn();
                ENS_CEVT(rcount, 1, 3);
                wg_wait<1>();
                wg_reg_fence(acc2a);
                release(2);
#pragma unroll
                for (int j = 0; j < 7; ++j) to_operand(acc2a, j, 0, q4, a2h[j], a2l[j], e2);
                wg_wait<0>();
                wg_reg_fence(acc2b);
                ENS_CEVT(rcount, 1, 4);
            }
            release(3);
#pragma unroll
            for (int j = 0; j < 6; ++j) to_operand(acc2b, j, kNA, q4, a2h[7 + j], a2l[7 + j], e2);
            ENS_CEVT(rcount, 1, 5);

            // ---------------- layer 3 (N 200 = 112 (units 4, 5) + 88 (units 6, 7), K 208) and the output layer w4 . h3 + b4
            float part[2] = {0.f, 0.f};
            // sigma'3 is the A operand of the first backward GEMM: saved operand-ready (tc_linear.cuh "packed": per k-step = unit
            // of 16 features [128 x 16 fp16 hi | 128 x 16 fp16 lo], core-matrix order), zeros in the K padding
            uint8_t *const pk = ACTS ? p.acts_packed_out + ((size_t)m * n_tiles + tile) * p.acts_packed_tile_steps * 8192
                                     : nullptr;
            auto out_layer = [&](const auto &acc, int col0, int units) {
                constexpr int kAcc = sizeof(acc) / sizeof(float);
#pragma unroll
                for (int j = 0; j < units; ++j)
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh)
#pragma unroll
                        for (int r = 0; r < 2; ++r) {
                            float v[2] = {0.f, 0.f};
                            if (4 * (2 * j + hh) < kAcc) {          // columns 200-207 have no accumulator (w4 is zero there)
#pragma unroll
                                for (int e = 0; e < 2; ++e) {
                                    const int col = col0 + 16 * j + 8 * hh + 2 * q4 + e;
                                    v[e] = sp_sel(acc[4 * (2 * j + hh) + 2 * r + e], e);
                                    part[r] = fmaf(v[e], rec[kRecW4 + col], part[r]);
                                    if (ACTS) {
                                        float ex;
                                        asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(ex) : "f"(-v[e]));
                                        v[e] = 1.0f - ex;
                                    }
                                }
                            }
                            if (ACTS) {
                                uint32_t hi, lo;
                                split2(v[0], v[1], hi, lo);
                                const int row = rl[r], u = (col0 >> 4) + j;
                                uint8_t *dst = pk + (size_t)u * 8192 + (size_t)(row >> 3) * 256 + (size_t)hh * 128 + (size_t)(row & 7) * 16 + 4 * q4;
                                *reinterpret_cast<uint32_t *>(dst) = hi;
                                *reinterpret_cast<uint32_t *>(dst + 4096) = lo;
                            }
                        }
            };
            {
                float acc3[kNA / 2];
#pragma unroll
                for (int i = 0; i < kNA / 2; ++i) acc3[i] = 0.f;
                ENS_CEVT(rcount, 2, 0);
                wait_unit(4);
                wait_unit(5);
                ENS_CEVT(rcount, 2, 1);
                take_turn();
                ENS_CEVT(rcount, 2, 2);
                wg_fence();
#pragma unroll
                for (int j = 0; j < kUnits208; ++j) {
                    kstep<kNA>(wgmma_rs_n112, acc3, a2h[j], a2l[j], unit_addr(j < 7 ? 4 : 5) + (j % 7) * kNA * 64, kNA * 32);
                }
                wg_commit();
                pass_turn();
                ENS_CEVT(rcount, 2, 3);
                wg_wait<0>();
                wg_reg_fence(acc3);
                ENS_CEVT(rcount, 2, 4);
                release(4);
                release(5);
                out_layer(acc3, 0, 7);
                ENS_CEVT(rcount, 2, 5);
            }
            {
                float acc3[kNB / 2];
#pragma unroll
                for (int i = 0; i < kNB / 2; ++i) acc3[i] = 0.f;
                ENS_CEVT(rcount, 3, 0);
                wait_unit(6);
                wait_unit(7);
                ENS_CEVT(rcount, 3, 1);
                take_turn();
                ENS_CEVT(rcount, 3, 2);
                wg_fence();
#pragma unroll
                for (int j = 0; j < kUnits208; ++j) {
                    kstep<kNB>(wgmma_rs_n88, acc3, a2h[j], a2l[j], unit_addr(j < 7 ? 6 : 7) + (j % 7) * kNB * 64, kNB * 32);
                }
                wg_commit();
                pass_turn();
                ENS_CEVT(rcount, 3, 3);
                wg_wait<0>();
                wg_reg_fence(acc3);
                ENS_CEVT(rcount, 3, 4);
                release(6);
                release(7);
                out_layer(acc3, kNA, 6);
                ENS_CEVT(rcount, 3, 5);
            }

            // ---------------- member output (reduced over the 4 lanes of a row) and the anchor blend
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                float s = part[r];
                s += __shfl_xor_sync(0xffffffffu, s, 1);
                s += __shfl_xor_sync(0xffffffffu, s, 2);
                s += rec[kRecMisc + 0];
                if (q4 == 0 && p.members_out && valid[r]) p.members_out[((size_t)qi * p.n_points + idx[r]) * p.n_members + m] = s;
                const float w = blend_weight(rec[kRecMisc + 4] != 0.f, rec[kRecMisc + 1], rec[kRecMisc + 2], rec[kRecMisc + 3],
                                             x[r], y[r], z[r]);
                num[r] = fmaf(w, quirk[r] ? 1.0f : s, num[r]);
                if (!PRUNE) den[r] += w;
            }
            release_rec(&sm.rec_empty[rslot]);
            ++rcount;
        }
#pragma unroll
        for (int r = 0; r < 2; ++r)
            if (q4 == 0 && valid[r] && n_groups == 1) p.out[(size_t)qi * p.n_points + idx[r]] = __fdiv_rn(num[r], den[r] + 1e-6f);
    }
    if (wgi == 0) take_turn();                   // the turn warpgroup 1 passed after its last phase
#ifdef NPHM_ENS_TRACE
    if (threadIdx.x == 0 && blockIdx.x < kTraceMaxCtas) {
        g_ens_ctas[1 + 2 * blockIdx.x] = rcount;
        g_ens_ctas[2 + 2 * blockIdx.x] = clock64() - cta_start;
    }
#endif
}

}  // namespace wg

int launch_ensemble_wgmma(const Params &p, bool prune, bool acts, int grid_x, cudaStream_t stream)
{
    if (prune || (!acts && p.zero_skip)) {
        const unsigned blocks = (unsigned)ceil_div(p.n_tiles, (long long)wg::kMaskWarps);
        if (prune) wg::tile_mask_kernel<true><<<blocks, 32 * wg::kMaskWarps, 0, stream>>>(p);
        else wg::tile_mask_kernel<false><<<blocks, 32 * wg::kMaskWarps, 0, stream>>>(p);
        NPHM_CUDA_CHECK(cudaGetLastError());
    }
    const int smem = (int)sizeof(wg::Smem);
    auto kern = acts ? wg::ensemble_wgmma_kernel<false, true>
                     : (prune ? wg::ensemble_wgmma_kernel<true, false> : wg::ensemble_wgmma_kernel<false, false>);
    NPHM_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    kern<<<grid_x, wg::kThreads, smem, stream>>>(p);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

}  // namespace tc
}  // namespace nphm

#ifdef NPHM_ENS_TRACE
// Debug entry of the timeline build (tools/ens_trace.py): copies the stamps of the last ensemble launch to host memory.
extern "C" int nphm_debug_ens_trace(long long *host, int n_ll)
{
    using namespace nphm;
    NPHM_REQUIRE(n_ll >= 1 && n_ll <= 1 + tc::wg::kTraceMembers * tc::wg::kTraceStride, "nphm_debug_ens_trace: bad length");
    NPHM_CUDA_CHECK(cudaDeviceSynchronize());
    NPHM_CUDA_CHECK(cudaMemcpyFromSymbol(host, tc::wg::g_ens_trace, (size_t)n_ll * 8));
    return NPHM_OK;
}

// Tile boundaries of CTA 0 (3 stamps per tile, kTraceTiles tiles) followed by the work of every CTA ([0] = CTAs, then per
// CTA member-tiles and cycles) of the last ensemble launch.
extern "C" int nphm_debug_ens_work(long long *host, int n_ll)
{
    using namespace nphm;
    constexpr int nt = 3 * tc::wg::kTraceTiles, nc = 1 + 2 * tc::wg::kTraceMaxCtas;
    NPHM_REQUIRE(n_ll == nt + nc, "nphm_debug_ens_work: bad length");
    NPHM_CUDA_CHECK(cudaDeviceSynchronize());
    NPHM_CUDA_CHECK(cudaMemcpyFromSymbol(host, tc::wg::g_ens_tiles, (size_t)nt * 8));
    NPHM_CUDA_CHECK(cudaMemcpyFromSymbol(host + nt, tc::wg::g_ens_ctas, (size_t)nc * 8));
    return NPHM_OK;
}
#endif
