// Warpgroup-MMA (wgmma, sm_90a) kernel for the identity-SDF ensemble.
//
// Reference semantics: FastEnsembleDeepSDFMirrored.forward  src/NPHM/models/EnsembledDeepSDF.py:203-267
// Math, weight slabs and per-(query, member) records are those of tc_ensemble.cu (see the header there).
//
// A CTA is persistent over 128-point tiles: two consumer warpgroups of 64 points each and one producer warpgroup, which
// hands most of its registers to the consumers (setmaxnreg: 24 / 240 per thread).
//   producer (warps 8-11; one thread unless the warpgroup decides an absorption): bulk async copies of the record of every member and of its 8 weight units (tc_ensemble.cuh)
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
// mask and passes the item to the consumers through a two-deep queue in shared memory, so that no SM idles while others
// still have tiles, and the producer streams the next tile's weights while the consumers finish the current one.  A mask
// pre-pass (tile_mask_kernel) computes which members each tile needs (dense: a blend weight that is not exactly zero at
// some valid point; pruned: the tau rule) and the producer streams only those; grid queries use compact tiles
// (Params::tbx, tby, tbz) so that a tile lies far from many anchors.  Dense grid queries also skip the members whose blend
// terms fp32 rounding absorbs (the producer warpgroup decides per point, see there); the producer tells the consumers which member
// each record slot holds and ends a tile with a record slot without a copy.
// Dense grid queries with absorption run member by member instead (MM variant): per member, member_pass_kernel decides
// every row on the exact state and lists the rows that need the member, and the kernel runs 128-row tiles of that list,
// whose rows the producer warpgroup gathers into shared memory one work item ahead.
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
// Work of every CTA: [0] = CTAs of the last launch, then per CTA the member-tiles it evaluated, its cycles, its tiles, the
// producer's cycles from the first wait of an absorption candidate to its decision (summed) and the part of them spent
// waiting for the consumers' |num|.
constexpr int kTraceMaxCtas = 1024, kTraceCtaWords = 5;
__device__ long long g_ens_ctas[1 + kTraceCtaWords * kTraceMaxCtas];
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
    // tile queue (producer -> consumers): work item of the next two tiles (-1 = no more work)
    uint64_t q_full[2], q_empty[2];
    long long q_item[2];
    // producer -> consumers: the member whose record a record slot holds, -1 = the tile has no more members
    int rec_member[kRecSlots];
    // consumers -> producer (absorption): per tile row, |num| after the member of record position r in pub_num[r % 4][row];
    // then the consumer warp that owns the row (rows 16 warp .. 16 warp + 15) sets pub_seq[warp] = r + 1
    float pub_num[4][128];
    unsigned int pub_seq[kConsumerWarps];
    // member-major: the rows of the queue's two work items, staged by the producer warpgroup (thread prow: row prow): point,
    // num, chunk state index (-1: past the end of the member's list)
    float mm_pt[2][4][128];
    int mm_pos[2][128];
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

__device__ __forceinline__ uint32_t ld_volatile_u32(const uint32_t *a) { return *reinterpret_cast<const volatile uint32_t *>(a); }
__device__ __forceinline__ float ld_volatile_f32(const float *a) { return *reinterpret_cast<const volatile float *>(a); }

// Named barrier of the 128 producer threads (warps 8-11).  The non-aligned barrier.cta forms: the lead thread of warp 8 may
// reach them after the rest of its warp.
constexpr int kProducerBar = 3;
__device__ __forceinline__ void producer_sync() { asm volatile("barrier.cta.sync %0, 128;" ::"n"(kProducerBar) : "memory"); }
// true when v holds on every producer thread
__device__ __forceinline__ bool producer_all(bool v)
{
    uint32_t r;
    asm volatile("{\n\t.reg .pred pv, pr;\n\tsetp.ne.u32 pv, %1, 0;\n\tbarrier.cta.red.and.pred pr, %2, 128, pv;\n\t"
                 "selp.u32 %0, 1, 0, pr;\n}" : "=r"(r) : "r"((uint32_t)v), "n"(kProducerBar) : "memory");
    return r != 0;
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
    unsigned long long mask = 1ull << (p.n_members - 1), absorbed = 0;
    // absorption (dense rule): the in-order partial sums den of the kernel's blend.  A member the kernel skips leaves den as
    // it was, so these are the sums the kernel sees whichever members it skips.
    const bool absorb = !PRUNE && p.absorb;
    float den[4] = {0.f, 0.f, 0.f, 0.f};
    for (int k = 0; k < p.n_members; ++k) {
        bool need = false, kept = false;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            if (!pt[i].valid) continue;
            const float w = member_weight(anc, k, p.n_members, pt[i].x, pt[i].y, pt[i].z);
            need |= PRUNE ? w >= thr[i] : w != 0.f;
            if (absorb) {
                kept |= den[i] + w != den[i];
                den[i] += w;
            }
        }
        if (k < p.n_members - 1 && __any_sync(0xffffffffu, need)) mask |= 1ull << k;
        if (absorb && !__any_sync(0xffffffffu, kept)) absorbed |= 1ull << k;
    }
    if (lane == 0) {
        p.tile_masks[tile] = mask;
        if (absorb) p.absorb_masks[tile] = absorbed & mask;
    }
}

// Member-major order (dense grid queries with absorption): before member k runs, every row of the chunk holds num and den
// after members 0 .. k-1 exactly, so the pass of member k decides per row with no lag.  One warp per tile, 4 rows per lane,
// only tiles whose pre-pass mask has bit k (elsewhere w_k = +0 at every valid point).  At a valid row with w = w_k != +0
// (member_weight(), bit for bit the blend's weight):
//   quirk row (every member outputs 1.0): blended here, num = fmaf(w, 1, num), den += w;
//   absorbed: den + w == den and w * B_k (rounded up) < ulp(|num|) / 4 with |s_k| <= B_k (member_bound_kernel), so that
//     fmaf(w, s_k, num) == num: nothing changes;
//   otherwise den += w and the row goes to member k's list (a warp-aggregated append), whose num the ensemble kernel
//     updates with fmaf(w, s_k, num).
// Each row's num and den see the same terms in the same order as in the tile-major kernel, whose skips are exact too:
// the outputs are the same bits.
__global__ void __launch_bounds__(32 * kMaskWarps) member_pass_kernel(const Params p)
{
    const long long lt = (long long)blockIdx.x * kMaskWarps + (threadIdx.x >> 5);
    if (lt >= p.mm_tiles) return;
    const long long tile = p.mm_t0 + lt;
    const int k = p.mm_member, lane = threadIdx.x & 31;
    if (!((p.tile_masks[tile] >> k) & 1)) return;
    const long long tiles_per_query = p.blocked ? p.n_tiles : (p.n_points + 127) / 128;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int row = lane + 32 * i;
        const int s = (int)(lt * 128 + row);
        const TilePoint t = tile_point(p, p.blocked, tile, 0, tiles_per_query, row);
        bool listed = false;
        if (t.valid) {
            const float B = p.sub_bounds ? p.sub_bounds[((size_t)(((t.ix >> 5) - p.sub_x0) * p.sub_n + (t.iy >> 5)) * p.sub_n +
                                                          (t.iz >> 5)) * p.n_members + k]
                                         : p.bounds[k];
            const float w = member_weight(p.anchors, k, p.n_members, t.x, t.y, t.z);
            if (w != 0.f) {
                const bool quirk = p.quirk_period > 0 && ((t.g % p.quirk_period) == p.quirk_period - 1 || t.g == p.total - 1);
                const float num = p.mm_num[s], den = p.mm_den[s];
                if (quirk) {
                    p.mm_num[s] = fmaf(w, 1.0f, num);
                    p.mm_den[s] = den + w;
                } else {
                    const float L = fabsf(num);
                    // ulp(L) / 4 = 2^(e(L) - 25), exact for L >= 2^-100; NaN, smaller L and B = +inf never certify
                    const bool absorbed = den + w == den && B < INFINITY && L >= 0x1p-100f &&
                                          __fmul_ru(w, B) < __uint_as_float(((__float_as_uint(L) >> 23) - 25) << 23);
                    if (!absorbed) {
                        p.mm_den[s] = den + w;
                        listed = true;
                    }
                }
            }
        }
        const unsigned int ballot = __ballot_sync(0xffffffffu, listed);
        if (ballot) {
            unsigned int base = 0;
            if (lane == 0) base = atomicAdd(p.mm_count + k, (unsigned int)__popc(ballot));
            base = __shfl_sync(0xffffffffu, base, 0);
            if (listed) p.mm_list[base + __popc(ballot & ((1u << lane) - 1))] = s;
        }
    }
}

// Member-major: the blend of every valid row of the chunk, out = num / (den + 1e-6), the tile-major kernel's expression
__global__ void __launch_bounds__(256) member_finalize_kernel(const Params p)
{
    const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= p.mm_tiles * 128) return;
    const long long tiles_per_query = p.blocked ? p.n_tiles : (p.n_points + 127) / 128;
    const TilePoint t = tile_point(p, p.blocked, p.mm_t0 + s / 128, 0, tiles_per_query, (int)(s % 128));
    if (t.valid) p.out[t.idx] = __fdiv_rn(p.mm_num[s], p.mm_den[s] + 1e-6f);
}

// LOG: the debug skip log (Params::skip_log) - a variant of its own, so that the kernel without it is not slowed by it.
// MM: member-major dense grid query - every work item is a tile of 128 listed rows of member p.mm_member (member_pass_kernel),
// which load num from the chunk's state and store it back after the blend (den and out are the pass's and finalize's)
template <bool PRUNE, bool ACTS, bool LOG = false, bool MM = false>
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
    // MM: the items of the member's row list, counted by the pass launched before on the stream
    const long long mm_rows = MM ? (long long)p.mm_count[p.mm_member] : 0;
    const long long n_items = MM ? (mm_rows + 127) / 128 : n_tiles * n_groups;
    // members 0 .. n - 1 as a mask, n <= 64 (a shift by 64 is undefined in C++)
    auto bits_below = [](int n) -> unsigned long long { return n >= 64 ? ~0ull : (1ull << n) - 1; };
    auto group_mask = [&](long long item) -> unsigned long long {
        if (!ACTS || n_groups == 1) return bits_below(p.n_members);
        const int per = (p.n_members + n_groups - 1) / n_groups, lo = (int)(item % n_groups) * per;
        const int hi = min(p.n_members, lo + per);
        return bits_below(hi) & ~bits_below(lo);
    };

    if (threadIdx.x == 0) {
        for (int i = 0; i < kSlots; ++i) { mbar_init(&sm.w_full[i], 1); mbar_init(&sm.w_empty[i], kConsumerWarps); }
        for (int i = 0; i < kRecSlots; ++i) { mbar_init(&sm.rec_full[i], 1); mbar_init(&sm.rec_empty[i], kConsumerWarps); }
        for (int i = 0; i < 2; ++i) { mbar_init(&sm.q_full[i], 1); mbar_init(&sm.q_empty[i], kConsumerWarps); }
        for (int i = 0; i < kConsumerWarps; ++i) sm.pub_seq[i] = 0;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
#ifdef NPHM_ENS_TRACE
    const long long cta_start = clock64();
    if (blockIdx.x == 0 && threadIdx.x == 0) { g_ens_trace[0] = cta_start; g_ens_ctas[0] = gridDim.x; }
#endif
    // tile masks from the pre-pass: the pruned rule, or (dense variant) exactly zero blend weights
    const bool premask = PRUNE || (!ACTS && p.zero_skip);
    // members absorbed by fp32 rounding (dense variant with the zero-weight masks only; member-major: decided by the pass)
    const bool absorb = !PRUNE && !ACTS && !MM && p.zero_skip && p.absorb;

    if (warp >= kConsumerWarps) {
        // =========================================================================== producer (tiles, bulk async copies)
        asm volatile("setmaxnreg.dec.sync.aligned.u32 24;" ::: "memory");
        {
            // thread 0 of the producer warpgroup (lead) takes the tiles, waits on the barriers and issues the copies; the
            // whole warpgroup decides absorption, thread `prow` for tile row prow, as in tile_mask_kernel
            const int prow = threadIdx.x - 32 * kConsumerWarps;
            const bool lead = prow == 0;
            uint32_t rcount = 0;
#ifdef NPHM_ENS_TRACE
            long long t_decide = 0, t_wait = 0;  // cycles from a candidate's first wait to its decision, of them waiting
#endif
            for (uint32_t tcount = 0;; ++tcount) {
                // take the next work item and pass it on (the end of the work as item -1), also to the other producer threads
                const int qs = tcount & 1;
                if (lead) {
                    const unsigned int item = atomicAdd(p.sched, 1u);
                    ENS_TILE(tcount, 1);
                    mbar_wait(&sm.q_empty[qs], ((tcount >> 1) & 1) ^ 1);
                    sm.q_item[qs] = item < n_items ? (long long)item : -1;
                    if (!MM) mbar_arrive(&sm.q_full[qs]);
                }
                __syncwarp();
                producer_sync();
                // q_item[qs] is rewritten two tiles later, after every producer thread has passed the next tile's sync
                const long long qitem = sm.q_item[qs];
                if (MM) {
                    // the item's listed rows, gathered here while the consumers still run the previous item: thread
                    // prow stages row prow (listed row qitem * 128 + prow of the member), then the lead publishes the item
                    if (qitem >= 0) {
                        const long long s = qitem * 128 + prow;
                        const int pos = s < mm_rows ? p.mm_list[s] : -1;
                        const TilePoint t = tile_point(p, p.blocked, p.mm_t0 + max(pos, 0) / 128, 0, tiles_per_query, max(pos, 0) % 128);
                        sm.mm_pt[qs][0][prow] = t.x;
                        sm.mm_pt[qs][1][prow] = t.y;
                        sm.mm_pt[qs][2][prow] = t.z;
                        sm.mm_pt[qs][3][prow] = pos >= 0 ? p.mm_num[pos] : 0.f;
                        sm.mm_pos[qs][prow] = pos;
                    }
                    producer_sync();
                    if (lead) mbar_arrive(&sm.q_full[qs]);
                }
                if (qitem < 0) {
#ifdef NPHM_ENS_TRACE
                    if (lead && blockIdx.x < kTraceMaxCtas) {
                        // member-major: every word summed over the member launches of the query (zeroed before the first;
                        // the decision words stay 0, the producer decides nothing there)
                        long long *w = g_ens_ctas + 1 + kTraceCtaWords * blockIdx.x;
                        if (MM) { w[2] += tcount; w[3] += t_decide; w[4] += t_wait; }
                        else { w[2] = tcount; w[3] = t_decide; w[4] = t_wait; }
                    }
#endif
                    break;
                }
                const unsigned int item = (unsigned int)qitem;
                const unsigned int tile = ACTS ? item / n_groups : item;
                const int qi = (MM || p.blocked) ? 0 : (int)(tile / (unsigned int)tiles_per_query);
                unsigned long long mask = MM ? 1ull << p.mm_member : (premask ? p.tile_masks[tile] : group_mask(item));
                // absorption: skip member m when den + w == den at every valid point (pre-pass) and, at every valid point p
                // with w_m(p) != 0, w_m(p) * B_m < ulp(L(p)) / 4 (so that fmaf(w, s, num) returns num), with |s_m| <= B_m
                // (member_bound_kernel) and |num(p)| >= L(p) = |num(p)| after the member two record positions back
                // (published by the consumer warps before they retire that member's successor's layer 2, i.e. before the
                // lead could issue the previous member's last unit) - w(p) * B of the member in between, rounded down.
                // Deterministic: each thread waits for that state of its row.  w_m(p) is member_weight(), bit for bit the
                // blend's weight.  The decision is a barrier reduction over the 128 producer threads.
                const unsigned long long amask = absorb ? p.absorb_masks[tile] : 0ull;
                const float *anc = p.anchors + (size_t)qi * (p.n_members - 1) * 3;
                float px = 0.f, py = 0.f, pz = 0.f;
                float lag = 0.f;                         // w * B of the member at record position rcount - 1, rounded up
                bool pvalid = false;
                if (amask) {
                    const TilePoint t = tile_point(p, p.blocked, tile, qi, tiles_per_query, prow);
                    px = t.x; py = t.y; pz = t.z; pvalid = t.valid;
                }
                const uint32_t rc0 = rcount;
                for (; mask; mask &= mask - 1) {         // the tile's members in ascending order
                    const int m = __ffsll((long long)mask) - 1;
                    const float bm = amask ? p.bounds[(size_t)qi * p.n_members + m] : 0.f;
                    float wb = -1.f;                     // w_m * B_m of this row, rounded up, once computed
                    if (((amask >> m) & 1) && rcount >= rc0 + 2 && bm < INFINITY) {
#ifdef NPHM_ENS_TRACE
                        const long long t0 = clock64();
#endif
                        // the consumer warp of row prow: rows 16 w .. 16 w + 15
                        while (ld_volatile_u32(&sm.pub_seq[prow >> 4]) < rcount - 1) { }
                        __threadfence_block();
#ifdef NPHM_ENS_TRACE
                        const long long t1 = clock64();
#endif
                        const float w = member_weight(anc, m, p.n_members, px, py, pz);
                        wb = __fmul_ru(w, bm);
                        const float L = __fsub_rd(ld_volatile_f32(&sm.pub_num[(rcount - 2) & 3][prow]), lag);
                        // ulp(L) / 4 = 2^(e(L) - 25), exact for L >= 2^-100; NaN and smaller L never certify
                        const bool ok = !pvalid || w == 0.f ||
                                        (L >= 0x1p-100f && wb < __uint_as_float(((__float_as_uint(L) >> 23) - 25) << 23));
                        const bool skip = producer_all(ok);
#ifdef NPHM_ENS_TRACE
                        if (lead) { const long long t2 = clock64(); t_decide += t2 - t0; t_wait += t1 - t0; }
#endif
                        if (skip) {
                            if (LOG && lead) atomicOr(p.skip_log + tile, 1ull << m);
                            continue;
                        }
                    }
                    // a later member is a candidate: the lag term of this one
                    if ((amask >> m) >> 1) lag = wb >= 0.f ? wb : __fmul_ru(member_weight(anc, m, p.n_members, px, py, pz), bm);
                    if (lead) {
                        const int rslot = rcount % kRecSlots;
                        mbar_wait(&sm.rec_empty[rslot], ((rcount / kRecSlots) & 1) ^ 1);
                        sm.rec_member[rslot] = m;
                        mbar_expect_tx(&sm.rec_full[rslot], kRecFloats * 4);
                        bulk_g2s(sm.rec[rslot], p.recs + ((size_t)qi * p.n_members + m) * kRecFloats, kRecFloats * 4, &sm.rec_full[rslot]);
                        const int set = m < 2 * p.n_symm ? (m >> 1) : m - p.n_symm;
                        const uint8_t *w = p.weights + (size_t)set * kSetBytes;
                        const uint8_t *l2 = p.l2_slabs + ((size_t)qi * p.n_members + m) * kL2SlabBytes;
#pragma unroll 1
                        for (int u = 0; u < kUnits; ++u) {
                            // every member has 8 units, so unit u always goes to slot u % 4, on its (u / 4)-th use per member
                            const int slot = u & 3;
                            const uint32_t bytes = unit_bytes(u);
                            ENS_PEVT(rcount, 8 + u);
                            mbar_wait(&sm.w_empty[slot], ((u >> 2) & 1) ^ 1);
                            ENS_PEVT(rcount, u);
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
                    __syncwarp();
                    ++rcount;
                }
                // the end of the tile's members: a record slot without a copy
                if (lead) {
                    const int rslot = rcount % kRecSlots;
                    mbar_wait(&sm.rec_empty[rslot], ((rcount / kRecSlots) & 1) ^ 1);
                    sm.rec_member[rslot] = -1;
                    mbar_arrive(&sm.rec_full[rslot]);
                }
                __syncwarp();
                ++rcount;
            }
            // every CTA has taken its last item once all have counted themselves finished: the last one resets the counter
            // for the next launch on the stream
            if (lead) {
                __threadfence();
                if (atomicAdd(p.sched + 1, 1u) == gridDim.x - 1) {
                    atomicExch(p.sched, 0u);
                    atomicExch(p.sched + 1, 0u);
                }
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
    uint32_t rcount = 0;                         // record positions: the members evaluated and one end marker per tile
#ifdef NPHM_ENS_TRACE
    uint32_t n_eval = 0;                         // member-tiles evaluated
#endif
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
        // (member-major: the slot's staged rows are read below, before the slot is released)
        if (!MM || item < 0) {
            __syncwarp();
            if (lane == 0) mbar_arrive(&sm.q_empty[qs]);
        }
        if (item < 0) break;
        if (threadIdx.x == 0) ENS_TILE(tcount, 0);
        const long long tile = ACTS ? item / n_groups : item;
        const int qi = (MM || p.blocked) ? 0 : (int)(tile / tiles_per_query);
        long long idx[2], g[2];
        bool valid[2], quirk[2];
        float x[2], y[2], z[2];
        float num[2] = {0.f, 0.f}, den[2] = {0.f, 0.f};
        int mpos[2];                             // MM: the rows' chunk state index
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            if (MM) {
                // listed row tile * 128 + rl[i] of the member, as the producer staged it: its point and num after the
                // members before; rows past the list end run on the chunk's first point and do not store
                mpos[i] = sm.mm_pos[qs][rl[i]];
                valid[i] = mpos[i] >= 0;
                x[i] = sm.mm_pt[qs][0][rl[i]]; y[i] = sm.mm_pt[qs][1][rl[i]]; z[i] = sm.mm_pt[qs][2][rl[i]];
                num[i] = sm.mm_pt[qs][3][rl[i]];
                idx[i] = g[i] = 0;
                quirk[i] = false;                // quirk rows are blended by the pass, never listed
                continue;
            }
            // (the fitting variant only runs linear tiles)
            const TilePoint t = tile_point(p, !ACTS && p.blocked, tile, qi, tiles_per_query, rl[i]);
            idx[i] = t.idx; g[i] = t.g; valid[i] = t.valid; x[i] = t.x; y[i] = t.y; z[i] = t.z;
            quirk[i] = p.quirk_period > 0 && ((g[i] % p.quirk_period) == p.quirk_period - 1 || g[i] == p.total - 1);
            // pruned rule: the blend divides by S = sum_k w_k over all members, evaluated or not
            if (PRUNE) den[i] = weight_sum(p.anchors + (size_t)qi * (p.n_members - 1) * 3, p.n_members, x[i], y[i], z[i]);
        }
        if (MM) {
            __syncwarp();
            if (lane == 0) mbar_arrive(&sm.q_empty[qs]);
        }
        const uint32_t tile_rc0 = rcount;        // the tile's first member (timeline build)

        for (;;) {
            // the tile's next member, as the producer hands it out (-1: no more)
            const uint32_t rslot = rcount % kRecSlots;
            ENS_CMARK(rcount, 24);
            mbar_wait(&sm.rec_full[rslot], (rcount / kRecSlots) & 1);
            const int m = sm.rec_member[rslot];
            if (m < 0) {
                release_rec(&sm.rec_empty[rslot]);
                ++rcount;
                break;
            }
#ifdef NPHM_ENS_TRACE
            ++n_eval;
#endif
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
            if (absorb) {
                // publish |num| of the warp's rows for the producer's absorption decisions (rows without a valid point
                // too: the producer passes them by itself); the rows are rl[0] and rl[1], recomputed from the warp
                if (q4 == 0) {
#pragma unroll
                    for (int r = 0; r < 2; ++r)
                        *reinterpret_cast<volatile float *>(&sm.pub_num[rcount & 3][16 * warp + (lane >> 2) + 8 * r]) = fabsf(num[r]);
                    __threadfence_block();
                }
                __syncwarp();
                if (lane == 0) {
                    __threadfence_block();
                    *reinterpret_cast<volatile unsigned int *>(&sm.pub_seq[warp]) = rcount + 1;
                }
            }
            release_rec(&sm.rec_empty[rslot]);
            ++rcount;
        }
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            if (MM) {
                if (q4 == 0 && valid[r]) p.mm_num[mpos[r]] = num[r];
            } else if (q4 == 0 && valid[r] && n_groups == 1) {
                p.out[(size_t)qi * p.n_points + idx[r]] = __fdiv_rn(num[r], den[r] + 1e-6f);
            }
        }
    }
    if (wgi == 0) take_turn();                   // the turn warpgroup 1 passed after its last phase
#ifdef NPHM_ENS_TRACE
    if (threadIdx.x == 0 && blockIdx.x < kTraceMaxCtas) {
        if (MM) {
            g_ens_ctas[1 + kTraceCtaWords * blockIdx.x] += n_eval;
            g_ens_ctas[2 + kTraceCtaWords * blockIdx.x] += clock64() - cta_start;
        } else {
            g_ens_ctas[1 + kTraceCtaWords * blockIdx.x] = n_eval;
            g_ens_ctas[2 + kTraceCtaWords * blockIdx.x] = clock64() - cta_start;
        }
    }
#endif
}

}  // namespace wg

int launch_ensemble_mask(const Params &p, bool prune, cudaStream_t stream)
{
    const unsigned blocks = (unsigned)ceil_div(p.n_tiles, (long long)wg::kMaskWarps);
    if (prune) wg::tile_mask_kernel<true><<<blocks, 32 * wg::kMaskWarps, 0, stream>>>(p);
    else wg::tile_mask_kernel<false><<<blocks, 32 * wg::kMaskWarps, 0, stream>>>(p);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

int launch_member_major_chunk(const Params &p0, int grid_x, cudaStream_t stream)
{
    const int smem = (int)sizeof(wg::Smem);
    auto kern = wg::ensemble_wgmma_kernel<false, false, false, true>;
    NPHM_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
#ifdef NPHM_ENS_TRACE
    if (p0.mm_t0 == 0) {                         // the work counts of the trace build sum over the query's member launches
        void *ctas = nullptr;
        NPHM_CUDA_CHECK(cudaGetSymbolAddress(&ctas, wg::g_ens_ctas));
        NPHM_CUDA_CHECK(cudaMemsetAsync(ctas, 0, sizeof(wg::g_ens_ctas), stream));
    }
#endif
    const unsigned pass_blocks = (unsigned)ceil_div(p0.mm_tiles, (long long)wg::kMaskWarps);
    Params p = p0;
    for (int k = 0; k < p.n_members; ++k) {
        p.mm_member = k;
        wg::member_pass_kernel<<<pass_blocks, 32 * wg::kMaskWarps, 0, stream>>>(p);
        NPHM_CUDA_CHECK(cudaGetLastError());
        kern<<<grid_x, wg::kThreads, smem, stream>>>(p);
        NPHM_CUDA_CHECK(cudaGetLastError());
    }
    wg::member_finalize_kernel<<<(unsigned)ceil_div(p.mm_tiles * 128, 256ll), 256, 0, stream>>>(p);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

int launch_ensemble_wgmma(const Params &p, bool prune, bool acts, int grid_x, cudaStream_t stream)
{
    int rc;
    if ((prune || (!acts && p.zero_skip)) && (rc = launch_ensemble_mask(p, prune, stream))) return rc;
    const int smem = (int)sizeof(wg::Smem);
    auto kern = acts ? wg::ensemble_wgmma_kernel<false, true>
                     : (prune ? wg::ensemble_wgmma_kernel<true, false>
                              : (p.skip_log ? wg::ensemble_wgmma_kernel<false, false, true> : wg::ensemble_wgmma_kernel<false, false>));
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
// CTA member-tiles, cycles, tiles, decision cycles, decision wait cycles) of the last ensemble launch.
extern "C" int nphm_debug_ens_work(long long *host, int n_ll)
{
    using namespace nphm;
    constexpr int nt = 3 * tc::wg::kTraceTiles, nc = 1 + tc::wg::kTraceCtaWords * tc::wg::kTraceMaxCtas;
    NPHM_REQUIRE(n_ll == nt + nc, "nphm_debug_ens_work: bad length");
    NPHM_CUDA_CHECK(cudaDeviceSynchronize());
    NPHM_CUDA_CHECK(cudaMemcpyFromSymbol(host, tc::wg::g_ens_tiles, (size_t)nt * 8));
    NPHM_CUDA_CHECK(cudaMemcpyFromSymbol(host + nt, tc::wg::g_ens_ctas, (size_t)nc * 8));
    return NPHM_OK;
}
#endif
