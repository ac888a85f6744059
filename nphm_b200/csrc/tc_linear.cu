// Generic fp32-accurate linear layer on Hopper warpgroup MMAs (wgmma):  C = epilogue( [A1 | A2] * W^T )
//
// One building block for everything on the hot path that is a chain of dense layers but does not fit the fully fused
// ensemble kernel (tc_ensemble_wgmma.cu, hidden 200): the forward pass, the forward-mode Jacobian and the
// backward pass of the forward-deformation network (reference src/NPHM/models/diff_operators.py:26-54 `jac`,
// src/NPHM/models/fitting.py:99-106,167 - implicit differentiation of the Broyden root and loss.backward()), and DeepSDF
// stacks of any width (NPM baseline 515 -> 1024 x 8, scripts/configs/npm.yaml:2-4).
//
// Arithmetic: fp16 MMAs with fp32 accumulation in registers, both operands split x = hi + lo in two fp16 terms, products
// hi*hi + hi*lo + lo*hi (3 MMAs per k-step) - the same fp32-level scheme as the fused kernel.  A is read as fp32 from
// global memory and split on the fly by eight "row" warps (thread = row of the 128-row tile x half of the k-step) into a
// 4-stage shared-memory ring in K-major core-matrix order; W comes pre-split and pre-packed (pack_linear_kernel) through
// bulk async copies.  The same eight warps are two warpgroups: each issues the SS-form wgmmas of its 64-row half of the tile
// (16 output columns per instruction), parks its accumulators in a shared-memory tile after the last k-step, and all eight
// run the epilogue from there (thread = row, every other 16-column unit).  Operands are row-major or `blocked` ([128-row tile][feature][128]: what the fused ensemble forward
// writes for the fitting backward); launches can be batched over gridDim.z with per-entry operands and weight sets.
//
//   A1 [M x K1] fp32 row-major, optional A2 [M x K2] appended along K (skip connection `cat([h, x])`, the 1/sqrt(2) is folded
//   into W), or a one-hot A2 (row r -> e_{r mod K2}: the input tangents of a forward-mode pass, never materialised)
//   W  [N x (K1 + K2)]  ->  slabs [n_tile][k-step][Nt x 16 hi | Nt x 16 lo]
//   epilogue modes:  LINEAR   C = t + bias[row / rows_per_bias][n]
//                    SOFTPLUS C = softplus_100(t + bias), optionally D = sigmoid(100 (t + bias))   (the activation's derivative)
//                    MULT     C = t * Mul[row / mul_div][n]                                         (tangent / adjoint passes)
//                             (+ coef (1 - Mul) z a: the second-order coupling of the SDF-gradient training backward)
#include "tc_linear.cuh"
#include <cuda_fp16.h>
#include <type_traits>

namespace nphm {
namespace tcl {
using namespace tc;

constexpr int kMaxStages = 4;                   // operand ring: as many stages (2..4) as fit next to the accumulator tile
constexpr int kMaxSmem = 227 * 1024;
constexpr int kARing = 4;                       // fp32 staging ring of A (independent of the operand ring)
constexpr int kRowWarps = 8;                      // two per 32-row quarter of the tile
constexpr int kThreads = 32 * (kRowWarps + 1);
constexpr int kMaxNt = 256;                     // accumulator columns held in registers: kMaxNt / 2 per thread
constexpr int kChunks = kMaxNt / 16;            // 64 x 16 MMAs per k-step and warpgroup
constexpr int kPackedStep = 2 * 128 * 32;       // bytes of one k-step of a packed A tile: 128 x 16 fp16 hi | 128 x 16 fp16 lo

constexpr int kAPitch = 20;                      // floats per staged fp32 row (16 + 4: 80-byte pitch spreads the banks)
constexpr int kADepth = 3;                       // k-steps of A kept in flight per thread (cp.async groups)
// dynamic shared memory: [Ctl | stages x (a_hi 4 KB | a_lo 4 KB | b Nt*64) | a32 ring | accumulator tile 128 x (Nt + 4) fp32]
#ifndef NPHM_TCL_MULSLOTS
#define NPHM_TCL_MULSLOTS 3
#endif
constexpr int kMulSlots = NPHM_TCL_MULSLOTS;                     // ring of multiplier units (16 features x 128 rows fp32 = 8 KB) in the a32 space
struct __align__(128) Ctl {
    uint64_t a_full[kMaxStages], b_full[kMaxStages], empty[kMaxStages];
    uint64_t mul_full[kMaxNt / 16], mul_empty[kMaxNt / 16];       // one single-use pair per 16-column unit (no phase bookkeeping)
};
constexpr int kCtlBytes = 512;
static_assert(kMulSlots * 16 * 128 * 4 <= kARing * 128 * kAPitch * 4, "multiplier ring must fit the fp32 staging area of A");
static_assert(sizeof(Ctl) <= kCtlBytes, "control block");
static_assert(kCtlBytes + 2 * (2 * 128 * 32 + kMaxNt * 64) + kARing * 128 * kAPitch * 4 + 128 * (kMaxNt + 4) * 4 <= kMaxSmem, "smem");
constexpr int kA32Bytes = kARing * 128 * kAPitch * 4;
__host__ __device__ inline int stage_bytes(int Nt) { return 2 * 128 * 32 + Nt * 64; }
constexpr int kMulRingBytes = kMulSlots * 16 * 128 * 4;
__host__ __device__ inline int dtile_pitch(int Nt) { return Nt + 4; }
// behind the operand stages: the fp32 staging ring of A, or (packed A: no staging) just the multiplier ring; then the accumulators
inline int smem_bytes(int Nt, int stages, bool packed_a)
{
    return kCtlBytes + stages * stage_bytes(Nt) + (packed_a ? kMulRingBytes : kA32Bytes) + 128 * dtile_pitch(Nt) * 4;
}

#ifdef NPHM_TCL_TRACE
#ifndef NPHM_TCL_TRACE_NT
#define NPHM_TCL_TRACE_NT 128          // which tile width to record (the chain uses 128, the fitting backward 208 / 112)
#endif
// timeline of CTA (0,0,0): [role field][k-step] clock64 stamps (tools/tcl_trace.py)
__device__ long long g_tcl_trace[16 * 64];
#define TCL_EVT(cond, field, j) do { if ((cond) && p.Nt == NPHM_TCL_TRACE_NT && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0 && (j) < 64) \
    g_tcl_trace[(field) * 64 + (j)] = clock64(); } while (0)
#else
#define TCL_EVT(cond, field, j) do { } while (0)
#endif


// MODE and PACKED_C (packed output present) are compile-time: the epilogue is the longest part of a latency-bound layer and
// loses ~a fifth of its instructions when the per-unit mode / layout tests disappear
template <int MODE, bool PACKED_C>
__global__ void __launch_bounds__(kThreads, 1) linear_tc_kernel(const LinearParams p)
{
    if (p.live && *p.live == 0) return;                 // uniform over the grid (Broyden: every sample of the search is frozen)
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    Ctl &sm = *reinterpret_cast<Ctl *>(smem_raw);
    const int kStages = p.stages;
    const int st_bytes = stage_bytes(p.Nt);
    uint8_t *const st0 = smem_raw + kCtlBytes;
    auto st_a_hi = [&](int s) { return st0 + (size_t)s * st_bytes; };
    auto st_a_lo = [&](int s) { return st0 + (size_t)s * st_bytes + 128 * 32; };
    auto st_b = [&](int s) { return st0 + (size_t)s * st_bytes + 2 * 128 * 32; };
    float (*a32)[128][kAPitch] = reinterpret_cast<float (*)[128][kAPitch]>(st0 + (size_t)kStages * st_bytes);
    const bool packed_a = p.Ap != nullptr;
    float *const dtile = reinterpret_cast<float *>(st0 + (size_t)kStages * st_bytes + (packed_a ? kMulRingBytes : kA32Bytes));
    const int dp = dtile_pitch(p.Nt);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long row0 = (long long)blockIdx.x * 128;
    const int nt_idx = blockIdx.y;
    const int z = blockIdx.z;                             // batch entry: own A / C / Mul / row scale, weights of set(z)
    const int wset = member_set(z, p.w_pairs);
    const int n0 = nt_idx * p.Nt;

    TCL_EVT(threadIdx.x == 0, 10, 0);
    if (threadIdx.x == 0) {
        for (int i = 0; i < kStages; ++i) { mbar_init(&sm.a_full[i], kRowWarps); mbar_init(&sm.b_full[i], 1); mbar_init(&sm.empty[i], 2); }
        for (int i = 0; i < kMaxNt / 16; ++i) { mbar_init(&sm.mul_full[i], 1); mbar_init(&sm.mul_empty[i], 4); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const int slab_bytes = p.Nt * 64;
    TCL_EVT(threadIdx.x == 0, 10, 1);

    // MULT epilogue with a blocked multiplier and packed A (the fp32 staging ring of A is idle then): the producer streams the
    // multiplier, unit by unit (16 features x 128 rows = 8 KB contiguous), into that ring while the MMAs run - read from global
    // memory inside the epilogue, every unit cost a full memory round trip (measured: 5 k cycles per unit)
    const bool mul_ring = p.Ap && MODE == kModeMult && p.Mul && (p.blocked || p.mul_blocked) && p.mul_div == 1;
    const int n_units = p.Nt / 16;
    float (*mring)[16][128] = reinterpret_cast<float (*)[16][128]>(a32);
    auto unit_in_ring = [&](int u) { return mul_ring && n0 + 16 * u + 16 <= p.ldmul; };     // whole unit inside the tile's block

    if (warp == kRowWarps) {
        // ================================================================ producer: weight slabs (bulk async copies)
        if (lane == 0) {
            const float *mul_tile = mul_ring ? p.Mul + (size_t)z * p.sMul + (size_t)blockIdx.x * p.ldmul * 128 + (size_t)n0 * 128 : nullptr;
            int mu = 0;                                    // next multiplier unit to fetch
            auto fetch_mul = [&](int limit) {
                for (; mu < limit && mu < n_units; ++mu) {
                    if (!unit_in_ring(mu)) continue;
                    const int slot = mu % kMulSlots;
                    if (mu >= kMulSlots) mbar_wait(&sm.mul_empty[mu - kMulSlots], 0);      // the unit that held this slot is consumed
                    mbar_expect_tx(&sm.mul_full[mu], 16 * 128 * 4);
                    bulk_g2s(&mring[slot][0][0], mul_tile + (size_t)mu * 16 * 128, 16 * 128 * 4, &sm.mul_full[mu]);
                }
            };
            const uint8_t *w = p.W + (size_t)wset * p.w_stride + (size_t)nt_idx * p.ksteps * slab_bytes;
            // packed A (operand-ready tiles written by the epilogue of the previous layer): one more bulk copy per k-step
            const uint8_t *ap = p.Ap ? p.Ap + (size_t)z * p.sAp + (size_t)blockIdx.x * p.a_tile_steps * kPackedStep : nullptr;
            for (int j = 0, s = 0, ph = 0; j < p.ksteps; ++j) {          // (stage, phase) counted, not divided: kStages is a runtime value
                mbar_wait(&sm.empty[s], ph ^ 1);
                TCL_EVT(true, 0, j);
                mbar_expect_tx(&sm.b_full[s], slab_bytes + (ap ? kPackedStep : 0));
                bulk_g2s(st_b(s), w + (size_t)j * slab_bytes, slab_bytes, &sm.b_full[s]);
                if (ap) bulk_g2s(st_a_hi(s), ap + (size_t)j * kPackedStep, kPackedStep, &sm.b_full[s]);   // a_hi | a_lo are adjacent
                if (++s == kStages) { s = 0; ph ^= 1; }
                if (j == kStages - 1 || j == p.ksteps - 1) fetch_mul(kMulSlots);   // behind the first operand stages: the first
                                                                                   // multiplier units travel while the MMAs run
            }
            fetch_mul(n_units);                            // the rest as the epilogue frees the slots
        }
    } else {
        // ================================================================ row warps: split A into the ring, MMAs, epilogue
        // Thread t of each warpgroup converts row t of the tile: `half` = warp / 4 converts inputs [8 half, 8 half + 8) of every
        // k-step and finishes the accumulator units u with u % 2 == half.  As MMA issuers, warpgroup `half` owns rows
        // [64 half, 64 half + 64) of the tile.
        const int t = threadIdx.x & 127;                  // row of the tile (conversion and epilogue)
        const int half = warp >> 2;
        const long long row = row0 + t;
        const bool row_ok = row < p.M;
        // row-major: element (row, k) at row * lda + k.  blocked: tiles of 128 rows, feature-major inside a tile,
        // (row, k) at (row / 128) * lda * 128 + k * 128 + row % 128 - what the fused ensemble forward writes (thread = point)
        const size_t kstr = p.blocked ? 128 : 1;
        const float *a1 = !p.A1 ? nullptr
                          : p.blocked ? p.A1 + (size_t)z * p.sA1 + (size_t)blockIdx.x * p.lda1 * 128 + t
                                      : p.A1 + (size_t)z * p.sA1 + (size_t)(row_ok ? row : 0) * p.lda1;
        const float *a2 = (p.A2 && !p.a2_onehot) ? p.A2 + (size_t)(row_ok ? row : 0) * p.lda2 : nullptr;
        const int hot = p.a2_onehot ? (int)(row % p.K2) : -1;
        const bool vec_ok = p.A1 && (p.blocked || ((p.lda1 % 4 == 0) && (p.sA1 % 4 == 0) && ((reinterpret_cast<uintptr_t>(p.A1) & 15) == 0)));
        const uint32_t off0 = (uint32_t)(t >> 3) * 256 + (uint32_t)(t & 7) * 16 + (uint32_t)half * 128;   // core-matrix slot of (row, 8 half)
        // this thread's 8 inputs of k-step j: cols [16 j + 8 half, + 8) of [A1 | A2], zero beyond the real width / the last row
        auto load_direct = [&](int j, float (&v)[8]) {
            const int k0 = 16 * j + 8 * half;
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                const int k = k0 + c;
                float x = 0.f;
                if (row_ok) {
                    if (k < p.K1) x = __ldg(a1 + (size_t)k * kstr);
                    else if (k < p.K1 + p.K2) x = p.a2_onehot ? (k - p.K1 == hot ? 1.f : 0.f) : __ldg(a2 + (k - p.K1));
                }
                v[c] = x;
            }
        };
        // inputs that lie inside A1 (and are 16-byte aligned) are staged through shared memory with cp.async, kADepth k-steps ahead
        // (a thread only ever reads what it copied itself, so cp.async.wait_group is all the synchronisation needed); the few
        // others (skip-connection tail, one-hot tangents, K padding) are loaded directly
        auto fast = [&](int j) { return row_ok && vec_ok && 16 * j + 8 * half + 8 <= p.K1; };
        auto prefetch = [&](int j) {
            if (j < p.ksteps && fast(j)) {
                const uint32_t dst = smem_u32(&a32[j % kARing][t][8 * half]);
                if (p.blocked) {
                    const float *src = a1 + (size_t)(16 * j + 8 * half) * 128;
#pragma unroll
                    for (int i = 0; i < 8; ++i)
                        asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst + 4 * i), "l"(src + (size_t)i * 128) : "memory");
                } else {
                    const float *src = a1 + 16 * j + 8 * half;
                    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
                    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + 16), "l"(src + 4) : "memory");
                }
            }
            asm volatile("cp.async.commit_group;" ::: "memory");
        };
        if (!p.Ap) for (int d = 0; d < kADepth; ++d) prefetch(d);
        float acc[kChunks][8];
#pragma unroll
        for (int c = 0; c < kChunks; ++c)
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[c][e] = 0.f;
        const uint32_t a_rows = (uint32_t)half * 2048;    // this warpgroup's 64 rows: 8 row groups of 256 B further
        int prev_s = 0;
        for (int j = 0, s = 0, ph = 0; j < p.ksteps; ++j) {
          if (!p.Ap) {
            const int sa = j % kARing;
            float cur[8];
            TCL_EVT(threadIdx.x == 0, 4, j);
            asm volatile("cp.async.wait_group %0;" ::"n"(kADepth - 1) : "memory");
            TCL_EVT(threadIdx.x == 0, 5, j);
            if (fast(j)) {
                const float4 f0 = *reinterpret_cast<const float4 *>(&a32[sa][t][8 * half]);
                const float4 f1 = *reinterpret_cast<const float4 *>(&a32[sa][t][8 * half + 4]);
                cur[0] = f0.x; cur[1] = f0.y; cur[2] = f0.z; cur[3] = f0.w; cur[4] = f1.x; cur[5] = f1.y; cur[6] = f1.z; cur[7] = f1.w;
            } else {
                load_direct(j, cur);
            }
            prefetch(j + kADepth);                             // slot (j + 3) % 4 was read by this thread at iteration j - 1
            uint32_t hi[4], lo[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) split2(cur[2 * i], cur[2 * i + 1], hi[i], lo[i]);
            TCL_EVT(threadIdx.x == 0, 6, j);
            mbar_wait(&sm.empty[s], ph ^ 1);
            TCL_EVT(threadIdx.x == 0, 7, j);
            *reinterpret_cast<uint4 *>(st_a_hi(s) + off0) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
            *reinterpret_cast<uint4 *>(st_a_lo(s) + off0) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncwarp();
            if (lane == 0) mbar_arrive(&sm.a_full[s]);
            TCL_EVT(threadIdx.x == 0, 8, j);
            mbar_wait(&sm.a_full[s], ph);
          }
            mbar_wait(&sm.b_full[s], ph);
            {
                const uint64_t a_hi = make_desc(smem_u32(st_a_hi(s)) + a_rows, 128, 256);
                const uint64_t a_lo = make_desc(smem_u32(st_a_lo(s)) + a_rows, 128, 256);
                const uint32_t b = smem_u32(st_b(s));
                wg_fence();
#pragma unroll
                for (int c = 0; c < kChunks; ++c) {
                    if (16 * c < p.Nt) {
                        const uint64_t b_hi = make_desc(b + 512 * c, 128, 256), b_lo = make_desc(b + 512 * c + p.Nt * 32, 128, 256);
                        wgmma_ss_n16(acc[c], a_hi, b_hi, 1);
                        wgmma_ss_n16(acc[c], a_hi, b_lo, 1);
                        wgmma_ss_n16(acc[c], a_lo, b_hi, 1);
                    }
                }
                wg_commit();
                wg_wait<1>();                              // k-step j - 1 is complete: its stage may be refilled
            }
            if (j > 0 && (threadIdx.x & 127) == 0) mbar_arrive(&sm.empty[prev_s]);
            prev_s = s;
            if (++s == kStages) { s = 0; ph ^= 1; }
        }
        wg_wait<0>();
#pragma unroll
        for (int c = 0; c < kChunks; ++c) wg_reg_fence(acc[c]);
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        {
            // accumulators -> shared tile [row][column] (fragment rows 16 (warp % 4) + lane / 4 (+ 8) of this warpgroup's half)
            const int fr = 64 * half + 16 * (warp & 3) + (lane >> 2), fc = 2 * (lane & 3);
#pragma unroll
            for (int c = 0; c < kChunks; ++c) {
                if (16 * c < p.Nt) {
                    float *d0 = dtile + (size_t)fr * dp + 16 * c + fc, *d1 = d0 + 8 * dp;
                    *reinterpret_cast<float2 *>(d0) = make_float2(acc[c][0], acc[c][1]);
                    *reinterpret_cast<float2 *>(d1) = make_float2(acc[c][2], acc[c][3]);
                    *reinterpret_cast<float2 *>(d0 + 8) = make_float2(acc[c][4], acc[c][5]);
                    *reinterpret_cast<float2 *>(d1 + 8) = make_float2(acc[c][6], acc[c][7]);
                }
            }
            asm volatile("bar.sync 1, %0;" ::"n"(32 * kRowWarps) : "memory");   // the row warps only
        }
        // ---------------- epilogue: thread = row, 16 accumulator columns at a time (units of this warp's parity)
        TCL_EVT(threadIdx.x == 0, 9, 1);
        const float *drow = dtile + (size_t)t * dp;
        const float *bias = p.bias ? p.bias + (size_t)z * p.sBias + (size_t)(row_ok ? row / p.rows_per_bias : 0) * p.ldb : nullptr;
        const bool mul_blk = p.blocked || p.mul_blocked;
        const long long mrow = row_ok ? row / p.mul_div : 0;                     // multiplier row (tangent passes: 3 rows per point)
        const float *mul = !p.Mul ? nullptr
                           : mul_blk ? p.Mul + (size_t)z * p.sMul + (size_t)(mrow >> 7) * p.ldmul * 128 + (mrow & 127)
                                     : p.Mul + (size_t)z * p.sMul + (size_t)mrow * p.ldmul;
        const float rscale = (p.row_scale && row_ok) ? __ldg(p.row_scale + (size_t)z * p.sRow + row) : 1.0f;
        float *const Cz = p.C ? p.C + (size_t)z * p.sC : nullptr;
        uint8_t *const cp = PACKED_C ? p.Cp + (size_t)z * p.sCp + (size_t)blockIdx.x * p.c_tile_steps * kPackedStep +
                                       (size_t)(t >> 3) * 256 + (size_t)(t & 7) * 16 : nullptr;
        const float *app = (p.app && row_ok) ? p.app + (size_t)z * p.sApp + (size_t)row * p.app_ld : nullptr;       // appended input columns (skip connection)
        const int app_hot = p.app_onehot ? (int)(row % p.app_w) : -1;
        const bool aux_blk = MODE == kModeMult ? mul_blk : false;
        const float *aux_src = MODE == kModeMult ? mul : bias;        // bias (LINEAR / SOFTPLUS) or multiplier (MULT)
        const int aux_ld = MODE == kModeMult ? p.ldmul : p.ldb;
        const bool aux_vec = aux_src && (aux_ld % 4 == 0) && ((n0 & 3) == 0) && ((reinterpret_cast<uintptr_t>(aux_src) & 15) == 0);
        const bool c_vec = (p.ldc % 4 == 0) && ((n0 & 3) == 0) && ((reinterpret_cast<uintptr_t>(Cz) & 15) == 0);
        const bool d_vec = p.Dv && (p.lddv % 4 == 0) && (p.sDv % 4 == 0) && ((n0 & 3) == 0) && ((reinterpret_cast<uintptr_t>(p.Dv) & 15) == 0);
        // FULL: all 16 columns of the unit exist (no per-column guards, constant address offsets)
        auto finish_unit = [&](int c0, auto full_c) {
            constexpr bool FULL = decltype(full_c)::value;
            float aux[16];
            const int unit = c0 >> 4;
            if (unit_in_ring(unit)) {
                const int slot = unit % kMulSlots;
                mbar_wait(&sm.mul_full[unit], 0);
#pragma unroll
                for (int e = 0; e < 16; ++e) aux[e] = mring[slot][e][t];
                __syncwarp();
                if (lane == 0) mbar_arrive(&sm.mul_empty[unit]);
            } else if (row_ok) {
                if (aux_blk) {
                    const float *ab = aux_src ? aux_src + (size_t)(n0 + c0) * 128 : nullptr;
#pragma unroll
                    for (int e = 0; e < 16; ++e) aux[e] = (ab && (FULL || n0 + c0 + e < p.N)) ? ab[e * 128] : 0.f;
                } else if (FULL && aux_vec && !aux_blk) {
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const float4 f = reinterpret_cast<const float4 *>(aux_src + n0 + c0)[i];      // plain loads: C may alias Mul
                        aux[4 * i] = f.x; aux[4 * i + 1] = f.y; aux[4 * i + 2] = f.z; aux[4 * i + 3] = f.w;
                    }
                } else {
#pragma unroll
                    for (int e = 0; e < 16; ++e) aux[e] = (aux_src && (FULL || n0 + c0 + e < p.N)) ? aux_src[n0 + c0 + e] : 0.f;
                }
            }
            TCL_EVT(threadIdx.x == 0, 11, c0 >> 4);
            if (!row_ok) return;
            // second-order coupling: cpl = coef * z * a of this row's 16 features (a: hi + lo of the packed operand)
            float cpl[16];
            const bool coupled = MODE == kModeMult && p.cpl_z && ((n0 + c0) >> 4) < p.cpl_a_steps;
            if (coupled) {
                const float *zb = p.cpl_z + (size_t)z * p.sCplZ + (size_t)blockIdx.x * p.ldmul * 128 + (size_t)(n0 + c0) * 128 + t;
                const uint8_t *ab = p.cpl_a + (size_t)z * p.sCplA + ((size_t)blockIdx.x * p.cpl_a_steps + ((n0 + c0) >> 4)) * kPackedStep +
                                    (size_t)(t >> 3) * 256 + (size_t)(t & 7) * 16;
                const uint4 h0 = *reinterpret_cast<const uint4 *>(ab), h1 = *reinterpret_cast<const uint4 *>(ab + 128);
                const uint4 l0 = *reinterpret_cast<const uint4 *>(ab + 4096), l1 = *reinterpret_cast<const uint4 *>(ab + 4096 + 128);
                const uint32_t hw[8] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
                const uint32_t lw[8] = {l0.x, l0.y, l0.z, l0.w, l1.x, l1.y, l1.z, l1.w};
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const float2 a = __half22float2(*reinterpret_cast<const __half2 *>(&hw[i]));
                    const float2 b = __half22float2(*reinterpret_cast<const __half2 *>(&lw[i]));
                    const bool ok0 = FULL || n0 + c0 + 2 * i < p.N, ok1 = FULL || n0 + c0 + 2 * i + 1 < p.N;
                    cpl[2 * i] = ok0 ? p.cpl_coef * zb[(size_t)(2 * i) * 128] * (a.x + b.x) : 0.f;
                    cpl[2 * i + 1] = ok1 ? p.cpl_coef * zb[(size_t)(2 * i + 1) * 128] * (a.y + b.y) : 0.f;
                }
            }
            float o[16], dv[16];
#pragma unroll
            for (int e = 0; e < 16; ++e) {
                float x = drow[c0 + e];
                dv[e] = 0.f;
                if (!FULL && n0 + c0 + e >= p.N) {
                    // beyond the layer's width: zero, or the columns appended for the next layer (`cat([h, xyz])`, tangent seeds)
                    const int a = n0 + c0 + e - p.N;
                    x = 0.f;
                    if (a < p.app_w) x = p.app_onehot ? (a == app_hot ? 1.f : 0.f) : (app ? app[a] : 0.f);
                }
                if (FULL || n0 + c0 + e < p.N) {
                    if (MODE == kModeMult) {
                        dv[e] = x;
                        x *= aux[e] * rscale;
                        if (coupled) x = fmaf(1.0f - aux[e], cpl[e], x);
                    } else {
                        x += aux[e];
                        if (MODE == kModeSoftplus) {
                            // softplus(beta = 100) and its derivative in log2 units: u = 100 log2(e) x
                            // log2(1 + 2^-|u|) by a degree-6 polynomial in 2^-|u| on the FMA pipe (the fused kernels' scheme) on
                            // every other element, by the second MUFU on the rest: the pass is bound by the MUFU pipe
                            const float u = x * kS;
                            float ex, lg;
                            asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(ex) : "f"(-fabsf(u)));
                            if (e & 1) {
                                float pl = fmaf(ex, -0.02645743577f, 0.1234514468f);
                                pl = fmaf(pl, ex, -0.2795380944f);
                                pl = fmaf(pl, ex, 0.4582707841f);
                                pl = fmaf(pl, ex, -0.7182819141f);
                                pl = fmaf(pl, ex, 1.442553145f);
                                lg = pl * ex;
                            } else {
                                asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(lg) : "f"(1.0f + ex));
                            }
                            x = (fmaxf(u, 0.0f) + lg) * (1.0f / kS);
                            if (p.Dv) dv[e] = __fdividef(u >= 0.f ? 1.0f : ex, 1.0f + ex);
                        }
                    }
                }
                o[e] = x;
            }
            TCL_EVT(threadIdx.x == 0, 13, c0 >> 4);
            if (PACKED_C && ((n0 + c0) >> 4) < p.c_ksteps) {
                // operand-ready output: this unit is k-step (n0 + c0) / 16 of the next layer's A tile, fp16 hi | lo, core-matrix order
                uint32_t hi[8], lo[8];
#pragma unroll
                for (int i = 0; i < 8; ++i) split2(o[2 * i], o[2 * i + 1], hi[i], lo[i]);
                uint8_t *dst = cp + (size_t)((n0 + c0) >> 4) * kPackedStep;
                *reinterpret_cast<uint4 *>(dst) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
                *reinterpret_cast<uint4 *>(dst + 128) = make_uint4(hi[4], hi[5], hi[6], hi[7]);
                *reinterpret_cast<uint4 *>(dst + 4096) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
                *reinterpret_cast<uint4 *>(dst + 4096 + 128) = make_uint4(lo[4], lo[5], lo[6], lo[7]);
            }
            TCL_EVT(threadIdx.x == 0, 14, c0 >> 4);
            if (p.Dv && (p.blocked || p.dv_blocked)) {
                float *db = p.Dv + (size_t)z * p.sDv + (size_t)blockIdx.x * p.lddv * 128 + (size_t)(n0 + c0) * 128 + t;
#pragma unroll
                for (int e = 0; e < 16; ++e)
                    if (FULL || n0 + c0 + e < p.N) db[e * 128] = dv[e];
            }
            TCL_EVT(threadIdx.x == 0, 15, c0 >> 4);
            if (!Cz) return;
            if (p.blocked) {
                float *cb = Cz + (size_t)blockIdx.x * p.ldc * 128 + (size_t)(n0 + c0) * 128 + t;
#pragma unroll
                for (int e = 0; e < 16; ++e)
                    if (FULL || n0 + c0 + e < p.N) cb[e * 128] = o[e];
                return;
            }
            float *crow = Cz + (size_t)row * p.ldc + n0 + c0;
            if (FULL && c_vec) {
#pragma unroll
                for (int i = 0; i < 4; ++i)
                    reinterpret_cast<float4 *>(crow)[i] = make_float4(o[4 * i], o[4 * i + 1], o[4 * i + 2], o[4 * i + 3]);
            } else {
#pragma unroll
                for (int e = 0; e < 16; ++e)
                    if (FULL || n0 + c0 + e < p.N) crow[e] = o[e];
            }
            if (p.Dv && !p.dv_blocked) {
                float *dvrow = p.Dv + (size_t)z * p.sDv + (size_t)row * p.lddv + n0 + c0;
                if (FULL && d_vec) {
#pragma unroll
                    for (int i = 0; i < 4; ++i)
                        reinterpret_cast<float4 *>(dvrow)[i] = make_float4(dv[4 * i], dv[4 * i + 1], dv[4 * i + 2], dv[4 * i + 3]);
                } else {
#pragma unroll
                    for (int e = 0; e < 16; ++e)
                        if (FULL || n0 + c0 + e < p.N) dvrow[e] = dv[e];
                }
            }
        };
        for (int c0 = 16 * half; c0 < p.Nt; c0 += 32) {
            if (n0 + c0 + 16 <= p.N) finish_unit(c0, std::true_type());
            else finish_unit(c0, std::false_type());
        }
        TCL_EVT(threadIdx.x == 0, 9, 2);
    }

}

// W [rows x ldw] fp32 (reference layout [out][in]) -> slabs.  B[n][k] = scale * (transpose ? W[k0 + k][n0w + n] : W[n0w + n][k0 + k])
// for n < N, k < K, zero elsewhere; n tiles of Nt, k-steps of 16; per slab Nt x 16 hi then Nt x 16 lo in core-matrix order.
__global__ void pack_linear_kernel(const float *__restrict__ W, int ldw, int N, int K, int n_off, int k_off, int transpose,
                                   float scale, const float *__restrict__ k_scale, int Nt, int n_tiles, int ksteps,
                                   uint8_t *__restrict__ out)
{
    const size_t total = (size_t)n_tiles * ksteps * Nt * 16;
    for (size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
        const int kk = (int)(t % 16);
        const int nn = (int)((t / 16) % Nt);
        const int j = (int)((t / (16 * (size_t)Nt)) % ksteps);
        const int tile = (int)(t / (16 * (size_t)Nt * ksteps));
        const int n = tile * Nt + nn, k = j * 16 + kk;
        float v = 0.f;
        if (n < N && k < K) {
            v = scale * (transpose ? W[(size_t)(k_off + k) * ldw + n_off + n] : W[(size_t)(n_off + n) * ldw + k_off + k]);
            if (k_scale) v *= k_scale[k];
        }
        const __half hi = __float2half_rn(v);
        const __half lo = __float2half_rn(v - __half2float(hi));
        const size_t off = (size_t)(nn >> 3) * 256 + (size_t)(kk >> 3) * 128 + (size_t)(nn & 7) * 16 + (size_t)(kk & 7) * 2;
        uint8_t *base = out + ((size_t)tile * ksteps + j) * Nt * 64;
        *reinterpret_cast<__half *>(base + off) = hi;
        *reinterpret_cast<__half *>(base + (size_t)Nt * 32 + off) = lo;
    }
}

int choose_nt(int N, int max_nt)
{
    // as few tiles of <= max_nt columns as possible, equally wide (277 -> 2 x 144, not 256 + 21), rounded up to 16
    const int tiles = (N + max_nt - 1) / max_nt;
    return ((N + tiles - 1) / tiles + 15) / 16 * 16;
}

int PackedLinear::pack(const float *W_dev, int ldw, int N_, int K_, int n_off, int k_off, bool transpose, float scale,
                       cudaStream_t stream, int sets_, long long w_set_stride, const float *k_scale_dev, long long k_scale_stride,
                       int n_extra_, int max_nt)
{
    N = N_; K = K_; n_extra = n_extra_;
    if (max_nt <= 0 || max_nt > kMaxNt) max_nt = kMaxNt;
    Nt = choose_nt(N + n_extra, max_nt);
    n_tiles = (N + n_extra + Nt - 1) / Nt;
    ksteps = (K + 15) / 16;
    sets = sets_ > 0 ? sets_ : 1;
    set_bytes = (size_t)n_tiles * ksteps * Nt * 64;
    int rc;
    if ((rc = slabs.reserve(set_bytes * sets))) return rc;
    for (int s = 0; s < sets; ++s) {
        pack_linear_kernel<<<64, 256, 0, stream>>>(W_dev + (size_t)s * w_set_stride, ldw, N, K, n_off, k_off, transpose ? 1 : 0, scale,
                                                   k_scale_dev ? k_scale_dev + (size_t)s * k_scale_stride : nullptr, Nt, n_tiles,
                                                   ksteps, slabs.as<uint8_t>() + (size_t)s * set_bytes);
        NPHM_CUDA_CHECK(cudaGetLastError());
    }
    return NPHM_OK;
}

int launch_linear(const PackedLinear &w, LinearParams p, cudaStream_t stream)
{
    NPHM_REQUIRE(w.slabs.ptr && (p.C || p.Cp) && p.M > 0, "tc_linear: unpacked weights or NULL output");
    if (p.Ap) {
        NPHM_REQUIRE(!p.A1 && !p.A2 && !p.a2_onehot && p.a_ksteps == w.ksteps,
                     "tc_linear: packed input of %d k-steps does not match the packed weights (%d)", p.a_ksteps, w.ksteps);
    } else {
        NPHM_REQUIRE(p.K1 + p.K2 == w.K, "tc_linear: input width %d + %d does not match the packed weights (%d)", p.K1, p.K2, w.K);
    }
    NPHM_REQUIRE(!p.Cp || (p.c_ksteps >= (w.N + p.app_w + 15) / 16 && p.app_w <= w.n_extra && (!p.Dv || p.dv_blocked || p.C)),
                 "tc_linear: packed output misconfigured");
    NPHM_REQUIRE(p.app_w == 0 || p.Cp, "tc_linear: appended columns need a packed output");
    NPHM_REQUIRE(p.mode != kModeMult || (p.Mul && p.mul_div > 0), "tc_linear: multiplier missing");
    NPHM_REQUIRE(!p.cpl_z || (p.mode == kModeMult && p.cpl_a && p.cpl_a_steps > 0 && (p.blocked || p.mul_blocked) && p.mul_div <= 1),
                 "tc_linear: the coupling term needs the multiplier epilogue with a blocked multiplier, one row per multiplier row");
    NPHM_REQUIRE(!p.blocked || (!p.bias && !p.A2 && !p.a2_onehot && p.mul_div <= 1),
                 "tc_linear: the blocked layout supports the plain and the multiplier epilogue only");
    NPHM_REQUIRE(p.batch >= 1 && (p.batch == 1 || (!p.A2 && !p.a2_onehot && !p.app_onehot)),
                 "tc_linear: batched launches take no second or one-hot input");
    if (p.batch > 1) {
        const int need = member_set(p.batch - 1, p.w_pairs) + 1;
        NPHM_REQUIRE(need <= w.sets, "tc_linear: batch of %d needs %d weight sets, %d packed", p.batch, need, w.sets);
    }
    if (p.a_tile_steps <= 0) p.a_tile_steps = p.a_ksteps;
    if (p.c_tile_steps <= 0) p.c_tile_steps = p.c_ksteps;
    p.W = w.slabs.as<uint8_t>();
    p.w_stride = (long long)w.set_bytes;
    p.N = w.N; p.Nt = w.Nt; p.ksteps = w.ksteps;
    if (p.rows_per_bias <= 0) p.rows_per_bias = p.M;
    if (p.mul_div <= 0) p.mul_div = 1;
    const bool packed_a = p.Ap != nullptr;
    p.stages = kMaxStages;
    while (p.stages > 2 && smem_bytes(p.Nt, p.stages, packed_a) > kMaxSmem) --p.stages;
    const int smem = smem_bytes(p.Nt, p.stages, packed_a);
    using Kernel = void (*)(const LinearParams);
    const bool pc = p.Cp != nullptr;
    Kernel kern = p.mode == kModeMult       ? (pc ? (Kernel)linear_tc_kernel<kModeMult, true> : (Kernel)linear_tc_kernel<kModeMult, false>)
                  : p.mode == kModeSoftplus ? (pc ? (Kernel)linear_tc_kernel<kModeSoftplus, true> : (Kernel)linear_tc_kernel<kModeSoftplus, false>)
                                            : (pc ? (Kernel)linear_tc_kernel<kModeLinear, true> : (Kernel)linear_tc_kernel<kModeLinear, false>);
    NPHM_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem));
    dim3 grid((unsigned)ceil_div(p.M, 128), (unsigned)w.n_tiles, (unsigned)p.batch);
    kern<<<grid, kThreads, smem, stream>>>(p);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

}  // namespace tcl
}  // namespace nphm

#ifdef NPHM_TCL_TRACE
extern "C" int nphm_debug_tcl_trace(long long *host, int n_ll)
{
    using namespace nphm;
    NPHM_CUDA_CHECK(cudaDeviceSynchronize());
    NPHM_CUDA_CHECK(cudaMemcpyFromSymbol(host, tcl::g_tcl_trace, (size_t)n_ll * 8));
    return NPHM_OK;
}
#endif

// Test entry (not part of the public ABI; tests/test_gpu_networks.py): three chained layers per batch entry on the generic layer,
//   H1 = A W1^T                      row-major fp32 in  -> packed out
//   H2 = (H1 W2^T) * Mul             packed in, blocked multiplier (streamed through the shared-memory ring) -> packed out
//   Z  = H2 W3^T                     packed in -> row-major fp32 out
// a [batch][M][K], w1 [sets][N1][K], w2 [sets][N2][N1], w3 [sets][N3][N2], mul [batch][ceil(M/128)][N2 rounded up to 4][128],
// z [batch][M][N3]; batch entry b uses weight set b/2 for b < 2 w_pairs, b - w_pairs beyond.
extern "C" int nphm_debug_linear_chain(const float *a_dev, const float *w1_dev, const float *w2_dev, const float *w3_dev,
                                       const float *mul_dev, int batch, int w_pairs, long long M, int K, int N1, int N2, int N3,
                                       float *z_dev, void *stream_)
{
    using namespace nphm;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    NPHM_REQUIRE(a_dev && w1_dev && w2_dev && w3_dev && mul_dev && z_dev && batch >= 1 && M > 0, "nphm_debug_linear_chain: bad arguments");
    const int sets = batch - w_pairs;
    tcl::PackedLinear l1, l2, l3;
    int rc;
    if ((rc = l1.pack(w1_dev, K, N1, K, 0, 0, false, 1.0f, stream, sets, (long long)N1 * K)) ||
        (rc = l2.pack(w2_dev, N1, N2, N1, 0, 0, false, 1.0f, stream, sets, (long long)N2 * N1)) ||
        (rc = l3.pack(w3_dev, N2, N3, N2, 0, 0, false, 1.0f, stream, sets, (long long)N3 * N2))) return rc;
    const long long tiles = ceil_div(M, 128);
    const int ks1 = l1.packed_ksteps_out(), ks2 = l2.packed_ksteps_out(), ldm = (N2 + 3) / 4 * 4;
    DeviceBuffer h1, h2;
    if ((rc = h1.reserve((size_t)batch * tiles * ks1 * 8192)) || (rc = h2.reserve((size_t)batch * tiles * ks2 * 8192))) return rc;
    tcl::LinearParams p{};
    p.M = M; p.batch = batch; p.w_pairs = w_pairs;
    p.A1 = a_dev; p.lda1 = K; p.K1 = K; p.sA1 = M * K;
    p.mode = tcl::kModeLinear; p.Cp = h1.as<uint8_t>(); p.c_ksteps = ks1; p.sCp = tiles * ks1 * 8192;
    if ((rc = tcl::launch_linear(l1, p, stream))) return rc;
    p = tcl::LinearParams{};
    p.M = M; p.batch = batch; p.w_pairs = w_pairs;
    p.Ap = h1.as<uint8_t>(); p.a_ksteps = ks1; p.sAp = tiles * ks1 * 8192;
    p.mode = tcl::kModeMult; p.Mul = mul_dev; p.ldmul = ldm; p.mul_blocked = 1; p.sMul = tiles * 128 * ldm;
    p.Cp = h2.as<uint8_t>(); p.c_ksteps = ks2; p.sCp = tiles * ks2 * 8192;
    if ((rc = tcl::launch_linear(l2, p, stream))) return rc;
    p = tcl::LinearParams{};
    p.M = M; p.batch = batch; p.w_pairs = w_pairs;
    p.Ap = h2.as<uint8_t>(); p.a_ksteps = ks2; p.sAp = tiles * ks2 * 8192;
    p.mode = tcl::kModeLinear; p.C = z_dev; p.ldc = N3; p.sC = M * N3;
    if ((rc = tcl::launch_linear(l3, p, stream))) return rc;
    NPHM_CUDA_CHECK(cudaStreamSynchronize(stream));          // the temporaries above are freed on return
    return NPHM_OK;
}
