// Marching cubes over an SDF slab on sm_90a, bit-exact (triangle ids, vertex order, double-precision vertex
// positions) with the sequential PyMCubes algorithm restated in oracle/mc_oracle.c.
//
// Reference call site: src/NPHM/utils/reconstruction.py:30  mcubes.marching_cubes(logits, 0.0)
//
// The sequential algorithm numbers vertices in creation order while sweeping cells x-major.  A vertex lives
// on a grid edge and is created by the first cell (in sweep order) that contains that edge, so the id of any
// vertex is   (number of vertices created by earlier cells) + (rank among the vertices its owner cell creates),
// both of which are pure functions of the 8-corner case index of the cells involved.
//
// Work decomposition: ONE WARP PER CELL ROW (all cells with the same (x, y), z running), a lane owns 8 consecutive
// cells of the row ("group"):
//   K1 classify : every voxel row is read with 128-bit loads (9 values per lane and voxel row, the 9th from the
//                 neighbour lane), 8 case indices per lane -> one 8-byte store; created-vertex counts are scanned
//                 inside the warp -> u16 prefix per group; per-row vertex / triangle counts            [HBM bound]
//   K2 scan     : exclusive scan of the row counts (chunks of 2048 rows, the last CTA scans the chunk sums)
//   K3 emit     : rows without a surface crossing exit at once (a 256^3 head: ~1.5 % of the cells are active).  Vertex
//                 base of ANY cell = row base + group prefix + popcounts of at most 7 case bytes of its group, so the
//                 owner-cell lookup of a triangle corner costs one 8-byte load instead of a per-cell u32 array.
// Algorithmic HBM traffic: 4 B/voxel read + 24 B/vertex + 24 B/triangle written; scratch: 1 B/cell (case index) +
// 2 B per 8 cells (group prefix) written once, read once by K3 (rows with a crossing and their neighbours only).
#include "common.cuh"
#include "mc_tables.h"
#include <cstring>

namespace nphm {

namespace {

constexpr int kWarpsPerCta = 8;
constexpr int kRowThreads = 32 * kWarpsPerCta;
constexpr int kRowChunk = 2048;               // rows per CTA of the scan kernel (256 threads x 8 rows)

__constant__ unsigned short c_edge_table[256];
__constant__ signed char c_tri_table[256][16];
__constant__ unsigned char c_num_tris[256];
// creation order inside a cell: edges 6, 5, 10, then 0, 1, 2, 3, 4, 7, 8, 9, 11
__constant__ unsigned short c_before_mask[12];     // edges created before edge e in that order
__constant__ unsigned char c_create_order[12];
// the same tables packed for the kernels' shared-memory staging: read with coalesced 128-bit loads from global memory (a
// per-thread-indexed read of __constant__ memory serialises 32-way; staging 4.8 KB that way cost more than the rest of the
// emit kernel): [0,512) edge table u16 | [512,768) triangle counts u8 | [768,4864) triangle table i8[256][16]
constexpr int kTabEdge = 0, kTabNtri = 512, kTabTri = 768, kTabBytes = 4864;
__device__ uint4 g_tables[kTabBytes / 16];
bool g_tables_loaded[64] = {false};

const int h_create_order[12] = {6, 5, 10, 0, 1, 2, 3, 4, 7, 8, 9, 11};
// corner offsets and edge end corners (Bourke order: edge e runs from corner A[e] to corner B[e])
__constant__ unsigned char c_corner[8][3] = {{0,0,0},{1,0,0},{1,1,0},{0,1,0},{0,0,1},{1,0,1},{1,1,1},{0,1,1}};
__constant__ unsigned char c_edge_a[12] = {0, 1, 2, 3, 4, 5, 6, 7, 0, 1, 2, 3};
__constant__ unsigned char c_edge_b[12] = {1, 2, 3, 0, 5, 6, 7, 4, 4, 5, 6, 7};
// edge id from (axis, offset of its low end point along the two other axes): [axis][d_first][d_second]
// x edges: (dj,dk); y edges: (di,dk); z edges: (di,dj)
__constant__ unsigned char c_edge_of[3][2][2] = {{{0, 4}, {2, 6}}, {{3, 7}, {1, 5}}, {{8, 11}, {9, 10}}};

struct Dims {
    int nx, ny, nz;          // planes
    int cx, cy, cz;          // cells = planes - 1
    long long ncells;
    int n_rows;              // cx * cy cell rows
    int pitch;               // bytes of one row of case indices (cz rounded up to 8)
    int ngrp;                // groups of 8 cells per row
    int x_global0, ghost_lo, negate;
    int cmp_float;           // the inside test can be done in fp32 (iso is exactly representable)
    float thr;               // fp32 threshold: inside <=> v <= thr  (negate: v >= thr)
    double iso;
};

// edges whose vertex this cell creates (it is the first cell in sweep order containing the edge)
__device__ __forceinline__ unsigned own_mask(int gi, int cj, int ck)
{
    unsigned m = (1u << 6) | (1u << 5) | (1u << 10);
    const bool i0 = gi == 0, j0 = cj == 0, k0 = ck == 0;
    if (j0 && k0) m |= 1u << 0;
    if (k0) m |= (1u << 2) | (1u << 1);
    if (j0) m |= (1u << 4) | (1u << 9);
    if (i0) m |= (1u << 7) | (1u << 11);
    if (i0 && k0) m |= 1u << 3;
    if (i0 && j0) m |= 1u << 8;
    return m;
}

// PyMCubes: corner bit set when value <= iso (on -vol when `negate`)
__device__ __forceinline__ unsigned inside(const Dims &d, float v)
{
    if (d.cmp_float) return d.negate ? (v >= d.thr) : (v <= d.thr);
    const double f = d.negate ? -(double)v : (double)v;
    return f <= d.iso;
}

__device__ __forceinline__ unsigned warp_inclusive_scan(unsigned v, int lane)
{
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned t = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += t;
    }
    return v;
}

// 9 consecutive voxels [kb, kb+8] of one voxel row as inside bits (bit p = voxel kb+p); out-of-range voxels read as 0
template <bool ALIGNED>
__device__ __forceinline__ unsigned row_bits(const Dims &d, const float *__restrict__ rowp, int kb, int lane)
{
    unsigned bits = 0;
    float first;
    if (ALIGNED && kb + 8 <= d.nz) {
        const float4 a = __ldg(reinterpret_cast<const float4 *>(rowp + kb));
        const float4 b = __ldg(reinterpret_cast<const float4 *>(rowp + kb + 4));
        first = a.x;
        bits = inside(d, a.x) | (inside(d, a.y) << 1) | (inside(d, a.z) << 2) | (inside(d, a.w) << 3) |
               (inside(d, b.x) << 4) | (inside(d, b.y) << 5) | (inside(d, b.z) << 6) | (inside(d, b.w) << 7);
    } else {
        first = kb < d.nz ? __ldg(rowp + kb) : 0.f;
        bits = kb < d.nz ? inside(d, first) : 0u;
#pragma unroll
        for (int p = 1; p < 8; ++p)
            if (kb + p < d.nz) bits |= inside(d, __ldg(rowp + kb + p)) << p;
    }
    // voxel kb + 8 is the neighbour lane's first voxel
    float nxt = __shfl_down_sync(0xffffffffu, first, 1);
    if (lane == 31) nxt = kb + 8 < d.nz ? __ldg(rowp + kb + 8) : 0.f;
    if (kb + 8 < d.nz) bits |= inside(d, nxt) << 8;
    return bits;
}

// K1 ---------------------------------------------------------------------------------------------
template <bool ALIGNED>
__global__ void __launch_bounds__(kRowThreads) mc_classify_rows_kernel(const float *__restrict__ vol, const Dims d,
                                                                       unsigned char *__restrict__ cube_out,
                                                                       unsigned short *__restrict__ grp_prefix,
                                                                       unsigned *__restrict__ row_nv, unsigned *__restrict__ row_nt)
{
    __shared__ uint4 s_tab[kTabTri / 16];
    for (int i = threadIdx.x; i < kTabTri / 16; i += kRowThreads) s_tab[i] = __ldg(g_tables + i);
    __syncthreads();
    const unsigned short *s_edge = reinterpret_cast<const unsigned short *>(s_tab);
    const unsigned char *s_ntri = reinterpret_cast<const unsigned char *>(s_tab) + kTabNtri;
    const int lane = threadIdx.x & 31;
    const int r = blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5);
    if (r >= d.n_rows) return;
    const int ci = r / d.cy, cj = r - ci * d.cy;
    const int gi = d.x_global0 + ci;
    const size_t sx = (size_t)d.ny * d.nz;
    const float *r00 = vol + (size_t)ci * sx + (size_t)cj * d.nz;
    const float *r10 = r00 + sx, *r01 = r00 + d.nz, *r11 = r10 + d.nz;
    unsigned carry_v = 0, tot_t = 0;
    for (int k0 = 0; k0 < d.cz; k0 += 256) {
        const int kb = k0 + 8 * lane;
        // corner order of a cell: v0 (i,j,k) v1 (i+1,j,k) v2 (i+1,j+1,k) v3 (i,j+1,k), v4..v7 the same at k+1
        const unsigned b00 = row_bits<ALIGNED>(d, r00, kb, lane), b10 = row_bits<ALIGNED>(d, r10, kb, lane);
        const unsigned b11 = row_bits<ALIGNED>(d, r11, kb, lane), b01 = row_bits<ALIGNED>(d, r01, kb, lane);
        unsigned cubes[8];
        unsigned nv = 0, nt = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const unsigned lo = ((b00 >> j) & 1) | (((b10 >> j) & 1) << 1) | (((b11 >> j) & 1) << 2) | (((b01 >> j) & 1) << 3);
            const unsigned hi = ((b00 >> (j + 1)) & 1) | (((b10 >> (j + 1)) & 1) << 1) | (((b11 >> (j + 1)) & 1) << 2) |
                                (((b01 >> (j + 1)) & 1) << 3);
            const unsigned cube = kb + j < d.cz ? (lo | (hi << 4)) : 0u;
            cubes[j] = cube;
            nv += __popc(s_edge[cube] & own_mask(gi, cj, kb + j));
            nt += s_ntri[cube];
        }
        const unsigned inc = warp_inclusive_scan(nv, lane);
        if (kb < d.pitch) {
            uint2 pk;
            pk.x = cubes[0] | (cubes[1] << 8) | (cubes[2] << 16) | (cubes[3] << 24);
            pk.y = cubes[4] | (cubes[5] << 8) | (cubes[6] << 16) | (cubes[7] << 24);
            *reinterpret_cast<uint2 *>(cube_out + (size_t)r * d.pitch + kb) = pk;
            grp_prefix[(size_t)r * d.ngrp + (kb >> 3)] = (unsigned short)(carry_v + inc - nv);
        }
        carry_v += __shfl_sync(0xffffffffu, inc, 31);
#pragma unroll
        for (int o = 16; o; o >>= 1) nt += __shfl_xor_sync(0xffffffffu, nt, o);
        tot_t += nt;
    }
    if (lane == 0) { row_nv[r] = carry_v; row_nt[r] = tot_t; }
}

// K2: exclusive scan of the row counts.  row_v/row_t receive the exclusive prefix INSIDE their chunk of kRowChunk rows,
// chunk_v/chunk_t the exclusive prefix of the chunk sums (written by the last CTA to finish), totals[0..1] the grand
// totals and totals[2..3] what the ghost layer (cell layer 0 of a slab with ghost_lo) creates.
__global__ void __launch_bounds__(256) mc_scan_rows_kernel(const unsigned *__restrict__ row_nv, const unsigned *__restrict__ row_nt,
                                                           unsigned *__restrict__ row_v, unsigned *__restrict__ row_t,
                                                           unsigned *__restrict__ chunk_v, unsigned *__restrict__ chunk_t,
                                                           int n_rows, int ghost_rows, unsigned long long *__restrict__ totals)
{
    __shared__ unsigned wsum[2][8];
    __shared__ bool last;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int r0 = blockIdx.x * kRowChunk + threadIdx.x * 8;
    unsigned v[8], t[8], sv = 0, st = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        v[i] = r0 + i < n_rows ? row_nv[r0 + i] : 0u;
        t[i] = r0 + i < n_rows ? row_nt[r0 + i] : 0u;
        sv += v[i]; st += t[i];
    }
    const unsigned iv = warp_inclusive_scan(sv, lane), it = warp_inclusive_scan(st, lane);
    if (lane == 31) { wsum[0][warp] = iv; wsum[1][warp] = it; }
    __syncthreads();
    unsigned bv = iv - sv, bt = it - st;
    for (int w = 0; w < warp; ++w) { bv += wsum[0][w]; bt += wsum[1][w]; }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        if (r0 + i < n_rows) { row_v[r0 + i] = bv; row_t[r0 + i] = bt; }
        bv += v[i]; bt += t[i];
    }
    if (threadIdx.x == 255) { chunk_v[blockIdx.x] = bv; chunk_t[blockIdx.x] = bt; }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned *ticket = reinterpret_cast<unsigned *>(totals + 8);
        last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last) return;
    __threadfence();
    if (warp == 0) {
        unsigned long long cv = 0, ct = 0;
        for (int base = 0; base < (int)gridDim.x; base += 32) {
            const int i = base + lane;
            const unsigned a = i < (int)gridDim.x ? __ldcg(chunk_v + i) : 0u, b = i < (int)gridDim.x ? __ldcg(chunk_t + i) : 0u;
            const unsigned ia = warp_inclusive_scan(a, lane), ib = warp_inclusive_scan(b, lane);
            if (i < (int)gridDim.x) { chunk_v[i] = (unsigned)cv + ia - a; chunk_t[i] = (unsigned)ct + ib - b; }
            cv += __shfl_sync(0xffffffffu, ia, 31);
            ct += __shfl_sync(0xffffffffu, ib, 31);
        }
        __threadfence();
        __syncwarp();
        if (lane == 0) {
            totals[0] = cv; totals[1] = ct;
            if (ghost_rows > 0 && ghost_rows < n_rows) {
                totals[2] = (unsigned long long)__ldcg(chunk_v + ghost_rows / kRowChunk) + __ldcg(row_v + ghost_rows);
                totals[3] = (unsigned long long)__ldcg(chunk_t + ghost_rows / kRowChunk) + __ldcg(row_t + ghost_rows);
            } else if (ghost_rows > 0) {
                totals[2] = cv; totals[3] = ct;
            }
        }
    }
}

// K3 ---------------------------------------------------------------------------------------------
__device__ __forceinline__ double mc_interp(double iso, double fa, double fb, double xa, double xb)
{
    if (fb == fa) return __ddiv_rn(__dadd_rn(xb, xa), 2.0);
    // (xb - xa) * (iso - fa) / (fb - fa) + xa, evaluated left to right without contraction
    const double num = __dmul_rn(__dsub_rn(xb, xa), __dsub_rn(iso, fa));
    return __dadd_rn(__ddiv_rn(num, __dsub_rn(fb, fa)), xa);
}

struct Scratch {
    const unsigned char *cube;
    const unsigned short *grp_prefix;
    const unsigned *row_nv, *row_nt, *row_v, *row_t, *chunk_v, *chunk_t;
    const unsigned long long *totals;
};

// One warp per cell row.  The active cells of the row (a handful out of 255 for a head) are processed ONE AT A TIME BY THE
// WHOLE WARP: lane e < 12 resolves the vertex id of cube edge e (owner cell lookup), lane o < 12 creates the o-th vertex
// of the cell's creation order, lane m < 3 * n_triangles writes one triangle index (ids travel by shuffle).  The per-edge
// constants (end corners, axis, creation rank mask) are therefore per-LANE constants held in registers.
__global__ void __launch_bounds__(kRowThreads) mc_emit_rows_kernel(const float *__restrict__ vol, const Dims d, const Scratch w,
                                                                   long long vert_id_base, double *__restrict__ verts,
                                                                   long long *__restrict__ tris)
{
    __shared__ uint4 s_tab[kTabBytes / 16];
    const int lane = threadIdx.x & 31;
    const int r = blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5);
    const int ci = r < d.n_rows ? r / d.cy : 0, cj = r < d.n_rows ? r - ci * d.cy : 0;
    // rows that emit nothing: beyond the end, the ghost layer (owner cells only), no surface crossing
    const bool idle = r >= d.n_rows || (d.ghost_lo && ci == 0) || (w.row_nv[r] == 0 && w.row_nt[r] == 0);
    if (__syncthreads_and(idle)) return;                     // most CTAs of a head volume: nothing to do, no table staging
    for (int i = threadIdx.x; i < kTabBytes / 16; i += kRowThreads) s_tab[i] = __ldg(g_tables + i);
    __syncthreads();
    if (idle) return;
    const unsigned short *s_edge = reinterpret_cast<const unsigned short *>(s_tab);
    const unsigned char *s_ntri = reinterpret_cast<const unsigned char *>(s_tab) + kTabNtri;
    const signed char (*s_tri)[16] = reinterpret_cast<const signed char (*)[16]>(reinterpret_cast<const unsigned char *>(s_tab) + kTabTri);
    const int gi = d.x_global0 + ci;
    const unsigned ghost_v = d.ghost_lo ? (unsigned)w.totals[2] : 0u;
    const unsigned ghost_t = d.ghost_lo ? (unsigned)w.totals[3] : 0u;
    auto base_v = [&](int row) { return w.chunk_v[row / kRowChunk] + w.row_v[row]; };
    // vertex bases of the four rows an owner cell can live in: [di][dj] = row (ci - di, cj - dj)
    unsigned rb[2][2];
    rb[0][0] = base_v(r);
    rb[0][1] = cj > 0 ? base_v(r - 1) : 0u;
    rb[1][0] = ci > 0 ? base_v(r - d.cy) : 0u;
    rb[1][1] = (ci > 0 && cj > 0) ? base_v(r - d.cy - 1) : 0u;
    const unsigned my_t = w.chunk_t[r / kRowChunk] + w.row_t[r] - ghost_t;

    // ---- per-lane constants.  Role T: lane e (< 12) looks up the vertex of cube edge e.  Role V: lane o (< 12) creates the
    // o-th vertex in creation order, i.e. the vertex of edge ev = c_create_order[o].
    const int e = lane < 12 ? lane : 0;
    const int ta = c_edge_a[e], tb = c_edge_b[e];
    const int t_axis = c_corner[ta][0] != c_corner[tb][0] ? 0 : (c_corner[ta][1] != c_corner[tb][1] ? 1 : 2);
    const int t_lo = c_corner[ta][t_axis] == 0 ? ta : tb;
    const int t_ox = c_corner[t_lo][0], t_oy = c_corner[t_lo][1], t_oz = c_corner[t_lo][2];
    const int ev = c_create_order[e];
    const int va = c_edge_a[ev], vb = c_edge_b[ev];
    const int v_axis = c_corner[va][0] != c_corner[vb][0] ? 0 : (c_corner[va][1] != c_corner[vb][1] ? 1 : 2);
    const int v_ax = c_corner[va][0], v_ay = c_corner[va][1], v_az = c_corner[va][2];
    const int v_bx = c_corner[vb][0], v_by = c_corner[vb][1], v_bz = c_corner[vb][2];
    const unsigned v_before = c_before_mask[ev];
    const size_t sx = (size_t)d.ny * d.nz, sy = d.nz;

    // absolute (un-shifted) id of the first vertex cell (fi, fj, fk) creates, and that cell's case index
    auto owner_cell = [&](int fi, int fj, int fk, unsigned &ocube) -> unsigned {
        const int ro = fi * d.cy + fj;
        const int g = fk >> 3;
        const uint2 grp = __ldg(reinterpret_cast<const uint2 *>(w.cube + (size_t)ro * d.pitch + 8 * g));
        unsigned n = rb[ci - fi][cj - fj] + w.grp_prefix[(size_t)ro * d.ngrp + g];
        const int gfi = d.x_global0 + fi;
        const int upto = fk & 7;
        for (int t = 0; t < upto; ++t) {
            const unsigned byte = ((t < 4 ? grp.x >> (8 * t) : grp.y >> (8 * (t - 4))) & 255u);
            n += __popc(s_edge[byte] & own_mask(gfi, fj, 8 * g + t));
        }
        ocube = ((upto < 4 ? grp.x >> (8 * upto) : grp.y >> (8 * (upto - 4))) & 255u);
        return n;
    };

    unsigned carry_t = 0;
    for (int k0 = 0; k0 < d.cz; k0 += 256) {
        const int kb = k0 + 8 * lane;
        uint2 grp = make_uint2(0u, 0u);
        if (kb < d.pitch) grp = __ldg(reinterpret_cast<const uint2 *>(w.cube + (size_t)r * d.pitch + kb));
        unsigned nt = 0, act = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const unsigned cb = (j < 4 ? grp.x >> (8 * j) : grp.y >> (8 * (j - 4))) & 255u;
            nt += s_ntri[cb];
            if (cb != 0u && cb != 255u) act |= 1u << j;
        }
        const unsigned inc_t = warp_inclusive_scan(nt, lane);
        unsigned t_run = my_t + carry_t + inc_t - nt;          // first triangle of this lane's next active cell
        carry_t += __shfl_sync(0xffffffffu, inc_t, 31);
        unsigned v_run = act ? rb[0][0] + w.grp_prefix[(size_t)r * d.ngrp + (kb >> 3)] : 0u;   // absolute id of its first vertex
        // ---- the warp walks over the active cells of this segment
        unsigned pending = __ballot_sync(0xffffffffu, act != 0u);
        while (pending) {
            const int L = __ffs(pending) - 1;
            const unsigned actL = __shfl_sync(0xffffffffu, act, L);
            const int j = __ffs(actL) - 1;
            const unsigned gx = __shfl_sync(0xffffffffu, grp.x, L), gy = __shfl_sync(0xffffffffu, grp.y, L);
            const unsigned cube = (j < 4 ? gx >> (8 * j) : gy >> (8 * (j - 4))) & 255u;
            const unsigned v_abs = __shfl_sync(0xffffffffu, v_run, L);
            const unsigned t_off = __shfl_sync(0xffffffffu, t_run, L);
            const int ck = k0 + 8 * L + j;
            const unsigned edges = s_edge[cube];
            const unsigned created = edges & own_mask(gi, cj, ck);
            const int n = s_ntri[cube];
            // ---- role V: vertices this cell creates, in the sequential algorithm's creation order
            if (lane < 12 && (created & (1u << ev))) {
                const float *p = vol + (size_t)ci * sx + (size_t)cj * sy + ck;
                double fa = (double)__ldg(p + v_ax * sx + v_ay * sy + v_az);
                double fb = (double)__ldg(p + v_bx * sx + v_by * sy + v_bz);
                if (d.negate) { fa = -fa; fb = -fb; }
                double pos[3] = {(double)(gi + v_ax), (double)(cj + v_ay), (double)(ck + v_az)};
                const double qa = pos[v_axis];
                const double qb = qa + (double)((v_axis == 0 ? v_bx - v_ax : (v_axis == 1 ? v_by - v_ay : v_bz - v_az)));
                pos[v_axis] = mc_interp(d.iso, fa, fb, qa, qb);
                const unsigned rank = __popc(created & v_before);
                double *dst = verts + (size_t)(v_abs - ghost_v + rank) * 3;
                dst[0] = pos[0]; dst[1] = pos[1]; dst[2] = pos[2];
            }
            // ---- role T: vertex id of cube edge `lane` (its owner = the first cell in sweep order that contains the grid edge)
            int local_id = 0;                                  // id relative to this slab's first vertex (negative: ghost-layer owner)
            if (lane < 12 && (edges & (1u << lane))) {
                const int ei = ci + t_ox, ej = cj + t_oy, ek = ck + t_oz;       // low end point of the grid edge (slab-local)
                int fi = ei, fj = ej, fk = ek;
                if (t_axis != 0) fi = (d.x_global0 + ei) > 0 ? ei - 1 : ei;
                if (t_axis != 1) fj = ej > 0 ? ej - 1 : 0;
                if (t_axis != 2) fk = ek > 0 ? ek - 1 : 0;
                int d1, d2;
                if (t_axis == 0)      { d1 = ej - fj; d2 = ek - fk; }
                else if (t_axis == 1) { d1 = ei - fi; d2 = ek - fk; }
                else                  { d1 = ei - fi; d2 = ej - fj; }
                const int eo = c_edge_of[t_axis][d1][d2];
                unsigned obase, ocube;
                if (fi == ci && fj == cj && fk == ck) { obase = v_abs; ocube = cube; }
                else obase = owner_cell(fi, fj, fk, ocube);
                const unsigned ocreated = s_edge[ocube] & own_mask(d.x_global0 + fi, fj, fk);
                local_id = (int)(obase + __popc(ocreated & c_before_mask[eo])) - (int)ghost_v;
            }
            // ---- triangles: lane m writes index m of the cell's 3 * n indices
            const int src = lane < 3 * n ? (int)s_tri[cube][lane & 15] : 0;
            const int idv = __shfl_sync(0xffffffffu, local_id, src);
            if (lane < 3 * n) tris[(size_t)t_off * 3 + lane] = vert_id_base + (long long)idv;
            if (lane == L) {
                act &= act - 1u;                              // this cell is done
                v_run += __popc(created);
                t_run += n;
            }
            pending = __ballot_sync(0xffffffffu, act != 0u);
        }
    }
}

int load_tables()
{
    int dev = 0;
    NPHM_CUDA_CHECK(cudaGetDevice(&dev));
    if (dev < 64 && g_tables_loaded[dev]) return NPHM_OK;
    NPHM_CUDA_CHECK(cudaMemcpyToSymbol(c_edge_table, MC_EDGE_TABLE, sizeof(MC_EDGE_TABLE)));
    NPHM_CUDA_CHECK(cudaMemcpyToSymbol(c_tri_table, MC_TRI_TABLE, sizeof(MC_TRI_TABLE)));
    NPHM_CUDA_CHECK(cudaMemcpyToSymbol(c_num_tris, MC_NUM_TRIS, sizeof(MC_NUM_TRIS)));
    unsigned short before[12];
    unsigned char order[12];
    unsigned short acc = 0;
    for (int o = 0; o < 12; ++o) {
        order[o] = (unsigned char)h_create_order[o];
        before[h_create_order[o]] = acc;
        acc |= (unsigned short)(1u << h_create_order[o]);
    }
    NPHM_CUDA_CHECK(cudaMemcpyToSymbol(c_before_mask, before, sizeof(before)));
    {
        static unsigned char packed[kTabBytes];
        memcpy(packed + kTabEdge, MC_EDGE_TABLE, sizeof(MC_EDGE_TABLE));
        memcpy(packed + kTabNtri, MC_NUM_TRIS, sizeof(MC_NUM_TRIS));
        memcpy(packed + kTabTri, MC_TRI_TABLE, sizeof(MC_TRI_TABLE));
        NPHM_CUDA_CHECK(cudaMemcpyToSymbol(g_tables, packed, kTabBytes));
    }
    NPHM_CUDA_CHECK(cudaMemcpyToSymbol(c_create_order, order, sizeof(order)));
    if (dev < 64) g_tables_loaded[dev] = true;
    return NPHM_OK;
}

int make_dims(const nphm_mc_params *p, Dims &d)
{
    NPHM_REQUIRE(p != nullptr, "nphm_mc: params is NULL");
    NPHM_REQUIRE(p->nx >= 0 && p->ny >= 0 && p->nz >= 0, "nphm_mc: negative dimensions");
    // a slab that does not start at the global x = 0 plane must bring the cell layer below it (its owner cells)
    NPHM_REQUIRE(p->x_global0 >= 0 && (p->x_global0 == 0 || p->ghost_lo), "nphm_mc: x_global0 > 0 needs ghost_lo = 1");
    d.nx = p->nx; d.ny = p->ny; d.nz = p->nz;
    d.cx = p->nx - 1; d.cy = p->ny - 1; d.cz = p->nz - 1;
    d.ncells = (d.cx > 0 && d.cy > 0 && d.cz > 0) ? (long long)d.cx * d.cy * d.cz : 0;
    d.x_global0 = p->x_global0; d.ghost_lo = p->ghost_lo ? 1 : 0; d.negate = p->negate ? 1 : 0;
    d.iso = p->iso;
    NPHM_REQUIRE(d.ncells == 0 || (long long)d.cx * d.cy < (1LL << 31), "nphm_mc: volume too large");
    NPHM_REQUIRE(d.ncells == 0 || d.cz <= 9000, "nphm_mc: rows longer than 9000 cells overflow the 16-bit group prefix");
    d.n_rows = d.ncells ? d.cx * d.cy : 0;
    d.pitch = d.ncells ? (d.cz + 7) / 8 * 8 : 0;
    d.ngrp = d.pitch / 8;
    // inside test: (negate ? -(double)v : (double)v) <= iso.  In fp32 when iso (resp. -iso) is exactly a float.
    const double t = d.negate ? -d.iso : d.iso;
    d.thr = (float)t;
    d.cmp_float = ((double)d.thr == t) ? 1 : 0;
    return NPHM_OK;
}

struct Workspace {
    unsigned long long *totals;     // [0..3] totals, [8] ticket of the scan kernel
    unsigned *row_nv, *row_nt, *row_v, *row_t, *chunk_v, *chunk_t;
    unsigned short *grp_prefix;
    unsigned char *cube;
    int n_chunks;
    long long bytes;
};

Workspace carve(void *ws, const Dims &d)
{
    auto align = [](long long x) { return (x + 255) / 256 * 256; };
    Workspace w;
    char *p = reinterpret_cast<char *>(ws);
    long long off = 0;
    const long long rows = d.n_rows > 0 ? d.n_rows : 1;
    w.n_chunks = (int)ceil_div(rows, kRowChunk);
    w.totals = reinterpret_cast<unsigned long long *>(p + off); off += 256;
    w.row_nv = reinterpret_cast<unsigned *>(p + off); off += align(rows * 4);
    w.row_nt = reinterpret_cast<unsigned *>(p + off); off += align(rows * 4);
    w.row_v = reinterpret_cast<unsigned *>(p + off); off += align(rows * 4);
    w.row_t = reinterpret_cast<unsigned *>(p + off); off += align(rows * 4);
    w.chunk_v = reinterpret_cast<unsigned *>(p + off); off += align((long long)w.n_chunks * 4);
    w.chunk_t = reinterpret_cast<unsigned *>(p + off); off += align((long long)w.n_chunks * 4);
    w.grp_prefix = reinterpret_cast<unsigned short *>(p + off); off += align(rows * (d.ngrp > 0 ? d.ngrp : 1) * 2);
    w.cube = reinterpret_cast<unsigned char *>(p + off); off += align(rows * (d.pitch > 0 ? d.pitch : 8));
    w.bytes = off;
    return w;
}

}  // namespace
}  // namespace nphm

using namespace nphm;

extern "C" long long nphm_mc_workspace_bytes(const nphm_mc_params *p)
{
    Dims d;
    if (make_dims(p, d) != NPHM_OK) return -1;
    return carve(nullptr, d).bytes;
}

extern "C" int nphm_mc_count(const float *vol_dev, const nphm_mc_params *p, void *workspace_dev,
                             long long *n_verts_host, long long *n_tris_host, void *stream_)
{
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    Dims d;
    int rc = make_dims(p, d);
    if (rc) return rc;
    NPHM_REQUIRE(n_verts_host && n_tris_host, "nphm_mc_count: NULL count pointers");
    *n_verts_host = 0; *n_tris_host = 0;
    if (d.ncells == 0) return NPHM_OK;
    NPHM_REQUIRE(vol_dev && workspace_dev, "nphm_mc_count: NULL volume / workspace");
    rc = load_tables();
    if (rc) return rc;
    Workspace w = carve(workspace_dev, d);
    NPHM_CUDA_CHECK(cudaMemsetAsync(w.totals, 0, 256, stream));
    const int grid = (int)ceil_div(d.n_rows, kWarpsPerCta);
    const bool aligned = (d.nz % 4 == 0) && ((reinterpret_cast<uintptr_t>(vol_dev) & 15) == 0);
    if (aligned)
        mc_classify_rows_kernel<true><<<grid, kRowThreads, 0, stream>>>(vol_dev, d, w.cube, w.grp_prefix, w.row_nv, w.row_nt);
    else
        mc_classify_rows_kernel<false><<<grid, kRowThreads, 0, stream>>>(vol_dev, d, w.cube, w.grp_prefix, w.row_nv, w.row_nt);
    NPHM_CUDA_CHECK(cudaGetLastError());
    mc_scan_rows_kernel<<<w.n_chunks, 256, 0, stream>>>(w.row_nv, w.row_nt, w.row_v, w.row_t, w.chunk_v, w.chunk_t, d.n_rows,
                                                        d.ghost_lo ? d.cy : 0, w.totals);
    NPHM_CUDA_CHECK(cudaGetLastError());
    unsigned long long totals[4];
    NPHM_CUDA_CHECK(cudaMemcpyAsync(totals, w.totals, sizeof(totals), cudaMemcpyDeviceToHost, stream));
    NPHM_CUDA_CHECK(cudaStreamSynchronize(stream));
    NPHM_REQUIRE(totals[0] < 0xffffffffull && totals[1] < 0xffffffffull, "nphm_mc_count: mesh too large for 32-bit scratch");
    *n_verts_host = (long long)(totals[0] - (d.ghost_lo ? totals[2] : 0));
    *n_tris_host = (long long)(totals[1] - (d.ghost_lo ? totals[3] : 0));
    return NPHM_OK;
}

extern "C" int nphm_mc_emit(const float *vol_dev, const nphm_mc_params *p, void *workspace_dev,
                            long long vert_id_base, double *verts_dev, long long *tris_dev, void *stream_)
{
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    Dims d;
    int rc = make_dims(p, d);
    if (rc) return rc;
    if (d.ncells == 0) return NPHM_OK;
    NPHM_REQUIRE(vol_dev && workspace_dev, "nphm_mc_emit: NULL volume / workspace");
    Workspace w = carve(workspace_dev, d);
    Scratch s{w.cube, w.grp_prefix, w.row_nv, w.row_nt, w.row_v, w.row_t, w.chunk_v, w.chunk_t, w.totals};
    mc_emit_rows_kernel<<<(int)ceil_div(d.n_rows, kWarpsPerCta), kRowThreads, 0, stream>>>(vol_dev, d, s, vert_id_base, verts_dev,
                                                                                          tris_dev);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

// Host-buffer convenience (== mcubes.marching_cubes on a host array).  The device staging buffers are kept between calls
// (grown on demand, per device) - a caller that extracts many meshes does not pay cudaMalloc/cudaFree every time.
namespace {
struct HostStaging {
    void *vol = nullptr, *ws = nullptr, *verts = nullptr, *tris = nullptr;
    size_t vol_cap = 0, ws_cap = 0, verts_cap = 0, tris_cap = 0;
    int device = -1;
};
HostStaging g_staging;

int grow(void **ptr, size_t *cap, size_t bytes)
{
    if (bytes <= *cap) return NPHM_OK;
    if (*ptr) cudaFree(*ptr);
    *ptr = nullptr; *cap = 0;
    if (cudaMalloc(ptr, bytes) != cudaSuccess) { set_error("nphm_marching_cubes_host: cudaMalloc(%zu) failed", bytes); return NPHM_ERR_CUDA; }
    *cap = bytes;
    return NPHM_OK;
}
}  // namespace

extern "C" int nphm_marching_cubes_host(const float *vol_host, int nx, int ny, int nz, double iso, int negate,
                                        double *verts_host, long long *tris_host,
                                        long long *n_verts, long long *n_tris)
{
    NPHM_REQUIRE(vol_host && n_verts && n_tris, "nphm_marching_cubes_host: NULL argument");
    nphm_mc_params p{nx, ny, nz, 0, 0, negate, iso};
    const long long ws_bytes = nphm_mc_workspace_bytes(&p);
    NPHM_REQUIRE(ws_bytes >= 0, "nphm_marching_cubes_host: bad dimensions");
    const size_t vol_bytes = (size_t)nx * ny * nz * sizeof(float);
    if (vol_bytes == 0) { *n_verts = 0; *n_tris = 0; return NPHM_OK; }
    int dev = 0;
    NPHM_CUDA_CHECK(cudaGetDevice(&dev));
    HostStaging &st = g_staging;
    if (st.device != dev) {                     // buffers belong to one device: start over on another one
        cudaFree(st.vol); cudaFree(st.ws); cudaFree(st.verts); cudaFree(st.tris);
        st = HostStaging();
        st.device = dev;
    }
    int rc;
    if ((rc = grow(&st.vol, &st.vol_cap, vol_bytes)) || (rc = grow(&st.ws, &st.ws_cap, (size_t)ws_bytes))) return rc;
    NPHM_CUDA_CHECK(cudaMemcpy(st.vol, vol_host, vol_bytes, cudaMemcpyHostToDevice));
    rc = nphm_mc_count(static_cast<const float *>(st.vol), &p, st.ws, n_verts, n_tris, nullptr);
    if (rc == NPHM_OK && verts_host && tris_host && (*n_verts > 0 || *n_tris > 0)) {
        if ((rc = grow(&st.verts, &st.verts_cap, (size_t)(*n_verts + 1) * 24)) ||
            (rc = grow(&st.tris, &st.tris_cap, (size_t)(*n_tris + 1) * 24))) return rc;
        rc = nphm_mc_emit(static_cast<const float *>(st.vol), &p, st.ws, 0, static_cast<double *>(st.verts),
                          static_cast<long long *>(st.tris), nullptr);
        if (rc == NPHM_OK) {
            NPHM_CUDA_CHECK(cudaMemcpy(verts_host, st.verts, (size_t)*n_verts * 24, cudaMemcpyDeviceToHost));
            NPHM_CUDA_CHECK(cudaMemcpy(tris_host, st.tris, (size_t)*n_tris * 24, cudaMemcpyDeviceToHost));
        }
    }
    return rc;
}
