// Narrow band with block-sparse storage on sm_90a: the protocol of narrowband.cu (the same steps on the same x-slab, DESIGN §4.13,
// §4.16, §4.17) with memory that follows the active blocks instead of the grid.  Nothing is stored per grid voxel:
//   frame (fixed, caller's workspace)  per block: its state byte and a u32 slot in the brick pool (~0: none); per block corner
//                                      ((l1-l0+1) (nb+1)^2): its value and mark; per shared plane X0 / X1: the values and
//                                      evaluated flags a neighbour sent (res^2 each); the ghost plane X0-1 (res^2 floats)
//   pool (grows, caller's buffers)     per slot: a brick of the (B+1)^3 voxels of its block (values and marks) and its block;
//                                      the list (brick-local indices slot (B+1)^3 + local, or corner indices) and compaction
//                                      scratch
// A voxel on a face shared by several allocated bricks has a copy in each; every write of a value (scatter) goes to all copies
// and to the corner array when it is a corner, so the copies never disagree.  A new brick starts from what the older bricks, the
// corners and the shared planes already hold.  Among the blocks being marked, the voxel is listed by the first (in x, y, z order)
// that contains it, so it is evaluated once.  A voxel held nowhere is not evaluated, and its value - wherever it is read - is that
// of corner 0 of the block min(x / B, nb - 1) (the dense fill), so `fill` writes nothing.  Growth is pushed from the bricks and the
// shared planes to the inactive blocks containing their voxels: on the whole grid the only evaluated voxels of an inactive block
// are its corners (all on one side, else classify had activated it) and voxels of active blocks' bricks or a neighbour's plane.
#include "common.cuh"
#include "simt.cuh"
#include "mc_tables.h"
#include <algorithm>
#include <vector>

namespace nphm {
namespace sband {

constexpr int kThreads = 256;
constexpr int kPerThread = 16;
constexpr int kChunk = kThreads * kPerThread;
constexpr int kScanThreads = 1024;
constexpr int kWarps = kThreads / 32;

enum : unsigned char { kIdle = 0, kWanted = 1, kDone = 2 };                          // voxel / corner marks
enum : unsigned char { kInactive = 0, kActivated = 1, kMarked = 2, kForced = 3 };     // block states (3: has a slot, not marked)
enum { H_LISTED = 0, H_ACTIVE = 1, H_USED = 2, H_NEED = 3, H_KIND = 4, H_OLD = 5, H_NEW = 6, H_OVER = 7 };   // header words
constexpr unsigned kNoSlot = 0xffffffffu;

struct Geo {
    int res, B, E, C, nb, nb1;    // grid points per axis, block edge in cells, brick edge (B + 1), cells per axis, blocks, nb + 1
    int L0, L1, X0, X1;
    bool lo, hi, ghost;           // plane X0 shared with a lower slab, plane X1 with an upper one, ghost plane X0 - 1 present
    long long rr, n_blocks, n_corners, V;      // voxels per plane, blocks, corners of the slab, voxels per brick
};

inline long long pad(long long n) { return std::max(ceil_div(n, kChunk), 1LL) * kChunk; }
inline long long al(long long x) { return (x + 255) / 256 * 256; }

inline Geo make_geo(int res, int block, int l0, int l1)
{
    Geo g;
    g.res = res; g.B = block; g.E = block + 1; g.C = res - 1;
    g.nb = (int)ceil_div(res - 1, block); g.nb1 = g.nb + 1;
    g.L0 = l0; g.L1 = l1;
    g.X0 = l0 * block; g.X1 = std::min(l1 * block, g.C);
    g.lo = l0 > 0; g.hi = g.X1 < g.C; g.ghost = l0 > 0;
    g.rr = (long long)res * res;
    g.n_blocks = (long long)(l1 - l0) * g.nb * g.nb;
    g.n_corners = (long long)(l1 - l0 + 1) * g.nb1 * g.nb1;
    g.V = (long long)g.E * g.E * g.E;
    return g;
}

struct Frame {
    long long hdr, axes, states, slot, cmarks, cvals, pvals, pdone, ghostv, bytes;
};

inline Frame frame_layout(const Geo &g)
{
    Frame f;
    long long off = 0;
    f.hdr = off; off += 256;
    f.axes = off; off += al(3LL * g.res * 4);
    f.states = off; off += al(pad(g.n_blocks));                 // padded to whole compaction chunks (the padding stays 0)
    f.slot = off; off += al(g.n_blocks * 4);
    f.cmarks = off; off += al(pad(g.n_corners));
    f.cvals = off; off += al(g.n_corners * 4);
    f.pvals = off; off += al(2 * g.rr * 4);
    f.pdone = off; off += al(2 * g.rr);
    f.ghostv = off; off += al(g.rr * 4);
    f.bytes = off;
    return f;
}

// pool sizes for `slots` bricks: {mark bytes, list entries, compaction chunks}
inline void pool_sizes(const Geo &g, long long slots, long long out[3])
{
    out[0] = pad(slots * g.V);
    out[1] = std::max(slots * g.V, g.n_corners);
    out[2] = std::max(std::max(out[0], pad(g.n_blocks)), pad(g.n_corners)) / kChunk;
}

struct Mem {
    unsigned long long *hdr;
    float *axes;
    unsigned char *states;
    unsigned *slot;
    unsigned char *cmarks;
    float *cvals, *pvals;
    unsigned char *pdone;
    float *ghostv;
    float *bvals;
    unsigned char *bmarks;
    unsigned *sblock, *list, *chunk_cnt, *chunk_off;
    long long slots;
};

inline Mem carve(void *ws, const Geo &g, const nphm_band_pool *p)
{
    const Frame f = frame_layout(g);
    char *b = static_cast<char *>(ws);
    Mem m;
    m.hdr = reinterpret_cast<unsigned long long *>(b + f.hdr);
    m.axes = reinterpret_cast<float *>(b + f.axes);
    m.states = reinterpret_cast<unsigned char *>(b + f.states);
    m.slot = reinterpret_cast<unsigned *>(b + f.slot);
    m.cmarks = reinterpret_cast<unsigned char *>(b + f.cmarks);
    m.cvals = reinterpret_cast<float *>(b + f.cvals);
    m.pvals = reinterpret_cast<float *>(b + f.pvals);
    m.pdone = reinterpret_cast<unsigned char *>(b + f.pdone);
    m.ghostv = reinterpret_cast<float *>(b + f.ghostv);
    m.bvals = p->vals; m.bmarks = p->marks; m.sblock = p->blocks; m.list = p->list;
    m.chunk_cnt = p->chunk_cnt; m.chunk_off = p->chunk_off;
    m.slots = p->slots;
    return m;
}

__device__ __forceinline__ bool side(float v) { return v >= 0.f; }

// blocks of one axis whose voxel range [bB, min(bB + B, C)] holds voxel x, limited to [lim0, lim1]
__device__ __forceinline__ void holders(const Geo &g, int x, int lim0, int lim1, int &b0, int &b1)
{
    const int hi = min(x / g.B, g.nb - 1);
    const int lo = (x % g.B == 0 && x > 0) ? x / g.B - 1 : hi;
    b0 = max(lo, lim0);
    b1 = min(hi, lim1);
}

__device__ __forceinline__ long long blk(const Geo &g, int bx, int by, int bz) { return ((long long)(bx - g.L0) * g.nb + by) * g.nb + bz; }

__device__ __forceinline__ void unblock(const Geo &g, long long b, int &bx, int &by, int &bz)
{
    bz = (int)(b % g.nb);
    const long long t = b / g.nb;
    by = (int)(t % g.nb);
    bx = g.L0 + (int)(t / g.nb);
}

__device__ __forceinline__ long long local(const Geo &g, int bx, int by, int bz, int x, int y, int z)
{
    return ((long long)(x - bx * g.B) * g.E + (y - by * g.B)) * g.E + (z - bz * g.B);
}

__device__ __forceinline__ long long corner(const Geo &g, int cx, int cy, int cz) { return ((long long)(cx - g.L0) * g.nb1 + cy) * g.nb1 + cz; }
__device__ __forceinline__ bool on_lattice(const Geo &g, int x) { return x % g.B == 0 || x == g.C; }
__device__ __forceinline__ int lattice(const Geo &g, int x) { return x == g.C ? g.nb : x / g.B; }
__device__ __forceinline__ long long corner0(const Geo &g, long long b)
{
    int bx, by, bz;
    unblock(g, b, bx, by, bz);
    return corner(g, bx, by, bz);
}

// voxel (x, y, z) of planes [X0, X1]: its value and whether it is evaluated, from the bricks of slot < slot_limit, the corners and
// the shared planes; a voxel not evaluated reads as the fill value, corner 0 of block min(x / B, nb - 1)
__device__ bool lookup(const Geo &g, const Mem &m, int x, int y, int z, unsigned slot_limit, float &val)
{
    int x0, x1, y0, y1, z0, z1;
    holders(g, x, g.L0, g.L1 - 1, x0, x1);
    holders(g, y, 0, g.nb - 1, y0, y1);
    holders(g, z, 0, g.nb - 1, z0, z1);
    for (int bx = x0; bx <= x1; ++bx)
        for (int by = y0; by <= y1; ++by)
            for (int bz = z0; bz <= z1; ++bz) {
                const unsigned s = m.slot[blk(g, bx, by, bz)];
                if (s >= slot_limit) continue;
                const long long e = s * g.V + local(g, bx, by, bz, x, y, z);
                if (m.bmarks[e] == kDone) { val = m.bvals[e]; return true; }
            }
    if (on_lattice(g, x) && on_lattice(g, y) && on_lattice(g, z)) {
        const long long c = corner(g, lattice(g, x), lattice(g, y), lattice(g, z));
        if (m.cmarks[c] == kDone) { val = m.cvals[c]; return true; }
    }
    const long long i = (long long)y * g.res + z;
    if (x == g.X0 && g.lo && m.pdone[i]) { val = m.pvals[i]; return true; }
    if (x == g.X1 && g.hi && m.pdone[g.rr + i]) { val = m.pvals[g.rr + i]; return true; }
    val = m.cvals[corner(g, min(x / g.B, g.nb - 1), min(y / g.B, g.nb - 1), min(z / g.B, g.nb - 1))];
    return false;
}

// the evaluated value of voxel (x, y, z) into every brick that holds it and into its corner
__device__ void store(const Geo &g, const Mem &m, int x, int y, int z, float val)
{
    int x0, x1, y0, y1, z0, z1;
    holders(g, x, g.L0, g.L1 - 1, x0, x1);
    holders(g, y, 0, g.nb - 1, y0, y1);
    holders(g, z, 0, g.nb - 1, z0, z1);
    for (int bx = x0; bx <= x1; ++bx)
        for (int by = y0; by <= y1; ++by)
            for (int bz = z0; bz <= z1; ++bz) {
                const unsigned s = m.slot[blk(g, bx, by, bz)];
                if (s == kNoSlot) continue;
                const long long e = s * g.V + local(g, bx, by, bz, x, y, z);
                m.bvals[e] = val;
                m.bmarks[e] = kDone;
            }
    if (on_lattice(g, x) && on_lattice(g, y) && on_lattice(g, z)) {
        const long long c = corner(g, lattice(g, x), lattice(g, y), lattice(g, z));
        m.cvals[c] = val;
        m.cmarks[c] = kDone;
    }
}

// the slot of the first block (x, y, z order) holding the voxel that is being marked (kForced); kNoSlot when none is
__device__ unsigned owner(const Geo &g, const Mem &m, int x, int y, int z, long long &e)
{
    int x0, x1, y0, y1, z0, z1;
    holders(g, x, g.L0, g.L1 - 1, x0, x1);
    holders(g, y, 0, g.nb - 1, y0, y1);
    holders(g, z, 0, g.nb - 1, z0, z1);
    for (int bx = x0; bx <= x1; ++bx)
        for (int by = y0; by <= y1; ++by)
            for (int bz = z0; bz <= z1; ++bz) {
                const long long b = blk(g, bx, by, bz);
                if (m.states[b] != kForced) continue;
                const unsigned s = m.slot[b];
                e = s * g.V + local(g, bx, by, bz, x, y, z);
                return s;
            }
    return kNoSlot;
}

// the inactive blocks holding an evaluated voxel of value v on the other side of the test from their corner 0 are activated
__device__ void push(const Geo &g, const Mem &m, int x, int y, int z, float v)
{
    int x0, x1, y0, y1, z0, z1;
    holders(g, x, g.L0, g.L1 - 1, x0, x1);
    holders(g, y, 0, g.nb - 1, y0, y1);
    holders(g, z, 0, g.nb - 1, z0, z1);
    for (int bx = x0; bx <= x1; ++bx)
        for (int by = y0; by <= y1; ++by)
            for (int bz = z0; bz <= z1; ++bz) {
                const long long b = blk(g, bx, by, bz);
                if (m.states[b] == kInactive && side(m.cvals[corner(g, bx, by, bz)]) != side(v)) m.states[b] = kActivated;
            }
}

// voxel (x, y, z) of a listed entry: a corner index (kind 1) or a brick-local index (kind 0)
__device__ __forceinline__ void entry_voxel(const Geo &g, const Mem &m, unsigned long long kind, unsigned e, int &x, int &y, int &z)
{
    if (kind) {
        const long long n1 = g.nb1;
        const int cz = (int)(e % n1), cy = (int)((e / n1) % n1), cx = g.L0 + (int)(e / (n1 * n1));
        x = min(cx * g.B, g.C); y = min(cy * g.B, g.C); z = min(cz * g.B, g.C);
        return;
    }
    const unsigned s = e / (unsigned)g.V, l = e % (unsigned)g.V;
    int bx, by, bz;
    unblock(g, m.sblock[s], bx, by, bz);
    z = bz * g.B + (int)(l % g.E);
    y = by * g.B + (int)((l / g.E) % g.E);
    x = bx * g.B + (int)(l / (g.E * g.E));
}

// ---------------------------------------------------------------------------------------------- ordered compaction of bytes == want
__device__ __forceinline__ unsigned match_bytes(uint4 m, unsigned want4, uint4 &eq)
{
    eq.x = __vcmpeq4(m.x, want4); eq.y = __vcmpeq4(m.y, want4);
    eq.z = __vcmpeq4(m.z, want4); eq.w = __vcmpeq4(m.w, want4);
    return (__popc(eq.x) + __popc(eq.y) + __popc(eq.z) + __popc(eq.w)) >> 3;
}

template <int N>
__device__ __forceinline__ unsigned cta_exclusive_scan(unsigned v, unsigned &total)
{
    __shared__ unsigned wsum[N / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    if (lane == 31) wsum[warp] = inc;
    __syncthreads();
    unsigned base = 0;
    total = 0;
    for (int w = 0; w < N / 32; ++w) {
        if (w < warp) base += wsum[w];
        total += wsum[w];
    }
    __syncthreads();
    return base + inc - v;
}

__device__ __forceinline__ void count_body(const unsigned char *__restrict__ bytes, unsigned want4, unsigned *__restrict__ cnt)
{
    const uint4 m = __ldg(reinterpret_cast<const uint4 *>(bytes + (size_t)blockIdx.x * kChunk) + threadIdx.x);
    uint4 eq;
    unsigned total;
    cta_exclusive_scan<kThreads>(match_bytes(m, want4, eq), total);
    if (threadIdx.x == 0) cnt[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kThreads) count_kernel(const unsigned char *__restrict__ bytes, unsigned want4, unsigned *__restrict__ cnt)
{
    count_body(bytes, want4, cnt);
}

__device__ __forceinline__ void scan_body(const unsigned *__restrict__ cnt, unsigned *__restrict__ off, long long n_chunks,
                                          unsigned long long *__restrict__ total_out)
{
    const long long per = (n_chunks + kScanThreads - 1) / kScanThreads;
    const long long c0 = threadIdx.x * per, c1 = min(c0 + per, n_chunks);
    unsigned s = 0;
    for (long long c = c0; c < c1; ++c) s += cnt[c];
    unsigned total;
    unsigned run = cta_exclusive_scan<kScanThreads>(s, total);
    for (long long c = c0; c < c1; ++c) {
        off[c] = run;
        run += cnt[c];
    }
    if (threadIdx.x == 0) *total_out = total;
}

__global__ void __launch_bounds__(kScanThreads) scan_kernel(const unsigned *__restrict__ cnt, unsigned *__restrict__ off, long long n_chunks,
                                                            unsigned long long *__restrict__ total_out)
{
    scan_body(cnt, off, n_chunks, total_out);
}

// chunk blockIdx.x of the compaction: list its bytes == want (from their chunk's offset on) and set them to `set`
__device__ __forceinline__ void emit_body(unsigned char *__restrict__ bytes, unsigned want4, unsigned set4, const unsigned *__restrict__ off,
                                          unsigned *__restrict__ list)
{
    uint4 *p = reinterpret_cast<uint4 *>(bytes + (size_t)blockIdx.x * kChunk) + threadIdx.x;
    uint4 m = *p, eq;
    const unsigned c = match_bytes(m, want4, eq);
    unsigned t;
    unsigned pos = off[blockIdx.x] + cta_exclusive_scan<kThreads>(c, t);
    if (c == 0) return;
    const unsigned v0 = blockIdx.x * (unsigned)kChunk + threadIdx.x * kPerThread;
    const unsigned e[4] = {eq.x, eq.y, eq.z, eq.w};
#pragma unroll
    for (int w = 0; w < 4; ++w)
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if ((e[w] >> (8 * j)) & 1u) list[pos++] = v0 + 4 * w + j;
    m.x = (m.x & ~eq.x) | (set4 & eq.x); m.y = (m.y & ~eq.y) | (set4 & eq.y);
    m.z = (m.z & ~eq.z) | (set4 & eq.z); m.w = (m.w & ~eq.w) | (set4 & eq.w);
    *p = m;
}

// list the indices of the bytes == want in ascending order and set them to `set`; nothing is written when *total + *used > cap
__global__ void __launch_bounds__(kThreads) emit_kernel(unsigned char *__restrict__ bytes, unsigned want4, unsigned set4,
                                                        const unsigned *__restrict__ cnt, const unsigned *__restrict__ off,
                                                        unsigned *__restrict__ list, const unsigned long long *__restrict__ total,
                                                        const unsigned long long *__restrict__ used, unsigned long long cap)
{
    if (cnt[blockIdx.x] == 0 || *total + (used ? *used : 0ull) > cap) return;
    emit_body(bytes, want4, set4, off, list);
}

// ---------------------------------------------------------------------------------------------- allocation and marking
__device__ __forceinline__ void quirk_states_body(const Geo g, long long period, long long k0, long long k1, unsigned char *__restrict__ states)
{
    const long long k = k0 + blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (k >= k1) return;
    const long long n_all = g.rr * g.res;
    const long long v = k < n_all / period ? (k + 1) * period - 1 : n_all - 1;
    int x0, x1, y0, y1, z0, z1;
    holders(g, (int)(v / g.rr), g.L0, g.L1 - 1, x0, x1);
    holders(g, (int)((v / g.res) % g.res), 0, g.nb - 1, y0, y1);
    holders(g, (int)(v % g.res), 0, g.nb - 1, z0, z1);
    for (int bx = x0; bx <= x1; ++bx)
        for (int by = y0; by <= y1; ++by)
            for (int bz = z0; bz <= z1; ++bz) states[blk(g, bx, by, bz)] = kActivated;
}

__global__ void quirk_states_kernel(const Geo g, long long period, long long k0, long long k1, unsigned char *__restrict__ states)
{
    quirk_states_body(g, period, k0, k1, states);
}

__device__ __forceinline__ void quirk_mark_body(const Geo g, const Mem m, long long period, long long k0, long long k1)
{
    const long long k = k0 + blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (k >= k1 || m.hdr[H_OVER]) return;
    const long long n_all = g.rr * g.res;
    const long long v = k < n_all / period ? (k + 1) * period - 1 : n_all - 1;
    long long e;
    if (owner(g, m, (int)(v / g.rr), (int)((v / g.res) % g.res), (int)(v % g.res), e) != kNoSlot) m.bmarks[e] = kWanted;
}

__global__ void quirk_mark_kernel(const Geo g, const Mem m, long long period, long long k0, long long k1)
{
    quirk_mark_body(g, m, period, k0, k1);
}

// after the compaction of the activated blocks into the list: take their slots, or flag that the pool is short
__global__ void commit_kernel(unsigned long long *hdr, unsigned long long cap)
{
    const unsigned long long used = hdr[H_USED], n = hdr[H_NEW];
    if (used + n > cap) {
        hdr[H_NEED] = used + n;
        hdr[H_OVER] = 1;
        return;
    }
    hdr[H_OLD] = used;
    hdr[H_USED] = used + n;
    hdr[H_OVER] = 0;
}

__device__ __forceinline__ void assign_body(const Mem m)
{
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (m.hdr[H_OVER] || i >= (long long)m.hdr[H_NEW]) return;
    const unsigned b = m.list[i], s = (unsigned)(m.hdr[H_OLD] + i);
    m.slot[b] = s;
    m.sblock[s] = b;
}

__global__ void assign_kernel(const Mem m)
{
    assign_body(m);
}

__device__ __forceinline__ void box(const Geo &g, long long b, int lo[3], int d[3])
{
    int bx, by, bz;
    unblock(g, b, bx, by, bz);
    const int bb[3] = {bx, by, bz};
    for (int a = 0; a < 3; ++a) {
        lo[a] = bb[a] * g.B;
        d[a] = min(lo[a] + g.B, g.C) - lo[a] + 1;
    }
}

// one warp per new brick: what the older bricks, the corners and the shared planes hold
__device__ __forceinline__ void init_body(const Geo g, const Mem m)
{
    const long long s = blockIdx.x * (long long)kWarps + (threadIdx.x >> 5);
    const unsigned long long old = m.hdr[H_OLD];
    if (m.hdr[H_OVER] || s < (long long)old || s >= (long long)m.hdr[H_USED]) return;
    int lo[3], d[3];
    box(g, m.sblock[s], lo, d);
    for (int i = threadIdx.x & 31; i < d[0] * d[1] * d[2]; i += 32) {
        const int lz = i % d[2], ly = (i / d[2]) % d[1], lx = i / (d[2] * d[1]);
        float v;
        const bool done = lookup(g, m, lo[0] + lx, lo[1] + ly, lo[2] + lz, (unsigned)old, v);
        const long long e = s * g.V + ((long long)lx * g.E + ly) * g.E + lz;
        m.bvals[e] = done ? v : 0.f;
        m.bmarks[e] = done ? kDone : kIdle;
    }
}

__global__ void __launch_bounds__(kThreads) init_kernel(const Geo g, const Mem m)
{
    init_body(g, m);
}

// one warp per brick of a block being marked: its voxels not evaluated are wanted, by the first marked block that holds them
__device__ __forceinline__ void mark_body(const Geo g, const Mem m)
{
    const long long s = blockIdx.x * (long long)kWarps + (threadIdx.x >> 5);
    if (m.hdr[H_OVER] || s >= (long long)m.hdr[H_USED] || m.states[m.sblock[s]] != kForced) return;
    int lo[3], d[3];
    box(g, m.sblock[s], lo, d);
    for (int i = threadIdx.x & 31; i < d[0] * d[1] * d[2]; i += 32) {
        const int lz = i % d[2], ly = (i / d[2]) % d[1], lx = i / (d[2] * d[1]);
        const long long e = s * g.V + ((long long)lx * g.E + ly) * g.E + lz;
        long long eo;
        if (m.bmarks[e] != kDone && owner(g, m, lo[0] + lx, lo[1] + ly, lo[2] + lz, eo) == (unsigned)s) m.bmarks[e] = kWanted;
    }
}

__global__ void __launch_bounds__(kThreads) mark_kernel(const Geo g, const Mem m)
{
    mark_body(g, m);
}

__device__ __forceinline__ void promote_body(const Mem m)
{
    const long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (m.hdr[H_OVER] || s >= (long long)m.hdr[H_USED]) return;
    const unsigned b = m.sblock[s];
    if (m.states[b] == kForced) {
        m.states[b] = kMarked;
        atomicAdd(m.hdr + H_ACTIVE, 1ull);
    }
}

__global__ void promote_kernel(const Mem m)
{
    promote_body(m);
}

// ---------------------------------------------------------------------------------------------- the band tests
__global__ void corners_kernel(long long n, unsigned char *__restrict__ cmarks)
{
    const long long c = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (c < n && cmarks[c] == kIdle) cmarks[c] = kWanted;
}

__device__ __forceinline__ void classify_body(const Geo g, float tau, const float *__restrict__ cvals, unsigned char *__restrict__ states)
{
    const long long b = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (b >= g.n_blocks || states[b] != kInactive) return;
    int bx, by, bz;
    unblock(g, b, bx, by, bz);
    bool near = false;
    int n_in = 0;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        const float v = __ldg(cvals + corner(g, bx + (c >> 2), by + ((c >> 1) & 1), bz + (c & 1)));
        near |= !(fabsf(v) > tau);
        n_in += side(v) ? 1 : 0;
    }
    if (near || (n_in != 0 && n_in != 8)) states[b] = kActivated;
}

__global__ void classify_kernel(const Geo g, float tau, const float *__restrict__ cvals, unsigned char *__restrict__ states)
{
    classify_body(g, tau, cvals, states);
}

// one warp per brick: its face voxels (all evaluated) push growth into the inactive blocks around it
__device__ __forceinline__ void grow_bricks_body(const Geo g, const Mem m)
{
    const long long s = blockIdx.x * (long long)kWarps + (threadIdx.x >> 5);
    if (s >= (long long)m.hdr[H_USED]) return;
    int lo[3], d[3];
    box(g, m.sblock[s], lo, d);
    for (int i = threadIdx.x & 31; i < d[0] * d[1] * d[2]; i += 32) {
        const int lz = i % d[2], ly = (i / d[2]) % d[1], lx = i / (d[2] * d[1]);
        if (lx != 0 && lx != d[0] - 1 && ly != 0 && ly != d[1] - 1 && lz != 0 && lz != d[2] - 1) continue;
        push(g, m, lo[0] + lx, lo[1] + ly, lo[2] + lz, m.bvals[s * g.V + ((long long)lx * g.E + ly) * g.E + lz]);
    }
}

__global__ void __launch_bounds__(kThreads) grow_bricks_kernel(const Geo g, const Mem m)
{
    grow_bricks_body(g, m);
}

// the voxels a neighbour evaluated on a shared plane push growth the same way
__global__ void grow_planes_kernel(const Geo g, const Mem m)
{
    const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (t >= 2 * g.rr) return;
    const bool upper = t >= g.rr;
    if (!(upper ? g.hi : g.lo) || !m.pdone[t]) return;
    const long long i = upper ? t - g.rr : t;
    push(g, m, upper ? g.X1 : g.X0, (int)(i / g.res), (int)(i % g.res), m.pvals[t]);
}

// ---------------------------------------------------------------------------------------------- lists <-> values, planes, volume
__global__ void gather_kernel(const Geo g, const Mem m, long long n, float *__restrict__ xyz)
{
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= n || i >= (long long)m.hdr[H_LISTED]) return;
    int x, y, z;
    entry_voxel(g, m, m.hdr[H_KIND], m.list[i], x, y, z);
    xyz[3 * i] = m.axes[x];
    xyz[3 * i + 1] = m.axes[g.res + y];
    xyz[3 * i + 2] = m.axes[2 * g.res + z];
}

__global__ void scatter_kernel(const Geo g, const Mem m, long long n, const float *__restrict__ values)
{
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= n || i >= (long long)m.hdr[H_LISTED]) return;
    int x, y, z;
    entry_voxel(g, m, m.hdr[H_KIND], m.list[i], x, y, z);
    store(g, m, x, y, z, values[i]);
}

__global__ void export_kernel(const Geo g, const Mem m, int plane, float *__restrict__ vals, unsigned char *__restrict__ done)
{
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= g.rr) return;
    float v;
    done[i] = lookup(g, m, plane, (int)(i / g.res), (int)(i % g.res), kNoSlot, v) ? 1 : 0;
    vals[i] = v;
}

__global__ void import_kernel(const Geo g, const Mem m, int plane, const float *__restrict__ vals, const unsigned char *__restrict__ done)
{
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= g.rr || !done[i]) return;
    float v;
    if (lookup(g, m, plane, (int)(i / g.res), (int)(i % g.res), kNoSlot, v)) return;
    const long long t = (plane == g.X0 ? 0 : g.rr) + i;
    m.pvals[t] = vals[i];
    m.pdone[t] = 1;
}

// planes [x_first, x_first + n_planes) of the filled slab volume (plane X0 - 1: the ghost plane)
__global__ void volume_kernel(const Geo g, const Mem m, int x_first, long long n, float *__restrict__ out)
{
    for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < n; v += (long long)gridDim.x * blockDim.x) {
        const int x = x_first + (int)(v / g.rr);
        const long long i = v % g.rr;
        if (x < g.X0) { out[v] = m.ghostv[i]; continue; }
        float val;
        lookup(g, m, x, (int)(i / g.res), (int)(i % g.res), kNoSlot, val);
        out[v] = val;
    }
}

// ---------------------------------------------------------------------------------------------- host side
// Index widths: block and corner indices are u32 (the lists of active blocks and of corners, the slot map's inverse), so
// (nb + 1)^3 < 2^32: with 4^3-cell blocks res <= 6497 (2048^3 uses 513^3 corners).  Brick-local list entries slot (B+1)^3 + local
// and the marching-cubes segment indices slot B^2 + row are u32, so a pool holds fewer than 2^32 / (B+1)^3 bricks (checked per
// pool).  res <= 8192 bounds the planes the band keeps whole (shared, ghost and exported planes, the ghost layer's per-cell vertex
// counts) to 2^26 entries; it decides over the corner bound for blocks of 6 cells or more.
int check_args(int res, int block, int l0, int l1, const char *who)
{
    NPHM_REQUIRE(res >= 2 && res <= 8192, "%s: res %d outside [2, 8192]", who, res);
    NPHM_REQUIRE(block >= 1 && block <= 64, "%s: block %d outside [1, 64]", who, block);
    const long long nb = ceil_div(res - 1, block);
    NPHM_REQUIRE((nb + 1) * (nb + 1) * (nb + 1) < (1LL << 32),
                 "%s: res %d with block %d has %lld^3 block corners; corner indices are u32 (use a larger block)", who, res, block,
                 nb + 1);
    NPHM_REQUIRE(l0 >= 0 && l0 < l1 && l1 <= nb, "%s: block layers [%d, %d) not a non-empty range of [0, %lld)", who, l0, l1, nb);
    return NPHM_OK;
}

int check_mem(const Geo &g, const void *ws, long long ws_bytes, const nphm_band_pool *p, const char *who)
{
    NPHM_REQUIRE(ws && p, "%s: NULL workspace or pool", who);
    const long long need = frame_layout(g).bytes;
    if (ws_bytes < need) {
        set_error("%s: sparse band workspace too small: %lld bytes for res %d, block %d, block layers [%d, %d), %lld needed", who,
                  ws_bytes, g.res, g.B, g.L0, g.L1, need);
        return NPHM_ERR_CAPACITY;
    }
    NPHM_REQUIRE(p->slots >= 0 && p->slots * g.V < (1LL << 32), "%s: pool of %lld bricks of %lld voxels: brick indices are u32", who,
                 p->slots, g.V);
    NPHM_REQUIRE(p->vals && p->marks && p->blocks && p->list && p->chunk_cnt && p->chunk_off, "%s: NULL pool buffer", who);
    long long s[3];
    pool_sizes(g, p->slots, s);
    if (p->marks_bytes < s[0] || p->list_len < s[1] || p->n_chunks < s[2]) {
        set_error("%s: pool buffers too small for %lld bricks: %lld mark bytes, %lld list entries, %lld chunks needed", who, p->slots,
                  s[0], s[1], s[2]);
        return NPHM_ERR_CAPACITY;
    }
    return NPHM_OK;
}

inline unsigned rep4(unsigned char b) { return 0x01010101u * b; }

int compact(const Mem &m, unsigned char *bytes, long long n_padded, unsigned char want, unsigned char set, unsigned long long *total,
            const unsigned long long *used, unsigned long long cap, unsigned *list, cudaStream_t stream)
{
    const long long n_chunks = n_padded / kChunk;
    count_kernel<<<(unsigned)n_chunks, kThreads, 0, stream>>>(bytes, rep4(want), m.chunk_cnt);
    NPHM_CUDA_CHECK(cudaGetLastError());
    scan_kernel<<<1, kScanThreads, 0, stream>>>(m.chunk_cnt, m.chunk_off, n_chunks, total);
    NPHM_CUDA_CHECK(cudaGetLastError());
    emit_kernel<<<(unsigned)n_chunks, kThreads, 0, stream>>>(bytes, rep4(want), rep4(set), m.chunk_cnt, m.chunk_off, list, total,
                                                             used, cap);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

int set_kind(const Mem &m, unsigned char kind, cudaStream_t stream)
{
    NPHM_CUDA_CHECK(cudaMemsetAsync(m.hdr + H_KIND, kind, 1, stream));
    return NPHM_OK;
}

// activated blocks -> slots (in block order) and bricks initialised from what is already evaluated
int allocate(const Geo &g, const Mem &m, cudaStream_t stream)
{
    int rc = compact(m, m.states, pad(g.n_blocks), kActivated, kForced, m.hdr + H_NEW, m.hdr + H_USED, (unsigned long long)m.slots,
                     m.list, stream);
    if (rc) return rc;
    commit_kernel<<<1, 1, 0, stream>>>(m.hdr, (unsigned long long)m.slots);
    NPHM_CUDA_CHECK(cudaGetLastError());
    const unsigned slot_ctas = (unsigned)std::max(ceil_div(m.slots, kThreads), 1LL);
    const unsigned warp_ctas = (unsigned)std::max(ceil_div(m.slots, kWarps), 1LL);
    assign_kernel<<<slot_ctas, kThreads, 0, stream>>>(m);
    NPHM_CUDA_CHECK(cudaGetLastError());
    init_kernel<<<warp_ctas, kThreads, 0, stream>>>(g, m);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

// bricks -> list (kind 0); counts_host = {listed, active blocks, slots used, slots needed}; NPHM_ERR_CAPACITY when the pool was short
int list_and_read(const Geo &g, const Mem &m, unsigned char *marks, long long n_padded, unsigned char kind, long long *counts_host,
                  cudaStream_t stream)
{
    int rc = set_kind(m, kind, stream);
    if (rc || (rc = compact(m, marks, n_padded, kWanted, kDone, m.hdr + H_LISTED, nullptr, ~0ull, m.list, stream))) return rc;
    unsigned long long h[8];
    NPHM_CUDA_CHECK(cudaMemcpyAsync(h, m.hdr, sizeof(h), cudaMemcpyDeviceToHost, stream));
    NPHM_CUDA_CHECK(cudaStreamSynchronize(stream));
    if (counts_host) {
        counts_host[0] = (long long)h[H_LISTED];
        counts_host[1] = (long long)h[H_ACTIVE];
        counts_host[2] = (long long)h[H_USED];
        counts_host[3] = (long long)(h[H_OVER] ? h[H_NEED] : h[H_USED]);
    }
    if (h[H_OVER]) {
        set_error("sparse band: the brick pool holds %lld bricks, %llu needed", m.slots, h[H_NEED]);
        return NPHM_ERR_CAPACITY;
    }
    return NPHM_OK;
}

int list_bricks(const Geo &g, const Mem &m, long long *counts_host, cudaStream_t stream)
{
    long long s[3];
    pool_sizes(g, m.slots, s);
    return list_and_read(g, m, m.bmarks, s[0], 0, counts_host, stream);
}

int mark_and_list(const Geo &g, const Mem &m, long long *counts_host, cudaStream_t stream)
{
    int rc = allocate(g, m, stream);
    if (rc) return rc;
    const unsigned warp_ctas = (unsigned)std::max(ceil_div(m.slots, kWarps), 1LL);
    mark_kernel<<<warp_ctas, kThreads, 0, stream>>>(g, m);
    NPHM_CUDA_CHECK(cudaGetLastError());
    promote_kernel<<<(unsigned)std::max(ceil_div(m.slots, kThreads), 1LL), kThreads, 0, stream>>>(m);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return list_bricks(g, m, counts_host, stream);
}

int begin(const Geo &g, const Mem &m, long long quirk_period, long long *counts_host, cudaStream_t stream)
{
    long long s[3];
    pool_sizes(g, m.slots, s);
    NPHM_CUDA_CHECK(cudaMemsetAsync(m.hdr, 0, 256, stream));
    NPHM_CUDA_CHECK(cudaMemsetAsync(m.states, 0, pad(g.n_blocks), stream));
    NPHM_CUDA_CHECK(cudaMemsetAsync(m.slot, 0xff, g.n_blocks * 4, stream));
    NPHM_CUDA_CHECK(cudaMemsetAsync(m.cmarks, 0, pad(g.n_corners), stream));
    NPHM_CUDA_CHECK(cudaMemsetAsync(m.pdone, 0, 2 * g.rr, stream));
    NPHM_CUDA_CHECK(cudaMemsetAsync(m.bmarks, 0, s[0], stream));
    if (quirk_period > 0) {
        // the quirk voxels of the slab's planes (as in narrowband.cu): their blocks are forced and take bricks now
        const long long n_all = g.rr * g.res, g1 = (g.X1 + 1) * g.rr;
        const long long k0 = g.X0 * g.rr / quirk_period;
        const long long k1 = g1 == n_all ? ceil_div(n_all, quirk_period) : g1 / quirk_period;
        if (k1 > k0) {
            const unsigned ctas = (unsigned)ceil_div(k1 - k0, kThreads);
            quirk_states_kernel<<<ctas, kThreads, 0, stream>>>(g, quirk_period, k0, k1, m.states);
            NPHM_CUDA_CHECK(cudaGetLastError());
            int rc = allocate(g, m, stream);
            if (rc) return rc;
            quirk_mark_kernel<<<ctas, kThreads, 0, stream>>>(g, m, quirk_period, k0, k1);
            NPHM_CUDA_CHECK(cudaGetLastError());
        }
    }
    return list_bricks(g, m, counts_host, stream);
}

// ---------------------------------------------------------------------------------------------- marching cubes on the bricks
// The mesh of the filled slab volume, bit for bit what nphm_mc_count / nphm_mc_emit give on it (negate, iso 0), reading only the
// bricks (and, for the ghost layer of a slab, the ghost plane and plane X0).  The id of a vertex is the number of vertices created
// by earlier cells in the x-major sweep plus its rank in its owner cell.  After closure every crossing cell - and so every owner
// cell of a crossing edge - lies in an active block (a cell of an inactive block has all corners on one side), so only the cells
// of active blocks create vertices.  A segment is one cell row (i, j) of one active block: its cells k in [bz B, min(bz B + B, C)).
// Segments in sweep order are (i, j, bz): row (i, j) holds one segment per active block of its column (i / B, j / B), and its
// first segment's index is an exclusive scan over the rows of those counts.  The vertex and triangle bases of the segments are
// exclusive scans of their counts in that order.  A slab's ghost layer (cells X0 - 1, owned by the neighbour below) creates the
// vertices of the edges on plane X0 that its triangles reference; they are counted per cell over the whole layer (res^2 cells) and
// get ids below the slab's first vertex, as in the slab kernels.
__constant__ unsigned short c_edge[256];
__constant__ signed char c_tri[256][16];
__constant__ unsigned char c_ntri[256];
__constant__ unsigned short c_before[12];        // edges created before edge e: creation order 6, 5, 10, 0, 1, 2, 3, 4, 7, 8, 9, 11
__constant__ unsigned char c_corner[8][3] = {{0,0,0},{1,0,0},{1,1,0},{0,1,0},{0,0,1},{1,0,1},{1,1,1},{0,1,1}};
__constant__ unsigned char c_edge_a[12] = {0, 1, 2, 3, 4, 5, 6, 7, 0, 1, 2, 3};
__constant__ unsigned char c_edge_b[12] = {1, 2, 3, 0, 5, 6, 7, 4, 4, 5, 6, 7};
__constant__ unsigned char c_edge_of[3][2][2] = {{{0, 4}, {2, 6}}, {{3, 7}, {1, 5}}, {{8, 11}, {9, 10}}};
bool g_mc_loaded[64] = {false};

int load_mc_tables()
{
    int dev = 0;
    NPHM_CUDA_CHECK(cudaGetDevice(&dev));
    if (dev < 64 && g_mc_loaded[dev]) return NPHM_OK;
    NPHM_CUDA_CHECK(cudaMemcpyToSymbol(c_edge, MC_EDGE_TABLE, sizeof(MC_EDGE_TABLE)));
    NPHM_CUDA_CHECK(cudaMemcpyToSymbol(c_tri, MC_TRI_TABLE, sizeof(MC_TRI_TABLE)));
    NPHM_CUDA_CHECK(cudaMemcpyToSymbol(c_ntri, MC_NUM_TRIS, sizeof(MC_NUM_TRIS)));
    const int order[12] = {6, 5, 10, 0, 1, 2, 3, 4, 7, 8, 9, 11};
    unsigned short before[12], acc = 0;
    for (int o = 0; o < 12; ++o) {
        before[order[o]] = acc;
        acc |= (unsigned short)(1u << order[o]);
    }
    NPHM_CUDA_CHECK(cudaMemcpyToSymbol(c_before, before, sizeof(before)));
    if (dev < 64) g_mc_loaded[dev] = true;
    return NPHM_OK;
}

// edges whose vertex cell (gi, cj, ck) creates: it is the first cell in sweep order that contains the edge
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

struct McWs {
    unsigned long long *hdr;       // [0] active blocks, [1] segments, [2] vertices, [3] triangles, [4] ghost-layer vertices
    unsigned *alist, *colcnt, *colstart, *rowbase, *segv, *segt, *gloc, *growv, *cnt, *off;
    float *px0;                    // plane X0 of the filled volume (slabs with a ghost layer)
    long long ncol, nrows, nseg, ngcell, bytes;
};

inline McWs mc_carve(void *ws, const Geo &g, long long slots)
{
    McWs w;
    char *p = static_cast<char *>(ws);
    long long off = 0;
    auto take = [&](long long bytes) { char *q = p + off; off += al(bytes); return q; };
    w.ncol = (long long)(g.L1 - g.L0) * g.nb;
    w.nrows = (long long)(g.X1 - g.X0) * g.C;
    w.nseg = std::max(slots, 1LL) * g.B * g.B;
    w.ngcell = g.ghost ? (long long)g.C * g.C : 1;
    const long long chunks = ceil_div(std::max(std::max(w.nseg, w.nrows), std::max(w.ncol, w.ngcell)), kChunk);
    w.hdr = reinterpret_cast<unsigned long long *>(take(256));
    w.alist = reinterpret_cast<unsigned *>(take(std::max(slots, 1LL) * 4));
    w.colcnt = reinterpret_cast<unsigned *>(take(w.ncol * 4));
    w.colstart = reinterpret_cast<unsigned *>(take(w.ncol * 4));
    w.rowbase = reinterpret_cast<unsigned *>(take(w.nrows * 4));
    w.segv = reinterpret_cast<unsigned *>(take(w.nseg * 4));
    w.segt = reinterpret_cast<unsigned *>(take(w.nseg * 4));
    w.gloc = reinterpret_cast<unsigned *>(take(w.ngcell * 4));
    w.growv = reinterpret_cast<unsigned *>(take((long long)g.C * 4));
    w.px0 = reinterpret_cast<float *>(take(g.ghost ? g.rr * 4 : 4));
    w.cnt = reinterpret_cast<unsigned *>(take(chunks * 4));
    w.off = reinterpret_cast<unsigned *>(take(chunks * 4));
    w.bytes = off;
    return w;
}

// exclusive scan of n u32 in place, total to *total: chunk sums, a one-CTA scan of those, then each chunk rescanned from its offset
__device__ __forceinline__ void sum_body(const unsigned *__restrict__ v, long long n, unsigned *__restrict__ cnt)
{
    const long long i0 = (long long)blockIdx.x * kChunk + threadIdx.x * kPerThread;
    unsigned s = 0, total;
    for (int t = 0; t < kPerThread; ++t) s += i0 + t < n ? v[i0 + t] : 0u;
    cta_exclusive_scan<kThreads>(s, total);
    if (threadIdx.x == 0) cnt[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kThreads) sum_kernel(const unsigned *__restrict__ v, long long n, unsigned *__restrict__ cnt)
{
    sum_body(v, n, cnt);
}

__device__ __forceinline__ void rescan_body(unsigned *__restrict__ v, long long n, const unsigned *__restrict__ off)
{
    const long long i0 = (long long)blockIdx.x * kChunk + threadIdx.x * kPerThread;
    unsigned s = 0, total;
    for (int t = 0; t < kPerThread; ++t) s += i0 + t < n ? v[i0 + t] : 0u;
    unsigned run = off[blockIdx.x] + cta_exclusive_scan<kThreads>(s, total);
    for (int t = 0; t < kPerThread; ++t)
        if (i0 + t < n) {
            const unsigned x = v[i0 + t];
            v[i0 + t] = run;
            run += x;
        }
}

__global__ void __launch_bounds__(kThreads) rescan_kernel(unsigned *__restrict__ v, long long n, const unsigned *__restrict__ off)
{
    rescan_body(v, n, off);
}

int scan_u32(const McWs &w, unsigned *v, long long n, unsigned long long *total, cudaStream_t stream)
{
    const long long chunks = std::max(ceil_div(n, kChunk), 1LL);
    sum_kernel<<<(unsigned)chunks, kThreads, 0, stream>>>(v, n, w.cnt);
    NPHM_CUDA_CHECK(cudaGetLastError());
    scan_kernel<<<1, kScanThreads, 0, stream>>>(w.cnt, w.off, chunks, total);
    NPHM_CUDA_CHECK(cudaGetLastError());
    rescan_kernel<<<(unsigned)chunks, kThreads, 0, stream>>>(v, n, w.off);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

__device__ __forceinline__ void col_count_body(const Geo g, const McWs w)
{
    const long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (p < (long long)w.hdr[0]) atomicAdd(w.colcnt + w.alist[p] / g.nb, 1u);
}

__global__ void col_count_kernel(const Geo g, const McWs w)
{
    col_count_body(g, w);
}

__device__ __forceinline__ void row_count_body(const Geo g, const McWs w)
{
    const long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (r >= w.nrows) return;
    const int i = g.X0 + (int)(r / g.C), j = (int)(r % g.C);
    w.rowbase[r] = w.colcnt[(long long)(i / g.B - g.L0) * g.nb + j / g.B];
}

__global__ void row_count_kernel(const Geo g, const McWs w)
{
    row_count_body(g, w);
}

// case index of cell (i, j, k) of the block at brick slot s whose voxel box starts at lo
__device__ __forceinline__ unsigned brick_case(const Geo &g, const Mem &m, unsigned s, const int lo[3], int i, int j, int k)
{
    const float *b = m.bvals + s * g.V + ((long long)(i - lo[0]) * g.E + (j - lo[1])) * g.E + (k - lo[2]);
    unsigned cube = 0;
#pragma unroll
    for (int c = 0; c < 8; ++c)
        if (side(b[((long long)c_corner[c][0] * g.E + c_corner[c][1]) * g.E + c_corner[c][2]])) cube |= 1u << c;
    return cube;
}

__device__ __forceinline__ float ghost_value(const Geo &g, const Mem &m, const McWs &w, int dx, int y, int z)
{
    const long long i = (long long)y * g.res + z;
    return dx ? w.px0[i] : m.ghostv[i];
}

__device__ __forceinline__ unsigned ghost_case(const Geo &g, const Mem &m, const McWs &w, int j, int k)
{
    unsigned cube = 0;
#pragma unroll
    for (int c = 0; c < 8; ++c)
        if (side(ghost_value(g, m, w, c_corner[c][0], j + c_corner[c][1], k + c_corner[c][2]))) cube |= 1u << c;
    return cube;
}

// one thread per segment (active block p, row il, jl of its cells): where it is in sweep order and its cells
struct Seg {
    unsigned slot;
    int lo[3], i, j, k0, k1;
    long long s;
};

__device__ __forceinline__ bool segment(const Geo &g, const Mem &m, const McWs &w, long long t, Seg &sg)
{
    const long long BB = (long long)g.B * g.B;
    const long long p = t / BB;
    if (p >= (long long)w.hdr[0]) return false;
    const unsigned b = w.alist[p];
    int bx, by, bz;
    unblock(g, b, bx, by, bz);
    sg.i = bx * g.B + (int)((t / g.B) % g.B);
    sg.j = by * g.B + (int)(t % g.B);
    if (sg.i >= g.C || sg.j >= g.C) return false;
    sg.slot = m.slot[b];
    sg.lo[0] = bx * g.B; sg.lo[1] = by * g.B; sg.lo[2] = bz * g.B;
    sg.k0 = bz * g.B;
    sg.k1 = min(sg.k0 + g.B, g.C);
    const unsigned col = b / g.nb;
    sg.s = (long long)w.rowbase[(long long)(sg.i - g.X0) * g.C + sg.j] + (p - w.colstart[col]);
    return true;
}

__device__ __forceinline__ void seg_count_body(const Geo g, const Mem m, const McWs w)
{
    Seg sg;
    if (!segment(g, m, w, blockIdx.x * (long long)blockDim.x + threadIdx.x, sg)) return;
    unsigned nv = 0, nt = 0;
    for (int k = sg.k0; k < sg.k1; ++k) {
        const unsigned cube = brick_case(g, m, sg.slot, sg.lo, sg.i, sg.j, k);
        nv += __popc(c_edge[cube] & own_mask(sg.i, sg.j, k));
        nt += c_ntri[cube];
    }
    w.segv[sg.s] = nv;
    w.segt[sg.s] = nt;
}

__global__ void seg_count_kernel(const Geo g, const Mem m, const McWs w)
{
    seg_count_body(g, m, w);
}

// one thread per row of the ghost layer: the vertices its cells create, as a running count within the row
__global__ void ghost_rows_kernel(const Geo g, const Mem m, const McWs w)
{
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= g.C) return;
    unsigned run = 0;
    for (int k = 0; k < g.C; ++k) {
        w.gloc[(long long)j * g.C + k] = run;
        run += __popc(c_edge[ghost_case(g, m, w, j, k)] & own_mask(g.X0 - 1, j, k));
    }
    w.growv[j] = run;
}

__device__ __forceinline__ double mc_interp(double fa, double fb, double xa, double xb)
{
    if (fb == fa) return __ddiv_rn(__dadd_rn(xb, xa), 2.0);
    const double num = __dmul_rn(__dsub_rn(xb, xa), __dsub_rn(0.0, fa));
    return __dadd_rn(__ddiv_rn(num, __dsub_rn(fb, fa)), xa);
}

__device__ int find_block(const McWs &w, unsigned b)
{
    int lo = 0, hi = (int)w.hdr[0] - 1;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (w.alist[mid] < b) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// id (relative to the slab's first vertex; negative: created by the ghost layer) of the vertex on edge e of cell (i, j, k)
__device__ long long vertex_id(const Geo &g, const Mem &m, const McWs &w, int i, int j, int k, unsigned cube, long long own_base, int e)
{
    const int a = c_edge_a[e], bb = c_edge_b[e];
    const int axis = c_corner[a][0] != c_corner[bb][0] ? 0 : (c_corner[a][1] != c_corner[bb][1] ? 1 : 2);
    const int lo = c_corner[a][axis] == 0 ? a : bb;
    const int ei = i + c_corner[lo][0], ej = j + c_corner[lo][1], ek = k + c_corner[lo][2];
    int fi = ei, fj = ej, fk = ek;
    if (axis != 0) fi = ei > 0 ? ei - 1 : ei;
    if (axis != 1) fj = ej > 0 ? ej - 1 : 0;
    if (axis != 2) fk = ek > 0 ? ek - 1 : 0;
    int d1, d2;
    if (axis == 0)      { d1 = ej - fj; d2 = ek - fk; }
    else if (axis == 1) { d1 = ei - fi; d2 = ek - fk; }
    else                { d1 = ei - fi; d2 = ej - fj; }
    const int eo = c_edge_of[axis][d1][d2];
    long long base;
    unsigned ocube;
    if (fi == i && fj == j && fk == k) {
        base = own_base;
        ocube = cube;
    } else if (fi < g.X0) {
        base = (long long)w.gloc[(long long)fj * g.C + fk] + w.growv[fj] - (long long)w.hdr[4];
        ocube = ghost_case(g, m, w, fj, fk);
    } else {
        const int obx = fi / g.B, oby = fj / g.B, obz = fk / g.B;
        const unsigned ob = (unsigned)blk(g, obx, oby, obz);
        const int p = find_block(w, ob);
        const int olo[3] = {obx * g.B, oby * g.B, obz * g.B};
        const unsigned s = m.slot[ob];
        base = (long long)w.segv[(long long)w.rowbase[(long long)(fi - g.X0) * g.C + fj] + (p - w.colstart[ob / g.nb])];
        for (int kk = olo[2]; kk < fk; ++kk) base += __popc(c_edge[brick_case(g, m, s, olo, fi, fj, kk)] & own_mask(fi, fj, kk));
        ocube = brick_case(g, m, s, olo, fi, fj, fk);
    }
    return base + __popc(c_edge[ocube] & own_mask(fi, fj, fk) & c_before[eo]);
}

__global__ void seg_emit_kernel(const Geo g, const Mem m, const McWs w, long long vert_id_base, double *__restrict__ verts,
                                long long *__restrict__ tris)
{
    Seg sg;
    if (!segment(g, m, w, blockIdx.x * (long long)blockDim.x + threadIdx.x, sg)) return;
    long long vrun = w.segv[sg.s], trun = w.segt[sg.s];
    const float *bv = m.bvals + sg.slot * g.V;
    for (int k = sg.k0; k < sg.k1; ++k) {
        const unsigned cube = brick_case(g, m, sg.slot, sg.lo, sg.i, sg.j, k);
        if (cube == 0u || cube == 255u) continue;
        const unsigned created = c_edge[cube] & own_mask(sg.i, sg.j, k);
        for (int e = 0; e < 12; ++e) {
            if (!(created & (1u << e))) continue;
            const int a = c_edge_a[e], b = c_edge_b[e];
            const int axis = c_corner[a][0] != c_corner[b][0] ? 0 : (c_corner[a][1] != c_corner[b][1] ? 1 : 2);
            auto val = [&](int c) {
                return -(double)bv[((long long)(sg.i + c_corner[c][0] - sg.lo[0]) * g.E + (sg.j + c_corner[c][1] - sg.lo[1])) * g.E +
                                   (k + c_corner[c][2] - sg.lo[2])];
            };
            double pos[3] = {(double)(sg.i + c_corner[a][0]), (double)(sg.j + c_corner[a][1]), (double)(k + c_corner[a][2])};
            const double qa = pos[axis], qb = qa + (double)(c_corner[b][axis] - c_corner[a][axis]);
            pos[axis] = mc_interp(val(a), val(b), qa, qb);
            double *dst = verts + (vrun + __popc(created & c_before[e])) * 3;
            dst[0] = pos[0]; dst[1] = pos[1]; dst[2] = pos[2];
        }
        const int n = c_ntri[cube];
        for (int q = 0; q < 3 * n; ++q)
            tris[trun * 3 + q] = vert_id_base + vertex_id(g, m, w, sg.i, sg.j, k, cube, vrun, c_tri[cube][q]);
        vrun += __popc(created);
        trun += n;
    }
}

int mc_count(const Geo &g, const Mem &m, const McWs &w, long long *n_verts, long long *n_tris, cudaStream_t stream)
{
    int rc = load_mc_tables();
    if (rc) return rc;
    NPHM_CUDA_CHECK(cudaMemsetAsync(w.hdr, 0, 256, stream));
    // the active blocks in block order (states are only read: kMarked stays kMarked)
    if ((rc = compact(m, m.states, pad(g.n_blocks), kMarked, kMarked, w.hdr, nullptr, ~0ull, w.alist, stream))) return rc;
    NPHM_CUDA_CHECK(cudaMemsetAsync(w.colcnt, 0, w.ncol * 4, stream));
    col_count_kernel<<<(unsigned)std::max(ceil_div(m.slots, kThreads), 1LL), kThreads, 0, stream>>>(g, w);
    NPHM_CUDA_CHECK(cudaGetLastError());
    NPHM_CUDA_CHECK(cudaMemcpyAsync(w.colstart, w.colcnt, w.ncol * 4, cudaMemcpyDeviceToDevice, stream));
    if ((rc = scan_u32(w, w.colstart, w.ncol, w.hdr + 5, stream))) return rc;
    row_count_kernel<<<(unsigned)ceil_div(w.nrows, kThreads), kThreads, 0, stream>>>(g, w);
    NPHM_CUDA_CHECK(cudaGetLastError());
    if ((rc = scan_u32(w, w.rowbase, w.nrows, w.hdr + 1, stream))) return rc;
    NPHM_CUDA_CHECK(cudaMemsetAsync(w.segv, 0, w.nseg * 4, stream));
    NPHM_CUDA_CHECK(cudaMemsetAsync(w.segt, 0, w.nseg * 4, stream));
    seg_count_kernel<<<(unsigned)ceil_div(w.nseg, kThreads), kThreads, 0, stream>>>(g, m, w);
    NPHM_CUDA_CHECK(cudaGetLastError());
    if ((rc = scan_u32(w, w.segv, w.nseg, w.hdr + 2, stream)) || (rc = scan_u32(w, w.segt, w.nseg, w.hdr + 3, stream))) return rc;
    if (g.ghost) {
        const long long ctas = std::min(ceil_div(g.rr, kThreads), 64LL * sm_count());
        volume_kernel<<<(unsigned)ctas, kThreads, 0, stream>>>(g, m, g.X0, g.rr, w.px0);
        NPHM_CUDA_CHECK(cudaGetLastError());
        ghost_rows_kernel<<<(unsigned)ceil_div(g.C, kThreads), kThreads, 0, stream>>>(g, m, w);
        NPHM_CUDA_CHECK(cudaGetLastError());
        if ((rc = scan_u32(w, w.growv, g.C, w.hdr + 4, stream))) return rc;
    }
    unsigned long long h[5];
    NPHM_CUDA_CHECK(cudaMemcpyAsync(h, w.hdr, sizeof(h), cudaMemcpyDeviceToHost, stream));
    NPHM_CUDA_CHECK(cudaStreamSynchronize(stream));
    NPHM_REQUIRE(h[2] < 0xffffffffull && h[3] < 0xffffffffull, "nphm_band_sparse_mc_count: mesh too large for 32-bit ids");
    *n_verts = (long long)h[2];
    *n_tris = (long long)h[3];
    return NPHM_OK;
}


// ---------------------------------------------------------------------------------------------- S heads of one whole grid
// The band of S heads in lockstep (DESIGN §4.21): every head runs the steps above on the whole grid (the slab [0, nb): no shared or
// ghost plane), the head being blockIdx.y of every launch.  Head h's frame (header, block states and slots, corner values and
// marks) lies h F bytes after head 0's, where F stops before the plane buffers the whole grid never reads; the axes are head 0's.
// Head h's pool is the h-th of S pools of equal size in the caller's buffers, each of the sizes nphm_band_pool gives, so a list
// entry slot (B+1)^3 + local stays local to its head and the u32 caps of the single band apply per head.  A step that allocates
// decides for all heads at once (commit_heads_kernel): when one head's pool is short, no head takes a brick or lists anything, so
// the caller can grow every pool and repeat the same call.  The heads record (256-byte aligned, before head 0's frame) holds that
// decision and a copy of each head's header, read back with one copy per listing step.
struct HeadStrides {
    long long frame, vals, marks, blocks, list, chunks;     // bytes between two heads' frames and pool buffers
};

template <class T> __host__ __device__ __forceinline__ T *shift(T *p, long long bytes) { return (T *)((const char *)p + bytes); }

__host__ __device__ __forceinline__ Mem head_mem(const Mem &m0, const HeadStrides &hs, long long h)
{
    Mem m = m0;
    const long long f = h * hs.frame;
    m.hdr = shift(m0.hdr, f); m.states = shift(m0.states, f); m.slot = shift(m0.slot, f);
    m.cmarks = shift(m0.cmarks, f); m.cvals = shift(m0.cvals, f);
    m.bvals = shift(m0.bvals, h * hs.vals); m.bmarks = shift(m0.bmarks, h * hs.marks); m.sblock = shift(m0.sblock, h * hs.blocks);
    m.list = shift(m0.list, h * hs.list);
    m.chunk_cnt = shift(m0.chunk_cnt, h * hs.chunks); m.chunk_off = shift(m0.chunk_off, h * hs.chunks);
    return m;
}

__host__ __device__ __forceinline__ McWs head_mc(const McWs &w0, long long stride, long long h)
{
    McWs w = w0;
    const long long o = h * stride;
    w.hdr = shift(w0.hdr, o); w.alist = shift(w0.alist, o); w.colcnt = shift(w0.colcnt, o); w.colstart = shift(w0.colstart, o);
    w.rowbase = shift(w0.rowbase, o); w.segv = shift(w0.segv, o); w.segt = shift(w0.segt, o); w.gloc = shift(w0.gloc, o);
    w.growv = shift(w0.growv, o); w.px0 = shift(w0.px0, o); w.cnt = shift(w0.cnt, o); w.off = shift(w0.off, o);
    return w;
}

inline long long heads_record_bytes(int S) { return al(64LL * (S + 1)); }     // word 0: pool short; words 8h + 8 ..: head h's header
inline long long heads_frame_bytes(const Geo &g) { return frame_layout(g).pvals; }
inline long long heads_bytes(const Geo &g, int S) { return heads_record_bytes(S) + S * heads_frame_bytes(g); }
inline long long heads_mc_record_bytes(int S) { return al(32LL * S); }         // S (n_verts, n_tris), then their exclusive scans

struct HeadsBand {
    Geo g;
    Mem m0;
    HeadStrides hs;
    int S;
    unsigned long long *rec;
};

__global__ void __launch_bounds__(kThreads) count_heads_kernel(const unsigned char *__restrict__ bytes, long long bstride, unsigned want4,
                                                               unsigned *__restrict__ cnt, long long cstride)
{
    count_body(shift(bytes, blockIdx.y * bstride), want4, shift(cnt, blockIdx.y * cstride));
}

__global__ void __launch_bounds__(kScanThreads) scan_heads_kernel(const unsigned *__restrict__ cnt, unsigned *__restrict__ off,
                                                                  long long cstride, long long n_chunks,
                                                                  unsigned long long *__restrict__ total, long long tstride)
{
    scan_body(shift(cnt, blockIdx.y * cstride), shift(off, blockIdx.y * cstride), n_chunks, shift(total, blockIdx.y * tstride));
}

// `short_flag`: nothing is listed or set when *short_flag (the allocation's decision for all heads)
__global__ void __launch_bounds__(kThreads) emit_heads_kernel(unsigned char *__restrict__ bytes, long long bstride, unsigned want4,
                                                              unsigned set4, const unsigned *__restrict__ cnt,
                                                              const unsigned *__restrict__ off, long long cstride,
                                                              unsigned *__restrict__ list, long long lstride,
                                                              const unsigned long long *__restrict__ short_flag)
{
    if (shift(cnt, blockIdx.y * cstride)[blockIdx.x] == 0 || (short_flag && *short_flag)) return;
    emit_body(shift(bytes, blockIdx.y * bstride), want4, set4, shift(off, blockIdx.y * cstride), shift(list, blockIdx.y * lstride));
}

// after the compaction counts of the activated blocks: every head takes its slots, or - when one head's pool is short - none does
__global__ void __launch_bounds__(kScanThreads) commit_heads_kernel(const Mem m0, const HeadStrides hs, int S, unsigned long long cap,
                                                                    unsigned long long *rec)
{
    bool over = false;
    for (int h = threadIdx.x; h < S; h += blockDim.x) {
        const unsigned long long *hdr = shift(m0.hdr, h * hs.frame);
        over |= hdr[H_USED] + hdr[H_NEW] > cap;
    }
    const int any = __syncthreads_or(over);
    for (int h = threadIdx.x; h < S; h += blockDim.x) {
        unsigned long long *hdr = shift(m0.hdr, h * hs.frame);
        const unsigned long long used = hdr[H_USED], n = hdr[H_NEW];
        if (any) {
            hdr[H_NEED] = used + n;
            hdr[H_OVER] = 1;
        } else {
            hdr[H_OLD] = used;
            hdr[H_USED] = used + n;
            hdr[H_OVER] = 0;
        }
    }
    if (threadIdx.x == 0) rec[0] = any ? 1ull : 0ull;
}

__global__ void set_kind_heads_kernel(const Mem m0, const HeadStrides hs, int S, unsigned long long kind)
{
    for (int h = blockIdx.x * blockDim.x + threadIdx.x; h < S; h += gridDim.x * blockDim.x) shift(m0.hdr, h * hs.frame)[H_KIND] = kind;
}

// each head's header words to the record, for the one read-back
__global__ void record_heads_kernel(const Mem m0, const HeadStrides hs, int S, unsigned long long *rec)
{
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < 8 * S; t += gridDim.x * blockDim.x) rec[8 + t] = shift(m0.hdr, (t / 8) * hs.frame)[t % 8];
}

__global__ void quirk_states_heads_kernel(const Geo g, long long period, long long k0, long long k1, unsigned char *__restrict__ states,
                                          long long fstride)
{
    quirk_states_body(g, period, k0, k1, shift(states, blockIdx.y * fstride));
}

__global__ void quirk_mark_heads_kernel(const Geo g, const Mem m0, const HeadStrides hs, long long period, long long k0, long long k1)
{
    quirk_mark_body(g, head_mem(m0, hs, blockIdx.y), period, k0, k1);
}

__global__ void assign_heads_kernel(const Mem m0, const HeadStrides hs) { assign_body(head_mem(m0, hs, blockIdx.y)); }
__global__ void __launch_bounds__(kThreads) init_heads_kernel(const Geo g, const Mem m0, const HeadStrides hs) { init_body(g, head_mem(m0, hs, blockIdx.y)); }
__global__ void __launch_bounds__(kThreads) mark_heads_kernel(const Geo g, const Mem m0, const HeadStrides hs) { mark_body(g, head_mem(m0, hs, blockIdx.y)); }
__global__ void promote_heads_kernel(const Mem m0, const HeadStrides hs) { promote_body(head_mem(m0, hs, blockIdx.y)); }
__global__ void __launch_bounds__(kThreads) grow_bricks_heads_kernel(const Geo g, const Mem m0, const HeadStrides hs)
{
    grow_bricks_body(g, head_mem(m0, hs, blockIdx.y));
}

__global__ void corners_heads_kernel(long long n, unsigned char *__restrict__ cmarks, long long fstride)
{
    const long long c = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    unsigned char *cm = shift(cmarks, blockIdx.y * fstride);
    if (c < n && cm[c] == kIdle) cm[c] = kWanted;
}

__global__ void classify_heads_kernel(const Geo g, float tau, const Mem m0, const HeadStrides hs)
{
    const Mem m = head_mem(m0, hs, blockIdx.y);
    classify_body(g, tau, m.cvals, m.states);
}

// rows [h n_pad, (h + 1) n_pad) of head h: its listed voxels, then rows that repeat its last listed voxel (voxel 0 when it listed
// nothing), so that every row is a grid point; the axes are head 0's
__global__ void gather_heads_kernel(const Geo g, const Mem m0, const HeadStrides hs, long long n_pad, float *__restrict__ xyz)
{
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= n_pad) return;
    const Mem m = head_mem(m0, hs, blockIdx.y);
    const long long cnt = (long long)m.hdr[H_LISTED];
    int x = 0, y = 0, z = 0;
    if (cnt > 0) entry_voxel(g, m, m.hdr[H_KIND], m.list[i < cnt ? i : cnt - 1], x, y, z);
    float *out = xyz + 3 * (blockIdx.y * n_pad + i);
    out[0] = m0.axes[x];
    out[1] = m0.axes[g.res + y];
    out[2] = m0.axes[2 * g.res + z];
}

__global__ void scatter_heads_kernel(const Geo g, const Mem m0, const HeadStrides hs, long long n_pad, const float *__restrict__ values)
{
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    const Mem m = head_mem(m0, hs, blockIdx.y);
    if (i >= n_pad || i >= (long long)m.hdr[H_LISTED]) return;
    int x, y, z;
    entry_voxel(g, m, m.hdr[H_KIND], m.list[i], x, y, z);
    store(g, m, x, y, z, values[blockIdx.y * n_pad + i]);
}

// ---- compaction, allocation and listing of S heads
// the bytes == want of every head (at bstride from head 0's) -> the heads' lists (at lstride), totals to each header word `word`
int compact_heads(const HeadsBand &b, unsigned char *bytes, long long bstride, long long n_padded, unsigned char want, unsigned char set,
                  int word, unsigned *list, long long lstride, bool allocating, cudaStream_t stream)
{
    const long long n_chunks = n_padded / kChunk;
    const dim3 grid((unsigned)n_chunks, (unsigned)b.S);
    count_heads_kernel<<<grid, kThreads, 0, stream>>>(bytes, bstride, rep4(want), b.m0.chunk_cnt, b.hs.chunks);
    NPHM_CUDA_CHECK(cudaGetLastError());
    scan_heads_kernel<<<dim3(1, (unsigned)b.S), kScanThreads, 0, stream>>>(b.m0.chunk_cnt, b.m0.chunk_off, b.hs.chunks, n_chunks,
                                                                            b.m0.hdr + word, b.hs.frame);
    NPHM_CUDA_CHECK(cudaGetLastError());
    if (allocating) {
        commit_heads_kernel<<<1, kScanThreads, 0, stream>>>(b.m0, b.hs, b.S, (unsigned long long)b.m0.slots, b.rec);
        NPHM_CUDA_CHECK(cudaGetLastError());
    }
    emit_heads_kernel<<<grid, kThreads, 0, stream>>>(bytes, bstride, rep4(want), rep4(set), b.m0.chunk_cnt, b.m0.chunk_off, b.hs.chunks,
                                                     list, lstride, allocating ? b.rec : nullptr);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

int allocate_heads(const HeadsBand &b, cudaStream_t stream)
{
    int rc = compact_heads(b, b.m0.states, b.hs.frame, pad(b.g.n_blocks), kActivated, kForced, H_NEW, b.m0.list, b.hs.list, true, stream);
    if (rc) return rc;
    const unsigned slot_ctas = (unsigned)std::max(ceil_div(b.m0.slots, kThreads), 1LL);
    const unsigned warp_ctas = (unsigned)std::max(ceil_div(b.m0.slots, kWarps), 1LL);
    assign_heads_kernel<<<dim3(slot_ctas, (unsigned)b.S), kThreads, 0, stream>>>(b.m0, b.hs);
    NPHM_CUDA_CHECK(cudaGetLastError());
    init_heads_kernel<<<dim3(warp_ctas, (unsigned)b.S), kThreads, 0, stream>>>(b.g, b.m0, b.hs);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

// the wanted marks of every head -> its list; counts_host[4h ..] = {listed, active blocks, bricks used, bricks needed} of head h,
// read back with one copy; NPHM_ERR_CAPACITY when the pools were short
int list_and_read_heads(const HeadsBand &b, unsigned char *marks, long long mstride, long long n_padded, unsigned char kind,
                        long long *counts_host, cudaStream_t stream)
{
    set_kind_heads_kernel<<<(unsigned)ceil_div(b.S, kThreads), kThreads, 0, stream>>>(b.m0, b.hs, b.S, kind);
    NPHM_CUDA_CHECK(cudaGetLastError());
    int rc = compact_heads(b, marks, mstride, n_padded, kWanted, kDone, H_LISTED, b.m0.list, b.hs.list, false, stream);
    if (rc) return rc;
    record_heads_kernel<<<(unsigned)ceil_div(8LL * b.S, kThreads), kThreads, 0, stream>>>(b.m0, b.hs, b.S, b.rec);
    NPHM_CUDA_CHECK(cudaGetLastError());
    std::vector<unsigned long long> h(8 * (size_t)(b.S + 1));
    NPHM_CUDA_CHECK(cudaMemcpyAsync(h.data(), b.rec, h.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost, stream));
    NPHM_CUDA_CHECK(cudaStreamSynchronize(stream));
    unsigned long long need = 0;
    for (int i = 0; i < b.S; ++i) {
        const unsigned long long *r = h.data() + 8 * (i + 1);
        const unsigned long long ni = r[H_OVER] ? r[H_NEED] : r[H_USED];
        need = std::max(need, ni);
        if (counts_host) {
            counts_host[4 * i] = (long long)r[H_LISTED];
            counts_host[4 * i + 1] = (long long)r[H_ACTIVE];
            counts_host[4 * i + 2] = (long long)r[H_USED];
            counts_host[4 * i + 3] = (long long)ni;
        }
    }
    if (h[0]) {
        set_error("sparse band of %d heads: each head's brick pool holds %lld bricks, %llu needed", b.S, b.m0.slots, need);
        return NPHM_ERR_CAPACITY;
    }
    return NPHM_OK;
}

int list_bricks_heads(const HeadsBand &b, long long *counts_host, cudaStream_t stream)
{
    long long s[3];
    pool_sizes(b.g, b.m0.slots, s);
    return list_and_read_heads(b, b.m0.bmarks, b.hs.marks, s[0], 0, counts_host, stream);
}

int mark_and_list_heads(const HeadsBand &b, long long *counts_host, cudaStream_t stream)
{
    int rc = allocate_heads(b, stream);
    if (rc) return rc;
    const unsigned warp_ctas = (unsigned)std::max(ceil_div(b.m0.slots, kWarps), 1LL);
    mark_heads_kernel<<<dim3(warp_ctas, (unsigned)b.S), kThreads, 0, stream>>>(b.g, b.m0, b.hs);
    NPHM_CUDA_CHECK(cudaGetLastError());
    promote_heads_kernel<<<dim3((unsigned)std::max(ceil_div(b.m0.slots, kThreads), 1LL), (unsigned)b.S), kThreads, 0, stream>>>(b.m0, b.hs);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return list_bricks_heads(b, counts_host, stream);
}

int begin_heads(const HeadsBand &b, long long quirk_period, long long *counts_host, cudaStream_t stream)
{
    const Geo &g = b.g;
    long long s[3];
    pool_sizes(g, b.m0.slots, s);
    NPHM_CUDA_CHECK(cudaMemsetAsync(b.rec, 0, heads_record_bytes(b.S), stream));
    for (int i = 0; i < b.S; ++i) {
        const Mem m = head_mem(b.m0, b.hs, i);
        NPHM_CUDA_CHECK(cudaMemsetAsync(m.hdr, 0, 256, stream));
        NPHM_CUDA_CHECK(cudaMemsetAsync(m.states, 0, pad(g.n_blocks), stream));
        NPHM_CUDA_CHECK(cudaMemsetAsync(m.slot, 0xff, g.n_blocks * 4, stream));
        NPHM_CUDA_CHECK(cudaMemsetAsync(m.cmarks, 0, pad(g.n_corners), stream));
        NPHM_CUDA_CHECK(cudaMemsetAsync(m.bmarks, 0, s[0], stream));
    }
    if (quirk_period > 0) {
        // the quirk voxels of the whole grid, the same for every head: their blocks are forced and take bricks now
        const long long k1 = ceil_div(g.rr * g.res, quirk_period);
        const dim3 grid((unsigned)ceil_div(k1, kThreads), (unsigned)b.S);
        quirk_states_heads_kernel<<<grid, kThreads, 0, stream>>>(g, quirk_period, 0, k1, b.m0.states, b.hs.frame);
        NPHM_CUDA_CHECK(cudaGetLastError());
        int rc = allocate_heads(b, stream);
        if (rc) return rc;
        quirk_mark_heads_kernel<<<grid, kThreads, 0, stream>>>(g, b.m0, b.hs, quirk_period, 0, k1);
        NPHM_CUDA_CHECK(cudaGetLastError());
    }
    return list_bricks_heads(b, counts_host, stream);
}

// ---- marching cubes of S heads: the single band's scans per head (blockIdx.y), one read-back of the S counts
__global__ void __launch_bounds__(kThreads) sum_heads_kernel(const unsigned *__restrict__ v, long long n, unsigned *__restrict__ cnt,
                                                             long long stride)
{
    sum_body(shift(v, blockIdx.y * stride), n, shift(cnt, blockIdx.y * stride));
}

__global__ void __launch_bounds__(kThreads) rescan_heads_kernel(unsigned *__restrict__ v, long long n, const unsigned *__restrict__ off,
                                                                long long stride)
{
    rescan_body(shift(v, blockIdx.y * stride), n, shift(off, blockIdx.y * stride));
}

__global__ void col_count_heads_kernel(const Geo g, const McWs w0, long long stride) { col_count_body(g, head_mc(w0, stride, blockIdx.y)); }
__global__ void row_count_heads_kernel(const Geo g, const McWs w0, long long stride) { row_count_body(g, head_mc(w0, stride, blockIdx.y)); }
__global__ void seg_count_heads_kernel(const Geo g, const Mem m0, const HeadStrides hs, const McWs w0, long long stride)
{
    seg_count_body(g, head_mem(m0, hs, blockIdx.y), head_mc(w0, stride, blockIdx.y));
}

// S (n_verts, n_tris) from the heads' headers to rec[0 .. 2S), their exclusive scans over the heads to rec[2S .. 4S)
__global__ void mc_record_heads_kernel(const McWs w0, long long stride, int S, unsigned long long *rec)
{
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    unsigned long long v = 0, t = 0;
    for (int h = 0; h < S; ++h) {
        const unsigned long long *hdr = shift(w0.hdr, h * stride);
        rec[2 * h] = hdr[2];
        rec[2 * h + 1] = hdr[3];
        rec[2 * S + 2 * h] = v;
        rec[2 * S + 2 * h + 1] = t;
        v += hdr[2];
        t += hdr[3];
    }
}

// seg_emit_kernel for head blockIdx.y, its vertices and triangles at the offsets of heads 0 .. h-1, ids local to the head.  The
// single band's kernel keeps its own copy of this body: its restrict-qualified outputs let it read the bricks through the
// read-only cache, which an inlined body loses.
__global__ void seg_emit_heads_kernel(const Geo g, const Mem m0, const HeadStrides hs, const McWs w0, long long stride,
                                      const unsigned long long *__restrict__ rec, int S, double *__restrict__ verts,
                                      long long *__restrict__ tris)
{
    const Mem m = head_mem(m0, hs, blockIdx.y);
    const McWs w = head_mc(w0, stride, blockIdx.y);
    Seg sg;
    if (!segment(g, m, w, blockIdx.x * (long long)blockDim.x + threadIdx.x, sg)) return;
    verts += 3 * (long long)rec[2 * S + 2 * blockIdx.y];
    tris += 3 * (long long)rec[2 * S + 2 * blockIdx.y + 1];
    long long vrun = w.segv[sg.s], trun = w.segt[sg.s];
    const float *bv = m.bvals + sg.slot * g.V;
    for (int k = sg.k0; k < sg.k1; ++k) {
        const unsigned cube = brick_case(g, m, sg.slot, sg.lo, sg.i, sg.j, k);
        if (cube == 0u || cube == 255u) continue;
        const unsigned created = c_edge[cube] & own_mask(sg.i, sg.j, k);
        for (int e = 0; e < 12; ++e) {
            if (!(created & (1u << e))) continue;
            const int a = c_edge_a[e], b = c_edge_b[e];
            const int axis = c_corner[a][0] != c_corner[b][0] ? 0 : (c_corner[a][1] != c_corner[b][1] ? 1 : 2);
            auto val = [&](int c) {
                return -(double)bv[((long long)(sg.i + c_corner[c][0] - sg.lo[0]) * g.E + (sg.j + c_corner[c][1] - sg.lo[1])) * g.E +
                                   (k + c_corner[c][2] - sg.lo[2])];
            };
            double pos[3] = {(double)(sg.i + c_corner[a][0]), (double)(sg.j + c_corner[a][1]), (double)(k + c_corner[a][2])};
            const double qa = pos[axis], qb = qa + (double)(c_corner[b][axis] - c_corner[a][axis]);
            pos[axis] = mc_interp(val(a), val(b), qa, qb);
            double *dst = verts + (vrun + __popc(created & c_before[e])) * 3;
            dst[0] = pos[0]; dst[1] = pos[1]; dst[2] = pos[2];
        }
        const int n = c_ntri[cube];
        for (int q = 0; q < 3 * n; ++q) tris[trun * 3 + q] = vertex_id(g, m, w, sg.i, sg.j, k, cube, vrun, c_tri[cube][q]);
        vrun += __popc(created);
        trun += n;
    }
}

int scan_u32_heads(const McWs &w0, long long stride, int S, unsigned *v, long long n, unsigned long long *total, cudaStream_t stream)
{
    const long long chunks = std::max(ceil_div(n, kChunk), 1LL);
    sum_heads_kernel<<<dim3((unsigned)chunks, (unsigned)S), kThreads, 0, stream>>>(v, n, w0.cnt, stride);
    NPHM_CUDA_CHECK(cudaGetLastError());
    scan_heads_kernel<<<dim3(1, (unsigned)S), kScanThreads, 0, stream>>>(w0.cnt, w0.off, stride, chunks, total, stride);
    NPHM_CUDA_CHECK(cudaGetLastError());
    rescan_heads_kernel<<<dim3((unsigned)chunks, (unsigned)S), kThreads, 0, stream>>>(v, n, w0.off, stride);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

int mc_count_heads(const HeadsBand &b, const McWs &w0, long long stride, unsigned long long *mrec, long long *counts_host,
                   cudaStream_t stream)
{
    const Geo &g = b.g;
    const int S = b.S;
    int rc = load_mc_tables();
    if (rc) return rc;
    for (int i = 0; i < S; ++i) {
        const McWs w = head_mc(w0, stride, i);
        NPHM_CUDA_CHECK(cudaMemsetAsync(w.hdr, 0, 256, stream));
        NPHM_CUDA_CHECK(cudaMemsetAsync(w.colcnt, 0, w.ncol * 4, stream));
        NPHM_CUDA_CHECK(cudaMemsetAsync(w.segv, 0, w.nseg * 4, stream));
        NPHM_CUDA_CHECK(cudaMemsetAsync(w.segt, 0, w.nseg * 4, stream));
    }
    // the active blocks of each head in block order (states are only read: kMarked stays kMarked); totals to each w.hdr[0]
    const long long n_chunks = pad(g.n_blocks) / kChunk;
    const dim3 grid((unsigned)n_chunks, (unsigned)S);
    count_heads_kernel<<<grid, kThreads, 0, stream>>>(b.m0.states, b.hs.frame, rep4(kMarked), b.m0.chunk_cnt, b.hs.chunks);
    NPHM_CUDA_CHECK(cudaGetLastError());
    scan_heads_kernel<<<dim3(1, (unsigned)S), kScanThreads, 0, stream>>>(b.m0.chunk_cnt, b.m0.chunk_off, b.hs.chunks, n_chunks, w0.hdr,
                                                                          stride);
    NPHM_CUDA_CHECK(cudaGetLastError());
    emit_heads_kernel<<<grid, kThreads, 0, stream>>>(b.m0.states, b.hs.frame, rep4(kMarked), rep4(kMarked), b.m0.chunk_cnt,
                                                     b.m0.chunk_off, b.hs.chunks, w0.alist, stride, nullptr);
    NPHM_CUDA_CHECK(cudaGetLastError());
    col_count_heads_kernel<<<dim3((unsigned)std::max(ceil_div(b.m0.slots, kThreads), 1LL), (unsigned)S), kThreads, 0, stream>>>(g, w0, stride);
    NPHM_CUDA_CHECK(cudaGetLastError());
    for (int i = 0; i < S; ++i) {
        const McWs w = head_mc(w0, stride, i);
        NPHM_CUDA_CHECK(cudaMemcpyAsync(w.colstart, w.colcnt, w.ncol * 4, cudaMemcpyDeviceToDevice, stream));
    }
    if ((rc = scan_u32_heads(w0, stride, S, w0.colstart, w0.ncol, w0.hdr + 5, stream))) return rc;
    row_count_heads_kernel<<<dim3((unsigned)ceil_div(w0.nrows, kThreads), (unsigned)S), kThreads, 0, stream>>>(g, w0, stride);
    NPHM_CUDA_CHECK(cudaGetLastError());
    if ((rc = scan_u32_heads(w0, stride, S, w0.rowbase, w0.nrows, w0.hdr + 1, stream))) return rc;
    seg_count_heads_kernel<<<dim3((unsigned)ceil_div(w0.nseg, kThreads), (unsigned)S), kThreads, 0, stream>>>(g, b.m0, b.hs, w0, stride);
    NPHM_CUDA_CHECK(cudaGetLastError());
    if ((rc = scan_u32_heads(w0, stride, S, w0.segv, w0.nseg, w0.hdr + 2, stream)) ||
        (rc = scan_u32_heads(w0, stride, S, w0.segt, w0.nseg, w0.hdr + 3, stream)))
        return rc;
    mc_record_heads_kernel<<<1, 1, 0, stream>>>(w0, stride, S, mrec);
    NPHM_CUDA_CHECK(cudaGetLastError());
    std::vector<unsigned long long> h(2 * (size_t)S);
    NPHM_CUDA_CHECK(cudaMemcpyAsync(h.data(), mrec, h.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost, stream));
    NPHM_CUDA_CHECK(cudaStreamSynchronize(stream));
    for (int i = 0; i < S; ++i) {
        NPHM_REQUIRE(h[2 * i] < 0xffffffffull && h[2 * i + 1] < 0xffffffffull,
                     "nphm_band_sparse_heads_mc_count: the mesh of head %d is too large for 32-bit ids", i);
        counts_host[2 * i] = (long long)h[2 * i];
        counts_host[2 * i + 1] = (long long)h[2 * i + 1];
    }
    return NPHM_OK;
}

int check_heads(int res, int block, int S, const char *who)
{
    int rc = check_args(res, block, 0, std::max((int)ceil_div(res - 1, std::max(block, 1)), 1), who);
    if (rc) return rc;
    NPHM_REQUIRE(S >= 1 && S <= 65535, "%s: %d heads outside [1, 65535]", who, S);
    return NPHM_OK;
}

// the S heads' band over the caller's workspace and pools (NPHM_ERR_CAPACITY when short, as check_mem)
int carve_heads(int res, int block, int S, const void *ws, long long ws_bytes, const nphm_band_pool *p, HeadsBand &b, const char *who)
{
    int rc = check_heads(res, block, S, who);
    if (rc) return rc;
    b.g = make_geo(res, block, 0, (int)ceil_div(res - 1, block));
    b.S = S;
    NPHM_REQUIRE(ws && p, "%s: NULL workspace or pool", who);
    const long long need = heads_bytes(b.g, S);
    if (ws_bytes < need) {
        set_error("%s: sparse band workspace too small: %lld bytes for %d heads of res %d, block %d, %lld needed", who, ws_bytes, S, res,
                  block, need);
        return NPHM_ERR_CAPACITY;
    }
    NPHM_REQUIRE(p->slots >= 0 && p->slots * b.g.V < (1LL << 32), "%s: pools of %lld bricks of %lld voxels: brick indices are u32", who,
                 p->slots, b.g.V);
    NPHM_REQUIRE(p->vals && p->marks && p->blocks && p->list && p->chunk_cnt && p->chunk_off, "%s: NULL pool buffer", who);
    long long s[3];
    pool_sizes(b.g, p->slots, s);
    if (p->marks_bytes < s[0] || p->list_len < s[1] || p->n_chunks < s[2]) {
        set_error("%s: pool buffers too small for %lld bricks: %lld mark bytes, %lld list entries, %lld chunks needed", who, p->slots,
                  s[0], s[1], s[2]);
        return NPHM_ERR_CAPACITY;
    }
    char *base = static_cast<char *>(const_cast<void *>(ws));
    b.rec = reinterpret_cast<unsigned long long *>(base);
    b.m0 = carve(base + heads_record_bytes(S), b.g, p);
    b.m0.pvals = nullptr;                        // the whole grid has no shared or ghost plane: never read
    b.m0.pdone = nullptr;
    b.m0.ghostv = nullptr;
    b.hs.frame = heads_frame_bytes(b.g);
    b.hs.vals = p->slots * b.g.V * 4;
    b.hs.marks = p->marks_bytes;
    b.hs.blocks = p->slots * 4;
    b.hs.list = p->list_len * 4;
    b.hs.chunks = p->n_chunks * 4;
    return NPHM_OK;
}

}  // namespace sband
}  // namespace nphm

using namespace nphm;

#define SPARSE_PROLOGUE(who)                                                         \
    int rc = sband::check_args(res, block, l0, l1, who);                             \
    if (rc) return rc;                                                               \
    const sband::Geo g = sband::make_geo(res, block, l0, l1);                        \
    if ((rc = sband::check_mem(g, ws, ws_bytes, pool, who))) return rc;              \
    const sband::Mem m = sband::carve(const_cast<void *>(static_cast<const void *>(ws)), g, pool); \
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);

// ---------------------------------------------------------------------------------------------- entry points
extern "C" long long nphm_band_sparse_workspace_bytes(int res, int block, int l0, int l1)
{
    if (sband::check_args(res, block, l0, l1, "nphm_band_sparse_workspace_bytes")) return -1;
    return sband::frame_layout(sband::make_geo(res, block, l0, l1)).bytes;
}

extern "C" int nphm_band_sparse_pool_sizes(int res, int block, int l0, int l1, long long slots, long long *sizes_host)
{
    int rc = sband::check_args(res, block, l0, l1, "nphm_band_sparse_pool_sizes");
    if (rc) return rc;
    NPHM_REQUIRE(sizes_host && slots >= 0, "nphm_band_sparse_pool_sizes: bad arguments");
    const sband::Geo g = sband::make_geo(res, block, l0, l1);
    NPHM_REQUIRE(slots * g.V < (1LL << 32), "nphm_band_sparse_pool_sizes: %lld bricks of %lld voxels: brick indices are u32", slots,
                 g.V);
    sband::pool_sizes(g, slots, sizes_host);
    return NPHM_OK;
}

extern "C" int nphm_band_sparse_begin(int res, int block, int l0, int l1, long long quirk_period, void *ws, long long ws_bytes,
                                      const nphm_band_pool *pool, long long *counts_host, void *stream_)
{
    SPARSE_PROLOGUE("nphm_band_sparse_begin")
    NPHM_REQUIRE(quirk_period >= 0, "nphm_band_sparse_begin: negative quirk period %lld", quirk_period);
    return sband::begin(g, m, quirk_period, counts_host, stream);
}

extern "C" int nphm_band_sparse_corners(int res, int block, int l0, int l1, void *ws, long long ws_bytes, const nphm_band_pool *pool,
                                        long long *counts_host, void *stream_)
{
    SPARSE_PROLOGUE("nphm_band_sparse_corners")
    sband::corners_kernel<<<(unsigned)ceil_div(g.n_corners, sband::kThreads), sband::kThreads, 0, stream>>>(g.n_corners, m.cmarks);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return sband::list_and_read(g, m, m.cmarks, sband::pad(g.n_corners), 1, counts_host, stream);
}

extern "C" int nphm_band_sparse_classify(int res, int block, int l0, int l1, float tau, void *ws, long long ws_bytes,
                                         const nphm_band_pool *pool, long long *counts_host, void *stream_)
{
    SPARSE_PROLOGUE("nphm_band_sparse_classify")
    NPHM_REQUIRE(tau >= 0.f, "nphm_band_sparse_classify: need tau >= 0 (got %g)", (double)tau);
    sband::classify_kernel<<<(unsigned)ceil_div(g.n_blocks, sband::kThreads), sband::kThreads, 0, stream>>>(g, tau, m.cvals, m.states);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return sband::mark_and_list(g, m, counts_host, stream);
}

extern "C" int nphm_band_sparse_grow(int res, int block, int l0, int l1, void *ws, long long ws_bytes, const nphm_band_pool *pool,
                                     long long *counts_host, void *stream_)
{
    SPARSE_PROLOGUE("nphm_band_sparse_grow")
    if (m.slots > 0) {
        sband::grow_bricks_kernel<<<(unsigned)ceil_div(m.slots, sband::kWarps), sband::kThreads, 0, stream>>>(g, m);
        NPHM_CUDA_CHECK(cudaGetLastError());
    }
    if (g.lo || g.hi) {
        sband::grow_planes_kernel<<<(unsigned)ceil_div(2 * g.rr, sband::kThreads), sband::kThreads, 0, stream>>>(g, m);
        NPHM_CUDA_CHECK(cudaGetLastError());
    }
    return sband::mark_and_list(g, m, counts_host, stream);
}

extern "C" int nphm_band_sparse_gather(int res, int block, int l0, int l1, const double grid_min[3], const double grid_max[3],
                                       long long n, float *xyz_dev, void *ws, long long ws_bytes, const nphm_band_pool *pool,
                                       void *stream_)
{
    SPARSE_PROLOGUE("nphm_band_sparse_gather")
    long long s[3];
    sband::pool_sizes(g, m.slots, s);
    NPHM_REQUIRE(grid_min && grid_max && n >= 0 && n <= s[1] && (n == 0 || xyz_dev), "nphm_band_sparse_gather: bad arguments");
    if (n == 0) return NPHM_OK;
    if ((rc = launch_grid_axes(grid_min, grid_max, g.res, m.axes, stream))) return rc;
    sband::gather_kernel<<<(unsigned)ceil_div(n, sband::kThreads), sband::kThreads, 0, stream>>>(g, m, n, xyz_dev);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

extern "C" int nphm_band_sparse_scatter(int res, int block, int l0, int l1, long long n, const float *values_dev, void *ws,
                                        long long ws_bytes, const nphm_band_pool *pool, void *stream_)
{
    SPARSE_PROLOGUE("nphm_band_sparse_scatter")
    long long s[3];
    sband::pool_sizes(g, m.slots, s);
    NPHM_REQUIRE(n >= 0 && n <= s[1] && (n == 0 || values_dev), "nphm_band_sparse_scatter: bad arguments");
    if (n == 0) return NPHM_OK;
    sband::scatter_kernel<<<(unsigned)ceil_div(n, sband::kThreads), sband::kThreads, 0, stream>>>(g, m, n, values_dev);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

extern "C" int nphm_band_sparse_fill(int res, int block, int l0, int l1, void *ws, long long ws_bytes, const nphm_band_pool *pool,
                                     void *stream_)
{
    (void)stream_;            // a voxel not evaluated reads as its fill value wherever it is read (lookup): nothing to write
    int rc = sband::check_args(res, block, l0, l1, "nphm_band_sparse_fill");
    return rc ? rc : sband::check_mem(sband::make_geo(res, block, l0, l1), ws, ws_bytes, pool, "nphm_band_sparse_fill");
}

extern "C" int nphm_band_sparse_block_states(int res, int block, int l0, int l1, const void *ws, long long ws_bytes,
                                             const nphm_band_pool *pool, unsigned char *states_dev, void *stream_)
{
    SPARSE_PROLOGUE("nphm_band_sparse_block_states")
    NPHM_REQUIRE(states_dev, "nphm_band_sparse_block_states: NULL output");
    NPHM_CUDA_CHECK(cudaMemcpyAsync(states_dev, m.states, g.n_blocks, cudaMemcpyDeviceToDevice, stream));
    return NPHM_OK;
}

extern "C" int nphm_band_sparse_export(int res, int block, int l0, int l1, int plane, const void *ws, long long ws_bytes,
                                       const nphm_band_pool *pool, unsigned char *buf_dev, void *stream_)
{
    SPARSE_PROLOGUE("nphm_band_sparse_export")
    NPHM_REQUIRE(buf_dev, "nphm_band_sparse_export: NULL buffer");
    NPHM_REQUIRE(plane >= g.X0 && plane <= g.X1, "nphm_band_sparse_export: plane %d outside the slab's planes [%d, %d]", plane, g.X0,
                 g.X1);
    sband::export_kernel<<<(unsigned)ceil_div(g.rr, sband::kThreads), sband::kThreads, 0, stream>>>(
        g, m, plane, reinterpret_cast<float *>(buf_dev), buf_dev + 4 * g.rr);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

extern "C" int nphm_band_sparse_import(int res, int block, int l0, int l1, int plane, const unsigned char *buf_dev, void *ws,
                                       long long ws_bytes, const nphm_band_pool *pool, void *stream_)
{
    SPARSE_PROLOGUE("nphm_band_sparse_import")
    NPHM_REQUIRE(buf_dev, "nphm_band_sparse_import: NULL buffer");
    const bool lower = plane == g.X0 && g.lo, upper = plane == g.X1 && g.hi, ghost = plane == g.X0 - 1 && g.ghost;
    NPHM_REQUIRE(lower || upper || ghost,
                 "nphm_band_sparse_import: plane %d is neither a plane shared with a neighbour nor the ghost plane of the slab of "
                 "block layers [%d, %d) (planes [%d, %d] of %d)", plane, l0, l1, g.X0, g.X1, g.res);
    const float *vals = reinterpret_cast<const float *>(buf_dev);
    if (ghost) {
        NPHM_CUDA_CHECK(cudaMemcpyAsync(m.ghostv, vals, g.rr * sizeof(float), cudaMemcpyDeviceToDevice, stream));
        return NPHM_OK;
    }
    sband::import_kernel<<<(unsigned)ceil_div(g.rr, sband::kThreads), sband::kThreads, 0, stream>>>(g, m, plane, vals,
                                                                                                   buf_dev + 4 * g.rr);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

extern "C" int nphm_band_sparse_volume(int res, int block, int l0, int l1, int x_first, int n_planes, float *out_dev, const void *ws,
                                       long long ws_bytes, const nphm_band_pool *pool, void *stream_)
{
    SPARSE_PROLOGUE("nphm_band_sparse_volume")
    const int first = g.X0 - (g.ghost ? 1 : 0);
    NPHM_REQUIRE(out_dev && n_planes >= 1 && x_first >= first && x_first + n_planes - 1 <= g.X1,
                 "nphm_band_sparse_volume: planes [%d, %d) outside the slab's planes [%d, %d]", x_first, x_first + n_planes, first, g.X1);
    const long long n = (long long)n_planes * g.rr;
    const long long ctas = std::min(ceil_div(n, sband::kThreads), 64LL * sm_count());
    sband::volume_kernel<<<(unsigned)ctas, sband::kThreads, 0, stream>>>(g, m, x_first, n, out_dev);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

extern "C" long long nphm_band_sparse_mc_workspace_bytes(int res, int block, int l0, int l1, long long slots)
{
    if (sband::check_args(res, block, l0, l1, "nphm_band_sparse_mc_workspace_bytes") || slots < 0) return -1;
    return sband::mc_carve(nullptr, sband::make_geo(res, block, l0, l1), slots).bytes;
}

#define SPARSE_MC_PROLOGUE(who)                                                                                       \
    SPARSE_PROLOGUE(who)                                                                                              \
    NPHM_REQUIRE(mc_ws, "%s: NULL marching-cubes workspace", who);                                                    \
    const sband::McWs w = sband::mc_carve(mc_ws, g, m.slots);                                                         \
    if (mc_ws_bytes < w.bytes) {                                                                                      \
        set_error("%s: marching-cubes workspace too small: %lld bytes, %lld needed", who, mc_ws_bytes, w.bytes);      \
        return NPHM_ERR_CAPACITY;                                                                                     \
    }

extern "C" int nphm_band_sparse_mc_count(int res, int block, int l0, int l1, const void *ws, long long ws_bytes,
                                         const nphm_band_pool *pool, void *mc_ws, long long mc_ws_bytes, long long *n_verts_host,
                                         long long *n_tris_host, void *stream_)
{
    SPARSE_MC_PROLOGUE("nphm_band_sparse_mc_count")
    NPHM_REQUIRE(n_verts_host && n_tris_host, "nphm_band_sparse_mc_count: NULL count pointers");
    return sband::mc_count(g, m, w, n_verts_host, n_tris_host, stream);
}

extern "C" int nphm_band_sparse_mc_emit(int res, int block, int l0, int l1, const void *ws, long long ws_bytes, const nphm_band_pool *pool,
                                        void *mc_ws, long long mc_ws_bytes, long long vert_id_base, double *verts_dev, long long *tris_dev,
                                        void *stream_)
{
    SPARSE_MC_PROLOGUE("nphm_band_sparse_mc_emit")
    NPHM_REQUIRE(verts_dev && tris_dev, "nphm_band_sparse_mc_emit: NULL output");
    sband::seg_emit_kernel<<<(unsigned)ceil_div(w.nseg, sband::kThreads), sband::kThreads, 0, stream>>>(g, m, w, vert_id_base, verts_dev,
                                                                                                      tris_dev);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

// ---------------------------------------------------------------------------------------------- entry points: S heads
#define HEADS_PROLOGUE(who)                                                                                         \
    sband::HeadsBand b;                                                                                             \
    int rc = sband::carve_heads(res, block, n_heads, ws, ws_bytes, pool, b, who);                                   \
    if (rc) return rc;                                                                                              \
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);

extern "C" long long nphm_band_sparse_heads_workspace_bytes(int res, int block, int n_heads)
{
    if (sband::check_heads(res, block, n_heads, "nphm_band_sparse_heads_workspace_bytes")) return -1;
    return sband::heads_bytes(sband::make_geo(res, block, 0, (int)ceil_div(res - 1, block)), n_heads);
}

extern "C" int nphm_band_sparse_heads_begin(int res, int block, int n_heads, long long quirk_period, void *ws, long long ws_bytes,
                                            const nphm_band_pool *pool, long long *counts_host, void *stream_)
{
    HEADS_PROLOGUE("nphm_band_sparse_heads_begin")
    NPHM_REQUIRE(quirk_period >= 0, "nphm_band_sparse_heads_begin: negative quirk period %lld", quirk_period);
    return sband::begin_heads(b, quirk_period, counts_host, stream);
}

extern "C" int nphm_band_sparse_heads_corners(int res, int block, int n_heads, void *ws, long long ws_bytes, const nphm_band_pool *pool,
                                              long long *counts_host, void *stream_)
{
    HEADS_PROLOGUE("nphm_band_sparse_heads_corners")
    const long long nc = b.g.n_corners;
    sband::corners_heads_kernel<<<dim3((unsigned)ceil_div(nc, sband::kThreads), (unsigned)n_heads), sband::kThreads, 0, stream>>>(
        nc, b.m0.cmarks, b.hs.frame);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return sband::list_and_read_heads(b, b.m0.cmarks, b.hs.frame, sband::pad(nc), 1, counts_host, stream);
}

extern "C" int nphm_band_sparse_heads_classify(int res, int block, int n_heads, float tau, void *ws, long long ws_bytes,
                                               const nphm_band_pool *pool, long long *counts_host, void *stream_)
{
    HEADS_PROLOGUE("nphm_band_sparse_heads_classify")
    NPHM_REQUIRE(tau >= 0.f, "nphm_band_sparse_heads_classify: need tau >= 0 (got %g)", (double)tau);
    sband::classify_heads_kernel<<<dim3((unsigned)ceil_div(b.g.n_blocks, sband::kThreads), (unsigned)n_heads), sband::kThreads, 0,
                                   stream>>>(b.g, tau, b.m0, b.hs);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return sband::mark_and_list_heads(b, counts_host, stream);
}

extern "C" int nphm_band_sparse_heads_grow(int res, int block, int n_heads, void *ws, long long ws_bytes, const nphm_band_pool *pool,
                                           long long *counts_host, void *stream_)
{
    HEADS_PROLOGUE("nphm_band_sparse_heads_grow")
    if (b.m0.slots > 0) {
        sband::grow_bricks_heads_kernel<<<dim3((unsigned)ceil_div(b.m0.slots, sband::kWarps), (unsigned)n_heads), sband::kThreads, 0,
                                          stream>>>(b.g, b.m0, b.hs);
        NPHM_CUDA_CHECK(cudaGetLastError());
    }
    return sband::mark_and_list_heads(b, counts_host, stream);
}

extern "C" int nphm_band_sparse_heads_gather(int res, int block, int n_heads, const double grid_min[3], const double grid_max[3],
                                             long long n_pad, float *xyz_dev, void *ws, long long ws_bytes, const nphm_band_pool *pool,
                                             void *stream_)
{
    HEADS_PROLOGUE("nphm_band_sparse_heads_gather")
    NPHM_REQUIRE(grid_min && grid_max && n_pad >= 0 && (n_pad == 0 || xyz_dev), "nphm_band_sparse_heads_gather: bad arguments");
    if (n_pad == 0) return NPHM_OK;
    if ((rc = launch_grid_axes(grid_min, grid_max, b.g.res, b.m0.axes, stream))) return rc;
    sband::gather_heads_kernel<<<dim3((unsigned)ceil_div(n_pad, sband::kThreads), (unsigned)n_heads), sband::kThreads, 0, stream>>>(
        b.g, b.m0, b.hs, n_pad, xyz_dev);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

extern "C" int nphm_band_sparse_heads_scatter(int res, int block, int n_heads, long long n_pad, const float *values_dev, void *ws,
                                              long long ws_bytes, const nphm_band_pool *pool, void *stream_)
{
    HEADS_PROLOGUE("nphm_band_sparse_heads_scatter")
    NPHM_REQUIRE(n_pad >= 0 && (n_pad == 0 || values_dev), "nphm_band_sparse_heads_scatter: bad arguments");
    if (n_pad == 0) return NPHM_OK;
    sband::scatter_heads_kernel<<<dim3((unsigned)ceil_div(n_pad, sband::kThreads), (unsigned)n_heads), sband::kThreads, 0, stream>>>(
        b.g, b.m0, b.hs, n_pad, values_dev);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

extern "C" int nphm_band_sparse_heads_fill(int res, int block, int n_heads, void *ws, long long ws_bytes, const nphm_band_pool *pool,
                                           void *stream_)
{
    (void)stream_;            // a voxel not evaluated reads as its fill value wherever it is read (lookup): nothing to write
    sband::HeadsBand b;
    return sband::carve_heads(res, block, n_heads, ws, ws_bytes, pool, b, "nphm_band_sparse_heads_fill");
}

extern "C" int nphm_band_sparse_heads_block_states(int res, int block, int n_heads, const void *ws, long long ws_bytes,
                                                   const nphm_band_pool *pool, unsigned char *states_dev, void *stream_)
{
    HEADS_PROLOGUE("nphm_band_sparse_heads_block_states")
    NPHM_REQUIRE(states_dev, "nphm_band_sparse_heads_block_states: NULL output");
    for (int i = 0; i < n_heads; ++i)
        NPHM_CUDA_CHECK(cudaMemcpyAsync(states_dev + i * b.g.n_blocks, sband::head_mem(b.m0, b.hs, i).states, b.g.n_blocks,
                                        cudaMemcpyDeviceToDevice, stream));
    return NPHM_OK;
}

extern "C" long long nphm_band_sparse_heads_mc_workspace_bytes(int res, int block, int n_heads, long long slots)
{
    if (sband::check_heads(res, block, n_heads, "nphm_band_sparse_heads_mc_workspace_bytes") || slots < 0) return -1;
    const sband::Geo g = sband::make_geo(res, block, 0, (int)ceil_div(res - 1, block));
    return sband::heads_mc_record_bytes(n_heads) + n_heads * sband::mc_carve(nullptr, g, slots).bytes;
}

#define HEADS_MC_PROLOGUE(who)                                                                                      \
    HEADS_PROLOGUE(who)                                                                                             \
    NPHM_REQUIRE(mc_ws, "%s: NULL marching-cubes workspace", who);                                                  \
    char *mc_base = static_cast<char *>(mc_ws);                                                                     \
    const long long mc_stride = sband::mc_carve(nullptr, b.g, b.m0.slots).bytes;                                    \
    const sband::McWs w0 = sband::mc_carve(mc_base + sband::heads_mc_record_bytes(n_heads), b.g, b.m0.slots);       \
    unsigned long long *mrec = reinterpret_cast<unsigned long long *>(mc_base);                                     \
    if (mc_ws_bytes < sband::heads_mc_record_bytes(n_heads) + n_heads * mc_stride) {                                \
        set_error("%s: marching-cubes workspace too small: %lld bytes, %lld needed", who, mc_ws_bytes,              \
                  sband::heads_mc_record_bytes(n_heads) + n_heads * mc_stride);                                      \
        return NPHM_ERR_CAPACITY;                                                                                   \
    }

extern "C" int nphm_band_sparse_heads_mc_count(int res, int block, int n_heads, const void *ws, long long ws_bytes,
                                               const nphm_band_pool *pool, void *mc_ws, long long mc_ws_bytes, long long *counts_host,
                                               void *stream_)
{
    HEADS_MC_PROLOGUE("nphm_band_sparse_heads_mc_count")
    NPHM_REQUIRE(counts_host, "nphm_band_sparse_heads_mc_count: NULL counts");
    return sband::mc_count_heads(b, w0, mc_stride, mrec, counts_host, stream);
}

extern "C" int nphm_band_sparse_heads_mc_emit(int res, int block, int n_heads, const void *ws, long long ws_bytes,
                                              const nphm_band_pool *pool, void *mc_ws, long long mc_ws_bytes, double *verts_dev,
                                              long long *tris_dev, void *stream_)
{
    HEADS_MC_PROLOGUE("nphm_band_sparse_heads_mc_emit")
    NPHM_REQUIRE(verts_dev && tris_dev, "nphm_band_sparse_heads_mc_emit: NULL output");
    sband::seg_emit_heads_kernel<<<dim3((unsigned)ceil_div(w0.nseg, sband::kThreads), (unsigned)n_heads), sband::kThreads, 0, stream>>>(
        b.g, b.m0, b.hs, w0, mc_stride, mrec, n_heads, verts_dev, tris_dev);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}
