// Narrow-band mesh extraction on sm_90a: the steps that decide WHICH voxels of a res^3 grid the decoder has to evaluate so that
// marching cubes on the filled volume gives the dense mesh, and that move values between the grid and compact point lists.
// The decoder itself runs through the existing query entry points on the gathered coordinates (see DESIGN §4.13, §4.16).
//
// The grid's (res - 1)^3 cells are split into blocks of B^3 cells (the last block of an axis may be partial); block b covers the
// voxels [bB, min(bB + B, res - 1)] of each axis, so neighbouring blocks share a face of voxels.  Every step works on an x-slab:
// the block layers [L0, L1) and their voxel planes [X0, X1] = [L0 B, min(L1 B, res - 1)]; the whole grid is the slab [0, nb).
// State lives in a caller-owned workspace, indexed from plane X0:
//   marks   1 byte per voxel: 0 not evaluated, 1 wanted (set by a marking kernel), 2 listed / evaluated
//   states  1 byte per block: 0 inactive, 1 activated (its voxels not yet marked), 2 active (marked)
//   list    u32 slab-local flat voxel indices of the last compaction, ascending
// Marching cubes runs on -sdf at 0, so a voxel is "inside" when -v <= 0, i.e. v >= 0 (NaN: outside) - `side()` below.
//
// Heads: S bands of the same slab (S latent codes of one decoder, DESIGN §4.18) step together.  Head h's workspace and volume lie
// h * Heads::ws bytes and h * Heads::vol floats past head 0's; every kernel takes its head from blockIdx.y, so one launch serves
// all S heads, and the single-band entry points are the S = 1 call of the same kernels.
#include "common.cuh"
#include "simt.cuh"
#include <algorithm>
#include <type_traits>
#include <vector>

namespace nphm {
namespace band {

constexpr int kThreads = 256;
constexpr int kPerThread = 16;                       // marks per thread of the compaction kernels (one 128-bit load)
constexpr int kChunk = kThreads * kPerThread;        // voxels per CTA of the compaction kernels
constexpr int kScanThreads = 1024;
constexpr int kWarpsPerCta = kThreads / 32;

enum : unsigned char { kIdle = 0, kWanted = 1, kDone = 2 };                 // voxel marks
enum : unsigned char { kInactive = 0, kActivated = 1, kMarked = 2 };        // block states

struct Geo {
    int res, B, C, nb;            // grid points per axis, block edge in cells, cells per axis (res - 1), blocks per axis
    int L0, L1, X0, X1;           // block layers [L0, L1) along x and their voxel planes [X0, X1]
    int ghost;                    // planes the caller's volume holds below X0 (1: a slab's ghost plane X0 - 1)
    long long rr, n_vox, n_blocks, n_chunks;    // voxels per plane; voxels, blocks and compaction chunks of the slab
};

struct Layout {
    long long hdr, axes, states, chunk_cnt, chunk_off, marks, list, bytes;
};

inline int blocks_per_axis(int res, int block) { return (int)ceil_div(res - 1, block); }

inline Geo make_geo(int res, int block, int l0, int l1)
{
    Geo g;
    g.res = res; g.B = block; g.C = res - 1;
    g.nb = blocks_per_axis(res, block);
    g.L0 = l0; g.L1 = l1;
    g.X0 = g.L0 * block; g.X1 = std::min(g.L1 * block, g.C);
    g.ghost = g.L0 > 0 ? 1 : 0;
    g.rr = (long long)res * res;
    g.n_vox = (long long)(g.X1 - g.X0 + 1) * g.rr;
    g.n_blocks = (long long)(g.L1 - g.L0) * g.nb * g.nb;
    g.n_chunks = ceil_div(g.n_vox, kChunk);
    return g;
}

inline Layout layout(const Geo &g)
{
    auto al = [](long long x) { return (x + 255) / 256 * 256; };
    Layout l;
    long long off = 0;
    l.hdr = off; off += 256;                                   // [0] voxels listed by the last compaction, [1] active blocks
    l.axes = off; off += al(3LL * g.res * 4);
    l.states = off; off += al(g.n_blocks);
    l.chunk_cnt = off; off += al(g.n_chunks * 4);
    l.chunk_off = off; off += al(g.n_chunks * 4);
    l.marks = off; off += g.n_chunks * kChunk;                 // padded to whole chunks (the padding stays 0)
    l.list = off; off += al(g.n_vox * 4);
    l.bytes = off;
    return l;
}

struct Heads {
    long long ws, vol;            // strides between heads: workspace bytes, volume floats (0, 0 for one band)
};

template <class T>
__device__ __forceinline__ T *head_at(T *p, long long stride_bytes)
{
    using B = typename std::conditional<std::is_const<T>::value, const char, char>::type;
    return reinterpret_cast<T *>(reinterpret_cast<B *>(p) + blockIdx.y * stride_bytes);
}

template <class T>
__device__ __forceinline__ T *head_vol(T *vol, const Heads &H) { return vol + blockIdx.y * H.vol; }

struct Ws {
    unsigned long long *hdr;
    float *axes;
    unsigned char *states, *marks;
    unsigned *chunk_cnt, *chunk_off, *list;
};

inline Ws carve(void *ws, const Layout &l)
{
    char *p = static_cast<char *>(ws);
    return Ws{reinterpret_cast<unsigned long long *>(p + l.hdr), reinterpret_cast<float *>(p + l.axes),
              reinterpret_cast<unsigned char *>(p + l.states), reinterpret_cast<unsigned char *>(p + l.marks),
              reinterpret_cast<unsigned *>(p + l.chunk_cnt), reinterpret_cast<unsigned *>(p + l.chunk_off),
              reinterpret_cast<unsigned *>(p + l.list)};
}

__device__ __forceinline__ bool side(float v) { return v >= 0.f; }

// slab-local flat index of the voxel at global plane x
__device__ __forceinline__ long long vox(const Geo &g, int x, int y, int z)
{
    return ((long long)(x - g.X0) * g.res + y) * g.res + z;
}

// voxel box of block b along one axis
__device__ __forceinline__ int blo(const Geo &g, int b) { return b * g.B; }
__device__ __forceinline__ int bhi(const Geo &g, int b) { return min(b * g.B + g.B, g.C); }

__device__ __forceinline__ void unblock(const Geo &g, long long b, int &bx, int &by, int &bz)
{
    bz = (int)(b % g.nb);
    const long long t = b / g.nb;
    by = (int)(t % g.nb);
    bx = g.L0 + (int)(t / g.nb);
}

// ---------------------------------------------------------------------------------------------- marking
// eval-mode quirk voxels g = (k + 1) p - 1 and g = res^3 - 1 (k in [k0, k1): those of the slab's planes): wanted, and every block
// of the slab owning a cell that touches one is forced
__global__ void quirk_kernel(const Geo g, long long period, long long k0, long long k1, unsigned char *__restrict__ marks,
                             unsigned char *__restrict__ states, const Heads H)
{
    const long long k = k0 + blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (k >= k1) return;
    marks = head_at(marks, H.ws);
    states = head_at(states, H.ws);
    const long long n_all = g.rr * g.res;
    const long long v = k < n_all / period ? (k + 1) * period - 1 : n_all - 1;
    const int x = (int)(v / g.rr), y = (int)((v / g.res) % g.res), z = (int)(v % g.res);
    marks[v - g.X0 * g.rr] = kWanted;
    // cells touching voxel x along an axis: [max(x - 1, 0), min(x, C - 1)]; along x only the slab's block layers
    const int bx0 = max(max(x - 1, 0) / g.B, g.L0), bx1 = min(min(x, g.C - 1) / g.B, g.L1 - 1);
    const int by0 = max(y - 1, 0) / g.B, by1 = min(y, g.C - 1) / g.B;
    const int bz0 = max(z - 1, 0) / g.B, bz1 = min(z, g.C - 1) / g.B;
    for (int bx = bx0; bx <= bx1; ++bx)
        for (int by = by0; by <= by1; ++by)
            for (int bz = bz0; bz <= bz1; ++bz) states[((long long)(bx - g.L0) * g.nb + by) * g.nb + bz] = kActivated;
}

// block corners (fine indices 0, B, 2B, ..., res - 1 on every axis; along x those of the slab's planes, L0 B ... X1)
__global__ void corners_kernel(const Geo g, unsigned char *__restrict__ marks, const Heads H)
{
    const long long n1 = g.nb + 1;
    const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (t >= (g.L1 - g.L0 + 1) * n1 * n1) return;
    marks = head_at(marks, H.ws);
    const int cz = (int)(t % n1), cy = (int)((t / n1) % n1), cx = g.L0 + (int)(t / (n1 * n1));
    const long long v = vox(g, min(cx * g.B, g.C), min(cy * g.B, g.C), min(cz * g.B, g.C));
    if (marks[v] == kIdle) marks[v] = kWanted;
}

// an inactive block becomes active when a corner has |sdf| <= tau (or is NaN) or its corners lie on both sides of the test
__global__ void classify_kernel(const Geo g, float tau, const float *__restrict__ vol, unsigned char *__restrict__ states,
                                const Heads H)
{
    const long long b = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    states = head_at(states, H.ws);
    vol = head_vol(vol, H);
    if (b >= g.n_blocks || states[b] != kInactive) return;
    int bx, by, bz;
    unblock(g, b, bx, by, bz);
    const int xs[2] = {blo(g, bx), bhi(g, bx)}, ys[2] = {blo(g, by), bhi(g, by)}, zs[2] = {blo(g, bz), bhi(g, bz)};
    bool near = false;
    int n_in = 0;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        const float v = __ldg(vol + vox(g, xs[c >> 2], ys[(c >> 1) & 1], zs[c & 1]));
        near |= !(fabsf(v) > tau);
        n_in += side(v) ? 1 : 0;
    }
    if (near || (n_in != 0 && n_in != 8)) states[b] = kActivated;
}

// one warp per block: the voxels of every activated block are wanted (those not evaluated yet); the block becomes active
__global__ void __launch_bounds__(kThreads) mark_blocks_kernel(const Geo g, unsigned char *__restrict__ states,
                                                               unsigned char *__restrict__ marks, unsigned long long *__restrict__ hdr,
                                                               const Heads H)
{
    const long long b = blockIdx.x * (long long)kWarpsPerCta + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    states = head_at(states, H.ws);
    marks = head_at(marks, H.ws);
    hdr = head_at(hdr, H.ws);
    if (b >= g.n_blocks || states[b] != kActivated) return;
    int bx, by, bz;
    unblock(g, b, bx, by, bz);
    const int x0 = blo(g, bx), y0 = blo(g, by), z0 = blo(g, bz);
    const int dx = bhi(g, bx) - x0 + 1, dy = bhi(g, by) - y0 + 1, dz = bhi(g, bz) - z0 + 1;
    for (int i = lane; i < dx * dy * dz; i += 32) {
        const int z = z0 + i % dz, y = y0 + (i / dz) % dy, x = x0 + i / (dz * dy);
        const long long v = vox(g, x, y, z);
        if (marks[v] == kIdle) marks[v] = kWanted;
    }
    __syncwarp();
    if (lane == 0) {
        states[b] = kMarked;
        atomicAdd(hdr + 1, 1ull);
    }
}

// one warp per inactive block: an evaluated voxel on its faces on the other side of the test from its corner 0 (the value its
// unevaluated voxels get) means the surface leaves the band there - the block is activated
__global__ void __launch_bounds__(kThreads) grow_kernel(const Geo g, const float *__restrict__ vol, const unsigned char *__restrict__ marks,
                                                        unsigned char *__restrict__ states, const Heads H)
{
    const long long b = blockIdx.x * (long long)kWarpsPerCta + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    states = head_at(states, H.ws);
    marks = head_at(marks, H.ws);
    vol = head_vol(vol, H);
    if (b >= g.n_blocks || states[b] != kInactive) return;
    int bx, by, bz;
    unblock(g, b, bx, by, bz);
    const int x0 = blo(g, bx), y0 = blo(g, by), z0 = blo(g, bz);
    const int x1 = bhi(g, bx), y1 = bhi(g, by), z1 = bhi(g, bz);
    const int dx = x1 - x0 + 1, dy = y1 - y0 + 1, dz = z1 - z0 + 1;
    const bool s0 = side(__ldg(vol + vox(g, x0, y0, z0)));
    bool leaves = false;
    for (int i = lane; i < dx * dy * dz; i += 32) {
        const int z = z0 + i % dz, y = y0 + (i / dz) % dy, x = x0 + i / (dz * dy);
        if (x != x0 && x != x1 && y != y0 && y != y1 && z != z0 && z != z1) continue;     // interior voxels are never evaluated
        const long long v = vox(g, x, y, z);
        if (marks[v] == kDone && side(__ldg(vol + v)) != s0) leaves = true;
    }
    if (__any_sync(0xffffffffu, leaves) && lane == 0) states[b] = kActivated;
}

// every voxel not evaluated takes the value of corner 0 of a block containing it (all such blocks are inactive and on one side)
// (on a slab the corner lies on the slab's planes too: plane X1 < res - 1 takes corner 0 of block L1, which is on plane X1)
__global__ void fill_kernel(const Geo g, const unsigned char *__restrict__ marks, float *__restrict__ vol, const Heads H)
{
    marks = head_at(marks, H.ws);
    vol = head_vol(vol, H);
    for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < g.n_vox; v += (long long)gridDim.x * blockDim.x) {
        if (marks[v] == kDone) continue;
        const int x = g.X0 + (int)(v / g.rr), y = (int)((v / g.res) % g.res), z = (int)(v % g.res);
        const int cx = min(x / g.B, g.nb - 1) * g.B, cy = min(y / g.B, g.nb - 1) * g.B, cz = min(z / g.B, g.nb - 1) * g.B;
        vol[v] = vol[vox(g, cx, cy, cz)];
    }
}

// ---------------------------------------------------------------------------------------------- ordered compaction of the wanted voxels
__device__ __forceinline__ unsigned wanted_bytes(uint4 m, uint4 &eq)
{
    eq.x = __vcmpeq4(m.x, 0x01010101u); eq.y = __vcmpeq4(m.y, 0x01010101u);
    eq.z = __vcmpeq4(m.z, 0x01010101u); eq.w = __vcmpeq4(m.w, 0x01010101u);
    return (__popc(eq.x) + __popc(eq.y) + __popc(eq.z) + __popc(eq.w)) >> 3;
}

// exclusive scan over the CTA; returns the CTA total through `total`
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

__global__ void __launch_bounds__(kThreads) count_kernel(const unsigned char *__restrict__ marks, unsigned *__restrict__ chunk_cnt,
                                                         const Heads H)
{
    marks = head_at(marks, H.ws);
    chunk_cnt = head_at(chunk_cnt, H.ws);
    const uint4 m = __ldg(reinterpret_cast<const uint4 *>(marks + (size_t)blockIdx.x * kChunk) + threadIdx.x);
    uint4 eq;
    unsigned total;
    cta_exclusive_scan<kThreads>(wanted_bytes(m, eq), total);
    if (threadIdx.x == 0) chunk_cnt[blockIdx.x] = total;
}

// one CTA per head; {listed, active blocks} also go to pairs[2h..2h+1] (the S heads' counts, read back with one copy)
__global__ void __launch_bounds__(kScanThreads) scan_kernel(const unsigned *__restrict__ chunk_cnt, unsigned *__restrict__ chunk_off,
                                                            long long n_chunks, unsigned long long *__restrict__ hdr, const Heads H,
                                                            unsigned long long *pairs)      // a single band: pairs == hdr
{
    chunk_cnt = head_at(chunk_cnt, H.ws);
    chunk_off = head_at(chunk_off, H.ws);
    hdr = head_at(hdr, H.ws);
    const long long per = (n_chunks + kScanThreads - 1) / kScanThreads;
    const long long c0 = threadIdx.x * per, c1 = min(c0 + per, n_chunks);
    unsigned s = 0;
    for (long long c = c0; c < c1; ++c) s += chunk_cnt[c];
    unsigned total;
    unsigned run = cta_exclusive_scan<kScanThreads>(s, total);
    for (long long c = c0; c < c1; ++c) {
        chunk_off[c] = run;
        run += chunk_cnt[c];
    }
    if (threadIdx.x == 0) {
        hdr[0] = total;
        pairs[2 * blockIdx.y] = total;
        pairs[2 * blockIdx.y + 1] = hdr[1];
    }
}

__global__ void __launch_bounds__(kThreads) emit_kernel(unsigned char *__restrict__ marks, const unsigned *__restrict__ chunk_cnt,
                                                        const unsigned *__restrict__ chunk_off, unsigned *__restrict__ list,
                                                        const Heads H)
{
    marks = head_at(marks, H.ws);
    chunk_cnt = head_at(chunk_cnt, H.ws);
    chunk_off = head_at(chunk_off, H.ws);
    list = head_at(list, H.ws);
    if (chunk_cnt[blockIdx.x] == 0) return;
    uint4 *p = reinterpret_cast<uint4 *>(marks + (size_t)blockIdx.x * kChunk) + threadIdx.x;
    uint4 m = *p, eq;
    const unsigned c = wanted_bytes(m, eq);
    unsigned total;
    unsigned pos = chunk_off[blockIdx.x] + cta_exclusive_scan<kThreads>(c, total);
    if (c == 0) return;
    const unsigned v0 = blockIdx.x * (unsigned)kChunk + threadIdx.x * kPerThread;
    const unsigned e[4] = {eq.x, eq.y, eq.z, eq.w};
#pragma unroll
    for (int w = 0; w < 4; ++w)
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if ((e[w] >> (8 * j)) & 1u) list[pos++] = v0 + 4 * w + j;
    m.x += eq.x & 0x01010101u; m.y += eq.y & 0x01010101u; m.z += eq.z & 0x01010101u; m.w += eq.w & 0x01010101u;   // 1 -> 2
    *p = m;
}

// ---------------------------------------------------------------------------------------------- lists <-> grid
// rows of head h: xyz / values rows [h n, h n + n), its listed voxels first.  `pad`: the rows past its count repeat its last listed
// voxel (voxel 0 of the slab when it listed nothing), so that every row is a grid point of the head; else they are not written.
// axes: those of head 0's workspace (every head has the same grid).
__global__ void gather_kernel(const Geo g, const unsigned *__restrict__ list, const unsigned long long *__restrict__ hdr, long long n,
                              bool pad, const float *__restrict__ axes, float *__restrict__ xyz, const Heads H)
{
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= n) return;
    list = head_at(list, H.ws);
    const long long cnt = (long long)head_at(hdr, H.ws)[0];
    if (i >= cnt && !pad) return;
    const long long v = i < cnt ? list[i] : (cnt > 0 ? list[cnt - 1] : 0);
    float *out = xyz + 3 * (blockIdx.y * n + i);
    out[0] = __ldg(axes + g.X0 + v / g.rr);
    out[1] = __ldg(axes + g.res + (v / g.res) % g.res);
    out[2] = __ldg(axes + 2 * g.res + v % g.res);
}

__global__ void scatter_kernel(const unsigned *__restrict__ list, const unsigned long long *__restrict__ hdr, long long n,
                               const float *__restrict__ values, float *__restrict__ vol, const Heads H)
{
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= n || i >= (long long)head_at(hdr, H.ws)[0]) return;
    head_vol(vol, H)[head_at(list, H.ws)[i]] = values[blockIdx.y * n + i];
}

// ---------------------------------------------------------------------------------------------- boundary planes between slabs
// buffer of plane p: res^2 floats (the volume), then res^2 bytes (1: evaluated)
__global__ void export_kernel(const Geo g, int plane, const float *__restrict__ vol, const unsigned char *__restrict__ marks,
                              float *__restrict__ vals, unsigned char *__restrict__ done)
{
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= g.rr) return;
    const long long v = (plane - g.X0) * g.rr + i;
    vals[i] = vol[v];
    done[i] = marks[v] == kDone ? 1 : 0;
}

// a voxel the neighbour evaluated and this slab did not takes the neighbour's value and counts as evaluated
__global__ void import_kernel(const Geo g, int plane, const float *__restrict__ vals, const unsigned char *__restrict__ done,
                              float *__restrict__ vol, unsigned char *__restrict__ marks)
{
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= g.rr) return;
    const long long v = (plane - g.X0) * g.rr + i;
    if (done[i] && marks[v] != kDone) {
        marks[v] = kDone;
        vol[v] = vals[i];
    }
}

// ---------------------------------------------------------------------------------------------- host side
int check_args(int res, int block, int l0, int l1, const char *who)
{
    NPHM_REQUIRE(res >= 2 && res <= 1024, "%s: res %d outside [2, 1024]", who, res);
    NPHM_REQUIRE(block >= 1 && block <= 64, "%s: block %d outside [1, 64]", who, block);
    const int nb = blocks_per_axis(res, block);
    NPHM_REQUIRE(l0 >= 0 && l0 < l1 && l1 <= nb, "%s: block layers [%d, %d) not a non-empty range of [0, %d)", who, l0, l1, nb);
    return NPHM_OK;
}

int check_ws(const Geo &g, const void *ws, long long ws_bytes, const char *who)
{
    NPHM_REQUIRE(ws, "%s: NULL workspace", who);
    const long long need = layout(g).bytes;
    if (ws_bytes < need) {
        set_error("%s: band workspace too small: %lld bytes for res %d, block %d, block layers [%d, %d), %lld needed", who, ws_bytes,
                  g.res, g.B, g.L0, g.L1, need);
        return NPHM_ERR_CAPACITY;
    }
    return NPHM_OK;
}

// the slab's own planes in a caller volume that starts at plane X0 - ghost
inline float *own(const Geo &g, float *vol) { return vol + g.ghost * g.rr; }
inline const float *own(const Geo &g, const float *vol) { return vol + g.ghost * g.rr; }

// S bands of one slab: head 0's geometry and carved workspace, the strides to the others, and where the listing steps put the S
// {listed, active blocks} pairs (a single band: its own header)
struct Band {
    Geo g;
    Ws w;
    Heads H;
    int S;
    unsigned long long *pairs;
};

inline dim3 grid2(long long x, int S) { return dim3((unsigned)x, (unsigned)S); }

// wanted voxels -> ascending list (and kDone); counts_host (may be NULL: no read-back) = the S pairs {listed, active blocks}, read
// back with one copy and one synchronisation whatever S is
int compact(const Band &b, long long *counts_host, cudaStream_t stream)
{
    const Geo &g = b.g;
    const Ws &w = b.w;
    count_kernel<<<grid2(g.n_chunks, b.S), kThreads, 0, stream>>>(w.marks, w.chunk_cnt, b.H);
    NPHM_CUDA_CHECK(cudaGetLastError());
    scan_kernel<<<grid2(1, b.S), kScanThreads, 0, stream>>>(w.chunk_cnt, w.chunk_off, g.n_chunks, w.hdr, b.H, b.pairs);
    NPHM_CUDA_CHECK(cudaGetLastError());
    emit_kernel<<<grid2(g.n_chunks, b.S), kThreads, 0, stream>>>(w.marks, w.chunk_cnt, w.chunk_off, w.list, b.H);
    NPHM_CUDA_CHECK(cudaGetLastError());
    if (counts_host) {
        std::vector<unsigned long long> h(2 * (size_t)b.S);
        NPHM_CUDA_CHECK(cudaMemcpyAsync(h.data(), b.pairs, h.size() * sizeof(h[0]), cudaMemcpyDeviceToHost, stream));
        NPHM_CUDA_CHECK(cudaStreamSynchronize(stream));
        for (size_t i = 0; i < h.size(); ++i) counts_host[i] = (long long)h[i];
    }
    return NPHM_OK;
}

// activated blocks -> their voxels not evaluated yet are wanted -> compact
int mark_and_compact(const Band &b, long long *counts_host, cudaStream_t stream)
{
    mark_blocks_kernel<<<grid2(ceil_div(b.g.n_blocks, kWarpsPerCta), b.S), kThreads, 0, stream>>>(b.g, b.w.states, b.w.marks,
                                                                                                  b.w.hdr, b.H);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return compact(b, counts_host, stream);
}

// ---- the steps on a slab (the entry points below check the arguments)
int begin(const Band &b, long long quirk_period, long long *counts_host, cudaStream_t stream)
{
    const Geo &g = b.g;
    const Ws &w = b.w;
    const Layout l = layout(g);
    for (int h = 0; h < b.S; ++h) {              // one memset per head and region: a 2D memset's pitch is capped below 2^31 bytes
        char *ws = reinterpret_cast<char *>(w.hdr) + h * b.H.ws;
        NPHM_CUDA_CHECK(cudaMemsetAsync(ws + l.hdr, 0, 256, stream));
        NPHM_CUDA_CHECK(cudaMemsetAsync(ws + l.states, 0, g.n_blocks, stream));
        NPHM_CUDA_CHECK(cudaMemsetAsync(ws + l.marks, 0, l.list - l.marks, stream));
    }
    if (quirk_period > 0) {
        // the quirk voxels of global flat indices [X0 res^2, (X1 + 1) res^2): k0 = the first with (k + 1) p - 1 >= X0 res^2; the
        // last voxel of the grid (k = n_all / p when p does not divide n_all) only on the slab that holds it.  They depend only on
        // res and p, so every head lists the same ones, which the caller evaluates as S queries of period 1.
        const long long n_all = g.rr * g.res, g1 = (g.X1 + 1) * g.rr;
        const long long k0 = g.X0 * g.rr / quirk_period;
        const long long k1 = g1 == n_all ? ceil_div(n_all, quirk_period) : g1 / quirk_period;
        if (k1 > k0) {
            quirk_kernel<<<grid2(ceil_div(k1 - k0, kThreads), b.S), kThreads, 0, stream>>>(g, quirk_period, k0, k1, w.marks, w.states,
                                                                                           b.H);
            NPHM_CUDA_CHECK(cudaGetLastError());
        }
    }
    // compaction only: the forced blocks' other voxels are listed with the first band pass
    return compact(b, counts_host, stream);
}

int corners(const Band &b, long long *counts_host, cudaStream_t stream)
{
    const Geo &g = b.g;
    const long long n1 = g.nb + 1;
    corners_kernel<<<grid2(ceil_div((g.L1 - g.L0 + 1) * n1 * n1, kThreads), b.S), kThreads, 0, stream>>>(g, b.w.marks, b.H);
    NPHM_CUDA_CHECK(cudaGetLastError());
    // the forced blocks stay activated until classify marks them with the blocks it activates
    return compact(b, counts_host, stream);
}

// n: rows per head; pad: see gather_kernel
int gather(const Band &b, const double grid_min[3], const double grid_max[3], long long n, bool pad, float *xyz_dev,
           cudaStream_t stream)
{
    if (n == 0) return NPHM_OK;
    int rc = launch_grid_axes(grid_min, grid_max, b.g.res, b.w.axes, stream);
    if (rc) return rc;
    gather_kernel<<<grid2(ceil_div(n, kThreads), b.S), kThreads, 0, stream>>>(b.g, b.w.list, b.w.hdr, n, pad, b.w.axes, xyz_dev, b.H);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

int scatter(const Band &b, long long n, const float *values_dev, float *vol_dev, cudaStream_t stream)
{
    if (n == 0) return NPHM_OK;
    scatter_kernel<<<grid2(ceil_div(n, kThreads), b.S), kThreads, 0, stream>>>(b.w.list, b.w.hdr, n, values_dev, own(b.g, vol_dev),
                                                                               b.H);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

int classify(const Band &b, float tau, const float *vol_dev, long long *counts_host, cudaStream_t stream)
{
    classify_kernel<<<grid2(ceil_div(b.g.n_blocks, kThreads), b.S), kThreads, 0, stream>>>(b.g, tau, own(b.g, vol_dev), b.w.states,
                                                                                           b.H);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return mark_and_compact(b, counts_host, stream);
}

int grow(const Band &b, const float *vol_dev, long long *counts_host, cudaStream_t stream)
{
    grow_kernel<<<grid2(ceil_div(b.g.n_blocks, kWarpsPerCta), b.S), kThreads, 0, stream>>>(b.g, own(b.g, vol_dev), b.w.marks,
                                                                                           b.w.states, b.H);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return mark_and_compact(b, counts_host, stream);
}

int fill(const Band &b, float *vol_dev, cudaStream_t stream)
{
    const long long ctas = std::min(ceil_div(b.g.n_vox, kThreads), 64LL * sm_count());
    fill_kernel<<<grid2(ctas, b.S), kThreads, 0, stream>>>(b.g, b.w.marks, own(b.g, vol_dev), b.H);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

// states_dev: S x n_blocks bytes
int block_states(const Band &b, unsigned char *states_dev, cudaStream_t stream)
{
    for (int h = 0; h < b.S; ++h)
        NPHM_CUDA_CHECK(cudaMemcpyAsync(states_dev + h * b.g.n_blocks, b.w.states + h * b.H.ws, b.g.n_blocks, cudaMemcpyDeviceToDevice,
                                        stream));
    return NPHM_OK;
}

}  // namespace band
}  // namespace nphm

using namespace nphm;

#define SLAB_PROLOGUE(who)                                                  \
    int rc = band::check_args(res, block, l0, l1, who);                     \
    if (rc) return rc;                                                      \
    const band::Geo g = band::make_geo(res, block, l0, l1);                 \
    if ((rc = band::check_ws(g, ws, ws_bytes, who))) return rc;             \
    const band::Ws w = band::carve(const_cast<void *>(static_cast<const void *>(ws)), band::layout(g)); \
    const band::Band b{g, w, band::Heads{band::layout(g).bytes, 0}, 1, w.hdr}; \
    (void)b;                                                                \
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);

// ---------------------------------------------------------------------------------------------- entry points
extern "C" long long nphm_band_slab_workspace_bytes(int res, int block, int l0, int l1)
{
    if (band::check_args(res, block, l0, l1, "nphm_band_slab_workspace_bytes")) return -1;
    return band::layout(band::make_geo(res, block, l0, l1)).bytes;
}

extern "C" int nphm_band_slab_begin(int res, int block, int l0, int l1, long long quirk_period, void *ws, long long ws_bytes,
                                    long long *counts_host, void *stream_)
{
    SLAB_PROLOGUE("nphm_band_slab_begin")
    NPHM_REQUIRE(quirk_period >= 0, "nphm_band_slab_begin: negative quirk period %lld", quirk_period);
    return band::begin(b, quirk_period, counts_host, stream);
}

extern "C" int nphm_band_slab_corners(int res, int block, int l0, int l1, void *ws, long long ws_bytes, long long *counts_host,
                                      void *stream_)
{
    SLAB_PROLOGUE("nphm_band_slab_corners")
    return band::corners(b, counts_host, stream);
}

extern "C" int nphm_band_slab_gather(int res, int block, int l0, int l1, const double grid_min[3], const double grid_max[3],
                                     long long n, float *xyz_dev, void *ws, long long ws_bytes, void *stream_)
{
    SLAB_PROLOGUE("nphm_band_slab_gather")
    NPHM_REQUIRE(grid_min && grid_max && n >= 0 && n <= g.n_vox && (n == 0 || xyz_dev), "nphm_band_slab_gather: bad arguments");
    return band::gather(b, grid_min, grid_max, n, false, xyz_dev, stream);
}

extern "C" int nphm_band_slab_scatter(int res, int block, int l0, int l1, long long n, const float *values_dev, float *vol_dev,
                                      void *ws, long long ws_bytes, void *stream_)
{
    SLAB_PROLOGUE("nphm_band_slab_scatter")
    NPHM_REQUIRE(n >= 0 && n <= g.n_vox && vol_dev && (n == 0 || values_dev), "nphm_band_slab_scatter: bad arguments");
    return band::scatter(b, n, values_dev, vol_dev, stream);
}

extern "C" int nphm_band_slab_classify(int res, int block, int l0, int l1, float tau, const float *vol_dev, void *ws,
                                       long long ws_bytes, long long *counts_host, void *stream_)
{
    SLAB_PROLOGUE("nphm_band_slab_classify")
    NPHM_REQUIRE(tau >= 0.f && vol_dev, "nphm_band_slab_classify: need tau >= 0 (got %g) and a volume", (double)tau);
    return band::classify(b, tau, vol_dev, counts_host, stream);
}

extern "C" int nphm_band_slab_grow(int res, int block, int l0, int l1, const float *vol_dev, void *ws, long long ws_bytes,
                                   long long *counts_host, void *stream_)
{
    SLAB_PROLOGUE("nphm_band_slab_grow")
    NPHM_REQUIRE(vol_dev, "nphm_band_slab_grow: NULL volume");
    return band::grow(b, vol_dev, counts_host, stream);
}

extern "C" int nphm_band_slab_fill(int res, int block, int l0, int l1, float *vol_dev, void *ws, long long ws_bytes, void *stream_)
{
    SLAB_PROLOGUE("nphm_band_slab_fill")
    NPHM_REQUIRE(vol_dev, "nphm_band_slab_fill: NULL volume");
    return band::fill(b, vol_dev, stream);
}

extern "C" int nphm_band_slab_block_states(int res, int block, int l0, int l1, const void *ws, long long ws_bytes,
                                           unsigned char *states_dev, void *stream_)
{
    SLAB_PROLOGUE("nphm_band_slab_block_states")
    NPHM_REQUIRE(states_dev, "nphm_band_slab_block_states: NULL output");
    return band::block_states(b, states_dev, stream);
}

extern "C" int nphm_band_slab_export(int res, int block, int l0, int l1, int plane, const float *vol_dev, const void *ws,
                                     long long ws_bytes, unsigned char *buf_dev, void *stream_)
{
    SLAB_PROLOGUE("nphm_band_slab_export")
    NPHM_REQUIRE(vol_dev && buf_dev, "nphm_band_slab_export: NULL volume or buffer");
    NPHM_REQUIRE(plane >= g.X0 && plane <= g.X1, "nphm_band_slab_export: plane %d outside the slab's planes [%d, %d]", plane, g.X0,
                 g.X1);
    float *vals = reinterpret_cast<float *>(buf_dev);
    band::export_kernel<<<(unsigned)ceil_div(g.rr, band::kThreads), band::kThreads, 0, stream>>>(
        g, plane, band::own(g, vol_dev), w.marks, vals, buf_dev + 4 * g.rr);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

extern "C" int nphm_band_slab_import(int res, int block, int l0, int l1, int plane, const unsigned char *buf_dev, float *vol_dev,
                                     void *ws, long long ws_bytes, void *stream_)
{
    SLAB_PROLOGUE("nphm_band_slab_import")
    NPHM_REQUIRE(vol_dev && buf_dev, "nphm_band_slab_import: NULL volume or buffer");
    const bool lower = plane == g.X0 && g.L0 > 0, upper = plane == g.X1 && g.X1 < g.C, ghost = plane == g.X0 - 1 && g.ghost;
    NPHM_REQUIRE(lower || upper || ghost,
                 "nphm_band_slab_import: plane %d is neither a plane shared with a neighbour nor the ghost plane of the slab of "
                 "block layers [%d, %d) (planes [%d, %d] of %d)", plane, l0, l1, g.X0, g.X1, g.res);
    const float *vals = reinterpret_cast<const float *>(buf_dev);
    if (ghost) {
        NPHM_CUDA_CHECK(cudaMemcpyAsync(vol_dev, vals, g.rr * sizeof(float), cudaMemcpyDeviceToDevice, stream));
        return NPHM_OK;
    }
    band::import_kernel<<<(unsigned)ceil_div(g.rr, band::kThreads), band::kThreads, 0, stream>>>(
        g, plane, vals, buf_dev + 4 * g.rr, band::own(g, vol_dev), w.marks);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

// ---------------------------------------------------------------------------------------------- S heads of one whole grid
namespace nphm {
namespace band {

// workspace of S heads: the S {listed, active blocks} pairs, then S band workspaces of the whole grid at a stride of their bytes
inline long long pairs_bytes(int S) { return (16LL * S + 255) / 256 * 256; }
inline long long heads_bytes(const Geo &g, int S) { return pairs_bytes(S) + S * layout(g).bytes; }

int check_heads(int res, int block, int S, const char *who)
{
    int rc = check_args(res, block, 0, 1, who);
    if (rc) return rc;
    NPHM_REQUIRE(S >= 1 && S <= 65535, "%s: %d heads outside [1, 65535]", who, S);
    return NPHM_OK;
}

}  // namespace band
}  // namespace nphm

#define HEADS_PROLOGUE(who)                                                                                   \
    int rc = band::check_heads(res, block, n_heads, who);                                                     \
    if (rc) return rc;                                                                                        \
    const band::Geo g = band::make_geo(res, block, 0, band::blocks_per_axis(res, block));                     \
    NPHM_REQUIRE(ws, "%s: NULL workspace", who);                                                              \
    if (ws_bytes < band::heads_bytes(g, n_heads)) {                                                           \
        set_error("%s: band workspace too small: %lld bytes for %d heads of res %d, block %d, %lld needed", who, ws_bytes, n_heads, \
                  res, block, band::heads_bytes(g, n_heads));                                                 \
        return NPHM_ERR_CAPACITY;                                                                             \
    }                                                                                                         \
    char *ws0 = static_cast<char *>(const_cast<void *>(static_cast<const void *>(ws)));                       \
    const band::Band b{g, band::carve(ws0 + band::pairs_bytes(n_heads), band::layout(g)),                     \
                       band::Heads{band::layout(g).bytes, g.n_vox}, n_heads, reinterpret_cast<unsigned long long *>(ws0)}; \
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);

extern "C" long long nphm_band_heads_workspace_bytes(int res, int block, int n_heads)
{
    if (band::check_heads(res, block, n_heads, "nphm_band_heads_workspace_bytes")) return -1;
    return band::heads_bytes(band::make_geo(res, block, 0, band::blocks_per_axis(res, block)), n_heads);
}

extern "C" int nphm_band_heads_begin(int res, int block, int n_heads, long long quirk_period, void *ws, long long ws_bytes,
                                     long long *counts_host, void *stream_)
{
    HEADS_PROLOGUE("nphm_band_heads_begin")
    NPHM_REQUIRE(quirk_period >= 0, "nphm_band_heads_begin: negative quirk period %lld", quirk_period);
    return band::begin(b, quirk_period, counts_host, stream);
}

extern "C" int nphm_band_heads_corners(int res, int block, int n_heads, void *ws, long long ws_bytes, long long *counts_host,
                                       void *stream_)
{
    HEADS_PROLOGUE("nphm_band_heads_corners")
    return band::corners(b, counts_host, stream);
}

extern "C" int nphm_band_heads_classify(int res, int block, int n_heads, float tau, const float *vols_dev, void *ws, long long ws_bytes,
                                        long long *counts_host, void *stream_)
{
    HEADS_PROLOGUE("nphm_band_heads_classify")
    NPHM_REQUIRE(tau >= 0.f && vols_dev, "nphm_band_heads_classify: need tau >= 0 (got %g) and volumes", (double)tau);
    return band::classify(b, tau, vols_dev, counts_host, stream);
}

extern "C" int nphm_band_heads_grow(int res, int block, int n_heads, const float *vols_dev, void *ws, long long ws_bytes,
                                    long long *counts_host, void *stream_)
{
    HEADS_PROLOGUE("nphm_band_heads_grow")
    NPHM_REQUIRE(vols_dev, "nphm_band_heads_grow: NULL volumes");
    return band::grow(b, vols_dev, counts_host, stream);
}

extern "C" int nphm_band_heads_gather(int res, int block, int n_heads, const double grid_min[3], const double grid_max[3],
                                      long long n_pad, float *xyz_dev, void *ws, long long ws_bytes, void *stream_)
{
    HEADS_PROLOGUE("nphm_band_heads_gather")
    NPHM_REQUIRE(grid_min && grid_max && n_pad >= 0 && n_pad <= g.n_vox && (n_pad == 0 || xyz_dev),
                 "nphm_band_heads_gather: bad arguments");
    return band::gather(b, grid_min, grid_max, n_pad, true, xyz_dev, stream);
}

extern "C" int nphm_band_heads_scatter(int res, int block, int n_heads, long long n_pad, const float *values_dev, float *vols_dev,
                                       void *ws, long long ws_bytes, void *stream_)
{
    HEADS_PROLOGUE("nphm_band_heads_scatter")
    NPHM_REQUIRE(n_pad >= 0 && n_pad <= g.n_vox && vols_dev && (n_pad == 0 || values_dev), "nphm_band_heads_scatter: bad arguments");
    return band::scatter(b, n_pad, values_dev, vols_dev, stream);
}

extern "C" int nphm_band_heads_fill(int res, int block, int n_heads, float *vols_dev, void *ws, long long ws_bytes, void *stream_)
{
    HEADS_PROLOGUE("nphm_band_heads_fill")
    NPHM_REQUIRE(vols_dev, "nphm_band_heads_fill: NULL volumes");
    return band::fill(b, vols_dev, stream);
}

extern "C" int nphm_band_heads_block_states(int res, int block, int n_heads, const void *ws, long long ws_bytes,
                                            unsigned char *states_dev, void *stream_)
{
    HEADS_PROLOGUE("nphm_band_heads_block_states")
    NPHM_REQUIRE(states_dev, "nphm_band_heads_block_states: NULL output");
    return band::block_states(b, states_dev, stream);
}
