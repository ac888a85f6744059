// Narrow-band mesh extraction on sm_90a: the steps that decide WHICH voxels of a res^3 grid the decoder has to evaluate so that
// marching cubes on the filled volume gives the dense mesh, and that move values between the grid and compact point lists.
// The decoder itself runs through the existing query entry points on the gathered coordinates (see DESIGN §4.13).
//
// The grid's (res - 1)^3 cells are split into blocks of B^3 cells (the last block of an axis may be partial); block b covers the
// voxels [bB, min(bB + B, res - 1)] of each axis, so neighbouring blocks share a face of voxels.  State lives in a caller-owned
// workspace:
//   marks   1 byte per voxel: 0 not evaluated, 1 wanted (set by a marking kernel), 2 listed / evaluated
//   states  1 byte per block: 0 inactive, 1 activated (its voxels not yet marked), 2 active (marked)
//   list    u32 flat voxel indices of the last compaction, ascending
// Marching cubes runs on -sdf at 0, so a voxel is "inside" when -v <= 0, i.e. v >= 0 (NaN: outside) - `side()` below.
#include "common.cuh"
#include "simt.cuh"
#include <algorithm>

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
    long long n_vox, n_blocks, n_chunks;
};

struct Layout {
    long long hdr, axes, states, chunk_cnt, chunk_off, marks, list, bytes;
};

inline Geo make_geo(int res, int block)
{
    Geo g;
    g.res = res; g.B = block; g.C = res - 1;
    g.nb = (int)ceil_div(g.C, block);
    g.n_vox = (long long)res * res * res;
    g.n_blocks = (long long)g.nb * g.nb * g.nb;
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

__device__ __forceinline__ long long vox(const Geo &g, int x, int y, int z)
{
    return ((long long)x * g.res + y) * g.res + z;
}

// voxel box of block b along one axis
__device__ __forceinline__ int blo(const Geo &g, int b) { return b * g.B; }
__device__ __forceinline__ int bhi(const Geo &g, int b) { return min(b * g.B + g.B, g.C); }

__device__ __forceinline__ void unblock(const Geo &g, long long b, int &bx, int &by, int &bz)
{
    bz = (int)(b % g.nb);
    const long long t = b / g.nb;
    by = (int)(t % g.nb);
    bx = (int)(t / g.nb);
}

// ---------------------------------------------------------------------------------------------- marking
// eval-mode quirk voxels g = (k + 1) p - 1 and g = res^3 - 1: wanted, and every block owning a cell that touches one is forced
__global__ void quirk_kernel(const Geo g, long long period, long long n_quirk, unsigned char *__restrict__ marks,
                             unsigned char *__restrict__ states)
{
    const long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (k >= n_quirk) return;
    const long long v = k < g.n_vox / period ? (k + 1) * period - 1 : g.n_vox - 1;
    const long long rr = (long long)g.res * g.res;
    const int x = (int)(v / rr), y = (int)((v / g.res) % g.res), z = (int)(v % g.res);
    marks[v] = kWanted;
    // cells touching voxel x along an axis: [max(x - 1, 0), min(x, C - 1)]
    const int bx0 = max(x - 1, 0) / g.B, bx1 = min(x, g.C - 1) / g.B;
    const int by0 = max(y - 1, 0) / g.B, by1 = min(y, g.C - 1) / g.B;
    const int bz0 = max(z - 1, 0) / g.B, bz1 = min(z, g.C - 1) / g.B;
    for (int bx = bx0; bx <= bx1; ++bx)
        for (int by = by0; by <= by1; ++by)
            for (int bz = bz0; bz <= bz1; ++bz) states[((long long)bx * g.nb + by) * g.nb + bz] = kActivated;
}

// block corners (fine indices 0, B, 2B, ..., res - 1 on every axis)
__global__ void corners_kernel(const Geo g, unsigned char *__restrict__ marks)
{
    const long long n1 = g.nb + 1;
    const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (t >= n1 * n1 * n1) return;
    const int cz = (int)(t % n1), cy = (int)((t / n1) % n1), cx = (int)(t / (n1 * n1));
    const long long v = vox(g, min(cx * g.B, g.C), min(cy * g.B, g.C), min(cz * g.B, g.C));
    if (marks[v] == kIdle) marks[v] = kWanted;
}

// an inactive block becomes active when a corner has |sdf| <= tau (or is NaN) or its corners lie on both sides of the test
__global__ void classify_kernel(const Geo g, float tau, const float *__restrict__ vol, unsigned char *__restrict__ states)
{
    const long long b = blockIdx.x * (long long)blockDim.x + threadIdx.x;
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
                                                               unsigned char *__restrict__ marks, unsigned long long *__restrict__ hdr)
{
    const long long b = blockIdx.x * (long long)kWarpsPerCta + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
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
                                                        unsigned char *__restrict__ states)
{
    const long long b = blockIdx.x * (long long)kWarpsPerCta + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
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
__global__ void fill_kernel(const Geo g, const unsigned char *__restrict__ marks, float *__restrict__ vol)
{
    const long long rr = (long long)g.res * g.res;
    for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < g.n_vox; v += (long long)gridDim.x * blockDim.x) {
        if (marks[v] == kDone) continue;
        const int x = (int)(v / rr), y = (int)((v / g.res) % g.res), z = (int)(v % g.res);
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

__global__ void __launch_bounds__(kThreads) count_kernel(const unsigned char *__restrict__ marks, unsigned *__restrict__ chunk_cnt)
{
    const uint4 m = __ldg(reinterpret_cast<const uint4 *>(marks + (size_t)blockIdx.x * kChunk) + threadIdx.x);
    uint4 eq;
    unsigned total;
    cta_exclusive_scan<kThreads>(wanted_bytes(m, eq), total);
    if (threadIdx.x == 0) chunk_cnt[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kScanThreads) scan_kernel(const unsigned *__restrict__ chunk_cnt, unsigned *__restrict__ chunk_off,
                                                            long long n_chunks, unsigned long long *__restrict__ hdr)
{
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
    if (threadIdx.x == 0) hdr[0] = total;
}

__global__ void __launch_bounds__(kThreads) emit_kernel(unsigned char *__restrict__ marks, const unsigned *__restrict__ chunk_cnt,
                                                        const unsigned *__restrict__ chunk_off, unsigned *__restrict__ list)
{
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
__global__ void gather_kernel(const Geo g, const unsigned *__restrict__ list, const unsigned long long *__restrict__ hdr, long long n,
                              const float *__restrict__ axes, float *__restrict__ xyz)
{
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= n || i >= (long long)hdr[0]) return;
    const long long v = list[i], rr = (long long)g.res * g.res;
    xyz[3 * i] = __ldg(axes + v / rr);
    xyz[3 * i + 1] = __ldg(axes + g.res + (v / g.res) % g.res);
    xyz[3 * i + 2] = __ldg(axes + 2 * g.res + v % g.res);
}

__global__ void scatter_kernel(const unsigned *__restrict__ list, const unsigned long long *__restrict__ hdr, long long n,
                               const float *__restrict__ values, float *__restrict__ vol)
{
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= n || i >= (long long)hdr[0]) return;
    vol[list[i]] = values[i];
}

// ---------------------------------------------------------------------------------------------- host side
int check_args(int res, int block, const char *who)
{
    NPHM_REQUIRE(res >= 2 && res <= 1024, "%s: res %d outside [2, 1024]", who, res);
    NPHM_REQUIRE(block >= 1 && block <= 64, "%s: block %d outside [1, 64]", who, block);
    return NPHM_OK;
}

int check_ws(const Geo &g, const void *ws, long long ws_bytes, const char *who)
{
    NPHM_REQUIRE(ws, "%s: NULL workspace", who);
    const long long need = layout(g).bytes;
    if (ws_bytes < need) {
        set_error("%s: band workspace too small: %lld bytes for res %d, block %d, %lld needed", who, ws_bytes, g.res, g.B, need);
        return NPHM_ERR_CAPACITY;
    }
    return NPHM_OK;
}

// wanted voxels -> ascending list (and kDone); counts_host (may be NULL: no read-back) = {listed, active blocks}
int compact(const Geo &g, const Ws &w, long long *counts_host, cudaStream_t stream)
{
    count_kernel<<<(unsigned)g.n_chunks, kThreads, 0, stream>>>(w.marks, w.chunk_cnt);
    NPHM_CUDA_CHECK(cudaGetLastError());
    scan_kernel<<<1, kScanThreads, 0, stream>>>(w.chunk_cnt, w.chunk_off, g.n_chunks, w.hdr);
    NPHM_CUDA_CHECK(cudaGetLastError());
    emit_kernel<<<(unsigned)g.n_chunks, kThreads, 0, stream>>>(w.marks, w.chunk_cnt, w.chunk_off, w.list);
    NPHM_CUDA_CHECK(cudaGetLastError());
    if (counts_host) {
        unsigned long long h[2];
        NPHM_CUDA_CHECK(cudaMemcpyAsync(h, w.hdr, sizeof(h), cudaMemcpyDeviceToHost, stream));
        NPHM_CUDA_CHECK(cudaStreamSynchronize(stream));
        counts_host[0] = (long long)h[0];
        counts_host[1] = (long long)h[1];
    }
    return NPHM_OK;
}

// activated blocks -> their voxels not evaluated yet are wanted -> compact
int mark_and_compact(const Geo &g, const Ws &w, long long *counts_host, cudaStream_t stream)
{
    mark_blocks_kernel<<<(unsigned)ceil_div(g.n_blocks, kWarpsPerCta), kThreads, 0, stream>>>(g, w.states, w.marks, w.hdr);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return compact(g, w, counts_host, stream);
}

}  // namespace band
}  // namespace nphm

using namespace nphm;

#define BAND_PROLOGUE(who)                                                  \
    int rc = band::check_args(res, block, who);                            \
    if (rc) return rc;                                                      \
    const band::Geo g = band::make_geo(res, block);                         \
    if ((rc = band::check_ws(g, ws, ws_bytes, who))) return rc;             \
    const band::Ws w = band::carve(ws, band::layout(g));                    \
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);

extern "C" long long nphm_band_workspace_bytes(int res, int block)
{
    if (band::check_args(res, block, "nphm_band_workspace_bytes")) return -1;
    return band::layout(band::make_geo(res, block)).bytes;
}

extern "C" int nphm_band_begin(int res, int block, long long quirk_period, void *ws, long long ws_bytes, long long *counts_host,
                               void *stream_)
{
    BAND_PROLOGUE("nphm_band_begin")
    NPHM_REQUIRE(quirk_period >= 0, "nphm_band_begin: negative quirk period %lld", quirk_period);
    const band::Layout l = band::layout(g);
    NPHM_CUDA_CHECK(cudaMemsetAsync(w.hdr, 0, 256, stream));
    NPHM_CUDA_CHECK(cudaMemsetAsync(w.states, 0, g.n_blocks, stream));
    NPHM_CUDA_CHECK(cudaMemsetAsync(w.marks, 0, l.list - l.marks, stream));
    if (quirk_period > 0) {
        const long long n_quirk = ceil_div(g.n_vox, quirk_period);
        band::quirk_kernel<<<(unsigned)ceil_div(n_quirk, band::kThreads), band::kThreads, 0, stream>>>(g, quirk_period, n_quirk, w.marks,
                                                                                                      w.states);
        NPHM_CUDA_CHECK(cudaGetLastError());
    }
    // compaction only: the forced blocks' other voxels are listed with the first band pass
    return band::compact(g, w, counts_host, stream);
}

extern "C" int nphm_band_corners(int res, int block, void *ws, long long ws_bytes, long long *counts_host, void *stream_)
{
    BAND_PROLOGUE("nphm_band_corners")
    const long long n1 = g.nb + 1;
    band::corners_kernel<<<(unsigned)ceil_div(n1 * n1 * n1, band::kThreads), band::kThreads, 0, stream>>>(g, w.marks);
    NPHM_CUDA_CHECK(cudaGetLastError());
    // the forced blocks stay activated until nphm_band_classify marks them with the blocks it activates
    return band::compact(g, w, counts_host, stream);
}

extern "C" int nphm_band_gather(int res, int block, const double grid_min[3], const double grid_max[3], long long n, float *xyz_dev,
                                void *ws, long long ws_bytes, void *stream_)
{
    BAND_PROLOGUE("nphm_band_gather")
    NPHM_REQUIRE(grid_min && grid_max && n >= 0 && n <= g.n_vox && (n == 0 || xyz_dev), "nphm_band_gather: bad arguments");
    if (n == 0) return NPHM_OK;
    if ((rc = launch_grid_axes(grid_min, grid_max, res, w.axes, stream))) return rc;
    band::gather_kernel<<<(unsigned)ceil_div(n, band::kThreads), band::kThreads, 0, stream>>>(g, w.list, w.hdr, n, w.axes, xyz_dev);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

extern "C" int nphm_band_scatter(int res, int block, long long n, const float *values_dev, float *vol_dev, void *ws, long long ws_bytes,
                                 void *stream_)
{
    BAND_PROLOGUE("nphm_band_scatter")
    NPHM_REQUIRE(n >= 0 && n <= g.n_vox && vol_dev && (n == 0 || values_dev), "nphm_band_scatter: bad arguments");
    if (n == 0) return NPHM_OK;
    band::scatter_kernel<<<(unsigned)ceil_div(n, band::kThreads), band::kThreads, 0, stream>>>(w.list, w.hdr, n, values_dev, vol_dev);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

extern "C" int nphm_band_classify(int res, int block, float tau, const float *vol_dev, void *ws, long long ws_bytes,
                                  long long *counts_host, void *stream_)
{
    BAND_PROLOGUE("nphm_band_classify")
    NPHM_REQUIRE(tau >= 0.f && vol_dev, "nphm_band_classify: need tau >= 0 (got %g) and a volume", (double)tau);
    band::classify_kernel<<<(unsigned)ceil_div(g.n_blocks, band::kThreads), band::kThreads, 0, stream>>>(g, tau, vol_dev, w.states);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return band::mark_and_compact(g, w, counts_host, stream);
}

extern "C" int nphm_band_grow(int res, int block, const float *vol_dev, void *ws, long long ws_bytes, long long *counts_host,
                              void *stream_)
{
    BAND_PROLOGUE("nphm_band_grow")
    NPHM_REQUIRE(vol_dev, "nphm_band_grow: NULL volume");
    band::grow_kernel<<<(unsigned)ceil_div(g.n_blocks, band::kWarpsPerCta), band::kThreads, 0, stream>>>(g, vol_dev, w.marks, w.states);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return band::mark_and_compact(g, w, counts_host, stream);
}

extern "C" int nphm_band_fill(int res, int block, float *vol_dev, void *ws, long long ws_bytes, void *stream_)
{
    BAND_PROLOGUE("nphm_band_fill")
    NPHM_REQUIRE(vol_dev, "nphm_band_fill: NULL volume");
    const long long ctas = std::min(ceil_div(g.n_vox, band::kThreads), 64LL * sm_count());
    band::fill_kernel<<<(unsigned)ctas, band::kThreads, 0, stream>>>(g, w.marks, vol_dev);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

extern "C" int nphm_band_block_states(int res, int block, const void *ws, long long ws_bytes, unsigned char *states_dev, void *stream_)
{
    int rc = band::check_args(res, block, "nphm_band_block_states");
    if (rc) return rc;
    const band::Geo g = band::make_geo(res, block);
    if ((rc = band::check_ws(g, ws, ws_bytes, "nphm_band_block_states"))) return rc;
    NPHM_REQUIRE(states_dev, "nphm_band_block_states: NULL output");
    const band::Layout l = band::layout(g);
    NPHM_CUDA_CHECK(cudaMemcpyAsync(states_dev, static_cast<const char *>(ws) + l.states, g.n_blocks, cudaMemcpyDeviceToDevice,
                                    static_cast<cudaStream_t>(stream_)));
    return NPHM_OK;
}
