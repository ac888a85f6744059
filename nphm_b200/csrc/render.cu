// Multi-view depth / face-normal rasterizer for triangle meshes: the images pyrender hands to the reference's `render_glcam`
// (src/NPHM/evaluation/render_utils.py:26-89), which `gen_render_samples` (:169-201) back-projects into the point clouds of the
// evaluation protocol (scripts/evaluation/eval.py:30-96) and generate_single_view_observations.py into fitting inputs.
//
// One call rasterizes one mesh into V views.  Conventions (DESIGN.md §4.12):
//  * pixel (row r, column c) samples the eye-space ray ((c + 0.5 - cx)/fx, (cy - r - 0.5)/fy, -1); row 0 is the top row;
//  * a triangle covers the pixel when that ray passes through it (the ray's direction lies in the cone the three eye-space
//    vertices span, so triangles with vertices behind the eye are exact); the edge test is inclusive, and every edge is
//    evaluated with its endpoints in vertex-index order and then negated as needed, so two triangles sharing an edge get
//    bit-identical values (no pixel centre falls between the triangles of a closed mesh); zero-area triangles cover nothing;
//  * depth is the eye depth -z_eye, kept when znear <= d <= zfar; the nearest fragment wins, ties go to the lower triangle index
//    (GL_LESS in draw order); no face culling;
//  * normal: the world-space face normal cross(v1 - v0, v2 - v0) in fp64, normalised, rounded to fp32, stored as
//    round(clamp(0.5 n + 0.5, 0, 1) * 255) (shaders/mesh.frag into an RGBA8 target), never flipped toward the camera.
//
// Z-buffer: one 64-bit word per pixel, atomicMin of (float bits of the depth << 32 | triangle index) - the depth is positive,
// so the bit pattern orders like the value, and the result does not depend on the order fragments arrive in.  A resolve pass
// then writes depth, normal and triangle index.  A (triangle, view) thread rasterizes its own screen box when the box holds at
// most kSmallBox pixels; a larger box is cut into kTile x kTile tiles that go to a list, and one CTA takes each tile, so a
// full-viewport triangle spreads over (H/32)(W/32) CTAs.  Should the list fill up (it holds 16 tiles per image tile of every
// view, plus 65536: 16 full-viewport triangles per view), the thread rasterizes its remaining tiles itself: slower, same result.
#include "common.cuh"

namespace nphm {
namespace render {

constexpr int kThreads = 256;
constexpr int kTile = 32;
constexpr int kTilePixelsPerThread = kTile * kTile / kThreads;
constexpr long long kSmallBox = 1024;
constexpr unsigned long long kEmpty = ~0ull;

struct Setup {
    double3 e[3];      // edge normals P_a x P_b of the edges (v0 v1), (v1 v2), (v2 v0), in index order, then signed
    double det;        // P0 . (P1 x P2): its sign is the side every edge value must have, det / sum(edge values) the depth
    int r0, r1, c0, c1;
    bool live;
};

struct ViewArgs {
    const double *w2e;    // V x 12: world-to-eye rows
    const double *intr;   // V x 4: fx fy cx cy
    int height, width;
    double znear, zfar;
};

__device__ __forceinline__ double3 eye_point(const double *m, const float *__restrict__ verts, int i)
{
    const double x = verts[3 * (long long)i], y = verts[3 * (long long)i + 1], z = verts[3 * (long long)i + 2];
    return make_double3(fma(m[0], x, fma(m[1], y, fma(m[2], z, m[3]))), fma(m[4], x, fma(m[5], y, fma(m[6], z, m[7]))),
                        fma(m[8], x, fma(m[9], y, fma(m[10], z, m[11]))));
}

// no contraction: P_b x P_a must be the exact negation of P_a x P_b
__device__ __forceinline__ double3 cross_rn(double3 a, double3 b)
{
    return make_double3(__dsub_rn(__dmul_rn(a.y, b.z), __dmul_rn(a.z, b.y)), __dsub_rn(__dmul_rn(a.z, b.x), __dmul_rn(a.x, b.z)),
                        __dsub_rn(__dmul_rn(a.x, b.y), __dmul_rn(a.y, b.x)));
}

__device__ __forceinline__ double3 edge_normal(double3 pa, int ia, double3 pb, int ib)
{
    if (ia < ib) return cross_rn(pa, pb);
    const double3 n = cross_rn(pb, pa);
    return make_double3(-n.x, -n.y, -n.z);
}

__device__ __forceinline__ double3 face_normal(const float *__restrict__ verts, int3 f)
{
    const double ax = verts[3 * (long long)f.x], ay = verts[3 * (long long)f.x + 1], az = verts[3 * (long long)f.x + 2];
    const double ux = verts[3 * (long long)f.y] - ax, uy = verts[3 * (long long)f.y + 1] - ay, uz = verts[3 * (long long)f.y + 2] - az;
    const double vx = verts[3 * (long long)f.z] - ax, vy = verts[3 * (long long)f.z + 1] - ay, vz = verts[3 * (long long)f.z + 2] - az;
    // differences and products of fp32 values are exact in fp64: a single rounding per component, contracted or not
    return make_double3(uy * vz - uz * vy, uz * vx - ux * vz, ux * vy - uy * vx);
}

__device__ __forceinline__ int clamp_floor(double x, int hi) { return x <= 0.0 ? 0 : (x >= (double)hi ? hi : (int)floor(x)); }
__device__ __forceinline__ int clamp_ceil(double x, int hi) { return x <= 0.0 ? 0 : (x >= (double)hi ? hi : (int)ceil(x)); }

__device__ Setup setup(const float *__restrict__ verts, const int *__restrict__ faces, int t, int v, const ViewArgs &a)
{
    Setup s;
    s.live = false;
    const int3 f = make_int3(faces[3 * (long long)t], faces[3 * (long long)t + 1], faces[3 * (long long)t + 2]);
    const double3 wn = face_normal(verts, f);
    if (wn.x == 0.0 && wn.y == 0.0 && wn.z == 0.0) return s;                  // zero area
    const double *m = a.w2e + 12 * (long long)v;
    const double3 p0 = eye_point(m, verts, f.x), p1 = eye_point(m, verts, f.y), p2 = eye_point(m, verts, f.z);
    const double d0 = -p0.z, d1 = -p1.z, d2 = -p2.z;
    if ((d0 < a.znear && d1 < a.znear && d2 < a.znear) || (d0 > a.zfar && d1 > a.zfar && d2 > a.zfar)) return s;
    s.e[0] = edge_normal(p0, f.x, p1, f.y);
    s.e[1] = edge_normal(p1, f.y, p2, f.z);
    s.e[2] = edge_normal(p2, f.z, p0, f.x);
    const double3 c12 = cross_rn(p1, p2);
    s.det = p0.x * c12.x + p0.y * c12.y + p0.z * c12.z;
    if (s.det == 0.0) return s;                                              // edge-on: the plane passes through the eye
    s.r0 = 0; s.r1 = a.height - 1; s.c0 = 0; s.c1 = a.width - 1;
    if (d0 >= a.znear && d1 >= a.znear && d2 >= a.znear) {                   // else: clipped by the near plane, whole viewport
        const double *k = a.intr + 4 * (long long)v;
        const double fx = k[0], fy = k[1], cx = k[2], cy = k[3];
        const double ca = fx * p0.x / d0 + cx - 0.5, cb = fx * p1.x / d1 + cx - 0.5, cc = fx * p2.x / d2 + cx - 0.5;
        const double ra = cy - fy * p0.y / d0 - 0.5, rb = cy - fy * p1.y / d1 - 0.5, rc = cy - fy * p2.y / d2 - 0.5;
        // one pixel of margin on each side: the box only bounds the work, coverage is decided by the exact edge test
        s.c0 = clamp_floor(fmin(ca, fmin(cb, cc)) - 1.0, a.width - 1);
        s.c1 = clamp_ceil(fmax(ca, fmax(cb, cc)) + 1.0, a.width - 1);
        s.r0 = clamp_floor(fmin(ra, fmin(rb, rc)) - 1.0, a.height - 1);
        s.r1 = clamp_ceil(fmax(ra, fmax(rb, rc)) + 1.0, a.height - 1);
        if (fmax(ca, fmax(cb, cc)) < -1.0 || fmin(ca, fmin(cb, cc)) > (double)a.width ||
            fmax(ra, fmax(rb, rc)) < -1.0 || fmin(ra, fmin(rb, rc)) > (double)a.height) return s;   // off screen
    }
    s.live = true;
    return s;
}

__device__ __forceinline__ void fragment(const Setup &s, int t, int v, int r, int c, const ViewArgs &a,
                                         unsigned long long *__restrict__ zbuf)
{
    const double *k = a.intr + 4 * (long long)v;
    // the same expression for every triangle, so a pixel's ray is bit-identical across them (no division per fragment)
    const double px = ((double)c + 0.5 - k[2]) * (1.0 / k[0]), py = (k[3] - (double)r - 0.5) * (1.0 / k[1]);
    const double e0 = fma(s.e[0].x, px, fma(s.e[0].y, py, -s.e[0].z));
    const double e1 = fma(s.e[1].x, px, fma(s.e[1].y, py, -s.e[1].z));
    const double e2 = fma(s.e[2].x, px, fma(s.e[2].y, py, -s.e[2].z));
    const bool inside = s.det > 0.0 ? (e0 >= 0.0 && e1 >= 0.0 && e2 >= 0.0) : (e0 <= 0.0 && e1 <= 0.0 && e2 <= 0.0);
    if (!inside) return;
    const double depth = s.det / ((e0 + e1) + e2);
    if (!(depth >= a.znear && depth <= a.zfar)) return;
    const unsigned long long key = ((unsigned long long)__float_as_uint(__double2float_rn(depth)) << 32) | (unsigned)t;
    unsigned long long *z = zbuf + ((long long)v * a.height + r) * a.width + c;
    if (key < *z) atomicMin(z, key);            // a stale read only ever holds a larger key: skipping is still correct
}

__device__ __forceinline__ void raster_box(const Setup &s, int t, int v, const ViewArgs &a, unsigned long long *zbuf)
{
    for (int r = s.r0; r <= s.r1; ++r)
        for (int c = s.c0; c <= s.c1; ++c) fragment(s, t, v, r, c, a, zbuf);
}

// one thread per (triangle, view): small boxes are rasterized here, large ones are cut into tiles for tile_kernel
__global__ void __launch_bounds__(kThreads) triangle_kernel(const float *__restrict__ verts, const int *__restrict__ faces, int n_faces,
                                                            ViewArgs a, unsigned long long *__restrict__ zbuf, int2 *__restrict__ tiles,
                                                            unsigned long long *__restrict__ n_tiles, long long capacity)
{
    const int t = blockIdx.x * kThreads + threadIdx.x, v = blockIdx.y;
    if (t >= n_faces) return;
    const Setup s = setup(verts, faces, t, v, a);
    if (!s.live) return;
    if ((long long)(s.r1 - s.r0 + 1) * (s.c1 - s.c0 + 1) <= kSmallBox) {
        raster_box(s, t, v, a, zbuf);
        return;
    }
    const int tx = (a.width + kTile - 1) / kTile, per_view = tx * ((a.height + kTile - 1) / kTile);
    const int tr0 = s.r0 / kTile, tr1 = s.r1 / kTile, tc0 = s.c0 / kTile, tc1 = s.c1 / kTile;
    const unsigned long long n = (unsigned long long)(tr1 - tr0 + 1) * (tc1 - tc0 + 1);
    // every reserved slot below the capacity is written (tile_kernel reads them all); tiles past it are rasterized here
    unsigned long long i = atomicAdd(n_tiles, n);
    for (int tr = tr0; tr <= tr1; ++tr)
        for (int tc = tc0; tc <= tc1; ++tc, ++i) {
            if (i < (unsigned long long)capacity) {
                tiles[i] = make_int2(t, v * per_view + tr * tx + tc);
                continue;
            }
            for (int r = max(s.r0, tr * kTile); r <= min(s.r1, tr * kTile + kTile - 1); ++r)
                for (int c = max(s.c0, tc * kTile); c <= min(s.c1, tc * kTile + kTile - 1); ++c) fragment(s, t, v, r, c, a, zbuf);
        }
}

// one CTA per listed tile of a large triangle, one pixel of the tile per thread and pass
__global__ void __launch_bounds__(kThreads) tile_kernel(const float *__restrict__ verts, const int *__restrict__ faces, ViewArgs a,
                                                        unsigned long long *__restrict__ zbuf, const int2 *__restrict__ tiles,
                                                        const unsigned long long *__restrict__ n_tiles, long long capacity)
{
    __shared__ Setup s;
    const long long n = (long long)min(*n_tiles, (unsigned long long)capacity);
    const int tx = (a.width + kTile - 1) / kTile, per_view = tx * ((a.height + kTile - 1) / kTile);
    for (long long i = blockIdx.x; i < n; i += gridDim.x) {
        const int2 e = tiles[i];
        const int v = e.y / per_view, tile = e.y - v * per_view;
        __syncthreads();                                    // the previous tile is done with s
        if (threadIdx.x == 0) s = setup(verts, faces, e.x, v, a);
        __syncthreads();
        const int rt = (tile / tx) * kTile, ct = (tile % tx) * kTile;
#pragma unroll
        for (int k = 0; k < kTilePixelsPerThread; ++k) {
            const int p = threadIdx.x + k * kThreads, r = rt + p / kTile, c = ct + p % kTile;
            if (r >= s.r0 && r <= s.r1 && c >= s.c0 && c <= s.c1) fragment(s, e.x, v, r, c, a, zbuf);
        }
    }
}

// z-buffer -> depth (0: background), uint8 face normal (0, 0, 0: background), triangle index (-1: background)
__global__ void __launch_bounds__(kThreads) resolve_kernel(const float *__restrict__ verts, const int *__restrict__ faces,
                                                           const unsigned long long *__restrict__ zbuf, long long n_pixels,
                                                           float *__restrict__ depth, unsigned char *__restrict__ normals,
                                                           int *__restrict__ tri)
{
    const long long p = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (p >= n_pixels) return;
    const unsigned long long key = zbuf[p];
    unsigned char q[3] = {0, 0, 0};
    float d = 0.f;
    int t = -1;
    if (key != kEmpty) {
        t = (int)(unsigned)(key & 0xffffffffull);
        d = __uint_as_float((unsigned)(key >> 32));
        const long long b = 3 * (long long)t;
        const double3 n = face_normal(verts, make_int3(faces[b], faces[b + 1], faces[b + 2]));
        const double len = sqrt(n.x * n.x + n.y * n.y + n.z * n.z);
        const float nf[3] = {__double2float_rn(n.x / len), __double2float_rn(n.y / len), __double2float_rn(n.z / len)};
#pragma unroll
        for (int j = 0; j < 3; ++j)
            q[j] = (unsigned char)__float2int_rn(fminf(fmaxf(fmaf(0.5f, nf[j], 0.5f), 0.f), 1.f) * 255.f);
    }
    depth[p] = d;
    normals[3 * p] = q[0]; normals[3 * p + 1] = q[1]; normals[3 * p + 2] = q[2];
    if (tri) tri[p] = t;
}

struct Layout {
    long long capacity, list_off, zbuf_off, bytes;
};

inline Layout layout(int n_views, int height, int width)
{
    Layout l;
    const long long per_view = ceil_div(height, kTile) * ceil_div(width, kTile);
    l.capacity = 16 * (long long)n_views * per_view + 65536;
    l.list_off = 256;                                       // [0, 8): tile counter
    l.zbuf_off = l.list_off + ceil_div(l.capacity * (long long)sizeof(int2), 256) * 256;
    l.bytes = l.zbuf_off + (long long)n_views * height * width * (long long)sizeof(unsigned long long);
    return l;
}

}  // namespace render
}  // namespace nphm

using namespace nphm;

extern "C" long long nphm_render_workspace_bytes(int n_views, int height, int width)
{
    if (n_views < 1 || height < 1 || width < 1) {
        set_error("nphm_render_workspace_bytes: n_views, height and width must be >= 1 (got %d, %d, %d)", n_views, height, width);
        return -1;
    }
    return render::layout(n_views, height, width).bytes;
}

extern "C" int nphm_render_depth_normals(const float *verts_dev, long long n_verts, const int *faces_dev, long long n_faces,
                                         const double *world_to_eye_dev, const double *intrinsics_dev, int n_views, double znear,
                                         double zfar, int height, int width, float *depth_dev, unsigned char *normals_dev,
                                         int *tri_dev, void *workspace_dev, long long workspace_bytes, void *stream_)
{
    NPHM_REQUIRE(n_views >= 1 && n_views <= 65535 && height >= 1 && width >= 1,
                 "nphm_render_depth_normals: need 1 <= n_views <= 65535 and height, width >= 1 (got %d, %d, %d)", n_views, height, width);
    NPHM_REQUIRE(n_faces >= 0 && n_faces < (1ll << 31) && n_verts >= 0 && (n_faces == 0 || (verts_dev && faces_dev && n_verts >= 1)),
                 "nphm_render_depth_normals: bad mesh (%lld vertices, %lld faces)", n_verts, n_faces);
    NPHM_REQUIRE(world_to_eye_dev && intrinsics_dev && depth_dev && normals_dev && workspace_dev,
                 "nphm_render_depth_normals: null camera, output or workspace pointer");
    NPHM_REQUIRE(znear > 0.0 && zfar > znear, "nphm_render_depth_normals: need 0 < znear < zfar (got %g, %g)", znear, zfar);
    NPHM_REQUIRE((long long)n_views * ceil_div(height, render::kTile) * ceil_div(width, render::kTile) < (1ll << 31),
                 "nphm_render_depth_normals: %d views of %d x %d pixels are too many tiles", n_views, height, width);
    const render::Layout l = render::layout(n_views, height, width);
    if (workspace_bytes < l.bytes) {
        set_error("render workspace too small: %lld bytes for %d views of %d x %d, %lld needed", workspace_bytes, n_views, height,
                  width, l.bytes);
        return NPHM_ERR_CAPACITY;
    }
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    unsigned char *ws = static_cast<unsigned char *>(workspace_dev);
    auto *n_tiles = reinterpret_cast<unsigned long long *>(ws);
    auto *tiles = reinterpret_cast<int2 *>(ws + l.list_off);
    auto *zbuf = reinterpret_cast<unsigned long long *>(ws + l.zbuf_off);
    const long long n_pixels = (long long)n_views * height * width;
    NPHM_CUDA_CHECK(cudaMemsetAsync(n_tiles, 0, sizeof(unsigned long long), stream));
    NPHM_CUDA_CHECK(cudaMemsetAsync(zbuf, 0xff, n_pixels * sizeof(unsigned long long), stream));
    const render::ViewArgs a{world_to_eye_dev, intrinsics_dev, height, width, znear, zfar};
    if (n_faces > 0) {
        render::triangle_kernel<<<dim3((unsigned)ceil_div(n_faces, render::kThreads), (unsigned)n_views), render::kThreads, 0, stream>>>(
            verts_dev, faces_dev, (int)n_faces, a, zbuf, tiles, n_tiles, l.capacity);
        NPHM_CUDA_CHECK(cudaGetLastError());
        render::tile_kernel<<<(unsigned)(16 * sm_count()), render::kThreads, 0, stream>>>(verts_dev, faces_dev, a, zbuf, tiles, n_tiles,
                                                                                         l.capacity);
        NPHM_CUDA_CHECK(cudaGetLastError());
    }
    render::resolve_kernel<<<(unsigned)ceil_div(n_pixels, render::kThreads), render::kThreads, 0, stream>>>(
        verts_dev, faces_dev, zbuf, n_pixels, depth_dev, normals_dev, tri_dev);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}
