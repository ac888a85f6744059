// Sphere tracing of SDF heads into the rasterizer's image format (DESIGN.md §4.23).  The network evaluation stays in the
// existing query entry points; this file owns the ray state and every step around them:
//   begin    per (head, view, pixel): the eye ray of render.cu, the world ray, its entry into and exit from the box, state LIVE
//            (or MISS without any query when the ray misses the box or the [znear, zfar] range);
//   compact  ordered list of the rays of each head that are LIVE (march) or BRACKET (refinement): flags, one exclusive scan over
//            all heads, a scatter; the per-head counts stay on the device;
//   gather   the scaled sample points of the listed rays, head h's at rows [h n_cols, h n_cols + count_h), the rest zero;
//   advance  one step of the state machine on the listed rays from the SDF (and the posed search's valid flag) at their points;
//   finish   depth, uint8 normal (render.cu's rounding), world point, status and step count of every ray into the images.
// A chunk holds n_rays consecutive pixels of the V x H x W images for each of the S heads; nothing in a step reads back to the
// host (nphm_trace_counts is the optional early exit).
#include <cub/cub.cuh>
#include "common.cuh"

namespace nphm {
namespace trace {

constexpr int kThreads = 256;
enum : unsigned char { kLive = 0, kBracket = 1, kHit = 2, kMiss = 3, kOutOfSteps = 4, kInvalid = 5 };

__host__ __device__ inline size_t align256(size_t x) { return (x + 255) / 256 * 256; }

struct Layout {
    size_t geo, s, lo, hi, flo, fhi, sgn, steps, status, flags, scan, rows, counts, scratch, scratch_bytes, bytes;
};

// per ray (shared by the heads): o[3], u[3], s_in, s_out, 1/|d_eye| in fp64; per (head, ray): the state
inline Layout layout(int n_heads, long long n_rays)
{
    const size_t R = (size_t)n_heads * n_rays;
    Layout l;
    size_t off = 0;
    auto take = [&](size_t bytes) { const size_t o = off; off += align256(bytes); return o; };
    l.geo = take((size_t)n_rays * 9 * sizeof(double));
    l.s = take(R * sizeof(double));
    l.lo = take(R * sizeof(double));
    l.hi = take(R * sizeof(double));
    l.flo = take(R * sizeof(float));
    l.fhi = take(R * sizeof(float));
    l.sgn = take(R * sizeof(float));
    l.steps = take(R * sizeof(int));
    l.status = take(R);
    l.flags = take(R * sizeof(int));
    l.scan = take(R * sizeof(int));
    l.rows = take(R * sizeof(int));
    l.counts = take((size_t)n_heads * sizeof(int));
    size_t scratch = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, scratch, (const int *)nullptr, (int *)nullptr, (int)R);
    l.scratch_bytes = scratch;
    l.scratch = take(scratch);
    l.bytes = off;
    return l;
}

struct State {
    const double *geo;
    double *s, *lo, *hi;
    float *flo, *fhi, *sgn;
    int *steps;
    unsigned char *status;
    int *flags, *scan, *rows, *counts;
};

inline State carve(void *ws, const Layout &l)
{
    unsigned char *b = static_cast<unsigned char *>(ws);
    return State{reinterpret_cast<const double *>(b + l.geo), reinterpret_cast<double *>(b + l.s), reinterpret_cast<double *>(b + l.lo),
                 reinterpret_cast<double *>(b + l.hi), reinterpret_cast<float *>(b + l.flo), reinterpret_cast<float *>(b + l.fhi),
                 reinterpret_cast<float *>(b + l.sgn), reinterpret_cast<int *>(b + l.steps), b + l.status, reinterpret_cast<int *>(b + l.flags),
                 reinterpret_cast<int *>(b + l.scan), reinterpret_cast<int *>(b + l.rows), reinterpret_cast<int *>(b + l.counts)};
}

// the refinement's next sample in the bracket [lo, hi] (f(lo) > 0 > f(hi)): the secant point, its fraction of the bracket
// clamped to [0.1, 0.9] so that every step shrinks the bracket by at least a tenth
__device__ __forceinline__ double secant(double lo, float flo, double hi, float fhi)
{
    double w = (double)flo / ((double)flo - (double)fhi);
    w = fmin(fmax(w, 0.1), 0.9);
    return lo + w * (hi - lo);
}

__global__ void __launch_bounds__(kThreads) begin_kernel(nphm_trace_params p, const double *__restrict__ c2w,
                                                         const double *__restrict__ intr, int height, int width, long long first_pixel,
                                                         double *__restrict__ geo, State st)
{
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= p.n_rays) return;
    const long long pix = first_pixel + i;
    const long long hw = (long long)height * width;
    const int v = (int)(pix / hw);
    const int r = (int)((pix - v * hw) / width), c = (int)(pix - v * hw - (long long)r * width);
    const double *k = intr + 4 * (long long)v, *m = c2w + 12 * (long long)v;
    // render.cu's pixel ray, bit for bit
    const double px = ((double)c + 0.5 - k[2]) * (1.0 / k[0]), py = (k[3] - (double)r - 0.5) * (1.0 / k[1]);
    const double dx = m[0] * px + m[1] * py - m[2], dy = m[4] * px + m[5] * py - m[6], dz = m[8] * px + m[9] * py - m[10];
    const double len = sqrt(dx * dx + dy * dy + dz * dz);
    const double o[3] = {m[3], m[7], m[11]}, u[3] = {dx / len, dy / len, dz / len};
    const double inv_cos = sqrt(px * px + py * py + 1.0);          // ray length per unit of eye depth
    double s_in = p.znear * inv_cos, s_out = p.zfar * inv_cos;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const double b0 = p.box_min[a] / p.scale, b1 = p.box_max[a] / p.scale;
        if (u[a] == 0.0) {
            if (o[a] < b0 || o[a] > b1) s_out = -1.0;
            continue;
        }
        const double t0 = (b0 - o[a]) / u[a], t1 = (b1 - o[a]) / u[a];
        s_in = fmax(s_in, fmin(t0, t1));
        s_out = fmin(s_out, fmax(t0, t1));
    }
    double *g = geo + 9 * i;
    g[0] = o[0]; g[1] = o[1]; g[2] = o[2]; g[3] = u[0]; g[4] = u[1]; g[5] = u[2];
    g[6] = s_in; g[7] = s_out; g[8] = 1.0 / inv_cos;
    const bool live = s_in <= s_out;
    for (int h = 0; h < p.n_heads; ++h) {
        const long long q = (long long)h * p.n_rays + i;
        st.s[q] = s_in;
        st.lo[q] = s_in;
        st.hi[q] = s_in;
        st.flo[q] = -1.f;                                           // no positive sample yet
        st.fhi[q] = 0.f;
        st.sgn[q] = 1.f;
        st.steps[q] = 0;
        st.status[q] = live ? kLive : kMiss;
    }
}

__global__ void __launch_bounds__(kThreads) flag_kernel(long long n, const unsigned char *__restrict__ status, unsigned char want,
                                                        int *__restrict__ flags)
{
    const long long q = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (q < n) flags[q] = status[q] == want;
}

__global__ void __launch_bounds__(kThreads) scatter_kernel(nphm_trace_params p, const int *__restrict__ flags,
                                                           const int *__restrict__ scan, int *__restrict__ rows)
{
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    const int h = blockIdx.y;
    if (i >= p.n_rays) return;
    const long long q = (long long)h * p.n_rays + i;
    if (flags[q]) rows[(long long)h * p.n_rays + (scan[q] - scan[(long long)h * p.n_rays])] = (int)i;
}

__global__ void count_kernel(nphm_trace_params p, const int *__restrict__ flags, const int *__restrict__ scan, int *__restrict__ counts)
{
    const int h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= p.n_heads) return;
    const long long last = (long long)(h + 1) * p.n_rays - 1;
    counts[h] = scan[last] + flags[last] - scan[(long long)h * p.n_rays];
}

__device__ __forceinline__ void point_at(const double *g, double s, double scale, float *out)
{
    out[0] = (float)(scale * (g[0] + s * g[3]));
    out[1] = (float)(scale * (g[1] + s * g[4]));
    out[2] = (float)(scale * (g[2] + s * g[5]));
}

__global__ void __launch_bounds__(kThreads) gather_kernel(nphm_trace_params p, long long n_cols, State st, float *__restrict__ pts)
{
    const long long j = (long long)blockIdx.x * kThreads + threadIdx.x;
    const int h = blockIdx.y;
    if (j >= n_cols) return;
    float *out = pts + 3 * ((long long)h * n_cols + j);
    if (j >= st.counts[h]) {
        out[0] = out[1] = out[2] = 0.f;
        return;
    }
    const int i = st.rows[(long long)h * p.n_rays + j];
    point_at(st.geo + 9 * (long long)i, st.s[(long long)h * p.n_rays + i], p.scale, out);
}

__global__ void __launch_bounds__(kThreads) advance_kernel(nphm_trace_params p, int refine, long long n_cols, State st,
                                                           const float *__restrict__ sdf, const unsigned char *__restrict__ valid)
{
    const long long j = (long long)blockIdx.x * kThreads + threadIdx.x;
    const int h = blockIdx.y;
    if (j >= n_cols || j >= st.counts[h]) return;
    const int i = st.rows[(long long)h * p.n_rays + j];
    const long long q = (long long)h * p.n_rays + i, in = (long long)h * n_cols + j;
    const double s = st.s[q];
    if (valid && !valid[in]) {
        st.status[q] = kInvalid;
        if (!refine) st.steps[q] += 1;
        return;
    }
    // the march runs on g = sign(f at the entry) f: a ray that enters the box inside the solid looks for the first crossing too
    float sg = st.sgn[q];
    if (!refine && st.steps[q] == 0) {
        sg = sdf[in] < 0.f ? -1.f : 1.f;
        st.sgn[q] = sg;
    }
    const float f = sg * sdf[in];
    if (refine) {
        if (f < 0.f) { st.hi[q] = s; st.fhi[q] = f; }
        else { st.lo[q] = s; st.flo[q] = f; }
        st.s[q] = secant(st.lo[q], st.flo[q], st.hi[q], st.fhi[q]);
        return;
    }
    const int steps = st.steps[q] + 1;
    st.steps[q] = steps;
    if (f < 0.f && st.flo[q] > 0.f) {                              // a crossing since the last (positive) sample
        st.hi[q] = s;
        st.fhi[q] = f;
        st.s[q] = secant(st.lo[q], st.flo[q], s, f);
        st.status[q] = kBracket;
        return;
    }
    if (f < p.hit_eps) {                                            // close enough
        st.status[q] = kHit;
        return;
    }
    st.lo[q] = s;
    st.flo[q] = f;
    const double next = s + (double)p.step_factor * fmax((double)f / p.scale, (double)p.min_step);
    const double s_out = st.geo[9 * (long long)i + 7];
    st.s[q] = next;
    if (next > s_out) st.status[q] = kMiss;
    else if (steps >= p.max_steps) st.status[q] = kOutOfSteps;
}

__global__ void __launch_bounds__(kThreads) points_kernel(nphm_trace_params p, State st, float *__restrict__ pts)
{
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    const int h = blockIdx.y;
    if (i >= p.n_rays) return;
    const long long q = (long long)h * p.n_rays + i;
    float *out = pts + 3 * q;
    const unsigned char stt = st.status[q];
    if (stt == kHit || stt == kBracket) point_at(st.geo + 9 * i, st.s[q], p.scale, out);
    else out[0] = out[1] = out[2] = 0.f;
}

__global__ void __launch_bounds__(kThreads) finish_kernel(nphm_trace_params p, State st, const float *__restrict__ grad,
                                                          const float *__restrict__ jinv, const unsigned char *__restrict__ valid,
                                                          long long n_pixels, long long first_pixel, float *__restrict__ depth,
                                                          unsigned char *__restrict__ normals, float *__restrict__ points,
                                                          unsigned char *__restrict__ status, int *__restrict__ steps)
{
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    const int h = blockIdx.y;
    if (i >= p.n_rays) return;
    const long long q = (long long)h * p.n_rays + i, out = (long long)h * n_pixels + first_pixel + i;
    unsigned char stt = st.status[q];
    if (stt == kBracket) stt = kHit;                                // refinement done: the last secant point is the hit
    if (stt == kHit && valid && !valid[q]) stt = kInvalid;          // the hit point's own search did not converge
    const double *g = st.geo + 9 * i;
    const double s = st.s[q];
    float d = 0.f;
    unsigned char nq[3] = {0, 0, 0};
    if (stt == kHit) {
        d = (float)(s * g[8]);
        const float *gr = grad + 3 * q;
        double n[3] = {gr[0], gr[1], gr[2]};
        if (jinv) {                                                 // posed: (I + dF/dx_c)^-T grad_{x_c} sdf
            const float *J = jinv + 9 * q;
            for (int a = 0; a < 3; ++a) n[a] = (double)J[a] * gr[0] + (double)J[3 + a] * gr[1] + (double)J[6 + a] * gr[2];
        }
        const double len = sqrt(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const float nf = len > 0.0 ? (float)(n[a] / len) : 0.f;
            nq[a] = (unsigned char)__float2int_rn(fminf(fmaxf(fmaf(0.5f, nf, 0.5f), 0.f), 1.f) * 255.f);   // render.cu's rounding
        }
    }
    depth[out] = d;
    normals[3 * out] = nq[0]; normals[3 * out + 1] = nq[1]; normals[3 * out + 2] = nq[2];
    if (points) {
        const bool at = stt == kHit || stt == kInvalid;
        points[3 * out] = at ? (float)(g[0] + s * g[3]) : 0.f;
        points[3 * out + 1] = at ? (float)(g[1] + s * g[4]) : 0.f;
        points[3 * out + 2] = at ? (float)(g[2] + s * g[5]) : 0.f;
    }
    if (status) status[out] = stt;
    if (steps) steps[out] = st.steps[q];
}

inline unsigned blocks(long long n) { return (unsigned)ceil_div(n, kThreads); }

}  // namespace trace
}  // namespace nphm

using namespace nphm;

#define TRACE_CHECK_PARAMS(p, what)                                                                                            \
    NPHM_REQUIRE(p && p->n_heads >= 1 && p->n_heads <= 65535 && p->n_rays >= 1 &&                                              \
                     (long long)p->n_heads * p->n_rays < (1ll << 31),                                                          \
                 what ": need 1 <= n_heads <= 65535, n_rays >= 1 and n_heads * n_rays < 2^31");                               \
    NPHM_REQUIRE(p->scale > 0.0 && p->znear > 0.0 && p->zfar > p->znear && p->step_factor > 0.f && p->hit_eps > 0.f &&         \
                     p->min_step >= 0.f && p->max_steps >= 1,                                                                  \
                 what ": need scale > 0, 0 < znear < zfar, step_factor > 0, hit_eps > 0, min_step >= 0, max_steps >= 1")

#define TRACE_WORKSPACE(p, ws, ws_bytes, what)                                                                                    \
    const trace::Layout l = trace::layout(p->n_heads, p->n_rays);                                                              \
    NPHM_REQUIRE(ws, what ": null workspace");                                                                                 \
    if (ws_bytes < (long long)l.bytes) {                                                                                       \
        set_error(what ": workspace of %lld bytes, %lld needed", ws_bytes, (long long)l.bytes);                                  \
        return NPHM_ERR_CAPACITY;                                                                                              \
    }                                                                                                                          \
    const trace::State st = trace::carve(ws, l);                                                                               \
    cudaStream_t stream = static_cast<cudaStream_t>(stream_)

extern "C" long long nphm_trace_workspace_bytes(int n_heads, long long n_rays)
{
    if (n_heads < 1 || n_heads > 65535 || n_rays < 1 || (long long)n_heads * n_rays >= (1ll << 31)) {
        set_error("nphm_trace_workspace_bytes: need 1 <= n_heads <= 65535, n_rays >= 1 and n_heads * n_rays < 2^31");
        return -1;
    }
    return (long long)trace::layout(n_heads, n_rays).bytes;
}

extern "C" int nphm_trace_begin(const nphm_trace_params *p, const double *cam_to_world_dev, const double *intrinsics_dev, int n_views,
                                int height, int width, long long first_pixel, void *workspace_dev, long long workspace_bytes,
                                void *stream_)
{
    TRACE_CHECK_PARAMS(p, "nphm_trace_begin");
    NPHM_REQUIRE(cam_to_world_dev && intrinsics_dev && n_views >= 1 && height >= 1 && width >= 1,
                 "nphm_trace_begin: need cameras and n_views, height, width >= 1");
    NPHM_REQUIRE(first_pixel >= 0 && first_pixel + p->n_rays <= (long long)n_views * height * width,
                 "nphm_trace_begin: pixels [%lld, %lld) outside the %d views of %d x %d", first_pixel, first_pixel + p->n_rays, n_views,
                 height, width);
    TRACE_WORKSPACE(p, workspace_dev, workspace_bytes, "nphm_trace_begin");
    trace::begin_kernel<<<trace::blocks(p->n_rays), trace::kThreads, 0, stream>>>(
        *p, cam_to_world_dev, intrinsics_dev, height, width, first_pixel, const_cast<double *>(st.geo), st);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

extern "C" int nphm_trace_compact(const nphm_trace_params *p, int refine, void *workspace_dev, long long workspace_bytes, void *stream_)
{
    TRACE_CHECK_PARAMS(p, "nphm_trace_compact");
    TRACE_WORKSPACE(p, workspace_dev, workspace_bytes, "nphm_trace_compact");
    const long long R = (long long)p->n_heads * p->n_rays;
    trace::flag_kernel<<<trace::blocks(R), trace::kThreads, 0, stream>>>(R, st.status, refine ? trace::kBracket : trace::kLive, st.flags);
    NPHM_CUDA_CHECK(cudaGetLastError());
    size_t scratch = l.scratch_bytes;
    NPHM_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(static_cast<unsigned char *>(workspace_dev) + l.scratch, scratch, st.flags, st.scan,
                                                  (int)R, stream));
    trace::scatter_kernel<<<dim3(trace::blocks(p->n_rays), p->n_heads), trace::kThreads, 0, stream>>>(*p, st.flags, st.scan, st.rows);
    NPHM_CUDA_CHECK(cudaGetLastError());
    trace::count_kernel<<<(unsigned)ceil_div(p->n_heads, 128), 128, 0, stream>>>(*p, st.flags, st.scan, st.counts);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

extern "C" int nphm_trace_counts(const nphm_trace_params *p, const void *workspace_dev, long long workspace_bytes, int *counts_host,
                                 void *stream_)
{
    TRACE_CHECK_PARAMS(p, "nphm_trace_counts");
    NPHM_REQUIRE(counts_host, "nphm_trace_counts: null counts");
    TRACE_WORKSPACE(p, const_cast<void *>(workspace_dev), workspace_bytes, "nphm_trace_counts");
    NPHM_CUDA_CHECK(cudaMemcpyAsync(counts_host, st.counts, p->n_heads * sizeof(int), cudaMemcpyDeviceToHost, stream));
    NPHM_CUDA_CHECK(cudaStreamSynchronize(stream));
    return NPHM_OK;
}

extern "C" int nphm_trace_gather(const nphm_trace_params *p, long long n_cols, void *workspace_dev, long long workspace_bytes,
                                 float *points_dev, void *stream_)
{
    TRACE_CHECK_PARAMS(p, "nphm_trace_gather");
    NPHM_REQUIRE(n_cols >= 1 && n_cols <= p->n_rays && points_dev, "nphm_trace_gather: need 1 <= n_cols <= n_rays and points");
    TRACE_WORKSPACE(p, workspace_dev, workspace_bytes, "nphm_trace_gather");
    trace::gather_kernel<<<dim3(trace::blocks(n_cols), p->n_heads), trace::kThreads, 0, stream>>>(*p, n_cols, st, points_dev);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

extern "C" int nphm_trace_advance(const nphm_trace_params *p, int refine, long long n_cols, const float *sdf_dev,
                                  const unsigned char *valid_dev, void *workspace_dev, long long workspace_bytes, void *stream_)
{
    TRACE_CHECK_PARAMS(p, "nphm_trace_advance");
    NPHM_REQUIRE(n_cols >= 1 && n_cols <= p->n_rays && sdf_dev, "nphm_trace_advance: need 1 <= n_cols <= n_rays and sdf");
    TRACE_WORKSPACE(p, workspace_dev, workspace_bytes, "nphm_trace_advance");
    trace::advance_kernel<<<dim3(trace::blocks(n_cols), p->n_heads), trace::kThreads, 0, stream>>>(*p, refine, n_cols, st, sdf_dev,
                                                                                                   valid_dev);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

extern "C" int nphm_trace_points(const nphm_trace_params *p, const void *workspace_dev, long long workspace_bytes, float *points_dev,
                                 void *stream_)
{
    TRACE_CHECK_PARAMS(p, "nphm_trace_points");
    NPHM_REQUIRE(points_dev, "nphm_trace_points: null points");
    TRACE_WORKSPACE(p, const_cast<void *>(workspace_dev), workspace_bytes, "nphm_trace_points");
    trace::points_kernel<<<dim3(trace::blocks(p->n_rays), p->n_heads), trace::kThreads, 0, stream>>>(*p, st, points_dev);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}

extern "C" int nphm_trace_finish(const nphm_trace_params *p, const void *workspace_dev, long long workspace_bytes, const float *grad_dev,
                                 const float *jinv_dev, const unsigned char *valid_dev, long long n_pixels, long long first_pixel,
                                 float *depth_dev, unsigned char *normals_dev, float *points_dev, unsigned char *status_dev,
                                 int *steps_dev, void *stream_)
{
    TRACE_CHECK_PARAMS(p, "nphm_trace_finish");
    NPHM_REQUIRE(grad_dev && depth_dev && normals_dev, "nphm_trace_finish: null gradient, depth or normals");
    NPHM_REQUIRE(first_pixel >= 0 && first_pixel + p->n_rays <= n_pixels, "nphm_trace_finish: pixels [%lld, %lld) outside [0, %lld)",
                 first_pixel, first_pixel + p->n_rays, n_pixels);
    TRACE_WORKSPACE(p, const_cast<void *>(workspace_dev), workspace_bytes, "nphm_trace_finish");
    trace::finish_kernel<<<dim3(trace::blocks(p->n_rays), p->n_heads), trace::kThreads, 0, stream>>>(
        *p, st, grad_dev, jinv_dev, valid_dev, n_pixels, first_pixel, depth_dev, normals_dev, points_dev, status_dev, steps_dev);
    NPHM_CUDA_CHECK(cudaGetLastError());
    return NPHM_OK;
}
