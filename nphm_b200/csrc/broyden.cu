// Batched Broyden root search for the canonical correspondences  x + F_ex(x; cond) = obs  (SURVEY §8 f1).
// Restates reference src/NPHM/models/iterative_root_finding.py:5-71 (`broyden`) with the residual of `search`
// (:142-147) on the device: the network evaluation of every step is one launch of the fused MLP kernel over ALL
// points (rows are independent, so frozen points are simply ignored), the 3x3 quasi-Newton algebra of a point lives in
// one thread, and the active masks are per-point flags instead of boolean-index gathers (no host synchronisation
// except one 4-byte "anyone still active?" read every `kCheckEvery` steps).
//
// Reference quirks kept: `x_opt` aliases `x` there (x_opt = x, then in-place updates), so 'result' is the point at
// which a sample stopped moving, not the best one seen; 'diff' is the smallest residual norm seen; a sample is frozen
// once diff <= cvg or its current norm >= dvg; b = vT.dgx is pushed away from zero by +-eps before the division.
#include "engine.cuh"
#include "simt.cuh"
#include <cub/device/device_select.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <climits>

namespace nphm {
int mlp_prepare(nphm_mlp *h, const float *cond_dev, int n_queries, cudaStream_t stream);
int mlp_run(nphm_mlp *h, const float *xyz_dev, int n_queries, long long n_points, float *out_dev, int impl, cudaStream_t stream);

namespace broyden {

constexpr int kCheckEvery = 3;

struct State {
    float *x;        // n*3   current iterate (also the result)
    float *jinv;     // n*9   row-major inverse-Jacobian estimate
    float *gx;       // n*3   residual at x
    float *upd;      // n*3   next step
    float *best;     // n     smallest residual norm seen
    unsigned char *active;   // n
    float *f;        // n*3   network output at x
    int *n_active;   // counter of the current step: samples still active after its update
};

__device__ __forceinline__ float norm3(float a, float b, float c) { return sqrtf(a * a + b * b + c * c); }

// gx = F(x) + x - obs; update = -J_inv gx; best = |gx|; everybody active
__global__ void init_kernel(State s, const float *__restrict__ obs, long long n)
{
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= n) return;
    float g[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) g[c] = (s.f[i * 3 + c] + s.x[i * 3 + c]) - obs[i * 3 + c];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        const float *J = s.jinv + i * 9 + r * 3;
        s.upd[i * 3 + r] = -(J[0] * g[0] + J[1] * g[1] + J[2] * g[2]);
        s.gx[i * 3 + r] = g[r];
    }
    s.best[i] = norm3(g[0], g[1], g[2]);
    s.active[i] = 1;
}

// x += update for active samples (the step the reference takes before evaluating g)
__global__ void advance_kernel(State s, long long n)
{
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= n || !s.active[i]) return;
#pragma unroll
    for (int c = 0; c < 3; ++c) s.x[i * 3 + c] += s.upd[i * 3 + c];
}

// after F(x) is available (f: the network output of sample i): residual bookkeeping, freeze test, rank-one update of J_inv,
// next step
__device__ __forceinline__ void update_sample(const State &s, long long i, const float *f, const float *__restrict__ obs,
                                              float cvg, float dvg, float eps)
{
    float dx[3], dg[3], g[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        dx[c] = s.upd[i * 3 + c];
        const float gnew = (f[c] + s.x[i * 3 + c]) - obs[i * 3 + c];
        const float gold = s.gx[i * 3 + c];
        dg[c] = gnew - gold;
        g[c] = gold + dg[c];                                  // gx[ids] += delta_gx[ids]
        s.gx[i * 3 + c] = g[c];
    }
    const float nrm = norm3(g[0], g[1], g[2]);
    float best = s.best[i];
    if (nrm < best) { best = nrm; s.best[i] = nrm; }
    const bool act = best > cvg && nrm < dvg;
    s.active[i] = act ? 1 : 0;
    if (!act) return;
    atomicAdd(s.n_active, 1);
    float J[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) J[k] = s.jinv[i * 9 + k];
    float vT[3], a[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) vT[c] = dx[0] * J[c] + dx[1] * J[3 + c] + dx[2] * J[6 + c];
#pragma unroll
    for (int r = 0; r < 3; ++r) a[r] = dx[r] - (J[r * 3] * dg[0] + J[r * 3 + 1] * dg[1] + J[r * 3 + 2] * dg[2]);
    float b = vT[0] * dg[0] + vT[1] * dg[1] + vT[2] * dg[2];
    b += b >= 0.0f ? eps : -eps;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        const float u = a[r] / b;
#pragma unroll
        for (int c = 0; c < 3; ++c) J[r * 3 + c] += u * vT[c];
    }
#pragma unroll
    for (int k = 0; k < 9; ++k) s.jinv[i * 9 + k] = J[k];
#pragma unroll
    for (int r = 0; r < 3; ++r) s.upd[i * 3 + r] = -(J[r * 3] * g[0] + J[r * 3 + 1] * g[1] + J[r * 3 + 2] * g[2]);
}

__global__ void update_kernel(State s, const float *__restrict__ obs, long long n, float cvg, float dvg, float eps)
{
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= n || !s.active[i]) return;
    update_sample(s, i, s.f + i * 3, obs, cvg, dvg, eps);
}

// ---- compacting variant: slot k < cnt[q] of query q (rows q * n_points + k of the row list) holds live sample
// q * n_points + idx[k]; the network reads xc and writes s.f in slot order

// the sample of slot k, or -1 beyond its query's live count
__device__ __forceinline__ long long slot_sample(const int *idx, const int *cnt, long long n_points, long long k)
{
    const long long q = k / n_points;
    return k - q * n_points < cnt[q] ? q * n_points + idx[k] : -1;
}

// x += update of every live sample (advance_kernel), and its copy into slot order
__global__ void gather_advance_kernel(State s, const int *__restrict__ idx, const int *__restrict__ cnt, long long n_points,
                                      long long n, float *__restrict__ xc)
{
    const long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (k >= n) return;
    const long long i = slot_sample(idx, cnt, n_points, k);
    if (i < 0) return;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        s.x[i * 3 + c] += s.upd[i * 3 + c];
        xc[k * 3 + c] = s.x[i * 3 + c];
    }
}

__global__ void update_compact_kernel(State s, const int *__restrict__ idx, const int *__restrict__ cnt, long long n_points,
                                      const float *__restrict__ obs, long long n, float cvg, float dvg, float eps)
{
    const long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (k >= n) return;
    const long long i = slot_sample(idx, cnt, n_points, k);
    if (i < 0) return;
    update_sample(s, i, s.f + k * 3, obs, cvg, dvg, eps);
}

__global__ void finish_kernel(State s, long long n, float cvg, float *diff, unsigned char *valid)
{
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float b = s.best[i];
    diff[i] = b;
    valid[i] = b < cvg ? 1 : 0;
}

}  // namespace broyden
}  // namespace nphm

using namespace nphm;

static inline size_t align256(size_t v) { return (v + 255) / 256 * 256; }

extern "C" long long nphm_broyden_workspace_bytes(long long n_total)
{
    if (n_total < 0) return NPHM_ERR_INVALID;
    const size_t n = (size_t)n_total;
    return (long long)(align256(n * 9 * 4) + 3 * align256(n * 3 * 4) + align256(n * 4) + align256(n) + 1024);
}

// the compacting search's buffers (Compact::carve): slot list, live counts, points in slot order, CUB scratch
struct Compact {
    int *idx = nullptr, *cnt = nullptr;
    float *xc = nullptr;
    void *scratch = nullptr;
    size_t scratch_bytes = 0;
};

static size_t select_scratch_bytes(long long n_points)
{
    size_t bytes = 0;
    cub::DeviceSelect::Flagged(nullptr, bytes, thrust::counting_iterator<int>(0), (const unsigned char *)nullptr, (int *)nullptr,
                               (int *)nullptr, (int)n_points);
    return bytes;
}

static size_t compact_extra_bytes(int n_queries, long long n_points)
{
    const size_t n = (size_t)n_queries * n_points;
    return align256(n * 4) + align256(n * 12) + align256((size_t)n_queries * 4) + align256(select_scratch_bytes(n_points));
}

extern "C" long long nphm_broyden_compact_workspace_bytes(int n_queries, long long n_points)
{
    if (n_queries < 1 || n_points < 0 || n_points > INT_MAX) return NPHM_ERR_INVALID;
    return nphm_broyden_workspace_bytes((long long)n_queries * n_points) + (long long)compact_extra_bytes(n_queries, n_points);
}

// the dense search (every step evaluates all samples, frozen ones are ignored) or the compacting one
static int broyden_search(const char *who, nphm_mlp *h, const float *cond_dev, int n_queries, long long n_points,
                          const float *obs_dev, float *x_dev, const float *jinv_init_dev, int max_steps, float cvg_thresh,
                          float dvg_thresh, float eps, float *diff_dev, unsigned char *valid_dev, int *steps_done,
                          void *workspace_dev, cudaStream_t stream, bool compact)
{
    NPHM_REQUIRE(h && h->loaded, "%s: weights not loaded", who);
    NPHM_REQUIRE(h->cfg.out_dim == 3, "%s: the field must have 3 outputs (has %d)", who, h->cfg.out_dim);
    NPHM_REQUIRE(n_queries >= 1 && n_points >= 0 && max_steps >= 0, "%s: bad sizes", who);
    NPHM_REQUIRE(!compact || n_points <= INT_MAX, "%s: at most 2^31 - 1 points per query", who);
    NPHM_REQUIRE(cond_dev && (n_points == 0 || (obs_dev && x_dev && jinv_init_dev && diff_dev && valid_dev && workspace_dev)),
                 "%s: NULL pointer", who);
    if (steps_done) *steps_done = 0;
    const long long n = n_points * n_queries;
    if (n == 0) return NPHM_OK;
    char *p = static_cast<char *>(workspace_dev);
    broyden::State s{};
    s.x = x_dev;
    s.jinv = reinterpret_cast<float *>(p); p += align256((size_t)n * 36);
    s.gx = reinterpret_cast<float *>(p); p += align256((size_t)n * 12);
    s.upd = reinterpret_cast<float *>(p); p += align256((size_t)n * 12);
    s.f = reinterpret_cast<float *>(p); p += align256((size_t)n * 12);
    s.best = reinterpret_cast<float *>(p); p += align256((size_t)n * 4);
    s.active = reinterpret_cast<unsigned char *>(p); p += align256((size_t)n);
    int *counters = reinterpret_cast<int *>(p);              // one counter per step (max 255), zeroed once
    p += 1024;
    Compact cmp;
    if (compact) {
        cmp.idx = reinterpret_cast<int *>(p); p += align256((size_t)n * 4);
        cmp.xc = reinterpret_cast<float *>(p); p += align256((size_t)n * 12);
        cmp.cnt = reinterpret_cast<int *>(p); p += align256((size_t)n_queries * 4);
        cmp.scratch = p;
        cmp.scratch_bytes = select_scratch_bytes(n_points);
    }
    NPHM_REQUIRE(max_steps < 255, "%s: max_steps must be < 255", who);
    NPHM_CUDA_CHECK(cudaMemsetAsync(counters, 0, 1024, stream));
    s.n_active = counters;
    NPHM_CUDA_CHECK(cudaMemcpyAsync(s.jinv, jinv_init_dev, (size_t)n * 36, cudaMemcpyDeviceToDevice, stream));

    int rc;
    if ((rc = mlp_prepare(h, cond_dev, n_queries, stream))) return rc;
    const unsigned blocks = (unsigned)ceil_div(n, 256);
    if ((rc = mlp_run(h, s.x, n_queries, n_points, s.f, NPHM_IMPL_AUTO, stream))) return rc;
    broyden::init_kernel<<<blocks, 256, 0, stream>>>(s, obs_dev, n);
    NPHM_CUDA_CHECK(cudaGetLastError());
    int done = 0;
    for (int step = 0; step < max_steps; ++step) {
        if (compact) {
            // ordered per-query compaction of the active flags: slot k of query q <- its k-th live sample; the launches below
            // keep their full grids and return at once beyond the counts, so no host synchronisation is needed
            for (int q = 0; q < n_queries; ++q) {
                size_t bytes = cmp.scratch_bytes;
                NPHM_CUDA_CHECK(cub::DeviceSelect::Flagged(cmp.scratch, bytes, thrust::counting_iterator<int>(0),
                                                           s.active + (size_t)q * n_points, cmp.idx + (size_t)q * n_points,
                                                           cmp.cnt + q, (int)n_points, stream));
            }
            broyden::gather_advance_kernel<<<blocks, 256, 0, stream>>>(s, cmp.idx, cmp.cnt, n_points, n, cmp.xc);
            NPHM_CUDA_CHECK(cudaGetLastError());
            h->live_rows = cmp.cnt;
            rc = mlp_run(h, cmp.xc, n_queries, n_points, s.f, NPHM_IMPL_AUTO, stream);
            h->live_rows = nullptr;
            if (rc) return rc;
            s.n_active = counters + step;
            broyden::update_compact_kernel<<<blocks, 256, 0, stream>>>(s, cmp.idx, cmp.cnt, n_points, obs_dev, n, cvg_thresh,
                                                                       dvg_thresh, eps);
        } else {
            broyden::advance_kernel<<<blocks, 256, 0, stream>>>(s, n);
            NPHM_CUDA_CHECK(cudaGetLastError());
            // once nobody is active (counter of the previous step == 0) the network evaluation returns at once: a device-side
            // early exit that needs no host synchronisation (the reference leaves its loop at that point)
            h->live = step > 0 ? counters + (step - 1) : nullptr;
            rc = mlp_run(h, s.x, n_queries, n_points, s.f, NPHM_IMPL_AUTO, stream);
            h->live = nullptr;
            if (rc) return rc;
            s.n_active = counters + step;
            broyden::update_kernel<<<blocks, 256, 0, stream>>>(s, obs_dev, n, cvg_thresh, dvg_thresh, eps);
        }
        NPHM_CUDA_CHECK(cudaGetLastError());
        done = step + 1;
        // optional host-side early exit (4-byte read-back + stream sync every kCheckEvery steps); a caller that passes
        // steps_done == NULL asks for a sync-free, CUDA-graph capturable call
        const bool check = steps_done != nullptr && (step % broyden::kCheckEvery) == broyden::kCheckEvery - 1 && step + 1 < max_steps;
        if (check) {
            int alive = 0;
            NPHM_CUDA_CHECK(cudaMemcpyAsync(&alive, s.n_active, sizeof(int), cudaMemcpyDeviceToHost, stream));
            NPHM_CUDA_CHECK(cudaStreamSynchronize(stream));
            if (alive == 0) break;
        }
    }
    broyden::finish_kernel<<<blocks, 256, 0, stream>>>(s, n, cvg_thresh, diff_dev, valid_dev);
    NPHM_CUDA_CHECK(cudaGetLastError());
    if (steps_done) *steps_done = done;
    return NPHM_OK;
}

extern "C" int nphm_mlp_broyden_search(nphm_mlp *h, const float *cond_dev, int n_queries, long long n_points,
                                       const float *obs_dev, float *x_dev, const float *jinv_init_dev, int max_steps,
                                       float cvg_thresh, float dvg_thresh, float eps, float *diff_dev,
                                       unsigned char *valid_dev, int *steps_done, void *workspace_dev, void *stream)
{
    return broyden_search("nphm_mlp_broyden_search", h, cond_dev, n_queries, n_points, obs_dev, x_dev, jinv_init_dev, max_steps,
                          cvg_thresh, dvg_thresh, eps, diff_dev, valid_dev, steps_done, workspace_dev,
                          static_cast<cudaStream_t>(stream), false);
}

extern "C" int nphm_mlp_broyden_search_compact(nphm_mlp *h, const float *cond_dev, int n_queries, long long n_points,
                                               const float *obs_dev, float *x_dev, const float *jinv_init_dev, int max_steps,
                                               float cvg_thresh, float dvg_thresh, float eps, float *diff_dev,
                                               unsigned char *valid_dev, int *steps_done, void *workspace_dev, void *stream)
{
    return broyden_search("nphm_mlp_broyden_search_compact", h, cond_dev, n_queries, n_points, obs_dev, x_dev, jinv_init_dev,
                          max_steps, cvg_thresh, dvg_thresh, eps, diff_dev, valid_dev, steps_done, workspace_dev,
                          static_cast<cudaStream_t>(stream), true);
}
