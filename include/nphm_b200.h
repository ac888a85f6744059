/* nphm_b200.h - C ABI of libnphm_b200.so, the H100 (sm_90a) engine behind NPHM's hot path.
 *
 * The reference (SimonGiebenhain/NPHM) has no FFI layer: its hot path sits behind Python call signatures
 * (SURVEY.md 8b).  This header is the boundary a binding would target; the Python mirror of the reference
 * modules in nphm_b200/ binds it with ctypes (nphm_b200/_native.py), see INTEGRATION.md.
 *
 * Conventions
 *   - every function returns NPHM_OK (0) or a negative error code; nphm_last_error() gives the message of the
 *     last failure on the calling thread.
 *   - pointers named *_dev are CUDA device pointers on the current device, *_host are host pointers.
 *   - `stream` is a cudaStream_t passed as void* (NULL = default stream); calls are asynchronous on that
 *     stream unless stated otherwise.  No torch types appear in any signature.
 *   - all network arithmetic is fp32 in / fp32 out; weights are given in the reference's state_dict layout.
 *   - handles are not thread safe; use one handle per host thread / stream.
 */
#ifndef NPHM_B200_H
#define NPHM_B200_H

#ifdef __cplusplus
extern "C" {
#endif

#define NPHM_OK               0
#define NPHM_ERR_INVALID     -1   /* bad argument */
#define NPHM_ERR_CUDA        -2   /* a CUDA runtime call failed */
#define NPHM_ERR_UNSUPPORTED -3   /* configuration not supported by the requested kernel */
#define NPHM_ERR_CAPACITY    -4   /* caller-provided buffer too small */

/* kernel selection for the network queries */
#define NPHM_IMPL_AUTO   0   /* tensor-core kernel when the configuration allows it, else SIMT */
#define NPHM_IMPL_SIMT   1   /* fp32 FFMA kernel (any configuration) */
#define NPHM_IMPL_TC     2   /* tensor-core (wgmma) kernel, 3-pass fp16 split (fp32-equivalent accuracy) */
#define NPHM_IMPL_TC_PRUNED 3 /* OPT-IN: tensor-core kernel that skips, per compact tile of 128 points, the ensemble members whose
                                normalised Gaussian blend weight is < tau for every point of the tile.  Not the dense
                                reference computation: |error| <= n_members * tau * max_k |s_k| (tau default 1e-8). */

const char *nphm_last_error(void);
int nphm_abi_version(void);
/* sm count and compute capability of the current device */
int nphm_device_info(int *sm_count, int *cc_major, int *cc_minor);

/* ------------------------------------------------------------------------------------------------
 * Identity SDF ensemble  == FastEnsembleDeepSDFMirrored (reference src/NPHM/models/EnsembledDeepSDF.py:153-267)
 * ---------------------------------------------------------------------------------------------- */
typedef struct nphm_ensemble nphm_ensemble;

typedef struct {
    int n_loc;          /* facial anchors (39); ensemble size is n_loc + 1              (:183)      */
    int n_symm_pairs;   /* mirrored anchor pairs sharing weights (16)                   (:184,:43)  */
    int lat_dim_glob;   /* 64                                                                        */
    int lat_dim_loc;    /* 32; latent = [z_glob, z_0 .. z_{n_loc-1}, z_global_member]   (:210-212)  */
    int hidden_dim;     /* 200                                                                       */
    int n_layers;       /* 4 hidden layers -> 5 linear layers, skip at n_layers/2       (:80-96)    */
    int pos_mlp_dim;    /* hidden width of mlp_pos (256)                                (:194-200)  */
} nphm_ensemble_config;

int nphm_ensemble_create(const nphm_ensemble_config *cfg, nphm_ensemble **out);
void nphm_ensemble_destroy(nphm_ensemble *h);
/* threshold tau of NPHM_IMPL_TC_PRUNED (relative blend weight below which a member is skipped), 0 <= tau < 1 */
int nphm_ensemble_set_prune_threshold(nphm_ensemble *h, float tau);

/* Replaces `load_state_dict` for the engine.  lin_w_dev[l]: (n_sets, out_l, in_l) row-major, lin_b_dev[l]:
 * (n_sets, out_l) for l = 0..n_layers (keys ensembled_deep_sdf.lin{l}.weight/bias, n_sets = n_loc+1-n_symm_pairs);
 * pos_w_dev/pos_b_dev: the three nn.Linear of mlp_pos (keys mlp_pos.{0,2,4}); mean_anchors_dev: n_loc*3.
 * Packs/splits the weights for every kernel; must be called again after the parameters change. */
int nphm_ensemble_load_weights(nphm_ensemble *h,
                               const float *const *lin_w_dev, const float *const *lin_b_dev,
                               const float *const *pos_w_dev, const float *const *pos_b_dev,
                               const float *mean_anchors_dev, void *stream);

/* == FastEnsembleDeepSDFMirrored.forward(xyz, lat_rep, None) for lat_rep constant over the points of a query.
 *   xyz_dev       n_queries * n_points * 3
 *   latents_dev   n_queries * lat_dim
 *   quirk_period  eval-mode quirk of :260-261 (`sdf_pred[:, :, -1, 0] = 1` hits the LAST POINT of a call):
 *                 0 = train mode (off); p > 0 = points with (i % p == p-1) or i == n_points-1 get s_k = 1 for all
 *                 members.  A plain forward call uses p = n_points; get_logits (models/reconstruction.py:13) uses
 *                 p = nbatch_points.
 *   out_sdf_dev   n_queries * n_points           out_anchors_dev  n_queries * n_loc * 3 (may be NULL)        */
int nphm_ensemble_query(nphm_ensemble *h, const float *xyz_dev, const float *latents_dev,
                        int n_queries, long long n_points, long long quirk_period,
                        float *out_sdf_dev, float *out_anchors_dev, int impl, void *stream);

/* Same for ONE latent over (a contiguous range of) the regular grid of
 * create_grid_points_from_bounds (utils/reconstruction.py:5-20): point g = first + i, i < count, has
 * (ix,iy,iz) = unravel(g, res^3), z fastest, coordinates float32(linspace_f64(min,max,res)[i*]).  The points are
 * generated in the kernel (no xyz traffic).  The quirk uses the GLOBAL index g, so shards agree with a
 * single-GPU run.  out_sdf_dev: count floats. */
int nphm_ensemble_query_grid(nphm_ensemble *h, const float *latent_dev,
                             const double grid_min[3], const double grid_max[3], int res,
                             long long first, long long count, long long quirk_period,
                             float *out_sdf_dev, float *out_anchors_dev, int impl, void *stream);

/* Host-buffer convenience used for end-to-end timing: latent_host (lat_dim floats) -> device, grid query of the
 * whole res^3 grid, volume -> out_host (res^3 floats).  Synchronous. */
int nphm_ensemble_get_logits_host(nphm_ensemble *h, const float *latent_host,
                                  const double grid_min[3], const double grid_max[3], int res,
                                  long long quirk_period, float *out_host, int impl);

/* ------------------------------------------------------------------------------------------------
 * Plain DeepSDF MLP == DeepSDF.forward (reference src/NPHM/models/deepSDF.py:6-89), also the backbone of
 * DeformationNetwork (:118-239) whose condition vector the host builds (compressor Linear, :218-223).
 * ---------------------------------------------------------------------------------------------- */
typedef struct nphm_mlp nphm_mlp;

typedef struct {
    int lat_dim;      /* condition width (232 for the deformation backbone)  */
    int hidden_dim;   /* 512                                                 */
    int n_layers;     /* hidden layers (6) -> n_layers+1 linear, skip at n_layers/2 */
    int out_dim;      /* 3                                                   */
} nphm_mlp_config;

/* accepts lat_dim >= 1, hidden_dim > lat_dim + 3, 2 <= n_layers <= 10, 1 <= out_dim <= 8 (else NPHM_ERR_INVALID) */
int nphm_mlp_create(const nphm_mlp_config *cfg, nphm_mlp **out);
void nphm_mlp_destroy(nphm_mlp *h);
/* w_dev[l]: (out_l, in_l) row-major, b_dev[l]: (out_l), l = 0..n_layers (keys lin{l}.weight/bias). */
int nphm_mlp_load_weights(nphm_mlp *h, const float *const *w_dev, const float *const *b_dev, void *stream);
/* xyz_dev n_queries*n_points*3, cond_dev n_queries*lat_dim -> out_dev n_queries*n_points*out_dim.
 * impl: NPHM_IMPL_AUTO picks the tensor-core path for the deformation-backbone configuration (hidden 512, 6 hidden layers,
 * condition 232, 3 outputs) and the fp32 FFMA kernel otherwise; NPHM_IMPL_SIMT / NPHM_IMPL_TC force one. */
int nphm_mlp_query(nphm_mlp *h, const float *xyz_dev, const float *cond_dev, int n_queries,
                   long long n_points, float *out_dev, int impl, void *stream);

/* Batched Broyden search for canonical correspondences: roots of  x + F(x; cond) - obs  per point, F = this MLP
 * (3 outputs).  Replaces the Python loop of models/iterative_root_finding.py:5-71 (`broyden`) with the residual of
 * `search` (:142-147): same update rule, thresholds and freeze logic, one fused-MLP launch per step, no host
 * round trips except a 4-byte "still active?" read every 3 steps (the reference's early exit).
 *   x_dev          in: start points, out: 'result' (n_queries*n_points*3) - like the reference this is the point at
 *                  which a sample stopped, not the best one seen (its x_opt aliases x)
 *   jinv_init_dev  n_queries*n_points*9 row-major initial inverse Jacobians (not modified)
 *   diff_dev       out: smallest residual norm seen per sample; valid_dev out: diff < cvg_thresh (1 byte each)
 *   steps_done     host int.  NULL = sync-free call (CUDA-graph capturable): no early-exit read-back, all max_steps run; frozen
 *                  samples do not move any more, so the result is identical.
 *   workspace_dev: nphm_broyden_workspace_bytes(n_queries*n_points) bytes. */
long long nphm_broyden_workspace_bytes(long long n_total);
int nphm_mlp_broyden_search(nphm_mlp *h, const float *cond_dev, int n_queries, long long n_points,
                            const float *obs_dev, float *x_dev, const float *jinv_init_dev, int max_steps,
                            float cvg_thresh, float dvg_thresh, float eps, float *diff_dev,
                            unsigned char *valid_dev, int *steps_done, void *workspace_dev, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Marching cubes == mcubes.marching_cubes(volume, iso) as called at utils/reconstruction.py:30
 * (PyMCubes semantics restated in oracle/mc_oracle.c: x-major cell order, `<=` classification, one vertex per
 * crossed grid edge numbered in creation order, double-precision interpolation, classic 256-case table).
 * The volume is a slab of nx planes (x slowest, z fastest) that may be a shard of a larger grid.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
    int nx, ny, nz;       /* planes / rows / columns of vol_dev                                               */
    int x_global0;        /* global x index of plane 0 (0 for a whole volume)                                 */
    int ghost_lo;         /* 1: the first cell layer belongs to the previous shard; it is classified so that
                             shared vertices resolve to the right ids, but emits nothing                      */
    int negate;           /* 1: run on -vol (mesh_from_logits negates the SDF, utils/reconstruction.py:25)    */
    double iso;
} nphm_mc_params;

/* bytes of scratch the two calls below need for this slab */
long long nphm_mc_workspace_bytes(const nphm_mc_params *p);
/* Pass 1: classify + count.  Writes the number of vertices / triangles this slab emits to the two host
 * integers (synchronises the stream). */
int nphm_mc_count(const float *vol_dev, const nphm_mc_params *p, void *workspace_dev,
                  long long *n_verts_host, long long *n_tris_host, void *stream);
/* Pass 2 (after nphm_mc_count on the same workspace): emit.  verts_dev: n_verts*3 doubles in GLOBAL index units;
 * tris_dev: n_tris*3 int64 vertex ids offset by vert_id_base (the number of vertices emitted by all earlier
 * shards; 0 for a whole volume). */
int nphm_mc_emit(const float *vol_dev, const nphm_mc_params *p, void *workspace_dev,
                 long long vert_id_base, double *verts_dev, long long *tris_dev, void *stream);
/* Host-buffer convenience == mcubes.marching_cubes on a host volume: two-call protocol, call with
 * verts_host == NULL to get the counts. Synchronous. */
int nphm_marching_cubes_host(const float *vol_host, int nx, int ny, int nz, double iso, int negate,
                             double *verts_host, long long *tris_host,
                             long long *n_verts, long long *n_tris);

/* ------------------------------------------------------------------------------------------------
 * Identity-space fitting step == one iteration of inference_identity_space
 * (reference src/NPHM/models/fitting.py:197-279): ensemble forward on the sampled observation points, clamped
 * |sdf| loss, latent regularisers, analytic gradient w.r.t. the latent (through the member inputs, the
 * anchors/mlp_pos and the blend weights), torch.optim.Adam update.  No autograd graph.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
    float lambda_surface, lambda_reg_global, lambda_reg_loc, lambda_reg_unobserved, lambda_symm_dist;
    float clamp;          /* keep |sdf| < clamp (0.1 / 0.05 / 0.0075 by iteration, :239-246)                */
    float lr;             /* current Adam lr                                                                 */
    int   step;           /* 1-based Adam step count                                                         */
} nphm_fit_params;

/* bytes of scratch for n_points observation points */
long long nphm_fit_workspace_bytes(const nphm_ensemble *h, long long n_points);
/* latent_dev (lat_dim) is updated in place; adam_m_dev / adam_v_dev are the optimiser state (lat_dim each,
 * zero-initialised by the caller).  loss_terms_dev (may be NULL) receives
 * [surface, reg_global, reg_loc, reg_unobserved, symm_dist, n_kept].  grad_out_dev (may be NULL) receives the
 * latent gradient (lat_dim). If `apply_update` is 0 only loss/gradient are produced. */
int nphm_fit_identity_step(nphm_ensemble *h, const float *points_dev, long long n_points,
                           float *latent_dev, float *adam_m_dev, float *adam_v_dev,
                           const nphm_fit_params *fp, int apply_update,
                           float *loss_terms_dev, float *grad_out_dev,
                           void *workspace_dev, void *stream);

/* Surface term of the joint fitter with gradients w.r.t. BOTH the identity code and the query points
 * (reference src/NPHM/models/fitting.py:114-125: `sdf = decoder(xc, lat_rep_shape)`, `sdf[valid_ids]`, `l[l < clamp].mean()`):
 *   loss = mean over { p : mask[p] != 0 and |sdf_p| < clamp } of |sdf_p|        (training-mode forward, no eval quirk)
 * mask_dev (n_points bytes, may be NULL = all valid).  loss_terms_dev[0] = loss (NaN if nothing is kept, like torch),
 * [5] = number of kept points, [1..4] = the latent regularisers (unweighted).  grad_latent_dev (lat_dim) and
 * grad_points_dev (n_points*3, may be NULL) receive d loss / d latent (member inputs + anchors/mlp_pos + blend weights) and
 * d loss / d point (local coordinates of every member + blend weights); both are zero when nothing is kept.
 * The latent is not modified.  Same workspace as nphm_fit_identity_step.  Needs the tensor-core configuration when
 * grad_points_dev is given. */
int nphm_fit_surface_grad(nphm_ensemble *h, const float *points_dev, long long n_points, const float *latent_dev,
                          const unsigned char *mask_dev, float clamp, float *loss_terms_dev,
                          float *grad_latent_dev, float *grad_points_dev, void *workspace_dev, void *stream);

/* ------------------------------------------------------------------------------------------------
 * DeepSDF-style stacks layer by layer on the generic fp32-accurate wgmma linear layer (csrc/tc_linear.cu, mlp_chain.cu).
 * ---------------------------------------------------------------------------------------------- */
/* == nphm_mlp_query for ANY width (DeepSDF.forward, reference src/NPHM/models/deepSDF.py:64-89; e.g. the NPM baseline
 * 515 -> 1024 x 8 of scripts/configs/npm.yaml:2-4, which no fused kernel takes). */
int nphm_mlp_query_layers(nphm_mlp *h, const float *xyz_dev, const float *cond_dev, int n_queries, long long n_points,
                          float *out_dev, void *stream);
/* Value and input Jacobian in one forward-mode pass == `jac` (reference src/NPHM/models/diff_operators.py:26-54: three
 * autograd passes) without the identity term:  out_dev [q][n][out_dim] (may be NULL), jac_dev [q][n][out_dim][3] = d out / d xyz.
 * Callers: iterative_root_finding.py:123 (initial inverse Jacobian of the Broyden search), fitting.py:104 (implicit
 * differentiation of the root). */
int nphm_mlp_jacobian(nphm_mlp *h, const float *xyz_dev, const float *cond_dev, int n_queries, long long n_points,
                      float *out_dev, float *jac_dev, void *stream);
/* Adjoint pass == what loss.backward() (reference src/NPHM/models/fitting.py:167) propagates through the deformation
 * network:  grad_cond_dev [q][lat_dim] = sum_n (d out_n / d cond_q)^T grad_out_n  (may be NULL),
 *           grad_xyz_dev [q][n][3]    = (d out_n / d xyz_n)^T grad_out_n            (may be NULL).   grad_out_dev: [q][n][out_dim].
 * xyz_dev == NULL: reuse the activations of the preceding nphm_mlp_jacobian / nphm_mlp_inverse_jacobian call on this handle
 * (same points, same condition) instead of recomputing the value pass.  grad_out may have any magnitude: each query's
 * upstream is scaled on the device by a power of two into the range of the fp16 adjoint, and the gradients scaled back. */
int nphm_mlp_backward_inputs(nphm_mlp *h, const float *xyz_dev, const float *cond_dev, int n_queries, long long n_points,
                             const float *grad_out_dev, float *grad_cond_dev, float *grad_xyz_dev, void *stream);
/* (I + d out / d xyz)^-1 per point for a 3-output stack == `jac(decoder_expr, x, ...).inverse()` of the reference
 * (iterative_root_finding.py:123, fitting.py:104): out_dev [q][n][3] (may be NULL), jinv_dev [q][n][3][3]. */
int nphm_mlp_inverse_jacobian(nphm_mlp *h, const float *xyz_dev, const float *cond_dev, int n_queries, long long n_points,
                              float *out_dev, float *jinv_dev, void *stream);

/* ---- training (first order): the stage-2 loss of the reference (src/NPHM/models/loss_functions.py:282-322, stepped by
 * training_corresp.py:154-176) differentiated to the weights on the tensor cores.  A forward keeps everything its backward
 * needs in a caller-owned device workspace, so several forwards may be alive at once; the backward reads nothing from the
 * handle except the packed weights.
 * Per-row condition noise: cond_noise_dev [q][n][noise_dim] is added to the leading noise_dim condition columns of every
 * point (the train-mode `compressed += randn(...) / 200` of deepSDF.py:220-221); noise_dim = 0: none. */
/* bytes of the workspace of one nphm_mlp_train_forward call (-1: bad arguments) */
long long nphm_mlp_train_workspace_bytes(const nphm_mlp *h, int n_queries, long long n_points, int noise_dim);
/* value pass of DeepSDF.forward (deepSDF.py:64-89): out_dev [q][n][out_dim]; activations, their derivatives, the staged
 * [xyz | noise] rows and a copy of cond_dev [q][lat_dim] go to workspace_dev (nphm_mlp_train_workspace_bytes bytes). */
int nphm_mlp_train_forward(nphm_mlp *h, const float *xyz_dev, const float *cond_dev, const float *cond_noise_dev, int noise_dim,
                           int n_queries, long long n_points, float *out_dev, void *workspace_dev, void *stream);
/* what autograd's backward of that forward gives for the upstream gradient grad_out_dev [q][n][out_dim]:
 * grad_w_dev[l] / grad_b_dev[l] in the state_dict layout of lin{l}.weight / bias (overwritten; the arrays or entries may be
 * NULL = not needed), grad_cond_dev [q][lat_dim] (summed over the points of a query), grad_xyz_dev [q][n][3] (may be NULL).
 * Deterministic: the same inputs give bitwise-identical gradients.  workspace_bytes / noise_dim / n_queries / n_points: the
 * size of the workspace and the shape of the forward that filled it; rejected (NPHM_ERR_INVALID) when the size does not match
 * that shape on this network.  Nothing is read back from the device: the call does not wait for the stream. */
int nphm_mlp_train_backward(nphm_mlp *h, const float *grad_out_dev, const void *workspace_dev, long long workspace_bytes,
                            int noise_dim, int n_queries, long long n_points,
                            float *const *grad_w_dev, float *const *grad_b_dev, float *grad_cond_dev, float *grad_xyz_dev,
                            void *stream);

/* ---- training through the spatial gradient: the stage-1 loss of the reference (src/NPHM/models/loss_functions.py:20-110,
 * scripts/training/train.py) reaches a one-output DeepSDF stack through s = f(x) and g = grad_x s, so its normal and eikonal
 * terms need second derivatives.  Stacks with out_dim != 1 are rejected with NPHM_ERR_UNSUPPORTED.  As for the first-order
 * calls, a forward keeps what its backward needs in a caller-owned device workspace. */
/* bytes of the workspace of one nphm_mlp_sdfgrad_forward call (-1: bad arguments) */
long long nphm_mlp_sdfgrad_workspace_bytes(const nphm_mlp *h, int n_queries, long long n_points);
/* sdf_out_dev [q][n] = f(xyz, cond), grad_out_dev [q][n][3] = d sdf / d xyz (value pass and one adjoint pass with unit
 * upstream); xyz_dev [q][n][3], cond_dev [q][lat_dim]. */
int nphm_mlp_sdfgrad_forward(nphm_mlp *h, const float *xyz_dev, const float *cond_dev, int n_queries, long long n_points,
                             float *sdf_out_dev, float *grad_out_dev, void *workspace_dev, void *stream);
/* what autograd's backward of that forward gives for upstream gradients grad_sdf_dev [q][n] and grad_grad_dev [q][n][3]:
 * grad_w_dev[l] / grad_b_dev[l] in the state_dict layout of lin{l}.weight / bias (overwritten; the arrays or entries may be
 * NULL), grad_cond_dev [q][lat_dim] (summed over the points of a query, may be NULL), grad_xyz_dev [q][n][3] (may be NULL).
 * The tail of the workspace is the call's scratch (its whole per-point memory; the handle only keeps buffers of the layer
 * widths), so the call writes to it; what the forward stored is left as it was.
 * Deterministic; workspace_bytes / n_queries / n_points state the forward that filled the workspace and are checked against
 * its size (NPHM_ERR_INVALID on a mismatch; a shape with the same workspace size is not detected).  Nothing is read back
 * from the device. */
int nphm_mlp_sdfgrad_backward(nphm_mlp *h, const float *grad_sdf_dev, const float *grad_grad_dev, void *workspace_dev,
                              long long workspace_bytes, int n_queries, long long n_points, float *const *grad_w_dev,
                              float *const *grad_b_dev, float *grad_cond_dev, float *grad_xyz_dev, void *stream);

/* ---- the same for the members of the ensemble (stage 1 of NPHM, train.py -local): every member k of the handle as a
 * one-output stack with its weight set, one launch per pass for all members.  Member-major layouts: xyz_local_dev and
 * grad_xyz_dev [members][B][N][3] in each member's frame (the caller applies the mirror), cond_dev and grad_cond_dev
 * [members][B][lat_dim_glob + lat_dim_loc], sdf_out_dev [members][B][N], grad_out_dev [members][B][N][3], grad_w_dev[l] /
 * grad_b_dev[l] in the state_dict layout of ensembled_deep_sdf.lin{l}.weight / bias ([sets][out][in], [sets][out]; a mirrored
 * set sums its two members).  Workspace contract and determinism as for nphm_mlp_sdfgrad_*; the upstream gradients are
 * scaled by one power of two per weight set, so a set whose upstream is all zero gets exactly zero gradients. */
long long nphm_ensemble_sdfgrad_workspace_bytes(const nphm_ensemble *h, int n_batch, long long n_points);
int nphm_ensemble_sdfgrad_forward(nphm_ensemble *h, const float *xyz_local_dev, const float *cond_dev, int n_batch,
                                  long long n_points, float *sdf_out_dev, float *grad_out_dev, void *workspace_dev, void *stream);
int nphm_ensemble_sdfgrad_backward(nphm_ensemble *h, const float *grad_sdf_dev, const float *grad_grad_dev, void *workspace_dev,
                                   long long workspace_bytes, int n_batch, long long n_points, float *const *grad_w_dev,
                                   float *const *grad_b_dev, float *grad_cond_dev, float *grad_xyz_dev, void *stream);

/* ---- fitting with a one-output DeepSDF stack (the NPM baseline's identity decoder): the surface term of
 * inference_identity_space and inference_iterative_root_finding_joint (reference src/NPHM/models/fitting.py:114-125, :229-247)
 *   loss = mean over { p : mask[p] != 0 and |s_p| < clamp } of |s_p|,   s = f(xyz, cond)
 * Stacks with out_dim != 1 are rejected with NPHM_ERR_UNSUPPORTED. */
/* bytes of the workspace of one nphm_mlp_fit_surface_grad call (-1: bad arguments) */
long long nphm_mlp_fit_workspace_bytes(const nphm_mlp *h, int n_queries, long long n_points);
/* xyz_dev [q][n][3], cond_dev [q][lat_dim], mask_dev [q*n] bytes (may be NULL = all valid).  loss_terms_dev[0] = loss (NaN if
 * nothing is kept, like torch), [5] = number of kept points, [1..4] = 0 (the layout of nphm_fit_surface_grad).
 * grad_cond_dev [q][lat_dim] = d loss / d cond_q (summed over the points of the query), grad_xyz_dev [q][n][3] (may be NULL);
 * both exactly zero when nothing is kept.  All per-point memory is the caller's workspace; workspace_bytes is checked against
 * the shape (NPHM_ERR_INVALID on a mismatch).  Bitwise deterministic; nothing is read back from the device. */
int nphm_mlp_fit_surface_grad(nphm_mlp *h, const float *xyz_dev, const float *cond_dev, int n_queries, long long n_points,
                              const unsigned char *mask_dev, float clamp, float *loss_terms_dev, float *grad_cond_dev,
                              float *grad_xyz_dev, void *workspace_dev, long long workspace_bytes, void *stream);
/* The same surface term per scan, for S scans of n points in one launch sequence (the scan-batched NPM fitters): scan k has its
 * own kept set (mask != 0 and |s| < clamp over its own rows), its own loss and its own gradients.  xyz_dev [S][n][3], cond_dev
 * [S][lat_dim], mask_dev [S][n] bytes (may be NULL = all valid).  loss_terms_dev [S][8] in the layout above; grad_cond_dev
 * [S][lat_dim] = d loss_k / d cond_k, grad_xyz_dev [S][n][3] (may be NULL) = d loss_k / d xyz over scan k's rows.  A scan with
 * nothing kept gets a NaN loss and exactly zero gradients and leaves the others unaffected.  The workspace is that of
 * nphm_mlp_fit_workspace_bytes(h, S, n) (checked: NPHM_ERR_INVALID on a mismatch).  Bitwise deterministic; nothing is read back
 * from the device.  Scan k's result equals a single call on its rows up to one rounding of the gradients (the factor 1 / n_kept
 * is applied after the chain). */
int nphm_mlp_fit_surface_grad_batched(nphm_mlp *h, const float *xyz_dev, const float *cond_dev, const unsigned char *mask_dev,
                                      int n_scans, long long n_points, float clamp, float *loss_terms_dev, float *grad_cond_dev,
                                      float *grad_xyz_dev, void *workspace_dev, long long workspace_bytes, void *stream);

/* anchors_dev [n_queries][n_loc][3] = mlp_pos(z_glob) + mean anchors (reference src/NPHM/models/EnsembledDeepSDF.py:228-229)
 * without evaluating the ensemble - what the fitters read from `decoder(zeros(1,1,3), lat)[1]` (fitting.py:59, :211). */
int nphm_ensemble_anchors(nphm_ensemble *h, const float *latents_dev, int n_queries, float *anchors_dev, void *stream);

/* Vector-Jacobian product of the ensemble forward w.r.t. its inputs == what torch.autograd computes for
 * `decoder(xyz, lat)[0].backward(grad_sdf)` on FastEnsembleDeepSDFMirrored in training mode (reference
 * src/NPHM/models/EnsembledDeepSDF.py:203-267; used by fitting.py:111-167 through loss.backward()):
 *   grad_points_dev[p] = grad_sdf[p] * d sdf_p / d xyz_p      (n_points * 3, may be NULL)
 *   grad_latent_dev    = sum_p grad_sdf[p] * d sdf_p / d latent  (lat_dim: member inputs + anchors/mlp_pos + blend weights)
 * sdf_out_dev (n_points, may be NULL) receives the forward values.  Same workspace as nphm_fit_identity_step. */
int nphm_ensemble_backward_inputs(nphm_ensemble *h, const float *points_dev, long long n_points, const float *latent_dev,
                                  const float *grad_sdf_dev, float *sdf_out_dev, float *grad_latent_dev,
                                  float *grad_points_dev, void *workspace_dev, void *stream);

/* ---- the same in eval mode: FastEnsembleDeepSDFMirrored.forward after decoder.eval() overwrites every member's output at the
 * last point of each decoder call with 1 (reference src/NPHM/models/EnsembledDeepSDF.py:260-261, `sdf_pred[:, :, -1, 0] = 1`).
 * Row i (0-based, within a scan) is such a quirk row when quirk_period p > 0 and i % p == p - 1; p = 0 is the training-mode
 * forward and gives the results of the calls above bit for bit.  At a quirk row s_k = 1 and grad s_k = 0 for all members k, so
 *   sdf = sum_k wt_k (the normalised blend weights, background included),   d sdf / d xyz = sum_k d wt_k / d xyz,
 * the member inputs get no gradient from the row, the anchors / mlp_pos / z_glob do, through the weights.  Only the
 * tensor-core configuration (hidden 200, 4 hidden layers, condition 96) takes p > 0 (else NPHM_ERR_UNSUPPORTED).
 * == nphm_fit_identity_step for one iteration of inference_identity_space with the decoder in eval mode (fitting.py:229-236:
 *    one call on the 5 sampled rows of n points each, so p = n) */
int nphm_fit_identity_step_quirk(nphm_ensemble *h, const float *points_dev, long long n_points, long long quirk_period,
                                 float *latent_dev, float *adam_m_dev, float *adam_v_dev, const nphm_fit_params *fp,
                                 int apply_update, float *loss_terms_dev, float *grad_out_dev, void *workspace_dev, void *stream);
/* == nphm_fit_surface_grad for the joint fitter in eval mode (fitting.py:111-125: `decoder(xc, ...)` on the 5 sampled rows of n
 *    points, p = n) */
int nphm_fit_surface_grad_quirk(nphm_ensemble *h, const float *points_dev, long long n_points, long long quirk_period,
                                const float *latent_dev, const unsigned char *mask_dev, float clamp, float *loss_terms_dev,
                                float *grad_latent_dev, float *grad_points_dev, void *workspace_dev, void *stream);
/* == nphm_ensemble_backward_inputs for `decoder.eval(); decoder(xyz, lat)[0].backward(grad_sdf)`: p = n_points is one call
 *    (the stage-1 losses, loss_functions.py:36-42, make one call per point set) */
int nphm_ensemble_backward_inputs_quirk(nphm_ensemble *h, const float *points_dev, long long n_points, long long quirk_period,
                                        const float *latent_dev, const float *grad_sdf_dev, float *sdf_out_dev,
                                        float *grad_latent_dev, float *grad_points_dev, void *workspace_dev, void *stream);

/* Second half of a fitting iteration (regularisers of fitting.py:252-268 + torch.optim.Adam, :278-279) for a surface
 * gradient that was evaluated elsewhere: the point-sharded fit of one head over several GPUs (north_star / SURVEY.md 8e)
 * evaluates nphm_fit_surface_grad on every rank's share of the sampled points, combines [n_r * grad_r, n_r * loss_r, n_r]
 * with ONE all-reduce and then calls this on every rank with the identical global result.
 * surface_grad_dev: d(mean |sdf| over the kept points)/d latent (lat_dim, un-weighted: lambda_surface is applied here);
 * surface_stats_dev: [n_kept, sum |sdf| over the kept points]; loss_terms_dev as in nphm_fit_identity_step (may be NULL).
 * grad_anchors_dev (n_loc*3, may be NULL): an additional gradient w.r.t. the anchors, back-propagated through mlp_pos into
 * z_glob (joint fitter: the deformation network is conditioned on the anchors, deepSDF.py:218-219); also scaled by
 * lambda_surface.  apply_update = 0: only the total gradient (grad_out_dev, lat_dim, may be NULL) and the loss terms. */
int nphm_fit_apply_gradient(nphm_ensemble *h, float *latent_dev, float *adam_m_dev, float *adam_v_dev,
                            const nphm_fit_params *fp, const float *surface_grad_dev, const float *surface_stats_dev,
                            const float *grad_anchors_dev, int apply_update, float *loss_terms_dev, float *grad_out_dev,
                            void *stream);

/* ---- scan-batched fitting: S independent scans (or subjects) in one launch sequence per iteration, each with its own latent
 * code, Adam moments and points; all scans share fp (schedule, clamp, lr, Adam step).  The result for scan s is what the
 * single-scan call gives on that scan alone (up to the order of floating-point sums): a scan is reduced only over its own
 * points, and a scan with nothing kept behaves as the single-scan call does (NaN surface loss, zero surface gradient).
 * Layouts: points_dev [S][n_points][3], mask_dev [S][n_points] bytes (may be NULL = all valid; rows with mask 0 are left out of
 * the loss - padding of a shorter scan, which should repeat one of its valid points so that it stays finite), latents_dev /
 * adam_m_dev / adam_v_dev / grad_out_dev / grad_latent_dev [S][lat_dim], loss_terms_dev [S][8], grad_points_dev [S][n_points][3].
 * The workspace is the caller's: workspace_bytes (checked, NPHM_ERR_CAPACITY when short) >= nphm_fit_batch_workspace_bytes.
 * The step and the surface gradient run only on the tensor-core configuration (hidden 200, 4 hidden layers, condition 96):
 * NPHM_ERR_UNSUPPORTED otherwise.  Nothing is read back from the device. */
/* bytes of scratch for n_scans scans of n_points observation points each (-1: bad arguments) */
long long nphm_fit_batch_workspace_bytes(const nphm_ensemble *h, int n_scans, long long n_points);
/* == nphm_fit_identity_step per scan, with an optional point mask */
int nphm_fit_identity_step_batched(nphm_ensemble *h, const float *points_dev, const unsigned char *mask_dev, int n_scans,
                                   long long n_points, float *latents_dev, float *adam_m_dev, float *adam_v_dev,
                                   const nphm_fit_params *fp, int apply_update, float *loss_terms_dev, float *grad_out_dev,
                                   void *workspace_dev, long long workspace_bytes, void *stream);
/* == nphm_fit_surface_grad per scan; loss_terms_dev and grad_latent_dev are required */
int nphm_fit_surface_grad_batched(nphm_ensemble *h, const float *points_dev, const unsigned char *mask_dev, int n_scans,
                                  long long n_points, const float *latents_dev, float clamp, float *loss_terms_dev,
                                  float *grad_latent_dev, float *grad_points_dev, void *workspace_dev, long long workspace_bytes,
                                  void *stream);
/* The same two in eval mode (see nphm_fit_identity_step_quirk): quirk_periods_dev [S] int32 on the device (may be NULL = all 0)
 * holds each scan's period, the points per sampled observation row of that scan (n_k = min(1000, |obs|), fitting.py:111/114,
 * :234/236); a scan's rows are numbered from 0 within the scan, so the padding after its last row is never a quirk row of it. */
int nphm_fit_identity_step_batched_quirk(nphm_ensemble *h, const float *points_dev, const unsigned char *mask_dev, int n_scans,
                                         long long n_points, const int *quirk_periods_dev, float *latents_dev, float *adam_m_dev,
                                         float *adam_v_dev, const nphm_fit_params *fp, int apply_update, float *loss_terms_dev,
                                         float *grad_out_dev, void *workspace_dev, long long workspace_bytes, void *stream);
int nphm_fit_surface_grad_batched_quirk(nphm_ensemble *h, const float *points_dev, const unsigned char *mask_dev, int n_scans,
                                        long long n_points, const int *quirk_periods_dev, const float *latents_dev, float clamp,
                                        float *loss_terms_dev, float *grad_latent_dev, float *grad_points_dev,
                                        void *workspace_dev, long long workspace_bytes, void *stream);
/* == nphm_fit_apply_gradient per scan: surface_grad_dev [S][lat_dim], surface_stats_dev [S][2], grad_anchors_dev
 * [S][n_loc*3] (may be NULL), loss_terms_dev [S][8] and grad_out_dev [S][lat_dim] (may be NULL).  Any ensemble configuration;
 * the scratch is the handle's. */
int nphm_fit_apply_gradient_batched(nphm_ensemble *h, int n_scans, float *latents_dev, float *adam_m_dev, float *adam_v_dev,
                                    const nphm_fit_params *fp, const float *surface_grad_dev, const float *surface_stats_dev,
                                    const float *grad_anchors_dev, int apply_update, float *loss_terms_dev, float *grad_out_dev,
                                    void *stream);
/* torch.optim.Adam.step() (lr, betas 0.9/0.999, eps 1e-8) on a dense fp32 tensor: the expression codes of the joint fitter
 * (reference src/NPHM/models/fitting.py:36,169).  step is the 1-based step count. */
int nphm_adam_step(float *param_dev, const float *grad_dev, float *adam_m_dev, float *adam_v_dev, long long n, float lr,
                   int step, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Evaluation metrics (SURVEY.md 8f-4): nearest-neighbour distances between two point clouds ==
 * scipy.spatial.cKDTree(tgt).query(src) as used by `distance_p2p` (reference src/NPHM/evaluation/metrics.py:171-194) on
 * 250 k-point clouds (scripts/evaluation/eval.py:111).  dist_dev: n_src fp64, idx_dev: n_src int64.
 * ---------------------------------------------------------------------------------------------- */
int nphm_nearest_neighbors(const float *src_dev, long long n_src, const float *tgt_dev, long long n_tgt,
                           double *dist_dev, long long *idx_dev, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Depth / normal rendering of a triangle mesh into V views in one call: the images pyrender hands to `render_glcam`
 * (reference src/NPHM/evaluation/render_utils.py:26-89), which `gen_render_samples` (:169-201) and
 * scripts/data_processing/generate_single_view_observations.py back-project into point clouds.
 * verts_dev: n_verts x 3 fp32 (world); faces_dev: n_faces x 3 int32, every index in [0, n_verts) - a PRECONDITION, not checked
 * here (the Python layer checks it); n_faces == 0 renders all background.  world_to_eye_dev: V x 3 x 4 fp64 (row-major, the
 * inverse of the camera pose; the camera looks down -z with +y up); intrinsics_dev: V x 4 fp64 (fx, fy, cx, cy).
 * Pixel (r, c) of a height x width image (row 0 at the top) samples the eye ray ((c + 0.5 - cx)/fx, (cy - r - 0.5)/fy, -1).
 * Outputs, V x height x width, row-major: depth_dev fp32 eye depth (-z_eye, fragments kept for znear <= d <= zfar; 0 =
 * background), normals_dev 3 bytes per pixel round(clamp(0.5 n + 0.5, 0, 1) * 255) of the unit world-space face normal
 * cross(v1 - v0, v2 - v0), not flipped toward the camera (0, 0, 0 = background), tri_dev (may be NULL) the winning face
 * (-1 = background).  Nearest depth wins, ties go to the lower face index; faces are not culled.  Bitwise deterministic.
 * workspace_bytes (checked, NPHM_ERR_CAPACITY when short) >= nphm_render_workspace_bytes(n_views, height, width).
 * Needs 1 <= n_views <= 65535, height, width >= 1, 0 < znear < zfar (else NPHM_ERR_INVALID).
 * ---------------------------------------------------------------------------------------------- */
/* bytes of scratch for n_views views of height x width (-1: bad arguments) */
long long nphm_render_workspace_bytes(int n_views, int height, int width);
int nphm_render_depth_normals(const float *verts_dev, long long n_verts, const int *faces_dev, long long n_faces,
                              const double *world_to_eye_dev, const double *intrinsics_dev, int n_views, double znear,
                              double zfar, int height, int width, float *depth_dev, unsigned char *normals_dev, int *tri_dev,
                              void *workspace_dev, long long workspace_bytes, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Narrow-band mesh extraction: the steps of extract_mesh_narrowband (nphm_b200/utils/reconstruction.py, DESIGN §4.13), which
 * gives the mesh of `mesh_from_logits(get_logits(...))` on a res^3 grid while evaluating the decoder only near the surface.
 * The (res-1)^3 cells are split into blocks of block^3 cells (the last block of an axis may be partial); block b covers the
 * voxels [b*block, min(b*block + block, res-1)] of every axis.  The decoder is evaluated by the caller, through the existing
 * query entry points, on coordinates these calls gather; the band state lives in the caller's workspace:
 *   nphm_band_begin      resets the state; quirk_period > 0: lists the eval-mode quirk voxels (g % p == p-1 or g == res^3-1,
 *                        which the caller evaluates in a query of period 1) and activates every block owning a cell that touches one
 *   nphm_band_corners    lists the block corners not evaluated yet (fine indices 0, block, 2 block, ..., res-1)
 *   nphm_band_classify   activates the blocks with a corner |sdf| <= tau (or NaN) or corners on both sides of the marching-cubes
 *                        test (-sdf <= 0), then lists the voxels of all newly activated blocks not evaluated yet
 *   nphm_band_grow       activates every inactive block with an evaluated face voxel on the other side of the test from its
 *                        corner 0, then lists as classify does (0 listed: the band is closed)
 *   nphm_band_fill       gives every voxel not evaluated the value of corner 0 of an (inactive) block containing it
 * A listing call writes its list, ascending in the flat index z + res (y + res x), to the workspace and, when counts_host is not
 * NULL, {voxels listed, blocks active so far} to counts_host[0..1] (synchronises the stream).  nphm_band_gather writes the
 * float32(linspace_f64(min, max, res)) coordinates of the first n listed voxels to xyz_dev (n x 3; those of
 * create_grid_points_from_bounds and nphm_ensemble_query_grid); nphm_band_scatter writes values_dev[i] to vol_dev[list[i]]
 * (i < n), and every listed voxel counts as evaluated.  vol_dev: res^3 floats, x slowest.
 * Needs 2 <= res <= 1024, 1 <= block <= 64, tau >= 0 (else NPHM_ERR_INVALID); workspace_bytes (checked, NPHM_ERR_CAPACITY when
 * short) >= nphm_band_workspace_bytes(res, block). */
/* bytes of the band workspace (-1: bad arguments) */
long long nphm_band_workspace_bytes(int res, int block);
int nphm_band_begin(int res, int block, long long quirk_period, void *workspace_dev, long long workspace_bytes,
                    long long *counts_host, void *stream);
int nphm_band_corners(int res, int block, void *workspace_dev, long long workspace_bytes, long long *counts_host, void *stream);
int nphm_band_gather(int res, int block, const double grid_min[3], const double grid_max[3], long long n, float *xyz_dev,
                     void *workspace_dev, long long workspace_bytes, void *stream);
int nphm_band_scatter(int res, int block, long long n, const float *values_dev, float *vol_dev, void *workspace_dev,
                      long long workspace_bytes, void *stream);
int nphm_band_classify(int res, int block, float tau, const float *vol_dev, void *workspace_dev, long long workspace_bytes,
                       long long *counts_host, void *stream);
int nphm_band_grow(int res, int block, const float *vol_dev, void *workspace_dev, long long workspace_bytes, long long *counts_host,
                   void *stream);
int nphm_band_fill(int res, int block, float *vol_dev, void *workspace_dev, long long workspace_bytes, void *stream);
/* states_dev (blocks^3 bytes, blocks = ceil((res-1)/block), x slowest): 0 inactive, 1 or 2 active */
int nphm_band_block_states(int res, int block, const void *workspace_dev, long long workspace_bytes, unsigned char *states_dev,
                           void *stream);

#ifdef __cplusplus
}
#endif
#endif /* NPHM_B200_H */
