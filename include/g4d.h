/*
 * g4d -- C-ABI of the H100-native fused deform + rasterize render path for 4D Gaussian Splatting.
 *
 * Plain C, plain pointers and sizes, no torch types.  Every pointer named `d_*` or documented as
 * "device" is a CUDA device pointer on the workspace's device; everything else is host memory.
 * All tensors are contiguous fp32 unless stated.  All entry points return 0 on success, a negative
 * G4D_ERR_* code otherwise (g4d_last_error() gives the text); nothing here ever falls back to a CPU
 * implementation.
 *
 * Reference interfaces replaced (file:line under /root/reference):
 *   g4d_rasterize_forward / _backward
 *       <- diff_gaussian_rasterization.GaussianRasterizer.forward / autograd backward, called at
 *          gaussian_renderer/__init__.py:120-128 with the settings built at :38-51
 *          (upstream: _C.rasterize_gaussians / _C.rasterize_gaussians_backward, SURVEY.md App. A.5)
 *   g4d_deform_forward / _backward (and _times: one time per row)
 *       <- scene/deformation.py:185-212 deform_network.forward (HexPlane scene/hexplane.py:73-106 +
 *          MLP scene/deformation.py:67-148) and its autograd backward
 *   g4d_render_forward / _backward
 *       <- gaussian_renderer/__init__.py:18-138 render(): deform (":87") + activations (":97-99") +
 *          rasterize (":120") as ONE fused device pass, no intermediate tensors through the caller
 *   G4DCamera
 *       <- GaussianRasterizationSettings (gaussian_renderer/__init__.py:38-51) + viewpoint_camera.time (":52")
 *   G4DDeformParams
 *       <- deform_network.state_dict() (SURVEY.md App. B.4); planes are channel-last views of the
 *          [1,C,H,W] checkpoint tensors, Linear weights are torch's [out,in] row-major
 */
#ifndef G4D_H_
#define G4D_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define G4D_ABI_VERSION 3
#define G4D_CAM_DEBUG 1
#define G4D_CAM_NO_GRAD 2
#define G4D_MAX_LEVELS 4
#define G4D_NUM_HEADS 5 /* pos, scales, rotations, opacity, shs (scene/deformation.py:61-65) */
#define G4D_MAX_DEPTH 8 /* defor_depth: Linear layers of the trunk feature_out (scene/deformation.py:55-60) */

enum {
    G4D_OK = 0,
    G4D_ERR_CUDA = -1,      /* a CUDA runtime call or kernel failed */
    G4D_ERR_ARG = -2,       /* invalid argument / unsupported configuration */
    G4D_ERR_NOMEM = -3,     /* device allocation failed */
    G4D_ERR_STATE = -4,     /* backward without a matching forward, ... */
    G4D_ERR_OVERFLOW = -5   /* tile-instance buffer overflowed in no-sync mode (re-run with sync), or an FP16x2 tensor-core
                             * launch met a value outside the f16 operand range (G4D_OPT_TENSOR_CORES = 2; 0 has no
                             * range limit) */
};

enum { /* bits of G4DDeformParams.head_mask: a set bit means the head is ACTIVE (not no_dx etc.) */
    G4D_HEAD_POS = 1, G4D_HEAD_SCALES = 2, G4D_HEAD_ROT = 4, G4D_HEAD_OPACITY = 8, G4D_HEAD_SHS = 16
};

typedef struct G4DWorkspace G4DWorkspace; /* per-device scratch, packed-parameter cache */
typedef struct G4DContext G4DContext;     /* state one forward keeps for its backward */

typedef struct G4DCamera {
    int32_t image_height, image_width;
    int32_t sh_degree; /* active SH degree 0..3 */
    int32_t debug;     /* bit 0: synchronise + check after every stage (settings.debug);
                        * bit 1 (G4D_CAM_NO_GRAD): no backward will follow this forward (torch.no_grad rendering):
                        *        g4d_render_forward skips saving state that only the backward reads */
    float tanfovx, tanfovy, scale_modifier;
    float time;        /* viewpoint_camera.time; ignored by the plain rasterizer entry points */
    float viewmatrix[16]; /* world_view_transform, row-vector convention (scene/cameras.py:59) */
    float projmatrix[16]; /* full_proj_transform (scene/cameras.py:63) */
    float campos[3];
    float bg[3];
    /* optional DEVICE sources; when non-NULL they override the host arrays above (the reference
     * passes these four as CUDA tensors) */
    const float *d_viewmatrix, *d_projmatrix, *d_campos, *d_bg;
    /* SH coefficients M = (max_sh_degree + 1)^2 every Gaussian stores (sh.size(1) upstream): 1, 4, 9 or 16; 0 means 16, so a
     * zero-filled tail is the degree-3 model.  (sh_degree + 1)^2 <= M; the SHS head of the network needs M = 16; the cameras
     * of one g4d_render_*_cameras call share M.  Otherwise G4D_ERR_ARG before any launch. */
    int32_t sh_coeffs;
    int32_t reserved;
} G4DCamera;

typedef struct G4DDeformParams {
    int32_t levels;    /* len(multires) <= G4D_MAX_LEVELS */
    int32_t channels;  /* kplanes output_coordinate_dim: multiple of 4, <= 32 */
    int32_t net_width; /* 64 or 128 */
    int32_t head_mask; /* G4D_HEAD_* bits */
    int32_t res[G4D_MAX_LEVELS][4]; /* per level: resolution of x, y, z, t */
    /* device: plane k of level l, CHANNEL-LAST [H][W][C]; (H,W) = (res[c1], res[c0]) for the k-th
     * pair (c0,c1) of combinations(range(4),2)  (scene/hexplane.py:48-70); H*W*C < 2^31, and the
     * spatial planes (k = 0, 1, 3) 16-byte aligned (else G4D_ERR_ARG before any launch) */
    const float *planes[G4D_MAX_LEVELS][6];
    const float *aabb;      /* device [2][3]: row 0 = xyz_max, row 1 = xyz_min */
    const float *w0, *b0;   /* device: feature_out.0  [Wd][F], [Wd] */
    const float *w1[G4D_NUM_HEADS], *b1[G4D_NUM_HEADS]; /* device: <head>.1  [Wd][Wd], [Wd] */
    const float *w2[G4D_NUM_HEADS], *b2[G4D_NUM_HEADS]; /* device: <head>.3  [k][Wd], [k]; k = 3,3,4,1,48 */
    uint64_t version; /* caller bumps it whenever any weight changed (packed copies are cached) */
    /* the trunk behind feature_out.0: h_j = W_j relu(h_{j-1}) + b_j for j = 1 .. depth-1, every head reads h_{depth-1}.
     * depth 0 and 1 both mean no trunk layer (feature_out.0 alone); at most G4D_MAX_DEPTH, with every levels / channels /
     * head_mask / net_width the other fields allow.  A zero-filled tail is the network without trunk layers, so a caller
     * zero-initialises the struct. */
    int32_t depth;     /* defor_depth */
    int32_t reserved;
    const float *wt[G4D_MAX_DEPTH - 1], *bt[G4D_MAX_DEPTH - 1]; /* device: wt[j-1], bt[j-1] = feature_out.{2j}  [Wd][Wd], [Wd],
                                                                 * j = 1 .. depth-1 (non-NULL); the rest are not read */
} G4DDeformParams;

/* gradient sinks mirroring G4DDeformParams (device, same layouts; ACCUMULATED into, caller zeroes); the backward entry
 * points need the spatial-plane sinks (k = 0, 1, 3) 16-byte aligned (else G4D_ERR_ARG before any launch) */
typedef struct G4DDeformGrads {
    float *planes[G4D_MAX_LEVELS][6];
    float *w0, *b0;
    float *w1[G4D_NUM_HEADS], *b1[G4D_NUM_HEADS];
    float *w2[G4D_NUM_HEADS], *b2[G4D_NUM_HEADS];
    float *wt[G4D_MAX_DEPTH - 1], *bt[G4D_MAX_DEPTH - 1]; /* the trunk layers j = 1 .. depth-1 */
} G4DDeformGrads;

/* the GaussianModel tensors render() reads (scene/gaussian_model.py:108-131), all device */
typedef struct G4DGaussians {
    int64_t n;
    const float *xyz;           /* [N,3] */
    const float *scaling;       /* [N,3] log-scale (pre-activation) */
    const float *rotation;      /* [N,4] raw quaternion, w first */
    const float *opacity;       /* [N,1] logit */
    const float *features_dc;   /* [N,1,3] */
    const float *features_rest; /* [N,M-1,3] (M: G4DCamera.sh_coeffs); NULL => features_dc points at a fused [N,M,3] tensor.
                                 * At M = 1 the two layouts are the same [N,1,3] in features_dc and features_rest is not read
                                 * (it may be NULL: an empty tensor's data pointer) */
} G4DGaussians;

typedef struct G4DGaussianGrads { /* device, OVERWRITTEN */
    float *xyz, *scaling, *rotation, *opacity, *features_dc, *features_rest;
    float *means2D; /* [N,3] screen-space gradient in NDC units (z = 0): viewspace_points.grad */
} G4DGaussianGrads;

typedef struct G4DStats { /* filled by g4d_context_stats (synchronises the context's stream) */
    int64_t num_rendered; /* R = number of (Gaussian, tile) instances */
    int64_t num_visible;  /* Gaussians with radius > 0 */
    int64_t instance_capacity;
    int32_t tiles_x, tiles_y;
} G4DStats;

int g4d_abi_version(void);
const char *g4d_last_error(void);

G4DWorkspace *g4d_workspace_create(int device);
void g4d_workspace_destroy(G4DWorkspace *ws);
G4DContext *g4d_context_create(G4DWorkspace *ws);
void g4d_context_destroy(G4DContext *ctx);
int g4d_context_stats(G4DContext *ctx, G4DStats *out);

/* ---- deformation network (drop-in for deform_network.forward) ----------------------------------
 * shs may be NULL when the SHS head is inactive (then out_shs is not written).  With the SHS head active, shs / out_shs (and
 * g_out_shs / g_in_shs of the backward) are [N,16,3]: these entry points take no G4DCamera, so no other M.  Outputs are the
 * PRE-activation tensors, same shapes as the inputs. */
int g4d_deform_forward(G4DWorkspace *ws, const G4DDeformParams *prm, int64_t n, const float *xyz,
                       const float *scaling, const float *rotation, const float *opacity, const float *shs,
                       float time, float *out_xyz, float *out_scaling, float *out_rotation, float *out_opacity,
                       float *out_shs, uint32_t *relu_bits, void *stream);
/* g_out_* are dL/d(outputs) (NULL = zero).  g_in_* are OVERWRITTEN with dL/d(inputs) including the
 * residual path; weight/plane gradients are ACCUMULATED into `grads`.
 * relu_bits (optional, G4D_RELU_BITS_WORDS(n) uint32 of device memory): what autograd would save for the
 * backward of the six ReLUs (deformation.py:85-148) -- one sign bit per hidden unit, written by the forward,
 * read by the backward, so that the gradient is the gradient of the forward that actually ran.  NULL on
 * either side: the backward derives the signs from its own recomputation of the pre-activations. */
int g4d_deform_backward(G4DWorkspace *ws, const G4DDeformParams *prm, G4DDeformGrads *grads, int64_t n,
                        const float *xyz, float time, const float *g_out_xyz, const float *g_out_scaling,
                        const float *g_out_rotation, const float *g_out_opacity, const float *g_out_shs,
                        float *g_in_xyz, float *g_in_scaling, float *g_in_rotation, float *g_in_opacity,
                        float *g_in_shs, const uint32_t *relu_bits, void *stream);
#define G4D_RELU_BITS_WORDS(n) ((size_t)24 * (size_t)(n) + 4) /* [6 layers][n][4 words] + validity tag */
/* The same network with one time per Gaussian (the reference's times_sel [N,1] with rows that differ): d_times is device [n]
 * fp32, row g deformed at d_times[g] -- the trajectory of every Gaussian over several frames in one call, per-Gaussian time
 * offsets.  Otherwise as g4d_deform_forward / _backward: the same checks, engine and relu_bits.  At equal times the results
 * are those of the entry points above, bit for bit (the weight and plane gradients up to the order of their atomic sums).
 * d_times NULL: G4D_ERR_ARG before any launch.  g_times (optional, device [n], OVERWRITTEN): dL/d(times), 0 on a row whose
 * time lies outside [-1, 1] (grid_sample's border clamp). */
int g4d_deform_forward_times(G4DWorkspace *ws, const G4DDeformParams *prm, int64_t n, const float *xyz,
                             const float *scaling, const float *rotation, const float *opacity, const float *shs,
                             const float *d_times, float *out_xyz, float *out_scaling, float *out_rotation,
                             float *out_opacity, float *out_shs, uint32_t *relu_bits, void *stream);
int g4d_deform_backward_times(G4DWorkspace *ws, const G4DDeformParams *prm, G4DDeformGrads *grads, int64_t n,
                              const float *xyz, const float *d_times, const float *g_out_xyz, const float *g_out_scaling,
                              const float *g_out_rotation, const float *g_out_opacity, const float *g_out_shs,
                              float *g_in_xyz, float *g_in_scaling, float *g_in_rotation, float *g_in_opacity,
                              float *g_in_shs, float *g_times, const uint32_t *relu_bits, void *stream);

/* ---- rasterizer (drop-in for GaussianRasterizer) ------------------------------------------------
 * Inputs are POST-activation (scales = exp, rotations normalised, opacities = sigmoid), shs [N,M,3] (M: cam->sh_coeffs).
 * out_color [3,H,W], out_depth [1,H,W], out_radii [N] int32. */
int g4d_rasterize_forward(G4DContext *ctx, const G4DCamera *cam, int64_t n, const float *means3D,
                          const float *shs, const float *opacities, const float *scales, const float *rotations,
                          float *out_color, float *out_depth, int32_t *out_radii, void *stream);
/* all g_* OVERWRITTEN: g_means3D [N,3], g_means2D [N,3], g_shs [N,M,3], g_opacities [N,1], g_scales [N,3],
 * g_rotations [N,4].  The gradients of coefficients >= (sh_degree + 1)^2 are 0.  A backward whose M differs from its
 * forward's returns G4D_ERR_STATE (also g4d_render_backward(_cameras)). */
int g4d_rasterize_backward(G4DContext *ctx, const G4DCamera *cam, int64_t n, const float *means3D,
                           const float *shs, const float *opacities, const float *scales, const float *rotations,
                           const float *dL_dcolor, float *g_means3D, float *g_means2D, float *g_shs,
                           float *g_opacities, float *g_scales, float *g_rotations, void *stream);

/* ---- fused render (drop-in for gaussian_renderer.render) ----------------------------------------
 * prm == NULL renders the "coarse" stage (no deformation, gaussian_renderer/__init__.py:80-81). */
int g4d_render_forward(G4DContext *ctx, const G4DCamera *cam, const G4DDeformParams *prm, const G4DGaussians *g,
                       float *out_color, float *out_depth, int32_t *out_radii, void *stream);
int g4d_render_backward(G4DContext *ctx, const G4DCamera *cam, const G4DDeformParams *prm, G4DDeformGrads *pgrads,
                        const G4DGaussians *g, const float *dL_dcolor, G4DGaussianGrads *ggrads, void *stream);

/* ---- one timestamp seen by several cameras (a camera rig at frame t) ------------------------------
 * k cameras, 1 <= k <= G4D_MAX_CAMERAS, on k pairwise distinct contexts of one workspace.  Every cams[i].time must be
 * bitwise equal to cams[0].time (else G4D_ERR_ARG before any launch); image sizes may differ.  The deformation network
 * runs ONCE: camera 0 runs the g4d_render_forward sequence on ctx[0] (k == 1 is g4d_render_forward), cameras 1..k-1 are
 * projected from ctx[0]'s deformed, activated tensors and binned / blended on their own contexts.  out_color[i] [3,H_i,W_i],
 * out_depth[i] [1,H_i,W_i], out_radii[i] [N].  G4D_CAM_NO_GRAD on cams[0] skips the state only the backward reads.
 * The backward takes the same k contexts: dL_dcolor[i] == NULL leaves camera i out of the loss unless ctx[i] has a depth
 * or an alpha gradient (g4d_context_set_depth_grad / _alpha_grad), which then makes dL_dcolor[i] == NULL a zero image
 * gradient; gg receives the per-Gaussian
 * gradients summed over the cameras (OVERWRITTEN; gg->means2D must be NULL), g_means2D[i] ([N,3], may be NULL) camera i's
 * screen-space gradient; the network's backward runs once, ACCUMULATED into pgrads.  It returns G4D_ERR_STATE when any of
 * the contexts ran another forward since; g4d_render_backward / g4d_rasterize_backward refuse a member context. */
#define G4D_MAX_CAMERAS 32
int g4d_render_forward_cameras(G4DContext *const *ctx, int32_t k, const G4DCamera *cams, const G4DDeformParams *prm,
                               const G4DGaussians *g, float *const *out_color, float *const *out_depth,
                               int32_t *const *out_radii, void *stream);
int g4d_render_backward_cameras(G4DContext *const *ctx, int32_t k, const G4DCamera *cams, const G4DDeformParams *prm,
                                G4DDeformGrads *pgrads, const G4DGaussians *g, const float *const *dL_dcolor,
                                G4DGaussianGrads *gg, float *const *g_means2D, void *stream);

/* ---- losses either side of the path (SURVEY.md 8f N2) -----------------------------------------------
 * Every `*_accum` is a DEVICE float that is ADDED to (caller zeroes); `upstream` is a DEVICE float holding dL/d(loss
 * term) (what autograd hands the backward of a scalar), NULL = 1.
 *   g4d_l1_loss            <- utils/loss_utils.py:20-21  l1_loss(network_output, gt) = |a - b|.mean(): scale = 1 / numel
 *   g4d_ssim               <- utils/loss_utils.py:37-66  ssim(img1, img2): 11x11 Gaussian window (sigma 1.5), zero padding,
 *                             mean over [channels, H, W]: scale = 1 / (channels * H * W); `saved` (3 * channels * H * W
 *                             floats, may be NULL when no backward follows) keeps the per-pixel partial derivatives
 *   g4d_plane_regulation   <- scene/gaussian_model.py:538-577 compute_regulation(time_smoothness_weight, l1_time_planes_weight,
 *                             plane_tv_weight) with scene/regulation.py:22-28 compute_plane_smoothness: value and, when
 *                             `grads` is given, the plane gradients ACCUMULATED into grads->planes (other fields unused)
 * Alignment: g4d_l1_loss / g4d_l1_loss_backward take `out`, `gt` and `grad_out` at any 4-byte alignment (a view at an odd
 * storage offset is fine); when all of them are 16-byte aligned they run with 128-bit loads, otherwise with scalar loads. */
int g4d_l1_loss(G4DWorkspace *ws, const float *out, const float *gt, int64_t numel, float scale, float *loss_accum,
                void *stream);
int g4d_l1_loss_backward(G4DWorkspace *ws, const float *out, const float *gt, int64_t numel, float scale,
                         const float *upstream, float *grad_out, void *stream);
int g4d_ssim(G4DWorkspace *ws, const float *img1, const float *img2, int32_t channels, int32_t height, int32_t width,
             float scale, float *ssim_accum, float *saved, void *stream);
int g4d_ssim_backward(G4DWorkspace *ws, const float *img1, const float *img2, int32_t channels, int32_t height,
                      int32_t width, float scale, const float *upstream, const float *saved, float *grad_img1,
                      void *stream);
int g4d_plane_regulation(G4DWorkspace *ws, const G4DDeformParams *prm, G4DDeformGrads *grads, float plane_tv_weight,
                         float time_smoothness_weight, float l1_time_planes_weight, const float *upstream,
                         float *loss_accum, void *stream);

/* ---- optimizer step of the data-parallel harness (SURVEY.md 8f N1) --------------------------------
 * g4d_adam_step <- gaussians.optimizer.step() (train.py:290-292; groups scene/gaussian_model.py:165-183): torch.optim.Adam
 * without weight decay over ONE flat buffer; segment i covers elements [begin, end) with its own learning rate (elements in
 * no segment are left untouched); `numel` must be a multiple of 4 (pad the buffers); `step` is the 1-based step count;
 * gradients are multiplied by grad_scale first (1 / world_size after a SUM all-reduce).  param, grad, exp_avg and exp_avg_sq
 * must each be 16-byte aligned (the kernel moves float4s); otherwise G4D_ERR_ARG before any launch. */
#define G4D_ADAM_MAX_SEGMENTS 16
typedef struct G4DAdamSegment { int64_t begin, end; float lr; float reserved; } G4DAdamSegment;
int g4d_adam_step(G4DWorkspace *ws, float *param, const float *grad, float *exp_avg, float *exp_avg_sq, int64_t numel,
                  const G4DAdamSegment *segments, int32_t num_segments, float beta1, float beta2, float eps, int64_t step,
                  float grad_scale, void *stream);
/* g4d_adam_step_device: the same update with the per-step scalars read from DEVICE memory when the kernel runs, so that a
 * captured CUDA graph applies each replay's values: d_scalars points at a G4DAdamScalars in device memory (lr[i] is segment
 * i's learning rate; the segments' own lr fields are not read; their begin / end are, and are checked as above).
 * g4d_adam_scalars fills a G4DAdamScalars on the host (no device needed) with exactly the values g4d_adam_step computes from
 * (segments[i].lr, beta1, beta2, step, grad_scale): the two updates are then bit-identical. */
typedef struct G4DAdamScalars {
    float lr[G4D_ADAM_MAX_SEGMENTS];
    float inv_bc1;        /* 1 / (1 - beta1^step) */
    float inv_sqrt_bc2;   /* 1 / sqrt(1 - beta2^step) */
    float grad_scale;
    float reserved;
} G4DAdamScalars;
int g4d_adam_scalars(const G4DAdamSegment *segments, int32_t num_segments, float beta1, float beta2, int64_t step,
                     float grad_scale, G4DAdamScalars *out);
int g4d_adam_step_device(G4DWorkspace *ws, float *param, const float *grad, float *exp_avg, float *exp_avg_sq, int64_t numel,
                         const G4DAdamSegment *segments, int32_t num_segments, float beta1, float beta2, float eps,
                         const G4DAdamScalars *d_scalars, void *stream);

/* ---- scene initialisation (SURVEY.md 8f N4) -------------------------------------------------------
 * g4d_dist2_knn3 <- simple_knn._C.distCUDA2(points) (scene/gaussian_model.py:22,148; submodule absent from the reference
 * tree): for every point the mean of the squared distances to its 3 nearest OTHER points, fp32, exact (not approximate).
 * xyz [N,3] device, out [N] device. */
int g4d_dist2_knn3(G4DWorkspace *ws, int64_t n, const float *xyz, float *out_mean_dist2, void *stream);

/* ---- options / introspection --------------------------------------------------------------------*/
enum { G4D_OPT_SYNC_MODE = 1,  /* 1 (default): size the instance buffer exactly (one host read of R per
                                  forward, like the reference); 0: R stays on the device, the placement is
                                  capacity-bounded (capacity learnt from the context's first forward + 50 %),
                                  an overflow is reported by the NEXT call on the context / g4d_context_stats */
       G4D_OPT_INSTANCE_CAPACITY = 2, /* minimum instance capacity for no-sync mode */
       G4D_OPT_TIGHT_CULL = 3, /* 0 (default): reference tile rects; 1: drop (Gaussian,tile) pairs that
                                  provably contribute nothing (images identical, fewer instances) */
       G4D_OPT_STAGE_TIMING = 4, /* 1: bracket every stage with CUDA events on the launching stream
                                   (bench.py's live per-kernel durations); 0 (default): off */
       G4D_OPT_TENSOR_CORES = 5, /* the deformation MLP's forward when the configuration allows tensor cores (net_width 128,
                                   C in {16,32}, F <= 64, and no trunk layers): 2 (default) wgmma with FP16x2 operands (hi + lo halves, 3 products,
                                   fp32-accurate; operands must stay below 65504 after scaling -- activations < 8188, features
                                   < 1023, weights < 255 -- else the NEXT call returns G4D_ERR_OVERFLOW); 0: FP32 FFMA
                                   kernels (no range limit).  1 (3xTF32, removed) returns G4D_ERR_ARG and changes nothing;
                                   any other value selects 2.  The tensor-core kernels take the network with
                                   no trunk layers (depth <= 1); a deeper one runs on the FFMA kernels whatever the value */
       G4D_OPT_TC_DEBUG = 6,     /* 1: the tensor-core forward records counters per CTA (g4d_debug_tc_cycles: [0] cycles of the
                                   whole kernel, [1] cycles waiting for W1 images, [2] the CTA's consumer warpgroups, [3..11]
                                   unused) */
       G4D_OPT_KEEP_DEFORMED = 8, /* 1: a no-grad fused forward (G4D_CAM_NO_GRAD) still stores the deformed + activated tensors
                                   * (G4D_BUF_DEFORMED / _SHS reads); default 0: it skips those 48-240 B / Gaussian of writes */
       G4D_OPT_WARP_CULL = 7,    /* 1 (default): the blend kernels skip, per warp, instances that cannot reach alpha >= 1/255
                                  *    on any pixel of the warp's 16 x 4 strip (results unchanged); 0 = test every pixel */
       G4D_OPT_PDL = 9,          /* 1 (default): the kernels of a forward are launched programmatically dependent on one another
                                  *    (a kernel's set-up overlaps the tail of its predecessor; results unchanged); 0: ordinary
                                  *    stream order.  PROCESS-wide, not per workspace (also: environment G4D_PDL=0) */
       G4D_OPT_GATHER_ORDER = 10 /* 1 (default): every path gathers the HexPlane features of the Gaussians in a spatial
                                  *    (Z) order, built on the device when the xyz pointer or N changes and kept otherwise (results
                                  *    unchanged: every Gaussian's features come from its own taps); 0: index order.  Per workspace;
                                  *    a workspace created with G4D_GATHER_ORDER=0 in the environment starts at 0 */ };
int g4d_workspace_set_option(G4DWorkspace *ws, int option, int64_t value);

/* copy an internal per-forward buffer to HOST memory (tests / debugging; synchronises).
 * Returns the number of bytes the buffer holds (>=0) or an error; copies min(bytes, held). */
enum { G4D_BUF_DEPTH = 1,      /* float  [N]  view-space depth                    */
       G4D_BUF_RECT = 2,       /* int32  [N,4] (min_x, min_y, max_x, max_y) tiles */
       G4D_BUF_TILES_TOUCHED = 3, /* uint32 [N]                                   */
       G4D_BUF_XY = 4,         /* float  [N,2] pixel centre                       */
       G4D_BUF_CONIC_OPACITY = 5, /* float [N,4]                                  */
       G4D_BUF_RGB = 6,        /* float  [N,3]                                    */
       G4D_BUF_SORTED_KEYS = 7,   /* uint64 [R]                                   */
       G4D_BUF_SORTED_IDS = 8,    /* uint32 [R]                                   */
       G4D_BUF_RANGES = 9,     /* uint32 [tiles,2]                                */
       G4D_BUF_FINAL_T = 10,   /* float  [H,W]                                    */
       G4D_BUF_N_CONTRIB = 11, /* uint32 [H,W]                                    */
       G4D_BUF_CLAMPED = 12,   /* uint8  [N,3]                                    */
       G4D_BUF_DEFORMED = 13,  /* float  [N,11] (xyz, scale, rot, opacity) post-activation, fused path */
       G4D_BUF_DEFORMED_SHS = 14, /* float [N,48] deformed SH coefficients (fused path with the SHS head active) */
       G4D_BUF_BIN_PHASES = 15, /* int64 [16] profiling: SM clock of CTA 0 at the phase boundaries of bin_sort (0 start,
                                  1 after the key range, 2 after the depth sort, 3 after chunking, 4 after counting,
                                  5 end), [15] = significant key bits */
       G4D_BUF_FEATURES = 16,  /* float [N,F] HexPlane features staged by a grad-enabled tensor-core fused forward */
       G4D_BUF_GATHER_ORDER = 17 /* uint32 [N'] the workspace's walk order of the HexPlane gather (G4D_OPT_GATHER_ORDER), built
                                  for the last N' Gaussians it was rebuilt for; 0 bytes when none was built.  The order of the
                                  Gaussians inside one grid cell may differ from one build to the next */ };
int64_t g4d_context_read(G4DContext *ctx, int which, void *host_dst, int64_t bytes);

/* per-stage device time (ms) of the LAST forward / backward on this context, measured with CUDA events on the
 * launching stream (needs G4D_OPT_STAGE_TIMING = 1; synchronises).  out_ms[G4D_STAGE_COUNT]; stages that did
 * not run hold 0.  Returns G4D_STAGE_COUNT or an error. */
enum { G4D_STAGE_PREP = 0,        /* camera pack, weight pack, time-row collapse            */
       G4D_STAGE_GEOM = 1,        /* deform+activate+project (fused) or preprocess           */
       G4D_STAGE_SCAN = 2,        /* bin_sort: depth order, per-(chunk,tile) counts, tile ranges, R (one cooperative launch) */
       G4D_STAGE_EMIT = 3,        /* bin_place: stable counting placement of the instances   */
       G4D_STAGE_SORT = 4, G4D_STAGE_RANGES = 5, /* unused since ABI 3 (no separate sort / range kernels) */
       G4D_STAGE_BLEND = 6,
       G4D_STAGE_BLEND_BWD = 7, G4D_STAGE_GEOM_BWD = 8, G4D_STAGE_DEFORM_BWD = 9,
       G4D_STAGE_COUNT = 10 };
int g4d_context_stage_times(G4DContext *ctx, float *out_ms, int capacity);

/* DEBUG: per-CTA counters of the last tensor-core deform launch (G4D_OPT_TC_DEBUG), averaged over the SMs (an SM without a
 * CTA of the launch counts as 0). */
int g4d_debug_tc_cycles(G4DWorkspace *ws, double *out12);

/* ---- CUDA-graph capture (opt-in; INTEGRATION.md "CUDA graphs") -------------------------------------
 * Every entry point that owns buffers or host-side state asks cudaStreamIsCapturing on its stream (the loss, regulariser and
 * Adam entry points own neither: they only launch kernels and capture as they are).  While the stream captures, nothing that a replay could not
 * re-run happens: no host events, no read of a pinned read-back slot, no host sync, no allocation.  An entry point returns
 * G4D_ERR_STATE (the message names the cause) before any launch when the workspace is in exact sync mode
 * (G4D_OPT_SYNC_MODE = 1), when a context has not learnt its instance capacity from an earlier forward, with G4D_CAM_DEBUG or
 * with G4D_OPT_STAGE_TIMING; and when one of its buffers would have to grow it returns G4D_ERR_STATE without freeing
 * anything.  Buffers are sized where each stage needs them, so that refusal can come after the call has enqueued (or, while
 * capturing, recorded) its first stages: a capture that met it is unusable (end it and drop the graph), and after an eager
 * refusal on a frozen workspace the context holds no forward (a backward on it returns G4D_ERR_STATE).
 *
 * g4d_context_set_time_source: while d_time (device, one float) is set, every forward and backward on ctx reads its
 * timestamp from there at run time instead of from G4DCamera.time: the time-row collapse, the network's backward and the
 * camera record.  NULL restores G4DCamera.time.  g4d_render_forward_cameras / _backward_cameras need either no source on any
 * of their contexts (the cameras' times are compared) or the same source on all of them.
 * g4d_workspace_freeze: while on, any call that would reallocate a buffer of ws or of one of its contexts returns
 * G4D_ERR_STATE and frees nothing (a captured graph keeps pointing at those buffers).
 * g4d_workspace_graph_status: what the forwards captured on ws met since the last call, then cleared: the no-sync forwards
 * whose tile instances exceeded the capacity they ran with (the placement clamps: those images are incomplete, nothing is
 * written out of bounds) and the FP16x2 range flag of G4D_OPT_TENSOR_CORES.  sync != 0: synchronise the device first;
 * sync == 0 is only valid when no replay on ws can still be running (the record is updated without atomics). */
typedef struct G4DGraphStatus {
    int64_t overflows;      /* captured forwards whose instance count exceeded their capacity */
    int64_t max_instances;  /* the largest such instance count (0 when overflows == 0) */
    int32_t f16_range;      /* 1: an FP16x2 tensor-core launch met a value outside the f16 operand range */
    int32_t reserved;
} G4DGraphStatus;
int g4d_context_set_time_source(G4DContext *ctx, const float *d_time);

/* ---- camera gradients ----------------------------------------------------------------------------------------------
 * g4d_context_set_camera_grad: while d_out (device, 35 floats) is set, every backward on ctx (g4d_rasterize_backward,
 * g4d_render_backward, and g4d_render_backward_cameras for the camera ctx holds) OVERWRITES it with dL/d of this camera:
 * view[16], proj[16], campos[3], each in the element order of G4DCamera.viewmatrix / projmatrix / campos.  Elements the
 * forward does not read (view 3, 7, 11, 15; proj 2, 6, 10, 14) are 0, and so is every element of a camera outside the loss
 * (image gradient NULL and no depth or alpha gradient).  The derivative is that of the forward as the kernels compute it: a
 * guard-band-clamped t.x / t.y is a constant, alpha's 0.99 clamp passes the gradient, a clamped colour channel passes none,
 * and the depth and alpha images pass their gradients when the context has them (g4d_context_set_depth_grad / _alpha_grad).  NULL turns it
 * off.  A backward on a stream that is capturing returns G4D_ERR_STATE before any launch while the pointer is set.  The
 * sink is zeroed on the stream after the backward's argument and state checks and before its first kernel: a backward that
 * returns an error after that point (a CUDA error, a buffer that cannot grow) leaves it zeroed or partly summed, not as it
 * was. */
int g4d_context_set_camera_grad(G4DContext *ctx, float *d_out);

/* ---- time gradients ------------------------------------------------------------------------------------------------
 * g4d_context_set_time_grad: while d_out (device, 1 float) is set, every backward on ctx OVERWRITES d_out[0] with dL/d of
 * the call's time (G4DCamera.time, or the value read through g4d_context_set_time_source).  g4d_render_backward_cameras
 * writes the one derivative the group shares into every context of the call that has a sink; a camera outside the loss (image
 * gradient NULL and no depth or alpha gradient) adds nothing to it.  g4d_rasterize_backward, a fused backward without deformation params (the coarse stage) and
 * n = 0 write 0.  The derivative is that of the forward as the kernels compute it: a time on a texel row of a time plane
 * takes the row above it, and a time at or past the plane's border (t <= -1 or t >= 1) gives 0.  It is summed with atomics,
 * so it is not bit-reproducible from run to run.  NULL turns it off.  Capture, zeroing and errors as for
 * g4d_context_set_camera_grad: a backward on a capturing stream returns G4D_ERR_STATE before any launch while it is set, and
 * a backward refused by its argument and state checks (e.g. after a G4D_CAM_NO_GRAD forward) leaves the sink untouched. */
int g4d_context_set_time_grad(G4DContext *ctx, float *d_out);

/* ---- depth gradients -----------------------------------------------------------------------------------------------
 * g4d_context_set_depth_grad: while d_dL_ddepth (device, [1,H,W] floats of the forward's image size) is set, every backward on
 * ctx (g4d_rasterize_backward, g4d_render_backward, and g4d_render_backward_cameras for the camera ctx holds) adds the
 * gradient of the forward's depth image out_depth to every gradient it computes, as if the loss had been differentiated
 * w.r.t. out_depth as well.  The depth image is D = sum_i w_i z_i over the pixel's colour instances (w_i = alpha_i T_i, the
 * colour weights; z_i the Gaussian's view-space depth; no background term, no normalisation).  The derivative is that of the
 * forward as the kernels compute it, with the conventions of the colour's (alpha's 0.99 clamp passes the gradient, only
 * Gaussians with radius > 0 get one).  It is summed with atomics, so it is not bit-reproducible from run to run.  The buffer
 * is read, never written.  NULL turns it off; with no pointer set a backward runs exactly as it did before this entry point
 * existed.  A backward on a capturing stream returns G4D_ERR_STATE before any launch while it is set. */
int g4d_context_set_depth_grad(G4DContext *ctx, const float *d_dL_ddepth);

/* ---- alpha maps ----------------------------------------------------------------------------------------------------
 * The alpha image of a forward is its accumulated opacity A = 1 - T per pixel, T the transmittance the blend leaves behind
 * the pixel's colour instances (the instance that would take T below 1e-4 stops the pixel and is not included; alpha < 1/255
 * is skipped; alpha is clamped to 0.99).  The image is then out_color = C_fg + (1 - A) bg, up to the fp32 rounding of
 * 1 - (1 - T): the kernel composites with T itself.
 * g4d_context_set_alpha_out: while d_out (device, [1,H,W] floats of the forward's image size) is set, every forward on ctx
 * (g4d_rasterize_forward, g4d_render_forward, and g4d_render_forward_cameras for the camera ctx holds) also writes A there,
 * G4D_CAM_NO_GRAD forwards included.  A forward captured in a CUDA graph keeps writing the pointer it was captured with.
 * NULL turns it off; with no pointer set a forward runs exactly as it did before this entry point existed.
 * g4d_context_set_alpha_grad: while d_dL_dalpha (device, [1,H,W] floats of the forward's image size) is set, every backward
 * on ctx (g4d_rasterize_backward, g4d_render_backward, and g4d_render_backward_cameras for the camera ctx holds) adds the
 * gradient of the forward's alpha image to every gradient it computes, as if the loss had been differentiated w.r.t. A as
 * well.  The backward derives it from the transmittance it keeps (G4D_BUF_FINAL_T), so the forward need not have written A.
 * The derivative is that of the forward as the kernels compute it, with the conventions of the colour's (alpha's 0.99 clamp
 * passes the gradient, only Gaussians with radius > 0 get one).  The buffer is read, never written.  NULL turns it off; with
 * no pointer set a backward runs exactly as it did before this entry point existed.  A backward on a capturing stream returns
 * G4D_ERR_STATE before any launch while it is set. */
int g4d_context_set_alpha_out(G4DContext *ctx, float *d_out);
int g4d_context_set_alpha_grad(G4DContext *ctx, const float *d_dL_dalpha);
int g4d_workspace_freeze(G4DWorkspace *ws, int on);
int g4d_workspace_graph_status(G4DWorkspace *ws, int sync, G4DGraphStatus *out);

#ifdef __cplusplus
}
#endif
#endif /* G4D_H_ */
