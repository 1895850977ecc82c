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
 *   g4d_deform_forward / _backward
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

enum {
    G4D_OK = 0,
    G4D_ERR_CUDA = -1,      /* a CUDA runtime call or kernel failed */
    G4D_ERR_ARG = -2,       /* invalid argument / unsupported configuration */
    G4D_ERR_NOMEM = -3,     /* device allocation failed */
    G4D_ERR_STATE = -4,     /* backward without a matching forward, ... */
    G4D_ERR_OVERFLOW = -5   /* tile-instance buffer overflowed in no-sync mode (re-run with sync), or an FP16x2 tensor-core
                             * launch met a value outside the f16 operand range (G4D_OPT_TENSOR_CORES) */
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
} G4DCamera;

typedef struct G4DDeformParams {
    int32_t levels;    /* len(multires) <= G4D_MAX_LEVELS */
    int32_t channels;  /* kplanes output_coordinate_dim: multiple of 4, <= 32 */
    int32_t net_width; /* 64, 128 or 256 */
    int32_t head_mask; /* G4D_HEAD_* bits */
    int32_t res[G4D_MAX_LEVELS][4]; /* per level: resolution of x, y, z, t */
    /* device: plane k of level l, CHANNEL-LAST [H][W][C]; (H,W) = (res[c1], res[c0]) for the k-th
     * pair (c0,c1) of combinations(range(4),2)  (scene/hexplane.py:48-70) */
    const float *planes[G4D_MAX_LEVELS][6];
    const float *aabb;      /* device [2][3]: row 0 = xyz_max, row 1 = xyz_min */
    const float *w0, *b0;   /* device: feature_out.0  [Wd][F], [Wd] */
    const float *w1[G4D_NUM_HEADS], *b1[G4D_NUM_HEADS]; /* device: <head>.1  [Wd][Wd], [Wd] */
    const float *w2[G4D_NUM_HEADS], *b2[G4D_NUM_HEADS]; /* device: <head>.3  [k][Wd], [k]; k = 3,3,4,1,48 */
    uint64_t version; /* caller bumps it whenever any weight changed (packed copies are cached) */
} G4DDeformParams;

/* gradient sinks mirroring G4DDeformParams (device, same layouts; ACCUMULATED into, caller zeroes) */
typedef struct G4DDeformGrads {
    float *planes[G4D_MAX_LEVELS][6];
    float *w0, *b0;
    float *w1[G4D_NUM_HEADS], *b1[G4D_NUM_HEADS];
    float *w2[G4D_NUM_HEADS], *b2[G4D_NUM_HEADS];
} G4DDeformGrads;

/* the GaussianModel tensors render() reads (scene/gaussian_model.py:108-131), all device */
typedef struct G4DGaussians {
    int64_t n;
    const float *xyz;           /* [N,3] */
    const float *scaling;       /* [N,3] log-scale (pre-activation) */
    const float *rotation;      /* [N,4] raw quaternion, w first */
    const float *opacity;       /* [N,1] logit */
    const float *features_dc;   /* [N,1,3] */
    const float *features_rest; /* [N,15,3]; NULL => features_dc points at a fused [N,16,3] tensor */
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
 * shs may be NULL when the SHS head is inactive (then out_shs is not written). Outputs are the
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

/* ---- rasterizer (drop-in for GaussianRasterizer) ------------------------------------------------
 * Inputs are POST-activation (scales = exp, rotations normalised, opacities = sigmoid), shs [N,16,3].
 * out_color [3,H,W], out_depth [1,H,W], out_radii [N] int32. */
int g4d_rasterize_forward(G4DContext *ctx, const G4DCamera *cam, int64_t n, const float *means3D,
                          const float *shs, const float *opacities, const float *scales, const float *rotations,
                          float *out_color, float *out_depth, int32_t *out_radii, void *stream);
/* all g_* OVERWRITTEN: g_means3D [N,3], g_means2D [N,3], g_shs [N,16,3], g_opacities [N,1], g_scales [N,3],
 * g_rotations [N,4] */
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
 * The backward takes the same k contexts: dL_dcolor[i] == NULL leaves camera i out of the loss; gg receives the per-Gaussian
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
 *                             `grads` is given, the plane gradients ACCUMULATED into grads->planes (other fields unused) */
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
 * gradients are multiplied by grad_scale first (1 / world_size after a SUM all-reduce). */
#define G4D_ADAM_MAX_SEGMENTS 16
typedef struct G4DAdamSegment { int64_t begin, end; float lr; float reserved; } G4DAdamSegment;
int g4d_adam_step(G4DWorkspace *ws, float *param, const float *grad, float *exp_avg, float *exp_avg_sq, int64_t numel,
                  const G4DAdamSegment *segments, int32_t num_segments, float beta1, float beta2, float eps, int64_t step,
                  float grad_scale, void *stream);

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
                                   C in {16,32}, F <= 64): 2 (default) wgmma with FP16x2 operands (hi + lo halves, 3 products,
                                   fp32-accurate; operands must stay below 65504 after scaling -- activations < 8188, features
                                   < 1023, weights < 255 -- else the NEXT call returns G4D_ERR_OVERFLOW); 1: wgmma 3xTF32 (no
                                   range limit); 0: FP32 FFMA kernels */
       G4D_OPT_TC_DEBUG = 6,     /* 1: the tensor-core forward records cycle counters per CTA (g4d_debug_tc_cycles: [0] whole
                                   kernel, [1] waiting for W1 images, [2..11] unused) */
       G4D_OPT_KEEP_DEFORMED = 8, /* 1: a no-grad fused forward (G4D_CAM_NO_GRAD) still stores the deformed + activated tensors
                                   * (G4D_BUF_DEFORMED / _SHS reads); default 0: it skips those 48-240 B / Gaussian of writes */
       G4D_OPT_WARP_CULL = 7,    /* 1 (default): the blend kernels skip, per warp, instances that cannot reach alpha >= 1/255
                                  *    on any pixel of the warp's 16 x 4 strip (results unchanged); 0 = test every pixel */
       G4D_OPT_PDL = 9           /* 1 (default): the kernels of a forward are launched programmatically dependent on one another
                                  *    (a kernel's set-up overlaps the tail of its predecessor; results unchanged); 0: ordinary
                                  *    stream order.  PROCESS-wide, not per workspace (also: environment G4D_PDL=0) */ };
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
       G4D_BUF_BIN_PHASES = 15 /* int64 [16] profiling: SM clock of CTA 0 at the phase boundaries of bin_sort (0 start,
                                  1 after the key range, 2 after the depth sort, 3 after chunking, 4 after counting,
                                  5 end), [15] = significant key bits */ };
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

/* DEBUG: mean per-CTA cycle counters of the last tensor-core deform launch (G4D_OPT_TC_DEBUG). */
int g4d_debug_tc_cycles(G4DWorkspace *ws, double *out12);

#ifdef __cplusplus
}
#endif
#endif /* G4D_H_ */
