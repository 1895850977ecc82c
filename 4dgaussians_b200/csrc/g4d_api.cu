// g4d_api.cu -- the C-ABI of libg4d.so (include/g4d.h): workspace / context management and stage orchestration.
// No torch types, no CPU fallback: every entry point either runs the CUDA path or returns an error code.
#include <cstdio>
#include <cstdlib>
#include <atomic>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "g4d_internal.h"

using namespace g4d;

namespace {

thread_local std::string t_last_error;

// What the entry point running on this thread allows (CallFrame): while its stream captures a CUDA graph nothing may run that
// a replay could not repeat, and while its workspace is frozen or its stream captures no buffer may be reallocated (a graph
// keeps the addresses it captured).
// growth_refused: set by the DevBuf::ensure that refused, so that its caller reports the refusal and not a CUDA error.
struct CallState { bool capturing = false, no_growth = false, growth_refused = false; };
thread_local CallState t_call;

int fail(int code, const char* what, const char* detail = nullptr) {
    t_last_error = what;
    if (detail) { t_last_error += ": "; t_last_error += detail; }
    return code;
}

int growth_refused(const char* what) {
    t_call.growth_refused = false;
    return fail(G4D_ERR_STATE, "a buffer would have to grow while the workspace is frozen or the stream is capturing", what);
}

#define G4D_CUDA(expr)                                                                      \
    do {                                                                                    \
        cudaError_t e__ = (expr);                                                           \
        if (e__ != cudaSuccess && t_call.growth_refused) return growth_refused(#expr);      \
        if (e__ != cudaSuccess) {                                                           \
            char buf__[64];                                                                 \
            snprintf(buf__, sizeof(buf__), " (%s:%d)", __FILE__, __LINE__);                 \
            std::string m__ = std::string(cudaGetErrorString(e__)) + buf__;                 \
            return fail(e__ == cudaErrorMemoryAllocation ? G4D_ERR_NOMEM : G4D_ERR_CUDA, #expr, m__.c_str()); \
        }                                                                                   \
    } while (0)

// device memory that grows by 1.5x on demand and is freed with its owner (on the owner's device); it refuses to grow (and
// frees nothing) under t_call.no_growth
struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    DevBuf(DevBuf&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
    ~DevBuf() { if (p) cudaFree(p); }
    cudaError_t ensure(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        if (t_call.no_growth) { t_call.growth_refused = true; return cudaErrorNotPermitted; }
        size_t want = bytes + bytes / 2 + 256;
        if (p) { cudaError_t e = cudaFree(p); p = nullptr; cap = 0; if (e != cudaSuccess) return e; }
        cudaError_t e = cudaMalloc(&p, want);
        if (e != cudaSuccess) { p = nullptr; cap = 0; return e; }
        cap = want;
        return cudaSuccess;
    }
    template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};

// grow `buf` to the size of a layout and place it there: layout(Carve&) takes the layout's ranges, and runs once to count
// the bytes and once on the buffer
template <class Layout> cudaError_t ensure_layout(DevBuf& buf, Layout layout) {
    Carve size;
    layout(size);
    const cudaError_t e = buf.ensure(size.bytes());
    if (e != cudaSuccess) return e;
    Carve place(buf.p);
    layout(place);
    return cudaSuccess;
}

// FP32 transposes of W0, of the active heads' W1 and of the trunk layers' W_j (the FFMA kernels' operands)
struct FfmaWeights {
    float* w0t;
    float* w1t[G4D_NUM_HEADS];
    float* wtt[G4D_MAX_DEPTH - 1];
};

// weight images derived from the caller's parameters, rebuilt when G4DDeformParams.version or the w0 pointer changes
template <class Images>
struct WeightCache {
    DevBuf buf;
    Images img{};   // where the images sit in buf
    uint64_t version = 0;
    const void* key = nullptr;
    bool valid = false;
    // pack(buf.p, &img) (re)builds the images unless they were built from these parameters; a capture always rebuilds them,
    // so that every replay packs the parameters as they are then
    template <class Pack> cudaError_t refresh(const G4DDeformParams* p, size_t bytes, Pack pack) {
        if (valid && !t_call.capturing && version == p->version && key == (const void*)p->w0) return cudaSuccess;
        valid = false;
        cudaError_t e = buf.ensure(bytes);
        if (e == cudaSuccess) e = pack(buf.p, &img);
        if (e != cudaSuccess) return e;
        version = p->version; key = (const void*)p->w0; valid = true;
        return cudaSuccess;
    }
};

// pinned host words of a workspace: the exact-mode read-back of R, the flag an FP16x2 tensor-core kernel sets (through
// the host mapping) when a value left the f16 operand range, and the overflow record of captured forwards (count, largest
// R: launch_record_overflow)
struct PinnedWords { uint32_t num_rendered, pad0[7], f16_range, pad1[7], overflow[2], pad2[6]; };

// The forward a context holds.  A forward entry point clears the record of every context it writes before its first launch
// and writes each one whole once the entry point has succeeded; an overflow found by a no-sync read-back clears it.  The
// backward entry points, g4d_context_read and g4d_context_stats decide from the record alone what the context holds.
struct ForwardRecord {
    enum Kind { kNone, kRaster, kFused };   // kRaster: g4d_rasterize_forward; kFused: g4d_render_forward(_cameras)
    Kind kind = kNone;
    int64_t n = 0;
    int H = 0, W = 0;
    bool deformed = false;    // the deformation network ran (fine stage)
    bool sh = false;          // the SHS head was active: the deformed SH coefficients are in fo.shs
    bool kept = false;        // fo holds the deformed, activated tensors
    int sh_coeffs = 0;        // M: SH coefficients per Gaussian of the forward's inputs (its camera's sh_coeffs)
    int feat_cols = 0;        // F of the HexPlane features in `feat` and the ReLU bits in `relu` kept for a backward (0: none)
    // g4d_render_forward_cameras: serial number of the call (0: a single-camera forward), this camera's position, the number
    // of cameras, and whether the group keeps what its backward reads
    uint64_t group = 0;
    int group_pos = 0, group_size = 0;
    bool group_grad = false;
};

}  // namespace

struct G4DWorkspace {
    int device = 0;
    int sm_count = 132;
    int sync_mode = 1;
    int64_t min_capacity = 0;
    int tight_cull = 0;
    int stage_timing = 0;
    int tensor_cores = 2;      // 0: FP32 FFMA kernels, 2 (default): wgmma FP16x2
    int warp_cull = 1;
    int keep_deformed = 0;
    int tc_debug = 0;
    int gather_order = 1;      // G4D_OPT_GATHER_ORDER: 1 spatial walk order of the HexPlane gather, 0 index order
    int frozen = 0;            // g4d_workspace_freeze
    DevBuf order_buf;          // the walk order and the scratch that builds it (GatherOrderBuffers)
    GatherOrderBuffers order{};
    const float* order_xyz = nullptr;   // the Gaussians the order was built for (nullptr: none)
    int64_t order_n = 0;
    WeightCache<FfmaWeights> packed;     // FFMA forward and backward
    WeightCache<TcWeights> tc;           // tensor-core forward (the weight fields and status of TcWeights)
    WeightCache<TcBwdWeights> tc_bwd;    // tensor-core backward
    DevBuf feat;        // the HexPlane features [N][F] of a forward that keeps none for its backward
    DevBuf tc_dbg;      // G4D_OPT_TC_DEBUG cycle counters
    DevBuf trow;        // time rows for the context-free deform entry points
    DevBuf scratch;     // misc per-call scratch (deform backward, kNN)
    PinnedWords* pinned = nullptr;
};

// What a context's view takes and gives beyond its colour image, one device pointer per g4d_context_set_* entry point
// (NULL: off).  A capture refuses every term a backward reads or writes: a graph would keep using a pointer the context
// may since have dropped.
struct ViewTerms {
    float* cam_grad = nullptr;           // g4d_context_set_camera_grad (kCamGradFloats)
    float* time_grad = nullptr;          // g4d_context_set_time_grad (1 float)
    const float* depth_grad = nullptr;   // g4d_context_set_depth_grad ([H,W] dL/d depth image)
    float* alpha_out = nullptr;          // g4d_context_set_alpha_out ([H,W] alpha image of every forward)
    const float* alpha_grad = nullptr;   // g4d_context_set_alpha_grad ([H,W] dL/d alpha image)

    // a backward takes the view into the loss: it has an image (dL_dcolor), a depth or an alpha gradient
    bool in_loss(const float* dL_dcolor) const { return dL_dcolor || depth_grad || alpha_grad; }

    // the refusal of a backward on a capturing stream, in the order the terms are checked (NULL: nothing to refuse)
    const char* capture_refusal() const {
        if (cam_grad) return "cannot capture a backward on a context with a camera gradient set (g4d_context_set_camera_grad)";
        if (time_grad) return "cannot capture a backward on a context with a time gradient set (g4d_context_set_time_grad)";
        if (depth_grad) return "cannot capture a backward on a context with a depth gradient set (g4d_context_set_depth_grad)";
        if (alpha_grad) return "cannot capture a backward on a context with an alpha gradient set (g4d_context_set_alpha_grad)";
        return nullptr;
    }
};

struct G4DContext {
    G4DWorkspace* ws = nullptr;
    DevBuf cam, geom, bin, binaux, img, fused, gscratch, gdeform, trow, relu, feat;
    ForwardRecord fwd;
    int grid_x = 0, grid_y = 0;
    int64_t R = 0, capacity = 0;
    const float* time_src = nullptr;  // g4d_context_set_time_source (device; NULL: G4DCamera.time)
    ViewTerms terms;
    const void* bin_ctl = nullptr;    // device BinCtl of the last forward
    bool learned = false;             // R of an earlier exact forward is known (no-sync mode needs a learnt capacity)
    GeomBuffers g{};
    BinBuffers b{};
    ImageBuffers im{};
    FusedOutputs fo{};
    float* trow_ptr[G4D_MAX_LEVELS][3] = {};
    // no-sync mode: the instance count of a forward is read back asynchronously (behind its blend kernel) into one of kSlots
    // slots (pinned word + event) used round robin: when forward v starts, the slot it is about to reuse holds forward
    // v - kSlots (complete unless the host is kSlots views ahead of the device -- then it waits, which bounds the run-ahead),
    // the others the newer forwards (looked at only if they are done)
    static constexpr int kSlots = 4;
    uint32_t* h_r = nullptr;          // pinned: [slot] instance count
    cudaEvent_t ev_r[kSlots] = {};
    bool pending[kSlots] = {};        // the slot's read-back has not been checked yet
    int64_t used_capacity[kSlots] = {};  // capacity the slot's forward ran with
    int slot = 0;                     // slot the NEXT no-sync forward uses
    cudaEvent_t ev[2 * G4D_STAGE_COUNT] = {};
    bool ev_used[G4D_STAGE_COUNT] = {};
    bool ev_created = false;
};

namespace g4d {
// programmatic dependent launch of the forward chain (g4d_common.cuh); G4D_OPT_PDL / env G4D_PDL=0 switch it off
int g_pdl = []() { const char* e = getenv("G4D_PDL"); return e ? atoi(e) != 0 : 1; }();
}  // namespace g4d

namespace {

// RAII bracket of one stage with CUDA events on the launching stream (only when G4D_OPT_STAGE_TIMING is on)
struct StageTimer {
    G4DContext* c; int stage; cudaStream_t st; bool on;
    StageTimer(G4DContext* c_, int stage_, cudaStream_t st_) : c(c_), stage(stage_), st(st_), on(c_->ws->stage_timing != 0) {
        if (!on) return;
        if (!c->ev_created) {
            for (int i = 0; i < 2 * G4D_STAGE_COUNT; ++i) cudaEventCreate(&c->ev[i]);
            c->ev_created = true;
        }
        cudaEventRecord(c->ev[2 * stage], st);
    }
    ~StageTimer() {
        if (!on) return;
        cudaEventRecord(c->ev[2 * stage + 1], st);
        c->ev_used[stage] = true;
    }
};
void reset_stage_flags(G4DContext* c, int first, int last) { for (int i = first; i <= last; ++i) c->ev_used[i] = false; }

// What a capture refuses, checked before any launch: host events (stage timing), host syncs (G4D_CAM_DEBUG) and, for a
// forward on the contexts fwd[0, k), the exact-mode read-back of R and a capacity that has not been learnt yet.
int refuse_capture(const G4DWorkspace* ws, const G4DCamera* cams, int k, G4DContext* const* fwd) {
    if (!t_call.capturing) return G4D_OK;
    if (ws->stage_timing) return fail(G4D_ERR_STATE, "cannot capture with G4D_OPT_STAGE_TIMING: it records host-managed events");
    for (int i = 0; i < k; ++i)
        if (cams[i].debug & G4D_CAM_DEBUG) return fail(G4D_ERR_STATE, "cannot capture with G4D_CAM_DEBUG: it synchronises after every stage");
    if (!fwd) return G4D_OK;
    if (ws->sync_mode)
        return fail(G4D_ERR_STATE, "cannot capture a forward in exact sync mode (G4D_OPT_SYNC_MODE = 1): it reads the instance count "
                                   "back on the host; set the option to 0");
    for (int i = 0; i < k; ++i)
        if (!fwd[i]->learned || fwd[i]->capacity <= 0)
            return fail(G4D_ERR_STATE, "cannot capture a forward on a context that has not learnt its instance capacity: run one "
                                       "forward on it outside the capture first");
    return G4D_OK;
}

int ensure_geom(G4DContext* c, int64_t n) {
    const size_t N = (size_t)(n > 0 ? n : 1);
    GeomBuffers& g = c->g;
    auto layout = [&](Carve& m) {
        g.rec0 = m.take<float4>(N); g.rec1 = m.take<float4>(N); g.rec2 = m.take<float2>(N); g.radii = m.take<int32_t>(N);
        g.rect = m.take<uint2>(N); g.tiles_touched = m.take<uint32_t>(N); g.clamped = m.take<uint8_t>(N); g.perm = m.take<uint32_t>(N);
    };
    G4D_CUDA(ensure_layout(c->geom, layout));
    g.depth_range = &c->cam.as<CameraDev>()->depth_min;
    return G4D_OK;
}

int ensure_image(G4DContext* c, int H, int W) {
    const size_t P = (size_t)H * W;
    const int gx = (W + kTile - 1) / kTile, gy = (H + kTile - 1) / kTile;
    auto layout = [&](Carve& m) {
        c->im.final_T = m.take<float>(P); c->im.n_contrib = m.take<uint32_t>(P);
        c->b.ranges = m.take<uint2>((size_t)gx * gy);
    };
    G4D_CUDA(ensure_layout(c->img, layout));
    c->grid_x = gx; c->grid_y = gy;
    return G4D_OK;
}

int ensure_bin(G4DContext* c, int64_t r) {
    const size_t R = (size_t)(r > 0 ? r : 1);
    if ((int64_t)R <= c->capacity && c->bin.p) return G4D_OK;
    G4D_CUDA(c->bin.ensure(R * 12 + 16));    // DevBuf grows by 1.5x: the one growth factor of the instance list
    c->capacity = (int64_t)((c->bin.cap - 16) / 12);
    c->b.kbuf = c->bin.as<uint2>();          // (8-byte entries first: alignment)
    c->b.ids_sorted = reinterpret_cast<uint32_t*>(c->b.kbuf + c->capacity);
    return G4D_OK;
}

int ensure_fused(G4DContext* c, int64_t n, bool with_sh) {
    const size_t N = (size_t)(n > 0 ? n : 1);
    FusedOutputs& fo = c->fo;
    auto layout = [&](Carve& m) {
        fo.means3D = m.take<float>(3 * N); fo.scales = m.take<float>(3 * N); fo.rotations = m.take<float>(4 * N);
        fo.opacities = m.take<float>(N); fo.rot_norm = m.take<float>(N);
        float* shs = m.take<float>(with_sh ? 48 * N : 4);
        fo.shs = with_sh ? shs : nullptr;
    };
    G4D_CUDA(ensure_layout(c->fused, layout));
    return G4D_OK;
}

// The set-up of one view on c: the buffers of n Gaussians and of the camera's image, the stage flags, and in the PREP stage
// the device camera (timestamp from d_time when set), then prep()
template <class Prep>
int setup_view(G4DContext* c, const G4DCamera* cam, const float* d_time, int64_t n, cudaStream_t st, Prep prep) {
    int rc;
    if ((rc = ensure_geom(c, n)) != G4D_OK) return rc;
    if ((rc = ensure_image(c, cam->image_height, cam->image_width)) != G4D_OK) return rc;
    reset_stage_flags(c, 0, G4D_STAGE_COUNT - 1);
    StageTimer tm(c, G4D_STAGE_PREP, st);
    G4D_CUDA(launch_pack_camera(*cam, d_time, c->cam.as<CameraDev>(), st));
    return prep();
}

int check_params(const G4DDeformParams* p) {
    if (!p) return fail(G4D_ERR_ARG, "deform params are NULL");
    if (p->levels < 1 || p->levels > G4D_MAX_LEVELS) return fail(G4D_ERR_ARG, "levels must be in 1..4");
    if (p->channels < 4 || p->channels > 32 || (p->channels & 3)) return fail(G4D_ERR_ARG, "channels must be a multiple of 4, <= 32");
    if (p->net_width != 64 && p->net_width != 128) return fail(G4D_ERR_ARG, "net_width must be 64 or 128");
    if (p->levels * p->channels > 128) return fail(G4D_ERR_ARG, "levels*channels must be <= 128");
    if (p->depth < 0 || p->depth > G4D_MAX_DEPTH) return fail(G4D_ERR_ARG, "depth (defor_depth) must be in 0..G4D_MAX_DEPTH (8)");
    for (int j = 1; j < p->depth; ++j)
        if (!p->wt[j - 1] || !p->bt[j - 1]) return fail(G4D_ERR_ARG, "trunk layer weight or bias (wt / bt) is NULL for a layer below depth");
    for (int l = 0; l < p->levels; ++l)
        for (int a = 0; a < 4; ++a)
            if (p->res[l][a] < 2 || p->res[l][a] > 65535) return fail(G4D_ERR_ARG, "plane resolution out of range");
    for (int l = 0; l < p->levels; ++l)
        for (int k = 0; k < 6; ++k) {
            // hexplane.cuh addresses a plane with 32-bit offsets: its scatter indexes floats, (Y*W + X)*C + c < 2^31
            if ((int64_t)p->res[l][plane_axis0(k)] * p->res[l][plane_axis1(k)] * p->channels >= (1ll << 31))
                return fail(G4D_ERR_ARG, "a plane has H*W*channels >= 2^31 floats: hexplane.cuh's 32-bit offsets cannot address it");
            // the gather reads the spatial planes' channel vectors as float4 (the time planes: scalar reads of the collapse)
            if (plane_axis1(k) != 3 && ((uintptr_t)p->planes[l][k] & 15u))
                return fail(G4D_ERR_ARG, "spatial planes must be 16-byte aligned");
        }
    return G4D_OK;
}

// The spatial-plane gradient sinks of the levels prm uses, which the network backward's scatter adds channel vectors to with
// red.v4.  (The time-plane sinks take the scalar atomics of the time-row distribution, the regulariser's sinks scalar adds.)
int check_plane_grads(const G4DDeformParams* p, const G4DDeformGrads* g) {
    for (int l = 0; l < p->levels; ++l)
        for (int k = 0; k < 6; ++k)
            if (plane_axis1(k) != 3 && ((uintptr_t)g->planes[l][k] & 15u))
                return fail(G4D_ERR_ARG, "spatial-plane gradient sinks must be 16-byte aligned (the scatter adds float4s)");
    return G4D_OK;
}

int refresh_packed(G4DWorkspace* ws, const G4DDeformParams* p, cudaStream_t st) {
    const size_t F = (size_t)p->levels * p->channels, WD = (size_t)p->net_width;
    const size_t ntrunk = p->depth > 1 ? (size_t)p->depth - 1 : 0;
    auto pack = [&](void* blob, FfmaWeights* w) {
        w->w0t = static_cast<float*>(blob);
        for (int h = 0; h < G4D_NUM_HEADS; ++h) w->w1t[h] = w->w0t + F * WD + h * WD * WD;
        for (size_t j = 0; j < G4D_MAX_DEPTH - 1; ++j) w->wtt[j] = j < ntrunk ? w->w0t + F * WD + (G4D_NUM_HEADS + j) * WD * WD : nullptr;
        return launch_pack_weights(*p, w->w0t, w->w1t, w->wtt, st);
    };
    G4D_CUDA(ws->packed.refresh(p, (F * WD + (G4D_NUM_HEADS + ntrunk) * WD * WD) * 4, pack));
    return G4D_OK;
}

int refresh_tc(G4DWorkspace* ws, const G4DDeformParams* p, cudaStream_t st) {
    if (!t_call.capturing && ws->pinned->f16_range) {   // (a capture leaves the flag to g4d_workspace_graph_status)
        ws->pinned->f16_range = 0;
        ws->tc.valid = false;      // re-pack (and re-check) the weights on the next call: they may be the out-of-range values
        return fail(G4D_ERR_OVERFLOW, "an earlier FP16x2 tensor-core launch met a value outside the f16 operand range (activation >= 8188, "
                                      "feature >= 1023 or weight >= 255): its results were saturated; set G4D_OPT_TENSOR_CORES = 0 (FFMA kernels, no range limit)");
    }
    auto pack = [&](void* blob, TcWeights* w) {
        w->status = &ws->pinned->f16_range;
        return launch_tc_pack_weights(*p, static_cast<float*>(blob), w, st);
    };
    G4D_CUDA(ws->tc.refresh(p, tc_packed_floats(*p) * 4, pack));
    return G4D_OK;
}

// w: the FP32 transposes, on the FFMA paths (the tensor-core kernels do not read them)
DeformDesc make_desc(const G4DDeformParams* p, float* const (*trow)[3], const FfmaWeights* w) {
    DeformDesc d{};
    d.levels = p->levels; d.C = p->channels; d.F = p->levels * p->channels; d.WD = p->net_width; d.head_mask = p->head_mask;
    for (int l = 0; l < p->levels; ++l) {
        for (int a = 0; a < 4; ++a) d.res[l][a] = p->res[l][a];
        for (int k = 0; k < 6; ++k) d.planes[l][k] = p->planes[l][k];
        for (int a = 0; a < 3; ++a) d.trow[l][a] = trow[l][a];
    }
    d.aabb = p->aabb; d.w0t = w ? w->w0t : nullptr; d.b0 = p->b0;
    for (int h = 0; h < G4D_NUM_HEADS; ++h) {
        d.w1t[h] = w ? w->w1t[h] : nullptr; d.b1[h] = p->b1[h]; d.w2[h] = p->w2[h]; d.b2[h] = p->b2[h];
    }
    d.ntrunk = p->depth > 1 ? p->depth - 1 : 0;
    for (int j = 0; j < d.ntrunk; ++j) { d.wtt[j] = w ? w->wtt[j] : nullptr; d.bt[j] = p->bt[j]; }
    return d;
}

// the deformation network of one forward call
struct DeformSetup {
    DeformDesc d;
    bool tc;              // the network runs on the tensor cores
    TcWeights tw;         // tc: weight images, range flag and debug counters; the caller adds its relu_bits buffer
    DeformGather gather;  // the walk order; the caller adds the feature buffer
};

// The walk order of the HexPlane gather over xyz [n] into *out (NULL: index order).  Rebuilt when the xyz pointer or n
// changes, kept otherwise -- also when xyz moved in place (a training step): the features do not depend on the order, so a
// stale one is still right and only costs L1 hits, but one built for another n is never used.  The rebuild is ordinary launches
// in stream order behind the earlier forwards that read the order (like the workspace's other buffers), issued ahead of the
// dependent chain of the forward that follows (DESIGN.md §4.6).
int gather_order(G4DWorkspace* ws, const float* aabb, const float* xyz, int64_t n, cudaStream_t st, const uint32_t** out) {
    *out = nullptr;
    if (!ws->gather_order || n <= 0) return G4D_OK;
    if (ws->order_xyz != xyz || ws->order_n != n) {
        ws->order_xyz = nullptr;
        GatherOrderBuffers& b = ws->order;
        auto layout = [&](Carve& m) {
            b.order = m.take<uint32_t>((size_t)n); b.key = m.take<uint2>((size_t)n);
            b.cell_start = m.take<uint32_t>(kOrderCells); b.block_total = m.take<uint32_t>(kOrderCells / 1024);
        };
        G4D_CUDA(ensure_layout(ws->order_buf, layout));
        G4D_CUDA(launch_gather_order(aabb, n, xyz, b, st));
        ws->order_xyz = xyz; ws->order_n = n;
    }
    *out = ws->order.order;
    return G4D_OK;
}

// the time planes interpolated at `time`, into `rows` (pointers in trow)
int collapse_time_rows(DevBuf& rows, float* (*trow)[3], const G4DDeformParams* p, TimeArg time, cudaStream_t st) {
    const TimeRows tr(p->levels, p->res, p->channels);
    if (rows.ensure(tr.total() * 4) != cudaSuccess)
        return t_call.growth_refused ? growth_refused("time-row buffer") : fail(G4D_ERR_NOMEM, "time-row buffer");
    tr.place(rows.as<float>(), trow);
    G4D_CUDA(launch_collapse_time_rows(*p, time, trow, st));
    return G4D_OK;
}

// Pick the forward's path from the params, bring the gather's walk order over xyz [n] up to date, collapse the time rows and
// bring the weight images the path reads up to date.  The desc is built after that refresh, which may move
// the transposes it embeds.  times (device [n], one time per Gaussian): no time rows; the gather samples each Gaussian at its
// own time, and `time` is not used.
int setup_deform(G4DWorkspace* ws, const G4DDeformParams* p, const float* xyz, int64_t n, DevBuf& rows, float* (*trow)[3],
                 TimeArg time, const float* times, cudaStream_t st, DeformSetup* out) {
    int rc;
    out->tc = ws->tensor_cores != 0 && tc_deform_supported(*p);
    if ((rc = gather_order(ws, p->aabb, xyz, n, st, &out->gather.order)) != G4D_OK) return rc;
    if (!times && (rc = collapse_time_rows(rows, trow, p, time, st)) != G4D_OK) return rc;
    if (!out->tc) {
        if ((rc = refresh_packed(ws, p, st)) != G4D_OK) return rc;
        out->d = make_desc(p, trow, &ws->packed.img);
        out->d.times = times;
        return G4D_OK;
    }
    if ((rc = refresh_tc(ws, p, st)) != G4D_OK) return rc;
    out->d = make_desc(p, trow, nullptr);
    out->d.times = times;
    out->tw = ws->tc.img;
    if (ws->tc_debug) {   // per-CTA phase cycle counters (g4d_debug_tc_cycles)
        G4D_CUDA(ws->tc_dbg.ensure((size_t)ws->sm_count * 12 * 8));
        G4D_CUDA(cudaMemsetAsync(ws->tc_dbg.p, 0, (size_t)ws->sm_count * 12 * 8, st));
        out->tw.dbg = ws->tc_dbg.as<long long>();
    }
    return G4D_OK;
}

// Buffers of this forward call.  feat: where the gather writes the HexPlane features [N][F] (NULL: the workspace's);
// relu_bits: where a tensor-core forward saves the ReLU signs for a backward, or NULL.  The tag word behind the bits tells
// the backward whether this forward wrote them.
int attach_forward_buffers(G4DWorkspace* ws, DeformSetup& s, float* feat, uint32_t* relu_bits, int64_t n, cudaStream_t st) {
    if (!feat) {
        G4D_CUDA(ws->feat.ensure((size_t)(n > 0 ? n : 1) * (size_t)s.d.F * 4 + 256));
        feat = ws->feat.as<float>();
    }
    s.gather.feat = feat;
    s.tw.relu_bits = relu_bits;
    if (relu_bits) G4D_CUDA(cudaMemsetAsync(relu_bits + (size_t)24 * (size_t)n, s.tc ? kReluBitsTagByte : 0, 16, st));
    return G4D_OK;
}

// backward of the deformation network with the time rows trow and dL/d(time) added into g_time (may be NULL) -- or, times
// set, at the per-Gaussian times [n] with dL/d(times) into g_times (may be NULL) -- picks the engine -- tensor-core when the configuration allows, FFMA otherwise -- and brings its
// weight images up to date; the desc is built after that refresh
int deform_backward_dispatch(G4DWorkspace* ws, const G4DDeformParams* prm, float* const (*trow)[3], const G4DDeformGrads* grads,
                             TimeArg time, const float* times, float* g_times, float* g_time, int64_t n, const float* xyz,
                             const float* const go[G4D_NUM_HEADS], float* const gi[G4D_NUM_HEADS], const uint32_t* relu_bits,
                             const float* saved_feat, cudaStream_t st) {
    int rc;
    const bool tc = ws->tensor_cores && tc_backward_supported(*prm);
    if (tc) {
        auto pack = [&](void* blob, TcBwdWeights* w) { return launch_tc_bwd_pack_weights(*prm, static_cast<uint8_t*>(blob), w, st); };
        G4D_CUDA(ws->tc_bwd.refresh(prm, tc_bwd_weight_bytes(*prm), pack));
    } else if ((rc = refresh_packed(ws, prm, st)) != G4D_OK) {
        return rc;
    }
    DeformDesc d = make_desc(prm, trow, tc ? nullptr : &ws->packed.img);
    d.times = times;
    const uint32_t* order = nullptr;   // the walk order of the backward's own gather (none when the forward's features are kept)
    if (!saved_feat && (rc = gather_order(ws, prm->aabb, xyz, n, st, &order)) != G4D_OK) return rc;
    G4D_CUDA(ws->scratch.ensure(deform_backward_scratch_bytes(d, n, tc)));
    G4D_CUDA(launch_deform_backward(d, *prm, *grads, tc ? &ws->tc_bwd.img : nullptr, time, n, xyz, go, gi, g_times, g_time, relu_bits, saved_feat,
                                    order, ws->scratch.p, ws->sm_count, st));
    return G4D_OK;
}

// M of a camera: the SH coefficients per Gaussian of the tensors it is rendered with (0 in G4DCamera.sh_coeffs means 16)
int sh_coeffs(const G4DCamera* cam) { return cam->sh_coeffs ? cam->sh_coeffs : kShCoeffs; }

int check_camera(const G4DCamera* cam) {
    if (!cam) return fail(G4D_ERR_ARG, "camera is NULL");
    if (cam->image_height <= 0 || cam->image_width <= 0 || cam->image_height > 16384 || cam->image_width > 16384)
        return fail(G4D_ERR_ARG, "image size out of range");
    if (cam->sh_degree < 0 || cam->sh_degree > 3) return fail(G4D_ERR_ARG, "sh_degree must be 0..3");
    const int m = sh_coeffs(cam);
    if (m != 1 && m != 4 && m != 9 && m != 16) return fail(G4D_ERR_ARG, "sh_coeffs must be 0, 1, 4, 9 or 16");
    if ((cam->sh_degree + 1) * (cam->sh_degree + 1) > m)
        return fail(G4D_ERR_ARG, "sh_degree needs more SH coefficients than sh_coeffs gives ((sh_degree + 1)^2 > M)");
    if (!(cam->tanfovx > 0.f) || !(cam->tanfovy > 0.f)) return fail(G4D_ERR_ARG, "tanfov must be positive");
    return G4D_OK;
}

int debug_sync(const G4DCamera* cam, cudaStream_t st, const char* stage) {
    if (!(cam->debug & G4D_CAM_DEBUG)) return G4D_OK;
    cudaError_t e = cudaStreamSynchronize(st);
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) return fail(G4D_ERR_CUDA, stage, cudaGetErrorString(e));
    return G4D_OK;
}

// no-sync mode: the previous forward's instance count arrives asynchronously; look at it before reusing the context
int check_pending(G4DContext* c) {
    if (t_call.capturing) return G4D_OK;   // (no host reads in a capture: its overflows go to g4d_workspace_graph_status)
    for (int k = 0; k < G4DContext::kSlots; ++k) {
        const int s = (c->slot + k) % G4DContext::kSlots;   // k = 0: the slot about to be reused (oldest forward: must be resolved), then the newer ones
        if (!c->pending[s]) continue;
        if (k == 0) {
            G4D_CUDA(cudaEventSynchronize(c->ev_r[s]));
        } else {
            const cudaError_t q = cudaEventQuery(c->ev_r[s]);
            if (q == cudaErrorNotReady) { (void)cudaGetLastError(); continue; }
            G4D_CUDA(q);
        }
        c->pending[s] = false;
        c->R = (int64_t)c->h_r[s];
        if (c->R > c->used_capacity[s]) {
            const int64_t need = c->R + c->R / 2;
            if (need > c->ws->min_capacity) c->ws->min_capacity = need;
            c->fwd = ForwardRecord{};
            char msg[160];
            snprintf(msg, sizeof(msg), "%lld tile instances did not fit the capacity of %lld used by an earlier no-sync forward; its image is incomplete",
                     (long long)c->R, (long long)c->used_capacity[s]);
            return fail(G4D_ERR_OVERFLOW, "instance buffer overflow", msg);
        }
    }
    return G4D_OK;
}

// stages after the per-Gaussian projection: bin_sort (depth order, per-tile counts, ranges, R) -> bin_place -> blend
int bin_and_blend(G4DContext* c, const G4DCamera* cam, int64_t n, float* out_color, float* out_depth, cudaStream_t st) {
    G4DWorkspace* ws = c->ws;
    const CameraDev* dcam = c->cam.as<CameraDev>();
    int rc;
    const int num_tiles = c->grid_x * c->grid_y;
    const uint32_t kNoCap = 0xFFFFFFFFu;
    const uint32_t* readback = nullptr;
    uint32_t cap_place = 0;
    if (n > 0) {
        if (ws->sm_count > 1024) return fail(G4D_ERR_ARG, "more than 1024 SMs are not supported by the binning kernel");
        G4D_CUDA(c->binaux.ensure(bin_aux_bytes(n, num_tiles, ws->sm_count)));
        // no-sync needs a capacity learnt from an earlier (exact) forward on this context
        const bool nosync = !ws->sync_mode && !(cam->debug & G4D_CAM_DEBUG) && c->capacity > 0 && c->learned;
        if (nosync && ws->min_capacity > c->capacity && (rc = ensure_bin(c, ws->min_capacity)) != G4D_OK) return rc;
        BinLayout lay{};
        {
            StageTimer tm(c, G4D_STAGE_SCAN, st);
            G4D_CUDA(launch_bin_sort(n, c->grid_x, c->grid_y, c->g, c->binaux.p, ws->tight_cull, ws->sm_count, &lay, st));
        }
        c->bin_ctl = lay.ctl;
        if (!nosync) {
            G4D_CUDA(cudaMemcpyAsync(&ws->pinned->num_rendered, &lay.ctl->R, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
            G4D_CUDA(cudaStreamSynchronize(st));   // exact mode: the one host sync of the path (as in the reference, A.2)
            const int64_t R = (int64_t)ws->pinned->num_rendered;
            c->R = R; c->learned = true;
            int64_t want = R;
            if (!ws->sync_mode) want = R + R / 2;                 // head-room for the asynchronous forwards that follow
            if (want < ws->min_capacity) want = ws->min_capacity;
            if ((rc = ensure_bin(c, want)) != G4D_OK) return rc;
        } else {
            // capacity-bounded, no host round trip: the placement clamps to the capacity, R arrives asynchronously and an
            // overflow is reported by the next call on this context
            // (the read-back itself is enqueued behind the blend kernel, below: a copy between bin_sort and the placement
            //  would keep the programmatically dependent launches of the chain from queueing up behind one another)
            readback = &lay.ctl->R;
        }
        if ((rc = debug_sync(cam, st, "bin_sort")) != G4D_OK) return rc;
        {
            StageTimer tm(c, G4D_STAGE_EMIT, st);
            cap_place = (uint32_t)(c->capacity < (int64_t)kNoCap ? c->capacity : (int64_t)kNoCap);
            G4D_CUDA(launch_bin_place(c->grid_x, c->grid_y, c->g, lay, c->b.ids_sorted, c->b.kbuf, c->b.ranges, cap_place, ws->tight_cull, st));
        }
    } else {
        c->R = 0;
        G4D_CUDA(cudaMemsetAsync(c->b.ranges, 0, sizeof(uint2) * (size_t)num_tiles, st));
        if ((rc = ensure_bin(c, 1)) != G4D_OK) return rc;
    }
    if ((rc = debug_sync(cam, st, "binning")) != G4D_OK) return rc;
    {
        StageTimer tm(c, G4D_STAGE_BLEND, st);
        G4D_CUDA(launch_blend_forward(dcam, c->grid_x, c->grid_y, c->g, c->b, c->im, out_color, out_depth, ws->warp_cull,
                                      c->terms.alpha_out, st));
    }
    if (readback && t_call.capturing) {
        G4D_CUDA(launch_record_overflow(static_cast<const BinCtl*>(c->bin_ctl), cap_place, ws->pinned->overflow, st));
    } else if (readback) {
        const int sl = c->slot;
        c->slot = (c->slot + 1) % G4DContext::kSlots;
        G4D_CUDA(cudaMemcpyAsync(c->h_r + sl, readback, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
        G4D_CUDA(cudaEventRecord(c->ev_r[sl], st));
        c->pending[sl] = true; c->used_capacity[sl] = c->capacity;
    }
    return debug_sync(cam, st, "blend_forward");
}

// A caller's SH tensors of M coefficients: fused [N,M,3] in dc, or (split) dc [N,1,3] + rest [N,M-1,3].  Sh = ShIn for the
// coefficients, ShOut for their gradient sinks.
template <class Sh, class T> Sh caller_sh(int m, bool split, T* dc, T* rest = nullptr) {
    return split ? Sh{nullptr, dc, rest, m} : Sh{dc, nullptr, nullptr, m};
}

// The terms of a backward on ctx[0, k): every context's capture refusal (ViewTerms::capture_refusal), then the camera and
// time gradient sinks zeroed on st; the backward adds into them, and a sink nothing adds into (a camera outside the loss, a
// backward without a deformation) keeps the zeros.  Called before the backward's first launch.
int zero_grad_sinks(G4DContext* const* ctx, int k, cudaStream_t st) {
    for (int i = 0; i < k && t_call.capturing; ++i)
        if (const char* why = ctx[i]->terms.capture_refusal()) return fail(G4D_ERR_STATE, why);
    for (int i = 0; i < k; ++i) {
        const ViewTerms& v = ctx[i]->terms;
        if (v.cam_grad) G4D_CUDA(cudaMemsetAsync(v.cam_grad, 0, kCamGradFloats * sizeof(float), st));
        if (v.time_grad) G4D_CUDA(cudaMemsetAsync(v.time_grad, 0, sizeof(float), st));
    }
    return G4D_OK;
}

// The frame of an entry point, built behind its argument checks and before its first launch: it makes ws's device current
// and sets t_call for the stream st (restored when the entry point returns; kRead synchronises the device instead).  Then,
// on the contexts ctx[0, k) and their cameras cams[0, k): a forward or backward refuses what a capture cannot repeat, every
// kind but kContextFree resolves the pending read-backs, a forward clears each context's record once its read-backs are
// resolved and a backward zeroes the gradient sinks.  rc != G4D_OK: the entry point returns it.
struct CallFrame {
    enum Kind { kContextFree, kRead, kForward, kBackward };
    CallState saved;
    int rc;
    CallFrame(Kind kind, const G4DWorkspace* ws, cudaStream_t st, G4DContext* const* ctx = nullptr, int k = 0,
              const G4DCamera* cams = nullptr)
        : saved(t_call), rc(open(kind, ws, st, ctx, k, cams)) {}
    ~CallFrame() { t_call = saved; }

  private:
    static int open(Kind kind, const G4DWorkspace* ws, cudaStream_t st, G4DContext* const* ctx, int k, const G4DCamera* cams) {
        G4D_CUDA(cudaSetDevice(ws->device));
        int rc = G4D_OK;
        if (kind == kRead) {
            G4D_CUDA(cudaDeviceSynchronize());
        } else {
            cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
            const cudaError_t e = cudaStreamIsCapturing(st, &cs);
            const bool capturing = cs != cudaStreamCaptureStatusNone;
            t_call = CallState{capturing, ws->frozen || capturing, false};
            if (e != cudaSuccess) {
                (void)cudaGetLastError();
                return fail(G4D_ERR_STATE, "cudaStreamIsCapturing", cudaGetErrorString(e));
            }
            if (kind != kContextFree) rc = refuse_capture(ws, cams, k, kind == kForward ? ctx : nullptr);
        }
        for (int i = 0; rc == G4D_OK && i < k; ++i)
            if ((rc = check_pending(ctx[i])) == G4D_OK && kind == kForward) ctx[i]->fwd = ForwardRecord{};
        return rc == G4D_OK && kind == kBackward ? zero_grad_sinks(ctx, k, st) : rc;
    }
};

// The blend backward of the forward on c: dL/d(mean2D, conic, rgb, opacity) into c->gscratch (BlendGradLayout, zeroed here),
// except that the opacity gradient lands in g_opacities (zeroed here) when it is set.  depth_block: the scratch has the depth
// block, which takes dL/d(view-space depth) when c has a depth gradient and stays zero otherwise.  c's alpha gradient, when
// set, is taken too.  dL_dcolor may be NULL when c has a depth or an alpha gradient.  *gb: the scratch.  n = 0 runs nothing.
int blend_backward(G4DContext* c, const G4DCamera* cam, int64_t n, const float* dL_dcolor, float* g_opacities, bool depth_block,
                   float** gb, cudaStream_t st) {
    using L = BlendGradLayout;
    const ViewTerms& v = c->terms;
    const size_t N = (size_t)(n > 0 ? n : 1);
    const size_t floats = N * (depth_block ? L::kDepthFloats : g_opacities ? L::kOpacity : L::kFloats);
    G4D_CUDA(c->gscratch.ensure(floats * 4 + 256));
    float* b = *gb = c->gscratch.as<float>();
    if (n == 0) return G4D_OK;
    G4D_CUDA(cudaMemsetAsync(b, 0, floats * 4, st));
    if (g_opacities) G4D_CUDA(cudaMemsetAsync(g_opacities, 0, N * 4, st));
    reset_stage_flags(c, G4D_STAGE_BLEND_BWD, G4D_STAGE_DEFORM_BWD);
    {
        StageTimer tm(c, G4D_STAGE_BLEND_BWD, st);
        G4D_CUDA(launch_blend_backward(c->cam.as<CameraDev>(), c->grid_x, c->grid_y, c->g, c->b, c->im, dL_dcolor, b + L::kMean2D * N,
                                       b + L::kConic * N, g_opacities ? g_opacities : b + L::kOpacity * N, b + L::kRgb * N,
                                       c->ws->warp_cull, v.depth_grad, v.depth_grad ? b + L::kDepth * N : nullptr, v.alpha_grad, st));
    }
    return debug_sync(cam, st, "blend_backward");
}

// blend backward + per-Gaussian backward on `in`; opacity gradient lands in g_opacities (zeroed here); the terms of c taken
// as they are set: the camera's gradient added into its sink, the depth and alpha images' gradients
int raster_backward_stages(G4DContext* c, const G4DCamera* cam, int64_t n, const RasterInputs& in, const float* dL_dcolor,
                           float* g_means3D, float* g_means2D, const ShOut& g_sh, float* g_opacities, float* g_scales,
                           float* g_rotations, cudaStream_t st) {
    using L = BlendGradLayout;
    const ViewTerms& v = c->terms;
    const size_t N = (size_t)n;
    float* gb;
    const int rc = blend_backward(c, cam, n, dL_dcolor, g_opacities, v.depth_grad != nullptr, &gb, st);
    if (rc != G4D_OK || n == 0) return rc;
    StageTimer tm(c, G4D_STAGE_GEOM_BWD, st);
    G4D_CUDA(launch_preprocess_backward(c->cam.as<CameraDev>(), n, in, c->g, gb + L::kMean2D * N, gb + L::kConic * N,
                                        gb + L::kRgb * N, g_means3D, g_means2D, g_scales, g_rotations, g_sh, v.cam_grad,
                                        v.depth_grad ? gb + L::kDepth * N : nullptr, st));
    return debug_sync(cam, st, "preprocess_backward");
}

}  // namespace

// ======================================================================================================
extern "C" {

int g4d_abi_version(void) { return G4D_ABI_VERSION; }
const char* g4d_last_error(void) { return t_last_error.c_str(); }

G4DWorkspace* g4d_workspace_create(int device) {
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || device < 0 || device >= count) {
        fail(G4D_ERR_CUDA, "g4d_workspace_create: no such CUDA device (the g4d path has no CPU fallback)");
        return nullptr;
    }
    if (cudaSetDevice(device) != cudaSuccess) { fail(G4D_ERR_CUDA, "cudaSetDevice"); return nullptr; }
    G4DWorkspace* ws = new G4DWorkspace();
    ws->device = device;
    if (const char* e = getenv("G4D_GATHER_ORDER")) ws->gather_order = atoi(e) != 0;
    cudaDeviceProp prop{};
    if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) ws->sm_count = prop.multiProcessorCount;
    if (cudaMallocHost((void**)&ws->pinned, sizeof(PinnedWords)) != cudaSuccess) { delete ws; fail(G4D_ERR_NOMEM, "cudaMallocHost"); return nullptr; }
    *ws->pinned = PinnedWords{};
    return ws;
}

void g4d_workspace_destroy(G4DWorkspace* ws) {
    if (!ws) return;
    cudaSetDevice(ws->device);
    if (ws->pinned) cudaFreeHost(ws->pinned);
    delete ws;
}

G4DContext* g4d_context_create(G4DWorkspace* ws) {
    if (!ws) { fail(G4D_ERR_ARG, "workspace is NULL"); return nullptr; }
    cudaSetDevice(ws->device);
    G4DContext* c = new G4DContext();
    c->ws = ws;
    if (c->cam.ensure(sizeof(CameraDev)) != cudaSuccess) { delete c; fail(G4D_ERR_NOMEM, "camera buffer"); return nullptr; }
    bool ok = cudaMallocHost((void**)&c->h_r, 64) == cudaSuccess;
    for (int i = 0; ok && i < G4DContext::kSlots; ++i) ok = cudaEventCreateWithFlags(&c->ev_r[i], cudaEventDisableTiming) == cudaSuccess;
    if (!ok) { g4d_context_destroy(c); fail(G4D_ERR_NOMEM, "pinned scalar / event"); return nullptr; }
    return c;
}

void g4d_context_destroy(G4DContext* c) {
    if (!c) return;
    cudaSetDevice(c->ws->device);
    if (c->ev_created) for (int i = 0; i < 2 * G4D_STAGE_COUNT; ++i) cudaEventDestroy(c->ev[i]);
    for (int i = 0; i < G4DContext::kSlots; ++i) if (c->ev_r[i]) cudaEventDestroy(c->ev_r[i]);
    if (c->h_r) cudaFreeHost(c->h_r);
    delete c;
}

int g4d_workspace_set_option(G4DWorkspace* ws, int option, int64_t value) {
    if (!ws) return fail(G4D_ERR_ARG, "workspace is NULL");
    switch (option) {
        case G4D_OPT_SYNC_MODE: ws->sync_mode = value ? 1 : 0; return G4D_OK;
        case G4D_OPT_INSTANCE_CAPACITY: ws->min_capacity = value; return G4D_OK;
        case G4D_OPT_TIGHT_CULL: ws->tight_cull = value ? 1 : 0; return G4D_OK;
        case G4D_OPT_STAGE_TIMING: ws->stage_timing = value ? 1 : 0; return G4D_OK;
        case G4D_OPT_TENSOR_CORES:
            if (value == 1) return fail(G4D_ERR_ARG, "G4D_OPT_TENSOR_CORES = 1 (3xTF32) was removed; 0 selects the FFMA kernels, which have no range limit");
            ws->tensor_cores = value == 0 ? 0 : 2;
            return G4D_OK;
        case G4D_OPT_WARP_CULL: ws->warp_cull = value ? 1 : 0; return G4D_OK;
        case G4D_OPT_TC_DEBUG: ws->tc_debug = value ? 1 : 0; return G4D_OK;
        case G4D_OPT_KEEP_DEFORMED: ws->keep_deformed = value ? 1 : 0; return G4D_OK;
        case G4D_OPT_PDL: g4d::g_pdl = value ? 1 : 0; return G4D_OK;
        case G4D_OPT_GATHER_ORDER: ws->gather_order = value ? 1 : 0; return G4D_OK;
        default: return fail(G4D_ERR_ARG, "unknown option");
    }
}

int g4d_context_stage_times(G4DContext* c, float* out_ms, int capacity) {
    if (!c || !out_ms || capacity < G4D_STAGE_COUNT) return fail(G4D_ERR_ARG, "need room for G4D_STAGE_COUNT floats");
    cudaSetDevice(c->ws->device);
    G4D_CUDA(cudaDeviceSynchronize());
    for (int i = 0; i < G4D_STAGE_COUNT; ++i) {
        out_ms[i] = 0.f;
        if (c->ev_created && c->ev_used[i]) {
            float ms = 0.f;
            if (cudaEventElapsedTime(&ms, c->ev[2 * i], c->ev[2 * i + 1]) == cudaSuccess) out_ms[i] = ms;
        }
    }
    return G4D_STAGE_COUNT;
}

int g4d_context_stats(G4DContext* c, G4DStats* out) {
    if (!c || !out) return fail(G4D_ERR_ARG, "NULL argument");
    if (c->fwd.kind == ForwardRecord::kNone) return fail(G4D_ERR_STATE, "no forward has run on this context");
    CallFrame call(CallFrame::kRead, c->ws, nullptr, &c, 1);
    if (call.rc != G4D_OK) return call.rc;
    out->num_rendered = c->R; out->instance_capacity = c->capacity; out->tiles_x = c->grid_x; out->tiles_y = c->grid_y;
    std::vector<int32_t> radii((size_t)c->fwd.n);
    if (c->fwd.n) G4D_CUDA(cudaMemcpy(radii.data(), c->g.radii, (size_t)c->fwd.n * 4, cudaMemcpyDeviceToHost));
    int64_t vis = 0;
    for (int32_t r : radii) vis += r > 0;
    out->num_visible = vis;
    return G4D_OK;
}

// ------------------------------------------------------------------------------------------------------
}  // extern "C"

namespace {

// g4d_deform_forward (times NULL: every Gaussian at `time`) and g4d_deform_forward_times (times [n], `time` unused)
int deform_forward(G4DWorkspace* ws, const G4DDeformParams* prm, int64_t n, const float* xyz, const float* scaling,
                   const float* rotation, const float* opacity, const float* shs, float time, const float* times, float* out_xyz,
                   float* out_scaling, float* out_rotation, float* out_opacity, float* out_shs, uint32_t* relu_bits, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    CallFrame call(CallFrame::kContextFree, ws, st);
    if (call.rc != G4D_OK) return call.rc;
    int rc;
    float* trow[G4D_MAX_LEVELS][3] = {};
    DeformSetup s{};
    if ((rc = setup_deform(ws, prm, xyz, n, ws->trow, trow, TimeArg{time, nullptr}, times, st, &s)) != G4D_OK) return rc;
    if ((rc = attach_forward_buffers(ws, s, nullptr, relu_bits, n, st)) != G4D_OK) return rc;
    const DeformIO io{xyz, scaling, rotation, opacity, caller_sh<ShIn>(kShCoeffs, false, shs), out_xyz, out_scaling, out_rotation, out_opacity,
                      out_shs, GeomBuffers{}, FusedOutputs{}, nullptr};
    G4D_CUDA(launch_deform(s.d, 0, nullptr, n, io, s.gather, ws->sm_count, st, s.tc ? &s.tw : nullptr));
    return G4D_OK;
}

// the argument checks of g4d_deform_forward / _forward_times
int check_deform_forward_args(G4DWorkspace* ws, const G4DDeformParams* prm, int64_t n, const float* xyz, const float* shs,
                              float* out_xyz, float* out_shs) {
    if (!ws) return fail(G4D_ERR_ARG, "workspace is NULL");
    int rc = check_params(prm);
    if (rc != G4D_OK) return rc;
    if (n < 0 || (n > 0 && (!xyz || !out_xyz))) return fail(G4D_ERR_ARG, "xyz / out_xyz required");
    if ((prm->head_mask & G4D_HEAD_SHS) && n > 0 && (!shs || !out_shs)) return fail(G4D_ERR_ARG, "shs / out_shs required when the SHS head is active");
    return G4D_OK;
}

}  // namespace

extern "C" {

int g4d_deform_forward(G4DWorkspace* ws, const G4DDeformParams* prm, int64_t n, const float* xyz, const float* scaling,
                       const float* rotation, const float* opacity, const float* shs, float time, float* out_xyz,
                       float* out_scaling, float* out_rotation, float* out_opacity, float* out_shs, uint32_t* relu_bits, void* stream) {
    const int rc = check_deform_forward_args(ws, prm, n, xyz, shs, out_xyz, out_shs);
    if (rc != G4D_OK) return rc;
    return deform_forward(ws, prm, n, xyz, scaling, rotation, opacity, shs, time, nullptr, out_xyz, out_scaling, out_rotation,
                          out_opacity, out_shs, relu_bits, stream);
}

int g4d_deform_forward_times(G4DWorkspace* ws, const G4DDeformParams* prm, int64_t n, const float* xyz, const float* scaling,
                             const float* rotation, const float* opacity, const float* shs, const float* d_times, float* out_xyz,
                             float* out_scaling, float* out_rotation, float* out_opacity, float* out_shs, uint32_t* relu_bits,
                             void* stream) {
    const int rc = check_deform_forward_args(ws, prm, n, xyz, shs, out_xyz, out_shs);
    if (rc != G4D_OK) return rc;
    if (!d_times) return fail(G4D_ERR_ARG, "d_times is NULL");
    return deform_forward(ws, prm, n, xyz, scaling, rotation, opacity, shs, 0.f, d_times, out_xyz, out_scaling, out_rotation,
                          out_opacity, out_shs, relu_bits, stream);
}

// ------------------------------------------------------------------------------------------------------
int g4d_rasterize_forward(G4DContext* c, const G4DCamera* cam, int64_t n, const float* means3D, const float* shs,
                          const float* opacities, const float* scales, const float* rotations, float* out_color,
                          float* out_depth, int32_t* out_radii, void* stream) {
    if (!c) return fail(G4D_ERR_ARG, "context is NULL");
    int rc = check_camera(cam);
    if (rc != G4D_OK) return rc;
    if (n < 0 || !out_color || !out_depth) return fail(G4D_ERR_ARG, "bad n / output pointers");
    if (n > 0 && (!means3D || !shs || !opacities || !scales || !rotations || !out_radii))
        return fail(G4D_ERR_ARG, "Please provide means3D, shs, opacities, scales and rotations");
    if (n >= (1ll << 31)) return fail(G4D_ERR_ARG, "n too large");
    cudaStream_t st = (cudaStream_t)stream;
    CallFrame call(CallFrame::kForward, c->ws, st, &c, 1, cam);
    if (call.rc != G4D_OK) return call.rc;
    if ((rc = setup_view(c, cam, nullptr, n, st, [] { return G4D_OK; })) != G4D_OK) return rc;
    const RasterInputs in{means3D, scales, rotations, opacities, caller_sh<ShIn>(sh_coeffs(cam), false, shs)};
    {
        StageTimer tm(c, G4D_STAGE_GEOM, st);
        G4D_CUDA(launch_preprocess(c->cam.as<CameraDev>(), n, in, c->g, out_radii, st));
    }
    if ((rc = bin_and_blend(c, cam, n, out_color, out_depth, st)) != G4D_OK) return rc;
    c->fwd = ForwardRecord{ForwardRecord::kRaster, n, cam->image_height, cam->image_width};
    c->fwd.sh_coeffs = sh_coeffs(cam);
    return G4D_OK;
}

int g4d_rasterize_backward(G4DContext* c, const G4DCamera* cam, int64_t n, const float* means3D, const float* shs,
                           const float* opacities, const float* scales, const float* rotations, const float* dL_dcolor,
                           float* g_means3D, float* g_means2D, float* g_shs, float* g_opacities, float* g_scales,
                           float* g_rotations, void* stream) {
    if (!c) return fail(G4D_ERR_ARG, "context is NULL");
    if (c->fwd.kind != ForwardRecord::kRaster || c->fwd.n != n) return fail(G4D_ERR_STATE, "g4d_rasterize_backward needs the matching g4d_rasterize_forward on this context");
    int rc = check_camera(cam);
    if (rc != G4D_OK) return rc;
    if (cam->image_height != c->fwd.H || cam->image_width != c->fwd.W) return fail(G4D_ERR_STATE, "camera differs from the forward's");
    if (sh_coeffs(cam) != c->fwd.sh_coeffs) return fail(G4D_ERR_STATE, "sh_coeffs differs from the forward's");
    if (!dL_dcolor || (n > 0 && (!g_means3D || !g_means2D || !g_shs || !g_opacities || !g_scales || !g_rotations)))
        return fail(G4D_ERR_ARG, "NULL gradient pointer");
    cudaStream_t st = (cudaStream_t)stream;
    CallFrame call(CallFrame::kBackward, c->ws, st, &c, 1, cam);
    if (call.rc != G4D_OK) return call.rc;
    (void)opacities;
    const int m = sh_coeffs(cam);
    const RasterInputs in{means3D, scales, rotations, opacities, caller_sh<ShIn>(m, false, shs)};
    return raster_backward_stages(c, cam, n, in, dL_dcolor, g_means3D, g_means2D, caller_sh<ShOut>(m, false, g_shs),
                                  g_opacities, g_scales, g_rotations, st);
}

// ------------------------------------------------------------------------------------------------------
int64_t g4d_context_read(G4DContext* c, int which, void* host_dst, int64_t bytes) {
    if (!c || c->fwd.kind == ForwardRecord::kNone) return fail(G4D_ERR_STATE, "no forward has run on this context");
    CallFrame call(CallFrame::kRead, c->ws, nullptr, &c, 1);
    if (call.rc != G4D_OK) return call.rc;
    const size_t N = (size_t)c->fwd.n, P = (size_t)c->fwd.H * c->fwd.W, R = (size_t)c->R, Tn = (size_t)c->grid_x * c->grid_y;
    std::vector<char> tmp;
    auto pull = [&](const void* src, size_t nbytes) -> bool {
        tmp.resize(nbytes ? nbytes : 1);
        return nbytes == 0 || cudaMemcpy(tmp.data(), src, nbytes, cudaMemcpyDeviceToHost) == cudaSuccess;
    };
    std::vector<char> outv;
    bool ok = true;
    switch (which) {
        case G4D_BUF_DEPTH: {
            ok = pull(c->g.rec2, N * 8); outv.resize(N * 4);
            for (size_t i = 0; i < N && ok; ++i) memcpy(&outv[i * 4], &tmp[i * 8 + 4], 4);
        } break;
        case G4D_BUF_RECT: {
            ok = pull(c->g.rect, N * 8); outv.resize(N * 16);
            for (size_t i = 0; i < N && ok; ++i) {
                uint32_t a, b; memcpy(&a, &tmp[i * 8], 4); memcpy(&b, &tmp[i * 8 + 4], 4);
                int32_t r[4] = {(int32_t)(a & 0xFFFF), (int32_t)(a >> 16), (int32_t)(b & 0xFFFF), (int32_t)(b >> 16)};
                memcpy(&outv[i * 16], r, 16);
            }
        } break;
        case G4D_BUF_TILES_TOUCHED: ok = pull(c->g.tiles_touched, N * 4); outv = tmp; outv.resize(N * 4); break;
        case G4D_BUF_XY: {
            ok = pull(c->g.rec0, N * 16); outv.resize(N * 8);
            for (size_t i = 0; i < N && ok; ++i) memcpy(&outv[i * 8], &tmp[i * 16], 8);
        } break;
        case G4D_BUF_CONIC_OPACITY: {
            ok = pull(c->g.rec0, N * 16); std::vector<char> t0 = tmp; ok = ok && pull(c->g.rec1, N * 16); outv.resize(N * 16);
            for (size_t i = 0; i < N && ok; ++i) { memcpy(&outv[i * 16], &t0[i * 16 + 8], 8); memcpy(&outv[i * 16 + 8], &tmp[i * 16], 8); }
        } break;
        case G4D_BUF_RGB: {
            ok = pull(c->g.rec1, N * 16); std::vector<char> t1 = tmp; ok = ok && pull(c->g.rec2, N * 8); outv.resize(N * 12);
            for (size_t i = 0; i < N && ok; ++i) { memcpy(&outv[i * 12], &t1[i * 16 + 8], 8); memcpy(&outv[i * 12 + 8], &tmp[i * 8], 4); }
        } break;
        case G4D_BUF_SORTED_KEYS: {
            // the (tile | depth bits) keys of the reference's sorted list are implicit in (ranges, ids, depth): rebuilt here
            ok = pull(c->b.ids_sorted, R * 4); std::vector<char> ids = tmp;
            ok = ok && pull(c->b.ranges, Tn * 8); std::vector<char> rg = tmp;
            ok = ok && pull(c->g.rec2, N * 8);
            outv.resize(R * 8);
            for (size_t t = 0; t < Tn && ok; ++t) {
                uint32_t lo, hi; memcpy(&lo, &rg[t * 8], 4); memcpy(&hi, &rg[t * 8 + 4], 4);
                for (size_t i = lo; i < hi && i < R; ++i) {
                    uint32_t id, db; memcpy(&id, &ids[i * 4], 4); memcpy(&db, &tmp[(size_t)id * 8 + 4], 4);
                    const uint64_t key = ((uint64_t)t << 32) | db;
                    memcpy(&outv[i * 8], &key, 8);
                }
            }
        } break;
        case G4D_BUF_SORTED_IDS: ok = pull(c->b.ids_sorted, R * 4); outv = tmp; outv.resize(R * 4); break;
        case G4D_BUF_RANGES: ok = pull(c->b.ranges, Tn * 8); outv = tmp; outv.resize(Tn * 8); break;
        case G4D_BUF_FINAL_T: ok = pull(c->im.final_T, P * 4); outv = tmp; outv.resize(P * 4); break;
        case G4D_BUF_N_CONTRIB: ok = pull(c->im.n_contrib, P * 4); outv = tmp; outv.resize(P * 4); break;
        case G4D_BUF_CLAMPED: {
            ok = pull(c->g.clamped, N); outv.resize(N * 3);
            for (size_t i = 0; i < N && ok; ++i) for (int ch = 0; ch < 3; ++ch) outv[i * 3 + ch] = (tmp[i] >> ch) & 1;
        } break;
        case G4D_BUF_DEFORMED: {
            if (!c->fwd.kept) return fail(G4D_ERR_STATE, "G4D_BUF_DEFORMED needs a fused forward that kept its tensors (grad-enabled, or G4D_OPT_KEEP_DEFORMED)");
            outv.resize(N * 44);
            std::vector<float> m(N * 3), s(N * 3), r(N * 4), o(N);
            ok = N == 0 || (cudaMemcpy(m.data(), c->fo.means3D, N * 12, cudaMemcpyDeviceToHost) == cudaSuccess &&
                            cudaMemcpy(s.data(), c->fo.scales, N * 12, cudaMemcpyDeviceToHost) == cudaSuccess &&
                            cudaMemcpy(r.data(), c->fo.rotations, N * 16, cudaMemcpyDeviceToHost) == cudaSuccess &&
                            cudaMemcpy(o.data(), c->fo.opacities, N * 4, cudaMemcpyDeviceToHost) == cudaSuccess);
            float* dst = reinterpret_cast<float*>(outv.data());
            for (size_t i = 0; i < N && ok; ++i) {
                memcpy(dst + i * 11, &m[i * 3], 12); memcpy(dst + i * 11 + 3, &s[i * 3], 12);
                memcpy(dst + i * 11 + 6, &r[i * 4], 16); dst[i * 11 + 10] = o[i];
            }
        } break;
        case G4D_BUF_DEFORMED_SHS: {
            if (!c->fwd.kept || !c->fwd.sh) return fail(G4D_ERR_STATE, "G4D_BUF_DEFORMED_SHS needs a fused forward with the SHS head active");
            ok = pull(c->fo.shs, N * 192); outv = tmp; outv.resize(N * 192);
        } break;
        case G4D_BUF_BIN_PHASES: {
            if (!c->bin_ctl) return fail(G4D_ERR_STATE, "no binning has run on this context");
            ok = pull(reinterpret_cast<const char*>(c->bin_ctl) + 16, 16 * 8); outv = tmp; outv.resize(16 * 8);
        } break;
        case G4D_BUF_FEATURES: {
            if (!c->fwd.feat_cols) return fail(G4D_ERR_STATE, "G4D_BUF_FEATURES needs a grad-enabled tensor-core fused forward");
            const size_t nb = N * (size_t)c->fwd.feat_cols * 4;
            ok = pull(c->feat.p, nb); outv = tmp; outv.resize(nb);
        } break;
        case G4D_BUF_GATHER_ORDER: {
            const G4DWorkspace* ws = c->ws;
            const size_t nb = ws->order_xyz ? (size_t)ws->order_n * 4 : 0;
            ok = pull(ws->order.order, nb); outv = tmp; outv.resize(nb);
        } break;
        default: return fail(G4D_ERR_ARG, "unknown buffer id");
    }
    if (!ok) return fail(G4D_ERR_CUDA, "cudaMemcpy in g4d_context_read");
    const int64_t held = (int64_t)outv.size();
    if (host_dst && bytes > 0) memcpy(host_dst, outv.data(), (size_t)(bytes < held ? bytes : held));
    return held;
}

// ------------------------------------------------------------------------------------------------------
}  // extern "C"

namespace {

// the argument checks of g4d_deform_backward / _backward_times
int check_deform_backward_args(G4DWorkspace* ws, const G4DDeformParams* prm, const G4DDeformGrads* grads, int64_t n, const float* xyz) {
    if (!ws) return fail(G4D_ERR_ARG, "workspace is NULL");
    int rc = check_params(prm);
    if (rc != G4D_OK) return rc;
    if (!grads) return fail(G4D_ERR_ARG, "grads is NULL");
    if ((rc = check_plane_grads(prm, grads)) != G4D_OK) return rc;
    if (n < 0 || (n > 0 && !xyz)) return fail(G4D_ERR_ARG, "xyz required");
    return G4D_OK;
}

// g4d_deform_backward (times NULL: the time rows at `time`) and g4d_deform_backward_times (times [n], dL/d(times) into g_times)
int deform_backward(G4DWorkspace* ws, const G4DDeformParams* prm, G4DDeformGrads* grads, int64_t n, const float* xyz, float time,
                    const float* times, const float* const go[G4D_NUM_HEADS], float* const gi[G4D_NUM_HEADS], float* g_times,
                    const uint32_t* relu_bits, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    CallFrame call(CallFrame::kContextFree, ws, st);
    if (call.rc != G4D_OK) return call.rc;
    int rc;
    float* trow[G4D_MAX_LEVELS][3] = {};
    if (!times && (rc = collapse_time_rows(ws->trow, trow, prm, TimeArg{time, nullptr}, st)) != G4D_OK) return rc;
    return deform_backward_dispatch(ws, prm, trow, grads, TimeArg{time, nullptr}, times, g_times, nullptr, n, xyz, go, gi, relu_bits,
                                    nullptr, st);
}

}  // namespace

extern "C" {

int g4d_deform_backward(G4DWorkspace* ws, const G4DDeformParams* prm, G4DDeformGrads* grads, int64_t n, const float* xyz,
                        float time, const float* g_out_xyz, const float* g_out_scaling, const float* g_out_rotation,
                        const float* g_out_opacity, const float* g_out_shs, float* g_in_xyz, float* g_in_scaling,
                        float* g_in_rotation, float* g_in_opacity, float* g_in_shs, const uint32_t* relu_bits, void* stream) {
    const int rc = check_deform_backward_args(ws, prm, grads, n, xyz);
    if (rc != G4D_OK) return rc;
    const float* go[G4D_NUM_HEADS] = {g_out_xyz, g_out_scaling, g_out_rotation, g_out_opacity, g_out_shs};
    float* gi[G4D_NUM_HEADS] = {g_in_xyz, g_in_scaling, g_in_rotation, g_in_opacity, g_in_shs};
    return deform_backward(ws, prm, grads, n, xyz, time, nullptr, go, gi, nullptr, relu_bits, stream);
}

int g4d_deform_backward_times(G4DWorkspace* ws, const G4DDeformParams* prm, G4DDeformGrads* grads, int64_t n, const float* xyz,
                              const float* d_times, const float* g_out_xyz, const float* g_out_scaling, const float* g_out_rotation,
                              const float* g_out_opacity, const float* g_out_shs, float* g_in_xyz, float* g_in_scaling,
                              float* g_in_rotation, float* g_in_opacity, float* g_in_shs, float* g_times, const uint32_t* relu_bits,
                              void* stream) {
    const int rc = check_deform_backward_args(ws, prm, grads, n, xyz);
    if (rc != G4D_OK) return rc;
    if (!d_times) return fail(G4D_ERR_ARG, "d_times is NULL");
    const float* go[G4D_NUM_HEADS] = {g_out_xyz, g_out_scaling, g_out_rotation, g_out_opacity, g_out_shs};
    float* gi[G4D_NUM_HEADS] = {g_in_xyz, g_in_scaling, g_in_rotation, g_in_opacity, g_in_shs};
    return deform_backward(ws, prm, grads, n, xyz, 0.f, d_times, go, gi, g_times, relu_bits, stream);
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------------
namespace {

// the SHS head adds a delta to all 16 coefficients (deformation.py:142): it needs models with all 16
int check_sh_head(const G4DCamera* cam, const G4DDeformParams* prm) {
    if (prm && (prm->head_mask & G4D_HEAD_SHS) && sh_coeffs(cam) != kShCoeffs)
        return fail(G4D_ERR_ARG, "the SHS head deforms 16 SH coefficients: it needs sh_coeffs 16");
    return G4D_OK;
}

int check_render_args(const G4DCamera* cam, const G4DDeformParams* prm, const G4DGaussians* g, const float* out_color,
                      const float* out_depth, const int32_t* out_radii) {
    int rc = check_camera(cam);
    if (rc != G4D_OK) return rc;
    if (prm && (rc = check_params(prm)) != G4D_OK) return rc;
    if ((rc = check_sh_head(cam, prm)) != G4D_OK) return rc;
    if (!g || g->n < 0 || g->n >= (1ll << 31) || !out_color || !out_depth) return fail(G4D_ERR_ARG, "bad gaussians / outputs");
    if (g->n > 0 && (!g->xyz || !g->scaling || !g->rotation || !g->opacity || !g->features_dc || !out_radii))
        return fail(G4D_ERR_ARG, "NULL gaussian tensor");
    return G4D_OK;
}

// The fused forward of one camera on c; *rec: the record of c once the calling entry point has succeeded.  keep_fo: store
// the deformed, activated tensors even under G4D_CAM_NO_GRAD (other cameras of the same call read them).
int fused_forward(G4DContext* c, const G4DCamera* cam, const G4DDeformParams* prm, const G4DGaussians* g, float* out_color,
                  float* out_depth, int32_t* out_radii, bool keep_fo, cudaStream_t st, ForwardRecord* rec) {
    const int64_t n = g->n;
    G4DWorkspace* ws = c->ws;
    int rc;
    const bool with_sh = prm && (prm->head_mask & G4D_HEAD_SHS);
    // a no-grad render needs none of the saved tensors: skip their stores (48 B + 192 B of deformed SH per Gaussian)
    const bool kept = !(cam->debug & G4D_CAM_NO_GRAD) || ws->keep_deformed || keep_fo;
    *rec = ForwardRecord{ForwardRecord::kFused, n, cam->image_height, cam->image_width, prm != nullptr, with_sh, kept,
                         sh_coeffs(cam)};
    if ((rc = ensure_fused(c, n, with_sh)) != G4D_OK) return rc;
    CameraDev* dcam = c->cam.as<CameraDev>();
    DeformSetup s{};
    auto prep = [&] {
        return prm ? setup_deform(ws, prm, g->xyz, n, c->trow, c->trow_ptr, TimeArg{cam->time, c->time_src}, nullptr, st, &s) : G4D_OK;
    };
    if ((rc = setup_view(c, cam, c->time_src, n, st, prep)) != G4D_OK) return rc;
    {
        StageTimer tm(c, G4D_STAGE_GEOM, st);
        const DeformIO io{g->xyz, g->scaling, g->rotation, g->opacity,
                          caller_sh<ShIn>(rec->sh_coeffs, g->features_rest != nullptr, g->features_dc, g->features_rest),
                          nullptr, nullptr, nullptr, nullptr, nullptr, c->g, kept ? c->fo : FusedOutputs{}, out_radii};
        if (prm) {
            const bool save = s.tc && !(cam->debug & G4D_CAM_NO_GRAD);
            if (save) {   // a backward will follow: it re-uses the ReLU signs and the staged HexPlane features
                G4D_CUDA(c->relu.ensure(G4D_RELU_BITS_WORDS(n) * 4));
                G4D_CUDA(c->feat.ensure((size_t)(n > 0 ? n : 1) * (size_t)s.d.F * 4 + 256));
                rec->feat_cols = s.d.F;
            }
            if ((rc = attach_forward_buffers(ws, s, save ? c->feat.as<float>() : nullptr, save ? c->relu.as<uint32_t>() : nullptr,
                                             n, st)) != G4D_OK) return rc;
            G4D_CUDA(launch_deform(s.d, 1, dcam, n, io, s.gather, ws->sm_count, st, s.tc ? &s.tw : nullptr));
        } else {
            G4D_CUDA(launch_activate_preprocess(dcam, n, io, st));
        }
    }
    if ((rc = debug_sync(cam, st, "deform+preprocess")) != G4D_OK) return rc;
    return bin_and_blend(c, cam, n, out_color, out_depth, st);
}

// the post-activation inputs of the rasterizer stages of the fused forward f on c: its stored deformed tensors, and the SH
// coefficients (deformed when the SHS head was active, the caller's otherwise)
RasterInputs deformed_inputs(const G4DContext* c, const ForwardRecord& f, const G4DGaussians* g) {
    RasterInputs in{c->fo.means3D, c->fo.scales, c->fo.rotations, c->fo.opacities,
                    caller_sh<ShIn>(f.sh_coeffs, g->features_rest != nullptr, g->features_dc, g->features_rest)};
    if (f.sh) in.sh = ShIn{c->fo.shs, nullptr, nullptr};
    return in;
}

// Gradients w.r.t. the deformed tensors of the backward of a fused forward on c: the caller's sinks in the coarse stage,
// scratch on c in the fine stage (the network's backward reads them)
struct DeformedGrads { float *xyz, *sc, *rot, *op, *sh; };
int deformed_grads(G4DContext* c, int64_t n, const G4DGaussianGrads* gg, DeformedGrads* out) {
    const size_t N = (size_t)n;
    DeformedGrads& d = *out;
    d = DeformedGrads{gg->xyz, gg->scaling, gg->rotation, gg->opacity, nullptr};
    if (!c->fwd.deformed) return G4D_OK;
    auto layout = [&](Carve& m) {
        d.xyz = m.take<float>(3 * N); d.sc = m.take<float>(3 * N); d.rot = m.take<float>(4 * N); d.op = m.take<float>(N);
        d.sh = m.take<float>(c->fwd.sh ? 48 * N : 4);
    };
    G4D_CUDA(ensure_layout(c->gdeform, layout));
    if (!c->fwd.sh) d.sh = nullptr;
    return G4D_OK;
}

// The SH gradient sinks of the backward of a fused forward on c: the caller's.  With the SHS head active the gradient also
// feeds the network's backward: the fused sink is then the scratch d_sh, which fused_backward_tail passes on to a caller
// sink in the fused layout.
ShOut fused_sh_sinks(const G4DContext* c, const G4DGaussians* g, const G4DGaussianGrads* gg, float* d_sh) {
    ShOut o = caller_sh<ShOut>(c->fwd.sh_coeffs, g->features_rest != nullptr, gg->features_dc, gg->features_rest);
    if (c->fwd.sh) o.shs = d_sh;
    return o;
}

// The tail of the backward of a fused forward on c, after its per-Gaussian backward wrote d: the SH gradient copy, the
// activation backward and, in the fine stage, the network's backward, which adds dL/d(time) into g_time when it is set.
// cam: the camera whose time and debug flag it uses.
int fused_backward_tail(G4DContext* c, const G4DCamera* cam, const G4DDeformParams* prm, G4DDeformGrads* pgrads,
                        const G4DGaussians* g, const G4DGaussianGrads* gg, const DeformedGrads& d, float* g_time, cudaStream_t st) {
    const int64_t n = g->n;
    int rc;
    if (c->fwd.sh && !g->features_rest)
        G4D_CUDA(cudaMemcpyAsync(gg->features_dc, d.sh, (size_t)n * 192, cudaMemcpyDeviceToDevice, st));
    G4D_CUDA(launch_activation_backward(n, c->fo, d.sc, d.rot, d.op, st));
    if (!c->fwd.deformed) return debug_sync(cam, st, "activation_backward");
    const float* go[G4D_NUM_HEADS] = {d.xyz, d.sc, d.rot, d.op, d.sh};
    float* gi[G4D_NUM_HEADS] = {gg->xyz, gg->scaling, gg->rotation, gg->opacity, nullptr};
    const bool saved = c->fwd.feat_cols != 0;
    {
        StageTimer tm(c, G4D_STAGE_DEFORM_BWD, st);
        if ((rc = deform_backward_dispatch(c->ws, prm, c->trow_ptr, pgrads, TimeArg{cam->time, c->time_src}, nullptr, nullptr, g_time,
                                           n, g->xyz, go, gi, saved ? c->relu.as<uint32_t>() : nullptr,
                                           saved ? c->feat.as<float>() : nullptr, st)) != G4D_OK) return rc;
    }
    return debug_sync(cam, st, "deform_backward");
}

// The backward of a fused forward of one camera on c (arguments checked by the caller).  gg->means2D may be NULL.
int fused_backward(G4DContext* c, const G4DCamera* cam, const G4DDeformParams* prm, G4DDeformGrads* pgrads, const G4DGaussians* g,
                   const float* dL_dcolor, const G4DGaussianGrads* gg, cudaStream_t st) {
    const int64_t n = g->n;
    int rc;
    if (n == 0) return G4D_OK;
    DeformedGrads d;
    if ((rc = deformed_grads(c, n, gg, &d)) != G4D_OK) return rc;
    // SH gradient: identity residual path -> written straight into the caller's sinks; the fused copy (when the SHS
    // head is active) additionally feeds the network's backward
    rc = raster_backward_stages(c, cam, n, deformed_inputs(c, c->fwd, g), dL_dcolor, d.xyz, gg->means2D,
                                fused_sh_sinks(c, g, gg, d.sh), d.op, d.sc, d.rot, st);
    if (rc != G4D_OK) return rc;
    return fused_backward_tail(c, cam, prm, pgrads, g, gg, d, c->terms.time_grad, st);
}

// k cameras on k contexts: 1 <= k <= G4D_MAX_CAMERAS, one time bit for bit (or, when ctx[0] has a time source, that same
// source on every context), pairwise distinct contexts of one workspace.  The cameras are checked before any context other
// than ctx[0] is looked at.
int check_camera_group(G4DContext* const* ctx, int32_t k, const G4DCamera* cams) {
    if (k < 1 || k > G4D_MAX_CAMERAS) return fail(G4D_ERR_ARG, "the number of cameras must be in 1..G4D_MAX_CAMERAS");
    if (!cams) return fail(G4D_ERR_ARG, "cameras are NULL");
    int rc;
    const float* src = ctx && ctx[0] ? ctx[0]->time_src : nullptr;
    for (int i = 0; i < k; ++i) {
        if ((rc = check_camera(&cams[i])) != G4D_OK) return rc;
        if (sh_coeffs(&cams[i]) != sh_coeffs(&cams[0])) return fail(G4D_ERR_ARG, "the cameras of one call must share sh_coeffs");
        if (!src && memcmp(&cams[i].time, &cams[0].time, sizeof(float)) != 0)
            return fail(G4D_ERR_ARG, "the cameras of one call must share their time bit for bit");
    }
    if (!ctx) return fail(G4D_ERR_ARG, "contexts are NULL");
    for (int i = 0; i < k; ++i) {
        if (!ctx[i]) return fail(G4D_ERR_ARG, "context is NULL");
        if (ctx[i]->ws != ctx[0]->ws) return fail(G4D_ERR_ARG, "the contexts of one call must belong to one workspace");
        if (ctx[i]->time_src != src)
            return fail(G4D_ERR_ARG, "the contexts of one call must share their time source (g4d_context_set_time_source), or have none");
        for (int j = 0; j < i; ++j)
            if (ctx[j] == ctx[i]) return fail(G4D_ERR_ARG, "the contexts of one call must be pairwise distinct");
    }
    return G4D_OK;
}

// The checks g4d_render_backward and g4d_render_backward_cameras share, behind each one's own checks of its arguments and of
// the records it matches: the forward on ctx[0, k) (saved: it kept what the backward reads; `who` names the entry point)
// deformed exactly when params are given now, cams[i] has the image size and M of the forward on ctx[i], and the params,
// their gradient sinks and the Gaussians' gradient sinks are usable.
int check_fused_backward(const char* who, bool saved, G4DContext* const* ctx, int k, const G4DCamera* cams,
                         const G4DDeformParams* prm, const G4DDeformGrads* pgrads, const G4DGaussians* g,
                         const G4DGaussianGrads* gg) {
    if (!saved) return fail(G4D_ERR_STATE, (std::string(who) + " after a G4D_CAM_NO_GRAD forward: nothing was saved for it").c_str());
    if ((prm != nullptr) != ctx[0]->fwd.deformed) return fail(G4D_ERR_STATE, "deform params differ from the forward's");
    int rc;
    if (prm && (rc = check_params(prm)) != G4D_OK) return rc;
    if ((rc = check_sh_head(&cams[0], prm)) != G4D_OK) return rc;
    if (prm && !pgrads) return fail(G4D_ERR_ARG, "pgrads is NULL");
    if (prm && (rc = check_plane_grads(prm, pgrads)) != G4D_OK) return rc;
    for (int i = 0; i < k; ++i) {
        const ForwardRecord& f = ctx[i]->fwd;
        if (cams[i].image_height != f.H || cams[i].image_width != f.W) return fail(G4D_ERR_STATE, "camera differs from the forward's");
        if (sh_coeffs(&cams[i]) != f.sh_coeffs) return fail(G4D_ERR_STATE, "sh_coeffs differs from the forward's");
    }
    const int64_t n = g->n;
    if (n > 0 && (!gg->xyz || !gg->scaling || !gg->rotation || !gg->opacity || !gg->features_dc))
        return fail(G4D_ERR_ARG, "NULL gradient pointer");
    if (g->features_rest && n > 0 && !gg->features_rest && sh_coeffs(&cams[0]) > 1)     // (M = 1: features_rest holds nothing)
        return fail(G4D_ERR_ARG, "features_rest gradient sink is NULL");
    return G4D_OK;
}

std::atomic<uint64_t> g_group_serial{0};

// The fused forward of cams[0, k) on ctx[0, k) (arguments checked by the caller).  group: the call is
// g4d_render_forward_cameras, whose records name the call, each camera's position in it and whether it kept what the group
// backward reads; g4d_render_forward's record (k = 1) has group 0.
int fused_forward_cameras(G4DContext* const* ctx, int k, const G4DCamera* cams, const G4DDeformParams* prm, const G4DGaussians* g,
                          float* const* out_color, float* const* out_depth, int32_t* const* out_radii, bool group,
                          cudaStream_t st) {
    G4DContext* c0 = ctx[0];
    CallFrame call(CallFrame::kForward, c0->ws, st, ctx, k, cams);
    if (call.rc != G4D_OK) return call.rc;
    int rc;
    // camera 0: the fused forward of one camera; it keeps the deformed tensors when other cameras read them
    ForwardRecord r0;
    if ((rc = fused_forward(c0, &cams[0], prm, g, out_color[0], out_depth[0], out_radii[0], k > 1, st, &r0)) != G4D_OK) return rc;
    const int64_t n = g->n;
    if (k > 1) {
        ExtraCameras ec{};
        ec.count = k - 1;
        for (int i = 1; i < k; ++i) {
            G4DContext* c = ctx[i];
            if ((rc = setup_view(c, &cams[i], c->time_src, n, st, [] { return G4D_OK; })) != G4D_OK) return rc;
            ec.cam[i - 1] = c->cam.as<CameraDev>(); ec.g[i - 1] = c->g; ec.out_radii[i - 1] = out_radii[i];
        }
        {
            StageTimer tm(ctx[1], G4D_STAGE_GEOM, st);
            G4D_CUDA(launch_project_cameras(ec, n, deformed_inputs(c0, r0, g), st));
        }
        if ((rc = debug_sync(&cams[1], st, "project_cameras")) != G4D_OK) return rc;
        for (int i = 1; i < k; ++i)
            if ((rc = bin_and_blend(ctx[i], &cams[i], n, out_color[i], out_depth[i], st)) != G4D_OK) return rc;
    }
    // cameras 1..k-1 keep nothing of their own for a backward: the group backward reads camera 0's tensors
    const uint64_t serial = group ? ++g_group_serial : 0;
    for (int i = 0; i < k; ++i) {
        ForwardRecord r = i == 0 ? r0 : ForwardRecord{ForwardRecord::kFused, n, cams[i].image_height, cams[i].image_width,
                                                      r0.deformed, r0.sh, false, r0.sh_coeffs};
        if (group) { r.group = serial; r.group_pos = i; r.group_size = k; r.group_grad = !(cams[0].debug & G4D_CAM_NO_GRAD); }
        ctx[i]->fwd = r;
    }
    return G4D_OK;
}

}  // namespace

extern "C" {

int g4d_render_forward(G4DContext* c, const G4DCamera* cam, const G4DDeformParams* prm, const G4DGaussians* g,
                       float* out_color, float* out_depth, int32_t* out_radii, void* stream) {
    if (!c) return fail(G4D_ERR_ARG, "context is NULL");
    const int rc = check_render_args(cam, prm, g, out_color, out_depth, out_radii);
    if (rc != G4D_OK) return rc;
    return fused_forward_cameras(&c, 1, cam, prm, g, &out_color, &out_depth, &out_radii, false, (cudaStream_t)stream);
}

int g4d_render_backward(G4DContext* c, const G4DCamera* cam, const G4DDeformParams* prm, G4DDeformGrads* pgrads,
                        const G4DGaussians* g, const float* dL_dcolor, G4DGaussianGrads* gg, void* stream) {
    if (!c) return fail(G4D_ERR_ARG, "context is NULL");
    if (c->fwd.kind != ForwardRecord::kFused || !g || c->fwd.n != g->n) return fail(G4D_ERR_STATE, "g4d_render_backward needs the matching g4d_render_forward on this context");
    if (c->fwd.group) return fail(G4D_ERR_STATE, "the last forward on this context was g4d_render_forward_cameras: use g4d_render_backward_cameras");
    int rc = check_camera(cam);
    if (rc != G4D_OK) return rc;
    if (!dL_dcolor || !gg || (g->n > 0 && !gg->means2D)) return fail(G4D_ERR_ARG, "NULL gradient pointer");
    if ((rc = check_fused_backward("g4d_render_backward", c->fwd.kept, &c, 1, cam, prm, pgrads, g, gg)) != G4D_OK) return rc;
    const cudaStream_t st = (cudaStream_t)stream;
    CallFrame call(CallFrame::kBackward, c->ws, st, &c, 1, cam);
    if (call.rc != G4D_OK) return call.rc;
    return fused_backward(c, cam, prm, pgrads, g, dL_dcolor, gg, st);
}

// ------------------------------------------------------------------------------------------------------
int g4d_render_forward_cameras(G4DContext* const* ctx, int32_t k, const G4DCamera* cams, const G4DDeformParams* prm,
                               const G4DGaussians* g, float* const* out_color, float* const* out_depth,
                               int32_t* const* out_radii, void* stream) {
    int rc = check_camera_group(ctx, k, cams);
    if (rc != G4D_OK) return rc;
    if (!out_color || !out_depth || !out_radii) return fail(G4D_ERR_ARG, "output arrays are NULL");
    for (int i = 0; i < k; ++i)
        if ((rc = check_render_args(&cams[i], prm, g, out_color[i], out_depth[i], out_radii[i])) != G4D_OK) return rc;
    return fused_forward_cameras(ctx, k, cams, prm, g, out_color, out_depth, out_radii, true, (cudaStream_t)stream);
}

int g4d_render_backward_cameras(G4DContext* const* ctx, int32_t k, const G4DCamera* cams, const G4DDeformParams* prm,
                                G4DDeformGrads* pgrads, const G4DGaussians* g, const float* const* dL_dcolor,
                                G4DGaussianGrads* gg, float* const* g_means2D, void* stream) {
    int rc = check_camera_group(ctx, k, cams);
    if (rc != G4D_OK) return rc;
    if (!g || !dL_dcolor || !gg) return fail(G4D_ERR_ARG, "NULL argument");
    if (gg->means2D) return fail(G4D_ERR_ARG, "gg->means2D must be NULL: the screen-space gradients go to g_means2D[i]");
    G4DContext* c0 = ctx[0];
    for (int i = 0; i < k; ++i) {
        const ForwardRecord& f = ctx[i]->fwd;
        if (f.kind == ForwardRecord::kNone || !f.group || f.group != c0->fwd.group || f.group_pos != i || f.group_size != k || f.n != g->n)
            return fail(G4D_ERR_STATE, "g4d_render_backward_cameras needs the matching g4d_render_forward_cameras on these contexts, "
                                       "with no other forward on any of them since");
    }
    if ((rc = check_fused_backward("g4d_render_backward_cameras", c0->fwd.group_grad && c0->fwd.kept, ctx, k, cams, prm, pgrads,
                                   g, gg)) != G4D_OK) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    CallFrame call(CallFrame::kBackward, c0->ws, st, ctx, k, cams);
    if (call.rc != G4D_OK) return call.rc;
    if (k == 1 && dL_dcolor[0]) {     // one camera: the single-camera backward
        G4DGaussianGrads g1 = *gg;
        g1.means2D = g_means2D ? g_means2D[0] : nullptr;
        return fused_backward(c0, &cams[0], prm, pgrads, g, dL_dcolor[0], &g1, st);
    }
    const int64_t n = g->n;
    if (n == 0) return G4D_OK;
    DeformedGrads d;
    if ((rc = deformed_grads(c0, n, gg, &d)) != G4D_OK) return rc;
    // blend backward of every camera in the loss, each into its own scratch; when any camera has a depth gradient, every
    // scratch has the depth block
    BackwardCameras bc{};
    CamGradSinks cs{};
    bool cam_grads = false, depth = false;
    for (int i = 0; i < k; ++i) depth |= ctx[i]->terms.depth_grad != nullptr;
    for (int i = 0; i < k; ++i) {
        G4DContext* c = ctx[i];
        if (!c->terms.in_loss(dL_dcolor[i])) {
            reset_stage_flags(c, G4D_STAGE_BLEND_BWD, G4D_STAGE_DEFORM_BWD);
            if (g_means2D && g_means2D[i]) G4D_CUDA(cudaMemsetAsync(g_means2D[i], 0, (size_t)n * 12, st));
            continue;
        }
        float* gb;
        if ((rc = blend_backward(c, &cams[i], n, dL_dcolor[i], nullptr, depth, &gb, st)) != G4D_OK) return rc;
        const int j = bc.count++;
        bc.cam[j] = c->cam.as<CameraDev>(); bc.radii[j] = c->g.radii; bc.clamped[j] = c->g.clamped; bc.grad[j] = gb;
        bc.g_means2D[j] = g_means2D ? g_means2D[i] : nullptr;
        cs.out[j] = c->terms.cam_grad;
        cam_grads |= c->terms.cam_grad != nullptr;
    }
    {
        StageTimer tm(c0, G4D_STAGE_GEOM_BWD, st);
        G4D_CUDA(launch_preprocess_backward_cameras(bc, n, deformed_inputs(c0, c0->fwd, g), d.xyz, d.sc, d.rot, d.op,
                                                    fused_sh_sinks(c0, g, gg, d.sh), cam_grads ? &cs : nullptr, depth, st));
    }
    if ((rc = debug_sync(&cams[0], st, "preprocess_backward_cameras")) != G4D_OK) return rc;
    // the network's backward, once, on the gradients summed over the cameras; the one dL/d(time) of the group goes to the
    // first context with a time sink and is copied into the others'
    float* g_time = nullptr;
    for (int i = 0; i < k && !g_time; ++i) g_time = ctx[i]->terms.time_grad;
    if ((rc = fused_backward_tail(c0, &cams[0], prm, pgrads, g, gg, d, g_time, st)) != G4D_OK) return rc;
    for (int i = 0; i < k; ++i)
        if (float* t = ctx[i]->terms.time_grad; t && t != g_time)
            G4D_CUDA(cudaMemcpyAsync(t, g_time, sizeof(float), cudaMemcpyDeviceToDevice, st));
    return G4D_OK;
}

// ------------------------------------------------------------------------------------------------------
int g4d_l1_loss(G4DWorkspace* ws, const float* out, const float* gt, int64_t numel, float scale, float* loss_accum, void* stream) {
    if (!ws || numel < 0 || (numel > 0 && (!out || !gt)) || !loss_accum) return fail(G4D_ERR_ARG, "g4d_l1_loss: bad argument");
    G4D_CUDA(cudaSetDevice(ws->device));
    G4D_CUDA(launch_l1_loss(out, gt, numel, scale, loss_accum, ws->sm_count, (cudaStream_t)stream));
    return G4D_OK;
}

int g4d_l1_loss_backward(G4DWorkspace* ws, const float* out, const float* gt, int64_t numel, float scale, const float* upstream,
                         float* grad_out, void* stream) {
    if (!ws || numel < 0 || (numel > 0 && (!out || !gt || !grad_out))) return fail(G4D_ERR_ARG, "g4d_l1_loss_backward: bad argument");
    G4D_CUDA(cudaSetDevice(ws->device));
    G4D_CUDA(launch_l1_grad(out, gt, numel, scale, upstream, grad_out, ws->sm_count, (cudaStream_t)stream));
    return G4D_OK;
}

int g4d_ssim(G4DWorkspace* ws, const float* img1, const float* img2, int32_t channels, int32_t height, int32_t width, float scale,
             float* ssim_accum, float* saved, void* stream) {
    if (!ws || channels < 0 || height < 0 || width < 0 || !img1 || !img2) return fail(G4D_ERR_ARG, "g4d_ssim: bad argument");
    if (channels > 65535) return fail(G4D_ERR_ARG, "g4d_ssim: more than 65535 channels");
    G4D_CUDA(cudaSetDevice(ws->device));
    const size_t P = (size_t)channels * height * width;
    G4D_CUDA(launch_ssim_forward(img1, img2, channels, height, width, scale, ssim_accum, saved, saved ? saved + P : nullptr,
                                 saved ? saved + 2 * P : nullptr, (cudaStream_t)stream));
    return G4D_OK;
}

int g4d_ssim_backward(G4DWorkspace* ws, const float* img1, const float* img2, int32_t channels, int32_t height, int32_t width,
                      float scale, const float* upstream, const float* saved, float* grad_img1, void* stream) {
    if (!ws || channels < 0 || height < 0 || width < 0 || !img1 || !img2 || !saved || !grad_img1)
        return fail(G4D_ERR_ARG, "g4d_ssim_backward: bad argument");
    if (channels > 65535) return fail(G4D_ERR_ARG, "g4d_ssim: more than 65535 channels");
    G4D_CUDA(cudaSetDevice(ws->device));
    const size_t P = (size_t)channels * height * width;
    G4D_CUDA(launch_ssim_backward(img1, img2, channels, height, width, scale, upstream, saved, saved + P, saved + 2 * P, grad_img1,
                                  (cudaStream_t)stream));
    return G4D_OK;
}

int g4d_plane_regulation(G4DWorkspace* ws, const G4DDeformParams* prm, G4DDeformGrads* grads, float plane_tv_weight,
                         float time_smoothness_weight, float l1_time_planes_weight, const float* upstream, float* loss_accum,
                         void* stream) {
    if (!ws) return fail(G4D_ERR_ARG, "workspace is NULL");
    int rc = check_params(prm);
    if (rc != G4D_OK) return rc;
    G4D_CUDA(cudaSetDevice(ws->device));
    G4D_CUDA(launch_plane_regulation(*prm, grads, plane_tv_weight, time_smoothness_weight, l1_time_planes_weight, upstream, loss_accum,
                                     ws->sm_count, (cudaStream_t)stream));
    return G4D_OK;
}

}  // extern "C"

namespace {
// the arguments g4d_adam_step and g4d_adam_step_device share (`who`: the entry point the message names)
int check_adam_args(const char* who, G4DWorkspace* ws, float* param, const float* grad, float* exp_avg, float* exp_avg_sq,
                    int64_t numel, const G4DAdamSegment* segments, int32_t num_segments) {
    if (!ws || numel < 0 || (numel > 0 && (!param || !grad || !exp_avg || !exp_avg_sq || !segments)))
        return fail(G4D_ERR_ARG, who, "bad argument");
    if ((numel & 3) || num_segments < 0 || num_segments > G4D_ADAM_MAX_SEGMENTS)
        return fail(G4D_ERR_ARG, who, "numel must be a multiple of 4 and at most 16 segments");
    if (((uintptr_t)param | (uintptr_t)grad | (uintptr_t)exp_avg | (uintptr_t)exp_avg_sq) & 15u)   // the kernel moves float4s
        return fail(G4D_ERR_ARG, who, "param, grad, exp_avg and exp_avg_sq must be 16-byte aligned");
    for (int i = 0; i < num_segments; ++i)
        if (segments[i].begin < 0 || segments[i].end < segments[i].begin || segments[i].end > numel || (i && segments[i].begin < segments[i - 1].end))
            return fail(G4D_ERR_ARG, who, "segments must be sorted, disjoint and inside [0, numel)");
    return G4D_OK;
}
}  // namespace

extern "C" {

int g4d_adam_step(G4DWorkspace* ws, float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t numel,
                  const G4DAdamSegment* segments, int32_t num_segments, float beta1, float beta2, float eps, int64_t step,
                  float grad_scale, void* stream) {
    if (step < 1) return fail(G4D_ERR_ARG, "g4d_adam_step: bad argument");
    const int rc = check_adam_args("g4d_adam_step", ws, param, grad, exp_avg, exp_avg_sq, numel, segments, num_segments);
    if (rc != G4D_OK) return rc;
    G4D_CUDA(cudaSetDevice(ws->device));
    G4D_CUDA(launch_adam_flat(param, grad, exp_avg, exp_avg_sq, numel, segments, num_segments, beta1, beta2, eps, step, grad_scale,
                              ws->sm_count, (cudaStream_t)stream));
    return G4D_OK;
}

int g4d_adam_scalars(const G4DAdamSegment* segments, int32_t num_segments, float beta1, float beta2, int64_t step, float grad_scale,
                     G4DAdamScalars* out) {
    if (!out || num_segments < 0 || num_segments > G4D_ADAM_MAX_SEGMENTS || (num_segments > 0 && !segments) || step < 1)
        return fail(G4D_ERR_ARG, "g4d_adam_scalars: bad argument");
    adam_scalars(segments, num_segments, beta1, beta2, step, grad_scale, out);
    return G4D_OK;
}

int g4d_adam_step_device(G4DWorkspace* ws, float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t numel,
                         const G4DAdamSegment* segments, int32_t num_segments, float beta1, float beta2, float eps,
                         const G4DAdamScalars* d_scalars, void* stream) {
    int rc = check_adam_args("g4d_adam_step_device", ws, param, grad, exp_avg, exp_avg_sq, numel, segments, num_segments);
    if (rc != G4D_OK) return rc;
    if (!d_scalars) return fail(G4D_ERR_ARG, "g4d_adam_step_device", "d_scalars is NULL");
    G4D_CUDA(cudaSetDevice(ws->device));
    G4D_CUDA(launch_adam_flat_device(param, grad, exp_avg, exp_avg_sq, numel, segments, num_segments, beta1, beta2, eps, d_scalars,
                                     ws->sm_count, (cudaStream_t)stream));
    return G4D_OK;
}

int g4d_dist2_knn3(G4DWorkspace* ws, int64_t n, const float* xyz, float* out_mean_dist2, void* stream) {
    if (!ws || n < 0 || (n > 0 && (!xyz || !out_mean_dist2))) return fail(G4D_ERR_ARG, "g4d_dist2_knn3: bad argument");
    if (n >= (1ll << 31)) return fail(G4D_ERR_ARG, "n too large");
    CallFrame call(CallFrame::kContextFree, ws, (cudaStream_t)stream);
    if (call.rc != G4D_OK) return call.rc;
    G4D_CUDA(ws->scratch.ensure(knn_scratch_bytes(n)));
    G4D_CUDA(launch_knn_dist2(n, xyz, out_mean_dist2, ws->scratch.p, ws->sm_count, (cudaStream_t)stream));
    return G4D_OK;
}

int g4d_context_set_time_source(G4DContext* c, const float* d_time) {
    if (!c) return fail(G4D_ERR_ARG, "context is NULL");
    c->time_src = d_time;
    return G4D_OK;
}

int g4d_context_set_camera_grad(G4DContext* c, float* d_out) {
    if (!c) return fail(G4D_ERR_ARG, "context is NULL");
    c->terms.cam_grad = d_out;
    return G4D_OK;
}

int g4d_context_set_time_grad(G4DContext* c, float* d_out) {
    if (!c) return fail(G4D_ERR_ARG, "context is NULL");
    c->terms.time_grad = d_out;
    return G4D_OK;
}

int g4d_context_set_depth_grad(G4DContext* c, const float* d_dL_ddepth) {
    if (!c) return fail(G4D_ERR_ARG, "context is NULL");
    c->terms.depth_grad = d_dL_ddepth;
    return G4D_OK;
}

int g4d_context_set_alpha_out(G4DContext* c, float* d_out) {
    if (!c) return fail(G4D_ERR_ARG, "context is NULL");
    c->terms.alpha_out = d_out;
    return G4D_OK;
}

int g4d_context_set_alpha_grad(G4DContext* c, const float* d_dL_dalpha) {
    if (!c) return fail(G4D_ERR_ARG, "context is NULL");
    c->terms.alpha_grad = d_dL_dalpha;
    return G4D_OK;
}

int g4d_workspace_freeze(G4DWorkspace* ws, int on) {
    if (!ws) return fail(G4D_ERR_ARG, "workspace is NULL");
    ws->frozen = on ? 1 : 0;
    return G4D_OK;
}

int g4d_workspace_graph_status(G4DWorkspace* ws, int sync, G4DGraphStatus* out) {
    if (!ws || !out) return fail(G4D_ERR_ARG, "NULL argument");
    if (sync) {
        G4D_CUDA(cudaSetDevice(ws->device));
        G4D_CUDA(cudaDeviceSynchronize());
    }
    volatile PinnedWords* w = ws->pinned;
    *out = G4DGraphStatus{};
    out->overflows = w->overflow[0];
    out->max_instances = w->overflow[1];
    out->f16_range = w->f16_range ? 1 : 0;
    w->overflow[0] = 0; w->overflow[1] = 0; w->f16_range = 0;
    return G4D_OK;
}

int g4d_debug_tc_cycles(G4DWorkspace* ws, double* out12) {
    if (!ws || !out12) return fail(G4D_ERR_ARG, "NULL argument");
    G4D_CUDA(cudaSetDevice(ws->device));
    G4D_CUDA(cudaDeviceSynchronize());
    for (int i = 0; i < 12; ++i) out12[i] = 0.0;
    if (!ws->tc_dbg.p) return G4D_OK;
    std::vector<long long> h((size_t)ws->sm_count * 12);
    G4D_CUDA(cudaMemcpy(h.data(), ws->tc_dbg.p, h.size() * 8, cudaMemcpyDeviceToHost));
    for (int c = 0; c < ws->sm_count; ++c)
        for (int i = 0; i < 12; ++i) out12[i] += (double)h[(size_t)c * 12 + i] / ws->sm_count;
    return G4D_OK;
}

}  // extern "C"
