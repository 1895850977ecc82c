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

int fail(int code, const char* what, const char* detail = nullptr) {
    t_last_error = what;
    if (detail) { t_last_error += ": "; t_last_error += detail; }
    return code;
}

#define G4D_CUDA(expr)                                                                      \
    do {                                                                                    \
        cudaError_t e__ = (expr);                                                           \
        if (e__ != cudaSuccess) {                                                           \
            char buf__[64];                                                                 \
            snprintf(buf__, sizeof(buf__), " (%s:%d)", __FILE__, __LINE__);                 \
            std::string m__ = std::string(cudaGetErrorString(e__)) + buf__;                 \
            return fail(e__ == cudaErrorMemoryAllocation ? G4D_ERR_NOMEM : G4D_ERR_CUDA, #expr, m__.c_str()); \
        }                                                                                   \
    } while (0)

// device memory that grows by 1.5x on demand and is freed with its owner (on the owner's device)
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

// FP32 transposes of W0 and of the active heads' W1 (the FFMA kernels' operands)
struct FfmaWeights {
    float* w0t;
    float* w1t[G4D_NUM_HEADS];
};

// weight images derived from the caller's parameters, rebuilt when G4DDeformParams.version or the w0 pointer changes (or,
// for the tensor-core forward, the arithmetic)
template <class Images>
struct WeightCache {
    DevBuf buf;
    Images img{};   // where the images sit in buf
    uint64_t version = 0;
    const void* key = nullptr;
    int arith = 0;
    bool valid = false;
    // pack(buf.p, &img) (re)builds the images unless they were built from these parameters
    template <class Pack> cudaError_t refresh(const G4DDeformParams* p, int arith_, size_t bytes, Pack pack) {
        if (valid && version == p->version && key == (const void*)p->w0 && arith == arith_) return cudaSuccess;
        valid = false;
        cudaError_t e = buf.ensure(bytes);
        if (e == cudaSuccess) e = pack(buf.p, &img);
        if (e != cudaSuccess) return e;
        version = p->version; key = (const void*)p->w0; arith = arith_; valid = true;
        return cudaSuccess;
    }
};

// pinned host words of a workspace: the exact-mode read-back of R, and the flag an FP16x2 tensor-core kernel sets (through
// the host mapping) when a value left the f16 operand range
struct PinnedWords { uint32_t num_rendered, pad0[7], f16_range, pad1[7]; };

}  // namespace

struct G4DWorkspace {
    int device = 0;
    int sm_count = 132;
    int sync_mode = 1;
    int64_t min_capacity = 0;
    int tight_cull = 0;
    int stage_timing = 0;
    int tensor_cores = 2;      // 0: FP32 FFMA kernels, 1: wgmma 3xTF32, 2 (default): wgmma FP16x2
    int warp_cull = 1;
    int keep_deformed = 0;
    int tc_debug = 0;
    WeightCache<FfmaWeights> packed;     // FFMA forward and backward
    WeightCache<TcWeights> tc;           // tensor-core forward (the weight fields and status of TcWeights)
    WeightCache<TcBwdWeights> tc_bwd;    // tensor-core backward
    DevBuf tc_feat;     // HexPlane feature staging of a tensor-core forward that keeps no features
    DevBuf tc_dbg;      // G4D_OPT_TC_DEBUG cycle counters
    DevBuf trow;        // time rows for the context-free deform entry points
    DevBuf scratch;     // misc per-call scratch (deform backward, kNN)
    PinnedWords* pinned = nullptr;
};

struct G4DContext {
    G4DWorkspace* ws = nullptr;
    DevBuf cam, geom, bin, binaux, img, fused, gscratch, gdeform, trow, relu, feat;
    bool relu_saved = false;
    int64_t n = 0;
    int H = 0, W = 0, grid_x = 0, grid_y = 0;
    int64_t R = 0, capacity = 0;
    const void* bin_ctl = nullptr;    // device BinCtl of the last forward
    bool learned = false;             // R of an earlier exact forward is known (no-sync mode needs a learnt capacity)
    bool has_forward = false, is_fused = false, fused_sh = false, deformed = false, fo_valid = false;
    // multi-camera forward (g4d_render_forward_cameras) whose state this context holds: serial number of that call (0: the
    // last forward was a single-camera one), this camera's position and the number of cameras; on camera 0, whether the
    // forward kept what the group backward reads
    uint64_t group = 0;
    int group_pos = 0, group_size = 0;
    bool group_grad = false;
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
    c->H = H; c->W = W; c->grid_x = gx; c->grid_y = gy;
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

int check_params(const G4DDeformParams* p) {
    if (!p) return fail(G4D_ERR_ARG, "deform params are NULL");
    if (p->levels < 1 || p->levels > G4D_MAX_LEVELS) return fail(G4D_ERR_ARG, "levels must be in 1..4");
    if (p->channels < 4 || p->channels > 32 || (p->channels & 3)) return fail(G4D_ERR_ARG, "channels must be a multiple of 4, <= 32");
    if (p->net_width != 64 && p->net_width != 128) return fail(G4D_ERR_ARG, "net_width must be 64 or 128");
    if (p->levels * p->channels > 128) return fail(G4D_ERR_ARG, "levels*channels must be <= 128");
    for (int l = 0; l < p->levels; ++l)
        for (int a = 0; a < 4; ++a)
            if (p->res[l][a] < 2 || p->res[l][a] > 65535) return fail(G4D_ERR_ARG, "plane resolution out of range");
    return G4D_OK;
}

int refresh_packed(G4DWorkspace* ws, const G4DDeformParams* p, cudaStream_t st) {
    const size_t F = (size_t)p->levels * p->channels, WD = (size_t)p->net_width;
    auto pack = [&](void* blob, FfmaWeights* w) {
        w->w0t = static_cast<float*>(blob);
        for (int h = 0; h < G4D_NUM_HEADS; ++h) w->w1t[h] = w->w0t + F * WD + h * WD * WD;
        return launch_pack_weights(*p, w->w0t, w->w1t, st);
    };
    G4D_CUDA(ws->packed.refresh(p, 0, (F * WD + G4D_NUM_HEADS * WD * WD) * 4, pack));
    return G4D_OK;
}

int refresh_tc(G4DWorkspace* ws, const G4DDeformParams* p, cudaStream_t st) {
    const int arith = ws->tensor_cores == 2 ? 2 : 1;
    if (arith == 2 && ws->pinned->f16_range) {
        ws->pinned->f16_range = 0;
        ws->tc.valid = false;      // re-pack (and re-check) the weights on the next call: they may be the out-of-range values
        return fail(G4D_ERR_OVERFLOW, "an earlier FP16x2 tensor-core launch met a value outside the f16 operand range (activation >= 8188, "
                                      "feature >= 1023 or weight >= 255): its results were saturated; set G4D_OPT_TENSOR_CORES = 1 (3xTF32)");
    }
    auto pack = [&](void* blob, TcWeights* w) {
        w->arith = arith;
        w->status = &ws->pinned->f16_range;
        return launch_tc_pack_weights(*p, arith, static_cast<float*>(blob), w, st);
    };
    G4D_CUDA(ws->tc.refresh(p, arith, tc_packed_floats(*p) * 4, pack));
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
    return d;
}

// the deformation network of one forward call
struct DeformSetup {
    DeformDesc d;
    bool tc;         // the forward runs on the tensor cores
    TcWeights tw;    // tc: weight images, range flag and debug counters; the caller adds its feat / relu_bits buffers
};

// the time planes interpolated at `time`, into `rows` (pointers in trow)
int collapse_time_rows(DevBuf& rows, float* (*trow)[3], const G4DDeformParams* p, float time, cudaStream_t st) {
    const TimeRows tr(p->levels, p->res, p->channels);
    if (rows.ensure(tr.total() * 4) != cudaSuccess) return fail(G4D_ERR_NOMEM, "time-row buffer");
    tr.place(rows.as<float>(), trow);
    G4D_CUDA(launch_collapse_time_rows(*p, time, trow, st));
    return G4D_OK;
}

// Collapse the time rows, pick the forward's path from the params and bring the weight images that path reads up to date.
// The desc is built after that refresh, which may move the transposes it embeds.
int setup_deform(G4DWorkspace* ws, const G4DDeformParams* p, DevBuf& rows, float* (*trow)[3], float time, cudaStream_t st,
                 DeformSetup* out) {
    int rc;
    if ((rc = collapse_time_rows(rows, trow, p, time, st)) != G4D_OK) return rc;
    out->tc = ws->tensor_cores != 0 && tc_deform_supported(*p, ws->tensor_cores);
    if (!out->tc) {
        if ((rc = refresh_packed(ws, p, st)) != G4D_OK) return rc;
        out->d = make_desc(p, trow, &ws->packed.img);
        return G4D_OK;
    }
    if ((rc = refresh_tc(ws, p, st)) != G4D_OK) return rc;
    out->d = make_desc(p, trow, nullptr);
    out->tw = ws->tc.img;
    if (ws->tc_debug) {   // per-CTA phase cycle counters (g4d_debug_tc_cycles)
        G4D_CUDA(ws->tc_dbg.ensure((size_t)ws->sm_count * 12 * 8));
        G4D_CUDA(cudaMemsetAsync(ws->tc_dbg.p, 0, (size_t)ws->sm_count * 12 * 8, st));
        out->tw.dbg = ws->tc_dbg.as<long long>();
    }
    return G4D_OK;
}

// Buffers of this forward call.  feat: where a tensor-core forward stages the HexPlane features [N][F] (NULL: the
// workspace's); relu_bits: where it saves the ReLU signs for a backward, or NULL.  The tag word behind the bits tells the
// backward whether this forward wrote them.
int attach_forward_buffers(G4DWorkspace* ws, DeformSetup& s, float* feat, uint32_t* relu_bits, int64_t n, cudaStream_t st) {
    if (s.tc && !feat) {
        G4D_CUDA(ws->tc_feat.ensure((size_t)(n > 0 ? n : 1) * 64 * 4 + 256));
        feat = ws->tc_feat.as<float>();
    }
    s.tw.feat = feat;
    s.tw.relu_bits = relu_bits;
    if (relu_bits) G4D_CUDA(cudaMemsetAsync(relu_bits + (size_t)24 * (size_t)n, s.tc ? kReluBitsTagByte : 0, 16, st));
    return G4D_OK;
}

// backward of the deformation network with the time rows trow: tensor-core path when the configuration allows, FFMA path
// otherwise; the desc is built after the weight images of that path are current
int deform_backward_dispatch(G4DWorkspace* ws, const G4DDeformParams* prm, float* const (*trow)[3], const G4DDeformGrads* grads,
                             float time, int64_t n, const float* xyz, const float* const go[G4D_NUM_HEADS],
                             float* const gi[G4D_NUM_HEADS], const uint32_t* relu_bits, const float* saved_feat, cudaStream_t st) {
    int rc;
    if (ws->tensor_cores && tc_backward_supported(*prm)) {
        auto pack = [&](void* blob, TcBwdWeights* w) { return launch_tc_bwd_pack_weights(*prm, static_cast<uint8_t*>(blob), w, st); };
        G4D_CUDA(ws->tc_bwd.refresh(prm, 0, tc_bwd_weight_bytes(*prm), pack));
        const DeformDesc d = make_desc(prm, trow, nullptr);
        G4D_CUDA(ws->scratch.ensure(tc_deform_backward_scratch_bytes(d, n)));
        G4D_CUDA(launch_deform_backward_tc(d, *prm, *grads, ws->tc_bwd.img, time, n, xyz, go, gi, relu_bits, saved_feat,
                                           ws->scratch.as<uint8_t>(), ws->sm_count, st));
        return G4D_OK;
    }
    if ((rc = refresh_packed(ws, prm, st)) != G4D_OK) return rc;
    const DeformDesc d = make_desc(prm, trow, &ws->packed.img);
    G4D_CUDA(ws->scratch.ensure(deform_backward_scratch_bytes(d, n)));
    G4D_CUDA(launch_deform_backward(d, *prm, *grads, time, n, xyz, go, gi, ws->scratch.as<float>(), ws->sm_count, st));
    return G4D_OK;
}

int check_camera(const G4DCamera* cam) {
    if (!cam) return fail(G4D_ERR_ARG, "camera is NULL");
    if (cam->image_height <= 0 || cam->image_width <= 0 || cam->image_height > 16384 || cam->image_width > 16384)
        return fail(G4D_ERR_ARG, "image size out of range");
    if (cam->sh_degree < 0 || cam->sh_degree > 3) return fail(G4D_ERR_ARG, "sh_degree must be 0..3");
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
            c->has_forward = false;
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
            const uint32_t cap_place = (uint32_t)(c->capacity < (int64_t)kNoCap ? c->capacity : (int64_t)kNoCap);
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
        G4D_CUDA(launch_blend_forward(dcam, c->grid_x, c->grid_y, c->g, c->b, c->im, out_color, out_depth, ws->warp_cull, st));
    }
    if (readback) {
        const int sl = c->slot;
        c->slot = (c->slot + 1) % G4DContext::kSlots;
        G4D_CUDA(cudaMemcpyAsync(c->h_r + sl, readback, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
        G4D_CUDA(cudaEventRecord(c->ev_r[sl], st));
        c->pending[sl] = true; c->used_capacity[sl] = c->capacity;
    }
    if ((rc = debug_sync(cam, st, "blend_forward")) != G4D_OK) return rc;
    c->n = n;
    c->has_forward = true;
    return G4D_OK;
}

// A caller's SH tensors: fused [N,16,3] in dc, or (split) dc [N,1,3] + rest [N,15,3].  Sh = ShIn for the coefficients,
// ShOut for their gradient sinks.
template <class Sh, class T> Sh caller_sh(bool split, T* dc, T* rest = nullptr) {
    return split ? Sh{nullptr, dc, rest} : Sh{dc, nullptr, nullptr};
}

// blend backward + per-Gaussian backward on `in`; opacity gradient lands in g_opacities (zeroed here)
int raster_backward_stages(G4DContext* c, const G4DCamera* cam, int64_t n, const RasterInputs& in, const float* dL_dcolor,
                           float* g_means3D, float* g_means2D, const ShOut& g_sh, float* g_opacities, float* g_scales,
                           float* g_rotations, cudaStream_t st) {
    const CameraDev* dcam = c->cam.as<CameraDev>();
    const size_t N = (size_t)(n > 0 ? n : 1);
    G4D_CUDA(c->gscratch.ensure(N * 8 * 4 + 256));
    float* g_mean2D = c->gscratch.as<float>();
    float* g_conic = g_mean2D + 2 * N;
    float* g_rgb = g_conic + 3 * N;
    if (n == 0) return G4D_OK;
    G4D_CUDA(cudaMemsetAsync(g_mean2D, 0, N * 8 * 4, st));
    G4D_CUDA(cudaMemsetAsync(g_opacities, 0, N * 4, st));
    reset_stage_flags(c, G4D_STAGE_BLEND_BWD, G4D_STAGE_DEFORM_BWD);
    {
        StageTimer tm(c, G4D_STAGE_BLEND_BWD, st);
        G4D_CUDA(launch_blend_backward(dcam, c->grid_x, c->grid_y, c->g, c->b, c->im, dL_dcolor, g_mean2D, g_conic, g_opacities,
                                       g_rgb, c->ws->warp_cull, st));
    }
    int rc;
    if ((rc = debug_sync(cam, st, "blend_backward")) != G4D_OK) return rc;
    StageTimer tm(c, G4D_STAGE_GEOM_BWD, st);
    G4D_CUDA(launch_preprocess_backward(dcam, n, in, c->g, g_mean2D, g_conic, g_rgb, g_means3D, g_means2D, g_scales,
                                        g_rotations, g_sh, st));
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
        case G4D_OPT_TENSOR_CORES: ws->tensor_cores = value < 0 || value > 2 ? 2 : (int)value; return G4D_OK;
        case G4D_OPT_WARP_CULL: ws->warp_cull = value ? 1 : 0; return G4D_OK;
        case G4D_OPT_TC_DEBUG: ws->tc_debug = value ? 1 : 0; return G4D_OK;
        case G4D_OPT_KEEP_DEFORMED: ws->keep_deformed = value ? 1 : 0; return G4D_OK;
        case G4D_OPT_PDL: g4d::g_pdl = value ? 1 : 0; return G4D_OK;
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
    if (!c->has_forward) return fail(G4D_ERR_STATE, "no forward has run on this context");
    cudaSetDevice(c->ws->device);
    G4D_CUDA(cudaDeviceSynchronize());
    { int rc_ = check_pending(c); if (rc_ != G4D_OK) return rc_; }
    out->num_rendered = c->R; out->instance_capacity = c->capacity; out->tiles_x = c->grid_x; out->tiles_y = c->grid_y;
    std::vector<int32_t> radii((size_t)c->n);
    if (c->n) G4D_CUDA(cudaMemcpy(radii.data(), c->g.radii, (size_t)c->n * 4, cudaMemcpyDeviceToHost));
    int64_t vis = 0;
    for (int32_t r : radii) vis += r > 0;
    out->num_visible = vis;
    return G4D_OK;
}

// ------------------------------------------------------------------------------------------------------
int g4d_deform_forward(G4DWorkspace* ws, const G4DDeformParams* prm, int64_t n, const float* xyz, const float* scaling,
                       const float* rotation, const float* opacity, const float* shs, float time, float* out_xyz,
                       float* out_scaling, float* out_rotation, float* out_opacity, float* out_shs, uint32_t* relu_bits, void* stream) {
    if (!ws) return fail(G4D_ERR_ARG, "workspace is NULL");
    int rc = check_params(prm);
    if (rc != G4D_OK) return rc;
    if (n < 0 || (n > 0 && (!xyz || !out_xyz))) return fail(G4D_ERR_ARG, "xyz / out_xyz required");
    if ((prm->head_mask & G4D_HEAD_SHS) && n > 0 && (!shs || !out_shs)) return fail(G4D_ERR_ARG, "shs / out_shs required when the SHS head is active");
    cudaStream_t st = (cudaStream_t)stream;
    G4D_CUDA(cudaSetDevice(ws->device));
    float* trow[G4D_MAX_LEVELS][3] = {};
    DeformSetup s{};
    if ((rc = setup_deform(ws, prm, ws->trow, trow, time, st, &s)) != G4D_OK) return rc;
    if ((rc = attach_forward_buffers(ws, s, nullptr, relu_bits, n, st)) != G4D_OK) return rc;
    const DeformIO io{xyz, scaling, rotation, opacity, caller_sh<ShIn>(false, shs), out_xyz, out_scaling, out_rotation, out_opacity,
                      out_shs, GeomBuffers{}, FusedOutputs{}, nullptr};
    G4D_CUDA(launch_deform(s.d, 0, nullptr, n, io, ws->sm_count, st, s.tc ? &s.tw : nullptr));
    return G4D_OK;
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
    G4D_CUDA(cudaSetDevice(c->ws->device));
    if ((rc = check_pending(c)) != G4D_OK) return rc;
    c->has_forward = false; c->is_fused = false; c->deformed = false; c->group = 0;
    if ((rc = ensure_geom(c, n)) != G4D_OK) return rc;
    if ((rc = ensure_image(c, cam->image_height, cam->image_width)) != G4D_OK) return rc;
    reset_stage_flags(c, 0, G4D_STAGE_COUNT - 1);
    {
        StageTimer tm(c, G4D_STAGE_PREP, st);
        G4D_CUDA(launch_pack_camera(*cam, c->cam.as<CameraDev>(), st));
    }
    const RasterInputs in{means3D, scales, rotations, opacities, caller_sh<ShIn>(false, shs)};
    {
        StageTimer tm(c, G4D_STAGE_GEOM, st);
        G4D_CUDA(launch_preprocess(c->cam.as<CameraDev>(), n, in, c->g, out_radii, st));
    }
    return bin_and_blend(c, cam, n, out_color, out_depth, st);
}

int g4d_rasterize_backward(G4DContext* c, const G4DCamera* cam, int64_t n, const float* means3D, const float* shs,
                           const float* opacities, const float* scales, const float* rotations, const float* dL_dcolor,
                           float* g_means3D, float* g_means2D, float* g_shs, float* g_opacities, float* g_scales,
                           float* g_rotations, void* stream) {
    if (!c) return fail(G4D_ERR_ARG, "context is NULL");
    if (!c->has_forward || c->is_fused || c->n != n) return fail(G4D_ERR_STATE, "g4d_rasterize_backward needs the matching g4d_rasterize_forward on this context");
    int rc = check_camera(cam);
    if (rc != G4D_OK) return rc;
    if (cam->image_height != c->H || cam->image_width != c->W) return fail(G4D_ERR_STATE, "camera differs from the forward's");
    if (!dL_dcolor || (n > 0 && (!g_means3D || !g_means2D || !g_shs || !g_opacities || !g_scales || !g_rotations)))
        return fail(G4D_ERR_ARG, "NULL gradient pointer");
    cudaStream_t st = (cudaStream_t)stream;
    G4D_CUDA(cudaSetDevice(c->ws->device));
    if ((rc = check_pending(c)) != G4D_OK) return rc;
    (void)opacities;
    const RasterInputs in{means3D, scales, rotations, opacities, caller_sh<ShIn>(false, shs)};
    return raster_backward_stages(c, cam, n, in, dL_dcolor, g_means3D, g_means2D, caller_sh<ShOut>(false, g_shs),
                                  g_opacities, g_scales, g_rotations, st);
}

// ------------------------------------------------------------------------------------------------------
int64_t g4d_context_read(G4DContext* c, int which, void* host_dst, int64_t bytes) {
    if (!c || !c->has_forward) return fail(G4D_ERR_STATE, "no forward has run on this context");
    cudaSetDevice(c->ws->device);
    if (cudaDeviceSynchronize() != cudaSuccess) return fail(G4D_ERR_CUDA, "cudaDeviceSynchronize");
    { int rc_ = check_pending(c); if (rc_ != G4D_OK) return rc_; }
    const size_t N = (size_t)c->n, P = (size_t)c->H * c->W, R = (size_t)c->R, Tn = (size_t)c->grid_x * c->grid_y;
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
            if (!c->is_fused || !c->fo_valid) return fail(G4D_ERR_STATE, "G4D_BUF_DEFORMED needs a fused forward that kept its tensors (grad-enabled, or G4D_OPT_KEEP_DEFORMED)");
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
            if (!c->is_fused || !c->fused_sh || !c->fo.shs || !c->fo_valid) return fail(G4D_ERR_STATE, "G4D_BUF_DEFORMED_SHS needs a fused forward with the SHS head active");
            ok = pull(c->fo.shs, N * 192); outv = tmp; outv.resize(N * 192);
        } break;
        case G4D_BUF_BIN_PHASES: {
            if (!c->bin_ctl) return fail(G4D_ERR_STATE, "no binning has run on this context");
            ok = pull(reinterpret_cast<const char*>(c->bin_ctl) + 16, 16 * 8); outv = tmp; outv.resize(16 * 8);
        } break;
        default: return fail(G4D_ERR_ARG, "unknown buffer id");
    }
    if (!ok) return fail(G4D_ERR_CUDA, "cudaMemcpy in g4d_context_read");
    const int64_t held = (int64_t)outv.size();
    if (host_dst && bytes > 0) memcpy(host_dst, outv.data(), (size_t)(bytes < held ? bytes : held));
    return held;
}

// ------------------------------------------------------------------------------------------------------
int g4d_deform_backward(G4DWorkspace* ws, const G4DDeformParams* prm, G4DDeformGrads* grads, int64_t n, const float* xyz,
                        float time, const float* g_out_xyz, const float* g_out_scaling, const float* g_out_rotation,
                        const float* g_out_opacity, const float* g_out_shs, float* g_in_xyz, float* g_in_scaling,
                        float* g_in_rotation, float* g_in_opacity, float* g_in_shs, const uint32_t* relu_bits, void* stream) {
    if (!ws) return fail(G4D_ERR_ARG, "workspace is NULL");
    int rc = check_params(prm);
    if (rc != G4D_OK) return rc;
    if (!grads) return fail(G4D_ERR_ARG, "grads is NULL");
    if (n < 0 || (n > 0 && !xyz)) return fail(G4D_ERR_ARG, "xyz required");
    cudaStream_t st = (cudaStream_t)stream;
    G4D_CUDA(cudaSetDevice(ws->device));
    float* trow[G4D_MAX_LEVELS][3] = {};
    if ((rc = collapse_time_rows(ws->trow, trow, prm, time, st)) != G4D_OK) return rc;
    const float* go[G4D_NUM_HEADS] = {g_out_xyz, g_out_scaling, g_out_rotation, g_out_opacity, g_out_shs};
    float* gi[G4D_NUM_HEADS] = {g_in_xyz, g_in_scaling, g_in_rotation, g_in_opacity, g_in_shs};
    return deform_backward_dispatch(ws, prm, trow, grads, time, n, xyz, go, gi, relu_bits, nullptr, st);
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------------
namespace {

int check_render_args(const G4DCamera* cam, const G4DDeformParams* prm, const G4DGaussians* g, const float* out_color,
                      const float* out_depth, const int32_t* out_radii) {
    int rc = check_camera(cam);
    if (rc != G4D_OK) return rc;
    if (prm && (rc = check_params(prm)) != G4D_OK) return rc;
    if (!g || g->n < 0 || g->n >= (1ll << 31) || !out_color || !out_depth) return fail(G4D_ERR_ARG, "bad gaussians / outputs");
    if (g->n > 0 && (!g->xyz || !g->scaling || !g->rotation || !g->opacity || !g->features_dc || !out_radii))
        return fail(G4D_ERR_ARG, "NULL gaussian tensor");
    return G4D_OK;
}

// The fused forward of one camera on c.  keep_fo: store the deformed, activated tensors even under G4D_CAM_NO_GRAD (other
// cameras of the same call read them).
int fused_forward(G4DContext* c, const G4DCamera* cam, const G4DDeformParams* prm, const G4DGaussians* g, float* out_color,
                  float* out_depth, int32_t* out_radii, bool keep_fo, cudaStream_t st) {
    const int64_t n = g->n;
    G4DWorkspace* ws = c->ws;
    int rc;
    G4D_CUDA(cudaSetDevice(ws->device));
    if ((rc = check_pending(c)) != G4D_OK) return rc;
    c->has_forward = false; c->group = 0;
    const bool with_sh = prm && (prm->head_mask & G4D_HEAD_SHS);
    if ((rc = ensure_geom(c, n)) != G4D_OK) return rc;
    if ((rc = ensure_image(c, cam->image_height, cam->image_width)) != G4D_OK) return rc;
    if ((rc = ensure_fused(c, n, with_sh)) != G4D_OK) return rc;
    CameraDev* dcam = c->cam.as<CameraDev>();
    reset_stage_flags(c, 0, G4D_STAGE_COUNT - 1);
    // a no-grad render needs none of the saved tensors: skip their stores (48 B + 192 B of deformed SH per Gaussian)
    c->fo_valid = !(cam->debug & G4D_CAM_NO_GRAD) || ws->keep_deformed || keep_fo;
    const FusedOutputs fo_arg = c->fo_valid ? c->fo : FusedOutputs{};
    DeformSetup s{};
    {
        StageTimer tm(c, G4D_STAGE_PREP, st);
        G4D_CUDA(launch_pack_camera(*cam, dcam, st));
        if (prm && (rc = setup_deform(ws, prm, c->trow, c->trow_ptr, cam->time, st, &s)) != G4D_OK) return rc;
    }
    {
        StageTimer tm(c, G4D_STAGE_GEOM, st);
        const DeformIO io{g->xyz, g->scaling, g->rotation, g->opacity,
                          caller_sh<ShIn>(g->features_rest != nullptr, g->features_dc, g->features_rest),
                          nullptr, nullptr, nullptr, nullptr, nullptr, c->g, fo_arg, out_radii};
        if (prm) {
            c->relu_saved = s.tc && !(cam->debug & G4D_CAM_NO_GRAD);
            if (c->relu_saved) {   // a backward will follow: it re-uses the ReLU signs and the staged HexPlane features
                G4D_CUDA(c->relu.ensure(G4D_RELU_BITS_WORDS(n) * 4));
                G4D_CUDA(c->feat.ensure((size_t)(n > 0 ? n : 1) * (size_t)s.d.F * 4 + 256));
            }
            if ((rc = attach_forward_buffers(ws, s, c->relu_saved ? c->feat.as<float>() : nullptr,
                                             c->relu_saved ? c->relu.as<uint32_t>() : nullptr, n, st)) != G4D_OK) return rc;
            G4D_CUDA(launch_deform(s.d, 1, dcam, n, io, ws->sm_count, st, s.tc ? &s.tw : nullptr));
        } else {
            G4D_CUDA(launch_activate_preprocess(dcam, n, io, st));
        }
    }
    if ((rc = debug_sync(cam, st, "deform+preprocess")) != G4D_OK) return rc;
    rc = bin_and_blend(c, cam, n, out_color, out_depth, st);
    if (rc != G4D_OK) return rc;
    c->is_fused = true; c->deformed = prm != nullptr; c->fused_sh = with_sh;
    return G4D_OK;
}

// the post-activation inputs of the rasterizer stages of a fused forward on c: its stored deformed tensors, and the SH
// coefficients (deformed when the SHS head is active, the caller's otherwise)
RasterInputs deformed_inputs(const G4DContext* c, const G4DGaussians* g) {
    RasterInputs in{c->fo.means3D, c->fo.scales, c->fo.rotations, c->fo.opacities,
                    caller_sh<ShIn>(g->features_rest != nullptr, g->features_dc, g->features_rest)};
    if (c->fused_sh) in.sh = ShIn{c->fo.shs, nullptr, nullptr};
    return in;
}

// gradients w.r.t. the deformed tensors of a fine-stage backward: scratch on c (the network's backward reads them)
struct DeformedGrads { float *xyz, *sc, *rot, *op, *sh; };
int deformed_grads(G4DContext* c, int64_t n, DeformedGrads* out) {
    const size_t N = (size_t)n;
    DeformedGrads& d = *out;
    auto layout = [&](Carve& m) {
        d.xyz = m.take<float>(3 * N); d.sc = m.take<float>(3 * N); d.rot = m.take<float>(4 * N); d.op = m.take<float>(N);
        d.sh = m.take<float>(c->fused_sh ? 48 * N : 4);
    };
    G4D_CUDA(ensure_layout(c->gdeform, layout));
    if (!c->fused_sh) d.sh = nullptr;
    return G4D_OK;
}

// The SH gradient sinks of the backward of a fused forward on c: the caller's.  With the SHS head active the gradient also
// feeds the network's backward: the fused sink is then the scratch d_sh, which copy_fused_sh_grad passes on to a caller sink
// in the fused layout.
ShOut fused_sh_sinks(const G4DContext* c, const G4DGaussians* g, const G4DGaussianGrads* gg, float* d_sh) {
    ShOut o = caller_sh<ShOut>(g->features_rest != nullptr, gg->features_dc, gg->features_rest);
    if (c->fused_sh) o.shs = d_sh;
    return o;
}
int copy_fused_sh_grad(const G4DContext* c, const G4DGaussians* g, const G4DGaussianGrads* gg, const float* d_sh, cudaStream_t st) {
    if (c->fused_sh && !g->features_rest)
        G4D_CUDA(cudaMemcpyAsync(gg->features_dc, d_sh, (size_t)g->n * 192, cudaMemcpyDeviceToDevice, st));
    return G4D_OK;
}

// The backward of a fused forward of one camera on c (arguments checked by the caller).  gg->means2D may be NULL.
int fused_backward(G4DContext* c, const G4DCamera* cam, const G4DDeformParams* prm, G4DDeformGrads* pgrads, const G4DGaussians* g,
                   const float* dL_dcolor, const G4DGaussianGrads* gg, cudaStream_t st) {
    const int64_t n = g->n;
    G4DWorkspace* ws = c->ws;
    int rc;
    G4D_CUDA(cudaSetDevice(ws->device));
    if ((rc = check_pending(c)) != G4D_OK) return rc;
    if (n == 0) return G4D_OK;
    const RasterInputs in = deformed_inputs(c, g);
    if (!c->deformed) {
        rc = raster_backward_stages(c, cam, n, in, dL_dcolor, gg->xyz, gg->means2D, fused_sh_sinks(c, g, gg, nullptr),
                                    gg->opacity, gg->scaling, gg->rotation, st);
        if (rc != G4D_OK) return rc;
        G4D_CUDA(launch_activation_backward(n, c->fo, gg->scaling, gg->rotation, gg->opacity, st));
        return debug_sync(cam, st, "activation_backward");
    }
    // gradients w.r.t. the deformed tensors land in scratch, then flow through the deformation network
    DeformedGrads d;
    if ((rc = deformed_grads(c, n, &d)) != G4D_OK) return rc;
    // SH gradient: identity residual path -> written straight into the caller's sinks; the fused copy (when the SHS
    // head is active) additionally feeds the network's backward
    rc = raster_backward_stages(c, cam, n, in, dL_dcolor, d.xyz, gg->means2D, fused_sh_sinks(c, g, gg, d.sh), d.op, d.sc, d.rot,
                                st);
    if (rc != G4D_OK) return rc;
    if ((rc = copy_fused_sh_grad(c, g, gg, d.sh, st)) != G4D_OK) return rc;
    G4D_CUDA(launch_activation_backward(n, c->fo, d.sc, d.rot, d.op, st));
    const float* go[G4D_NUM_HEADS] = {d.xyz, d.sc, d.rot, d.op, d.sh};
    float* gi[G4D_NUM_HEADS] = {gg->xyz, gg->scaling, gg->rotation, gg->opacity, nullptr};
    {
        StageTimer tm(c, G4D_STAGE_DEFORM_BWD, st);
        if ((rc = deform_backward_dispatch(ws, prm, c->trow_ptr, pgrads, cam->time, n, g->xyz, go, gi,
                                           c->relu_saved ? c->relu.as<uint32_t>() : nullptr,
                                           c->relu_saved ? c->feat.as<float>() : nullptr, st)) != G4D_OK) return rc;
    }
    return debug_sync(cam, st, "deform_backward");
}

// k cameras on k contexts: 1 <= k <= G4D_MAX_CAMERAS, one time bit for bit, pairwise distinct contexts of one workspace.
// The cameras are checked before any context is looked at.
int check_camera_group(G4DContext* const* ctx, int32_t k, const G4DCamera* cams) {
    if (k < 1 || k > G4D_MAX_CAMERAS) return fail(G4D_ERR_ARG, "the number of cameras must be in 1..G4D_MAX_CAMERAS");
    if (!cams) return fail(G4D_ERR_ARG, "cameras are NULL");
    int rc;
    for (int i = 0; i < k; ++i) {
        if ((rc = check_camera(&cams[i])) != G4D_OK) return rc;
        if (memcmp(&cams[i].time, &cams[0].time, sizeof(float)) != 0)
            return fail(G4D_ERR_ARG, "the cameras of one call must share their time bit for bit");
    }
    if (!ctx) return fail(G4D_ERR_ARG, "contexts are NULL");
    for (int i = 0; i < k; ++i) {
        if (!ctx[i]) return fail(G4D_ERR_ARG, "context is NULL");
        if (ctx[i]->ws != ctx[0]->ws) return fail(G4D_ERR_ARG, "the contexts of one call must belong to one workspace");
        for (int j = 0; j < i; ++j)
            if (ctx[j] == ctx[i]) return fail(G4D_ERR_ARG, "the contexts of one call must be pairwise distinct");
    }
    return G4D_OK;
}

std::atomic<uint64_t> g_group_serial{0};

}  // namespace

extern "C" {

int g4d_render_forward(G4DContext* c, const G4DCamera* cam, const G4DDeformParams* prm, const G4DGaussians* g,
                       float* out_color, float* out_depth, int32_t* out_radii, void* stream) {
    if (!c) return fail(G4D_ERR_ARG, "context is NULL");
    int rc = check_render_args(cam, prm, g, out_color, out_depth, out_radii);
    if (rc != G4D_OK) return rc;
    return fused_forward(c, cam, prm, g, out_color, out_depth, out_radii, false, (cudaStream_t)stream);
}

int g4d_render_backward(G4DContext* c, const G4DCamera* cam, const G4DDeformParams* prm, G4DDeformGrads* pgrads,
                        const G4DGaussians* g, const float* dL_dcolor, G4DGaussianGrads* gg, void* stream) {
    if (!c) return fail(G4D_ERR_ARG, "context is NULL");
    if (!c->has_forward || !c->is_fused || !g || c->n != g->n) return fail(G4D_ERR_STATE, "g4d_render_backward needs the matching g4d_render_forward on this context");
    if (c->group) return fail(G4D_ERR_STATE, "the last forward on this context was g4d_render_forward_cameras: use g4d_render_backward_cameras");
    if (!c->fo_valid) return fail(G4D_ERR_STATE, "g4d_render_backward after a G4D_CAM_NO_GRAD forward: nothing was saved for it");
    if ((prm != nullptr) != c->deformed) return fail(G4D_ERR_STATE, "deform params differ from the forward's");
    int rc = check_camera(cam);
    if (rc != G4D_OK) return rc;
    if (prm && (rc = check_params(prm)) != G4D_OK) return rc;
    if (prm && !pgrads) return fail(G4D_ERR_ARG, "pgrads is NULL");
    if (cam->image_height != c->H || cam->image_width != c->W) return fail(G4D_ERR_STATE, "camera differs from the forward's");
    const int64_t n = g->n;
    if (!dL_dcolor || !gg || (n > 0 && (!gg->xyz || !gg->scaling || !gg->rotation || !gg->opacity || !gg->features_dc || !gg->means2D)))
        return fail(G4D_ERR_ARG, "NULL gradient pointer");
    if (g->features_rest && n > 0 && !gg->features_rest) return fail(G4D_ERR_ARG, "features_rest gradient sink is NULL");
    return fused_backward(c, cam, prm, pgrads, g, dL_dcolor, gg, (cudaStream_t)stream);
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
    cudaStream_t st = (cudaStream_t)stream;
    G4DContext* c0 = ctx[0];
    G4D_CUDA(cudaSetDevice(c0->ws->device));
    for (int i = 0; i < k; ++i) {
        if ((rc = check_pending(ctx[i])) != G4D_OK) return rc;
        ctx[i]->has_forward = false; ctx[i]->group = 0;
    }
    // camera 0: the fused forward of g4d_render_forward; it keeps the deformed tensors when other cameras read them
    if ((rc = fused_forward(c0, &cams[0], prm, g, out_color[0], out_depth[0], out_radii[0], k > 1, st)) != G4D_OK) return rc;
    const int64_t n = g->n;
    if (k > 1) {
        ExtraCameras ec{};
        ec.count = k - 1;
        for (int i = 1; i < k; ++i) {
            G4DContext* c = ctx[i];
            if ((rc = ensure_geom(c, n)) != G4D_OK) return rc;
            if ((rc = ensure_image(c, cams[i].image_height, cams[i].image_width)) != G4D_OK) return rc;
            reset_stage_flags(c, 0, G4D_STAGE_COUNT - 1);
            {
                StageTimer tm(c, G4D_STAGE_PREP, st);
                G4D_CUDA(launch_pack_camera(cams[i], c->cam.as<CameraDev>(), st));
            }
            ec.cam[i - 1] = c->cam.as<CameraDev>(); ec.g[i - 1] = c->g; ec.out_radii[i - 1] = out_radii[i];
        }
        {
            StageTimer tm(ctx[1], G4D_STAGE_GEOM, st);
            G4D_CUDA(launch_project_cameras(ec, n, deformed_inputs(c0, g), st));
        }
        if ((rc = debug_sync(&cams[1], st, "project_cameras")) != G4D_OK) return rc;
        for (int i = 1; i < k; ++i) {
            G4DContext* c = ctx[i];
            if ((rc = bin_and_blend(c, &cams[i], n, out_color[i], out_depth[i], st)) != G4D_OK) return rc;
            c->is_fused = true; c->deformed = c0->deformed; c->fused_sh = c0->fused_sh; c->fo_valid = false;
        }
    }
    const uint64_t serial = ++g_group_serial;
    for (int i = 0; i < k; ++i) { ctx[i]->group = serial; ctx[i]->group_pos = i; ctx[i]->group_size = k; }
    c0->group_grad = !(cams[0].debug & G4D_CAM_NO_GRAD);
    return G4D_OK;
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
        const G4DContext* c = ctx[i];
        if (!c->has_forward || !c->group || c->group != c0->group || c->group_pos != i || c->group_size != k || c->n != g->n)
            return fail(G4D_ERR_STATE, "g4d_render_backward_cameras needs the matching g4d_render_forward_cameras on these contexts, "
                                       "with no other forward on any of them since");
        if (cams[i].image_height != c->H || cams[i].image_width != c->W) return fail(G4D_ERR_STATE, "camera differs from the forward's");
    }
    if (!c0->group_grad || !c0->fo_valid) return fail(G4D_ERR_STATE, "g4d_render_backward_cameras after a G4D_CAM_NO_GRAD forward: nothing was saved for it");
    if ((prm != nullptr) != c0->deformed) return fail(G4D_ERR_STATE, "deform params differ from the forward's");
    if (prm && (rc = check_params(prm)) != G4D_OK) return rc;
    if (prm && !pgrads) return fail(G4D_ERR_ARG, "pgrads is NULL");
    const int64_t n = g->n;
    if (n > 0 && (!gg->xyz || !gg->scaling || !gg->rotation || !gg->opacity || !gg->features_dc))
        return fail(G4D_ERR_ARG, "NULL gradient pointer");
    if (g->features_rest && n > 0 && !gg->features_rest) return fail(G4D_ERR_ARG, "features_rest gradient sink is NULL");
    cudaStream_t st = (cudaStream_t)stream;
    G4DWorkspace* ws = c0->ws;
    G4D_CUDA(cudaSetDevice(ws->device));
    for (int i = 0; i < k; ++i)
        if ((rc = check_pending(ctx[i])) != G4D_OK) return rc;
    if (k == 1 && dL_dcolor[0]) {     // one camera: the single-camera backward
        G4DGaussianGrads g1 = *gg;
        g1.means2D = g_means2D ? g_means2D[0] : nullptr;
        return fused_backward(c0, &cams[0], prm, pgrads, g, dL_dcolor[0], &g1, st);
    }
    if (n == 0) return G4D_OK;
    const size_t N = (size_t)n;
    DeformedGrads d{gg->xyz, gg->scaling, gg->rotation, gg->opacity, nullptr};   // coarse: straight into the caller's sinks
    if (c0->deformed && (rc = deformed_grads(c0, n, &d)) != G4D_OK) return rc;
    // blend backward of every camera in the loss, each into its own scratch: d(mean2D), d(conic), d(rgb), d(opacity)
    BackwardCameras bc{};
    for (int i = 0; i < k; ++i) {
        G4DContext* c = ctx[i];
        reset_stage_flags(c, G4D_STAGE_BLEND_BWD, G4D_STAGE_DEFORM_BWD);
        if (!dL_dcolor[i]) {
            if (g_means2D && g_means2D[i]) G4D_CUDA(cudaMemsetAsync(g_means2D[i], 0, N * 12, st));
            continue;
        }
        G4D_CUDA(c->gscratch.ensure(N * 9 * 4 + 256));
        float* gb = c->gscratch.as<float>();
        G4D_CUDA(cudaMemsetAsync(gb, 0, N * 9 * 4, st));
        {
            StageTimer tm(c, G4D_STAGE_BLEND_BWD, st);
            G4D_CUDA(launch_blend_backward(c->cam.as<CameraDev>(), c->grid_x, c->grid_y, c->g, c->b, c->im, dL_dcolor[i], gb,
                                           gb + 2 * N, gb + 8 * N, gb + 5 * N, ws->warp_cull, st));
        }
        if ((rc = debug_sync(&cams[i], st, "blend_backward")) != G4D_OK) return rc;
        const int j = bc.count++;
        bc.cam[j] = c->cam.as<CameraDev>(); bc.radii[j] = c->g.radii; bc.clamped[j] = c->g.clamped; bc.grad[j] = gb;
        bc.g_means2D[j] = g_means2D ? g_means2D[i] : nullptr;
    }
    {
        StageTimer tm(c0, G4D_STAGE_GEOM_BWD, st);
        G4D_CUDA(launch_preprocess_backward_cameras(bc, n, deformed_inputs(c0, g), d.xyz, d.sc, d.rot, d.op,
                                                    fused_sh_sinks(c0, g, gg, d.sh), st));
    }
    if ((rc = debug_sync(&cams[0], st, "preprocess_backward_cameras")) != G4D_OK) return rc;
    if ((rc = copy_fused_sh_grad(c0, g, gg, d.sh, st)) != G4D_OK) return rc;
    G4D_CUDA(launch_activation_backward(n, c0->fo, d.sc, d.rot, d.op, st));
    if (!c0->deformed) return debug_sync(&cams[0], st, "activation_backward");
    // the network's backward, once, on the gradients summed over the cameras
    const float* go[G4D_NUM_HEADS] = {d.xyz, d.sc, d.rot, d.op, d.sh};
    float* gi[G4D_NUM_HEADS] = {gg->xyz, gg->scaling, gg->rotation, gg->opacity, nullptr};
    {
        StageTimer tm(c0, G4D_STAGE_DEFORM_BWD, st);
        if ((rc = deform_backward_dispatch(ws, prm, c0->trow_ptr, pgrads, cams[0].time, n, g->xyz, go, gi,
                                           c0->relu_saved ? c0->relu.as<uint32_t>() : nullptr,
                                           c0->relu_saved ? c0->feat.as<float>() : nullptr, st)) != G4D_OK) return rc;
    }
    return debug_sync(&cams[0], st, "deform_backward");
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

int g4d_adam_step(G4DWorkspace* ws, float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t numel,
                  const G4DAdamSegment* segments, int32_t num_segments, float beta1, float beta2, float eps, int64_t step,
                  float grad_scale, void* stream) {
    if (!ws || numel < 0 || (numel > 0 && (!param || !grad || !exp_avg || !exp_avg_sq || !segments)) || step < 1)
        return fail(G4D_ERR_ARG, "g4d_adam_step: bad argument");
    if ((numel & 3) || num_segments < 0 || num_segments > G4D_ADAM_MAX_SEGMENTS)
        return fail(G4D_ERR_ARG, "g4d_adam_step: numel must be a multiple of 4 and at most 16 segments");
    for (int i = 0; i < num_segments; ++i)
        if (segments[i].begin < 0 || segments[i].end < segments[i].begin || segments[i].end > numel || (i && segments[i].begin < segments[i - 1].end))
            return fail(G4D_ERR_ARG, "g4d_adam_step: segments must be sorted, disjoint and inside [0, numel)");
    G4D_CUDA(cudaSetDevice(ws->device));
    G4D_CUDA(launch_adam_flat(param, grad, exp_avg, exp_avg_sq, numel, segments, num_segments, beta1, beta2, eps, step, grad_scale,
                              ws->sm_count, (cudaStream_t)stream));
    return G4D_OK;
}

int g4d_dist2_knn3(G4DWorkspace* ws, int64_t n, const float* xyz, float* out_mean_dist2, void* stream) {
    if (!ws || n < 0 || (n > 0 && (!xyz || !out_mean_dist2))) return fail(G4D_ERR_ARG, "g4d_dist2_knn3: bad argument");
    if (n >= (1ll << 31)) return fail(G4D_ERR_ARG, "n too large");
    G4D_CUDA(cudaSetDevice(ws->device));
    G4D_CUDA(ws->scratch.ensure(knn_scratch_bytes(n)));
    G4D_CUDA(launch_knn_dist2(n, xyz, out_mean_dist2, ws->scratch.p, ws->sm_count, (cudaStream_t)stream));
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
