// g4d_api.cu -- the C-ABI of libg4d.so (include/g4d.h): workspace / context management and stage orchestration.
// No torch types, no CPU fallback: every entry point either runs the CUDA path or returns an error code.
#include <cstdio>
#include <cstdlib>
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

struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    cudaError_t ensure(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        size_t want = bytes + bytes / 2 + 256;
        if (p) { cudaError_t e = cudaFree(p); p = nullptr; cap = 0; if (e != cudaSuccess) return e; }
        cudaError_t e = cudaMalloc(&p, want);
        if (e != cudaSuccess) { p = nullptr; cap = 0; return e; }
        cap = want;
        return cudaSuccess;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
    template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};

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
    DevBuf tc_packed;
    TcWeights tcw{};
    DevBuf tc_bwd_packed, tc_feat;
    TcBwdWeights tcbw{};
    uint64_t tc_bwd_version = 0;
    const void* tc_bwd_key = nullptr;
    uint64_t tc_version = ~0ull;
    const void* tc_key = nullptr;
    DevBuf tc_dbg;
    int tc_debug = 0;
    // packed (transposed) MLP weights, refreshed when G4DDeformParams.version changes
    uint64_t packed_version = ~0ull;
    const void* packed_key = nullptr;
    DevBuf packed;
    float* w0t = nullptr;
    float* w1t[G4D_NUM_HEADS] = {nullptr, nullptr, nullptr, nullptr, nullptr};
    DevBuf trow;        // time rows for the context-free deform entry points
    DevBuf scratch;     // misc per-call scratch (deform backward)
    uint32_t* h_pinned = nullptr;
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

size_t align_up(size_t v, size_t a = 256) { return (v + a - 1) / a * a; }

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
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off += align_up(bytes); return o; };
    const size_t o0 = take(N * 16), o1 = take(N * 16), o2 = take(N * 8), o3 = take(N * 4), o4 = take(N * 8), o5 = take(N * 4),
                 o7 = take(N), o8 = take(N * 4);
    G4D_CUDA(c->geom.ensure(off));
    char* base = c->geom.as<char>();
    c->g.rec0 = (float4*)(base + o0); c->g.rec1 = (float4*)(base + o1); c->g.rec2 = (float2*)(base + o2);
    c->g.radii = (int32_t*)(base + o3); c->g.rect = (uint2*)(base + o4); c->g.tiles_touched = (uint32_t*)(base + o5);
    c->g.clamped = (uint8_t*)(base + o7);
    c->g.perm = (uint32_t*)(base + o8);
    c->g.depth_range = &c->cam.as<CameraDev>()->depth_min;
    return G4D_OK;
}

int ensure_image(G4DContext* c, int H, int W) {
    const size_t P = (size_t)H * W;
    const int gx = (W + kTile - 1) / kTile, gy = (H + kTile - 1) / kTile;
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off += align_up(bytes); return o; };
    const size_t o0 = take(P * 4), o1 = take(P * 4), o2 = take((size_t)gx * gy * 8);
    G4D_CUDA(c->img.ensure(off));
    char* base = c->img.as<char>();
    c->im.final_T = (float*)(base + o0); c->im.n_contrib = (uint32_t*)(base + o1);
    c->b.ranges = (uint2*)(base + o2);
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
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off += align_up(bytes); return o; };
    const size_t o0 = take(N * 12), o1 = take(N * 12), o2 = take(N * 16), o3 = take(N * 4), o5 = take(N * 4),
                 o4 = take(with_sh ? N * 192 : 16);
    G4D_CUDA(c->fused.ensure(off));
    char* base = c->fused.as<char>();
    c->fo.means3D = (float*)(base + o0); c->fo.scales = (float*)(base + o1); c->fo.rotations = (float*)(base + o2);
    c->fo.opacities = (float*)(base + o3); c->fo.rot_norm = (float*)(base + o5);
    c->fo.shs = with_sh ? (float*)(base + o4) : nullptr;
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

// (re)build the transposed weight copies when the caller bumped the version
int refresh_packed(G4DWorkspace* ws, const G4DDeformParams* p, cudaStream_t st) {
    const int F = p->levels * p->channels, WD = p->net_width;
    if (ws->packed_version == p->version && ws->packed_key == (const void*)p->w0 && ws->w0t) return G4D_OK;
    size_t floats = (size_t)F * WD + (size_t)G4D_NUM_HEADS * WD * WD;
    G4D_CUDA(ws->packed.ensure(floats * 4));
    float* base = ws->packed.as<float>();
    ws->w0t = base;
    for (int h = 0; h < G4D_NUM_HEADS; ++h) ws->w1t[h] = base + (size_t)F * WD + (size_t)h * WD * WD;
    G4D_CUDA(launch_pack_weights(*p, ws->w0t, ws->w1t, st));
    ws->packed_version = p->version;
    ws->packed_key = (const void*)p->w0;
    return G4D_OK;
}

bool forward_on_tensor_cores(const G4DWorkspace* ws, const DeformDesc& d) {
    return ws->tensor_cores != 0 && tc_deform_supported(d, ws->tensor_cores);
}

// tensor-core weight images, same caching rule as refresh_packed
int refresh_tc(G4DWorkspace* ws, const G4DDeformParams* p, cudaStream_t st) {
    const int arith = ws->tensor_cores == 2 ? 2 : 1;
    ws->tcw.status = ws->h_pinned + 8;
    if (arith == 2 && ws->h_pinned[8]) {
        ws->h_pinned[8] = 0;
        ws->tc_version = ~0ull;      // re-pack (and re-check) the weights on the next call: they may be the out-of-range values
        return fail(G4D_ERR_OVERFLOW, "an earlier FP16x2 tensor-core launch met a value outside the f16 operand range (activation >= 8188, "
                                      "feature >= 1023 or weight >= 255): its results were saturated; set G4D_OPT_TENSOR_CORES = 1 (3xTF32)");
    }
    if (ws->tc_version == p->version && ws->tc_key == (const void*)p->w0 && ws->tc_packed.p && ws->tcw.arith == arith) return G4D_OK;
    G4D_CUDA(ws->tc_packed.ensure(tc_packed_floats(*p) * 4));
    G4D_CUDA(launch_tc_pack_weights(*p, arith, ws->tc_packed.as<float>(), &ws->tcw, st));
    ws->tcw.arith = arith;
    ws->tc_version = p->version;
    ws->tc_key = (const void*)p->w0;
    return G4D_OK;
}

int refresh_tc_bwd(G4DWorkspace* ws, const G4DDeformParams* p, cudaStream_t st) {
    if (ws->tc_bwd_version == p->version && ws->tc_bwd_key == (const void*)p->w0 && ws->tc_bwd_packed.p) return G4D_OK;
    G4D_CUDA(ws->tc_bwd_packed.ensure(tc_bwd_weight_bytes(*p)));
    G4D_CUDA(launch_tc_bwd_pack_weights(*p, ws->tc_bwd_packed.as<uint8_t>(), &ws->tcbw, st));
    ws->tc_bwd_version = p->version;
    ws->tc_bwd_key = (const void*)p->w0;
    return G4D_OK;
}

// backward of the deformation network: tensor-core path when the configuration allows, FFMA path otherwise
int deform_backward_dispatch(G4DWorkspace* ws, const DeformDesc& d, const G4DDeformParams* prm, const G4DDeformGrads* grads,
                             float time, int64_t n, const float* xyz, const float* const go[G4D_NUM_HEADS],
                             float* const gi[G4D_NUM_HEADS], const uint32_t* relu_bits, const float* saved_feat, cudaStream_t st) {
    int rc;
    if (ws->tensor_cores && tc_backward_supported(d)) {
        if ((rc = refresh_tc_bwd(ws, prm, st)) != G4D_OK) return rc;
        G4D_CUDA(ws->scratch.ensure(tc_deform_backward_scratch_bytes(d, n)));
        G4D_CUDA(launch_deform_backward_tc(d, *prm, *grads, ws->tcbw, time, n, xyz, go, gi, relu_bits, saved_feat, ws->scratch.as<uint8_t>(),
                                           ws->sm_count, st));
        return G4D_OK;
    }
    if ((rc = refresh_packed(ws, prm, st)) != G4D_OK) return rc;
    DeformDesc df = d;                       // the transposes may just have been (re)allocated: take the current pointers
    df.w0t = ws->w0t;
    for (int h = 0; h < G4D_NUM_HEADS; ++h) df.w1t[h] = ws->w1t[h];
    G4D_CUDA(ws->scratch.ensure(deform_backward_scratch_bytes(df, n)));
    G4D_CUDA(launch_deform_backward(df, *prm, *grads, time, n, xyz, go, gi, ws->scratch.as<float>(), ws->sm_count, st));
    return G4D_OK;
}

// ReLU sign bits saved by the tensor-core forward for its backward; the trailing tag word says whether they were written
constexpr int kReluTagByte = 0x5A;
int attach_relu_bits(G4DWorkspace* ws, bool use_tc, bool save, uint32_t* relu_bits, int64_t n, cudaStream_t st) {
    const bool tc = use_tc;
    use_tc = use_tc && save;
    ws->tcw.relu_bits = use_tc ? relu_bits : nullptr;
    ws->tcw.feat = nullptr;
    if (tc) {   // feature staging buffer of the tensor-core forward
        G4D_CUDA(ws->tc_feat.ensure((size_t)(n > 0 ? n : 1) * 64 * 4 + 256));
        ws->tcw.feat = ws->tc_feat.as<float>();
    }
    if (relu_bits) G4D_CUDA(cudaMemsetAsync(relu_bits + (size_t)24 * (size_t)n, use_tc ? kReluTagByte : 0, 16, st));
    return G4D_OK;
}

int attach_tc_debug(G4DWorkspace* ws, cudaStream_t st) {
    ws->tcw.dbg = nullptr;
    if (!ws->tc_debug) return G4D_OK;
    G4D_CUDA(ws->tc_dbg.ensure((size_t)ws->sm_count * 12 * 8));
    G4D_CUDA(cudaMemsetAsync(ws->tc_dbg.p, 0, (size_t)ws->sm_count * 12 * 8, st));
    ws->tcw.dbg = ws->tc_dbg.as<long long>();
    return G4D_OK;
}

int setup_trow(DevBuf& buf, float* (*ptrs)[3], const G4DDeformParams* p) {
    size_t floats = 0;
    for (int l = 0; l < p->levels; ++l)
        for (int a = 0; a < 3; ++a) floats += (size_t)p->res[l][a] * p->channels;
    cudaError_t e = buf.ensure(floats * 4);
    if (e != cudaSuccess) return fail(G4D_ERR_NOMEM, "time-row buffer");
    float* q = buf.as<float>();
    for (int l = 0; l < p->levels; ++l)
        for (int a = 0; a < 3; ++a) { ptrs[l][a] = q; q += (size_t)p->res[l][a] * p->channels; }
    return G4D_OK;
}

DeformDesc make_desc(const G4DWorkspace* ws, const G4DDeformParams* p, float* const (*trow)[3]) {
    DeformDesc d{};
    d.levels = p->levels; d.C = p->channels; d.F = p->levels * p->channels; d.WD = p->net_width; d.head_mask = p->head_mask;
    for (int l = 0; l < p->levels; ++l) {
        for (int a = 0; a < 4; ++a) d.res[l][a] = p->res[l][a];
        for (int k = 0; k < 6; ++k) d.planes[l][k] = p->planes[l][k];
        for (int a = 0; a < 3; ++a) d.trow[l][a] = trow[l][a];
    }
    d.aabb = p->aabb; d.w0t = ws->w0t; d.b0 = p->b0;
    for (int h = 0; h < G4D_NUM_HEADS; ++h) { d.w1t[h] = ws->w1t[h]; d.b1[h] = p->b1[h]; d.w2[h] = p->w2[h]; d.b2[h] = p->b2[h]; }
    return d;
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
            G4D_CUDA(cudaMemcpyAsync(ws->h_pinned, &lay.ctl->R, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
            G4D_CUDA(cudaStreamSynchronize(st));   // exact mode: the one host sync of the path (as in the reference, A.2)
            const int64_t R = (int64_t)ws->h_pinned[0];
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

// blend backward + per-Gaussian backward on `in`; opacity gradient lands in g_opacities (zeroed here)
int raster_backward_stages(G4DContext* c, const G4DCamera* cam, int64_t n, const RasterInputs& in, const float* dL_dcolor,
                           float* g_means3D, float* g_means2D, float* g_shs, float* g_sh_dc, float* g_sh_rest,
                           float* g_opacities, float* g_scales, float* g_rotations, cudaStream_t st) {
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
                                        g_rotations, g_shs, g_sh_dc, g_sh_rest, st));
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
    if (cudaMallocHost((void**)&ws->h_pinned, 64) != cudaSuccess) { delete ws; fail(G4D_ERR_NOMEM, "cudaMallocHost"); return nullptr; }
    for (int i = 0; i < 16; ++i) ws->h_pinned[i] = 0;      // [0]: R read-back, [8]: FP16x2 range flag (written by the kernel)
    return ws;
}

void g4d_workspace_destroy(G4DWorkspace* ws) {
    if (!ws) return;
    cudaSetDevice(ws->device);
    ws->packed.release(); ws->tc_packed.release(); ws->tc_bwd_packed.release(); ws->tc_feat.release(); ws->trow.release(); ws->scratch.release();
    if (ws->h_pinned) cudaFreeHost(ws->h_pinned);
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
    c->cam.release(); c->geom.release(); c->bin.release(); c->binaux.release(); c->img.release(); c->fused.release(); c->gscratch.release(); c->gdeform.release(); c->relu.release(); c->feat.release();
    c->trow.release();
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
    if ((rc = setup_trow(ws->trow, trow, prm)) != G4D_OK) return rc;
    G4D_CUDA(launch_collapse_time_rows(*prm, nullptr, time, false, trow, st));
    const bool use_tc = forward_on_tensor_cores(ws, make_desc(ws, prm, trow));
    if (!use_tc && (rc = refresh_packed(ws, prm, st)) != G4D_OK) return rc;     // FP32 transposes: only the FFMA kernels read them
    const DeformDesc d = make_desc(ws, prm, trow);
    GeomBuffers g{};
    FusedOutputs fo{};
    if (use_tc && (rc = refresh_tc(ws, prm, st)) != G4D_OK) return rc;
    if (use_tc && (rc = attach_tc_debug(ws, st)) != G4D_OK) return rc;
    if ((rc = attach_relu_bits(ws, use_tc, true, relu_bits, n, st)) != G4D_OK) return rc;
    G4D_CUDA(launch_deform(d, 0, nullptr, time, false, n, xyz, scaling, rotation, opacity, shs, nullptr, nullptr, out_xyz,
                           out_scaling, out_rotation, out_opacity, out_shs, g, fo, nullptr, ws->sm_count, st,
                           use_tc ? &ws->tcw : nullptr));
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
    c->has_forward = false; c->is_fused = false; c->deformed = false;
    if ((rc = ensure_geom(c, n)) != G4D_OK) return rc;
    if ((rc = ensure_image(c, cam->image_height, cam->image_width)) != G4D_OK) return rc;
    reset_stage_flags(c, 0, G4D_STAGE_COUNT - 1);
    {
        StageTimer tm(c, G4D_STAGE_PREP, st);
        G4D_CUDA(launch_pack_camera(*cam, c->cam.as<CameraDev>(), st));
    }
    RasterInputs in{means3D, scales, rotations, opacities, shs, nullptr, nullptr};
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
    RasterInputs in{means3D, scales, rotations, opacities, shs, nullptr, nullptr};
    return raster_backward_stages(c, cam, n, in, dL_dcolor, g_means3D, g_means2D, g_shs, nullptr, nullptr, g_opacities,
                                  g_scales, g_rotations, st);
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
    if ((rc = setup_trow(ws->trow, trow, prm)) != G4D_OK) return rc;
    G4D_CUDA(launch_collapse_time_rows(*prm, nullptr, time, false, trow, st));
    const DeformDesc d = make_desc(ws, prm, trow);      // (the dispatcher refreshes the weight images its path needs)
    const float* go[G4D_NUM_HEADS] = {g_out_xyz, g_out_scaling, g_out_rotation, g_out_opacity, g_out_shs};
    float* gi[G4D_NUM_HEADS] = {g_in_xyz, g_in_scaling, g_in_rotation, g_in_opacity, g_in_shs};
    return deform_backward_dispatch(ws, d, prm, grads, time, n, xyz, go, gi, relu_bits, nullptr, st);
}

// ------------------------------------------------------------------------------------------------------
int g4d_render_forward(G4DContext* c, const G4DCamera* cam, const G4DDeformParams* prm, const G4DGaussians* g,
                       float* out_color, float* out_depth, int32_t* out_radii, void* stream) {
    if (!c) return fail(G4D_ERR_ARG, "context is NULL");
    int rc = check_camera(cam);
    if (rc != G4D_OK) return rc;
    if (prm && (rc = check_params(prm)) != G4D_OK) return rc;
    if (!g || g->n < 0 || g->n >= (1ll << 31) || !out_color || !out_depth) return fail(G4D_ERR_ARG, "bad gaussians / outputs");
    const int64_t n = g->n;
    if (n > 0 && (!g->xyz || !g->scaling || !g->rotation || !g->opacity || !g->features_dc || !out_radii))
        return fail(G4D_ERR_ARG, "NULL gaussian tensor");
    cudaStream_t st = (cudaStream_t)stream;
    G4DWorkspace* ws = c->ws;
    G4D_CUDA(cudaSetDevice(ws->device));
    if ((rc = check_pending(c)) != G4D_OK) return rc;
    c->has_forward = false;
    const bool with_sh = prm && (prm->head_mask & G4D_HEAD_SHS);
    if ((rc = ensure_geom(c, n)) != G4D_OK) return rc;
    if ((rc = ensure_image(c, cam->image_height, cam->image_width)) != G4D_OK) return rc;
    if ((rc = ensure_fused(c, n, with_sh)) != G4D_OK) return rc;
    CameraDev* dcam = c->cam.as<CameraDev>();
    reset_stage_flags(c, 0, G4D_STAGE_COUNT - 1);
    const float* shs = g->features_rest ? nullptr : g->features_dc;
    const float* dc = g->features_rest ? g->features_dc : nullptr;
    // a no-grad render needs none of the saved tensors: skip their stores (48 B + 192 B of deformed SH per Gaussian)
    c->fo_valid = !(cam->debug & G4D_CAM_NO_GRAD) || ws->keep_deformed;
    const FusedOutputs fo_arg = c->fo_valid ? c->fo : FusedOutputs{};
    {
        StageTimer tm(c, G4D_STAGE_PREP, st);
        G4D_CUDA(launch_pack_camera(*cam, dcam, st));
        if (prm) {
            if ((rc = setup_trow(c->trow, c->trow_ptr, prm)) != G4D_OK) return rc;
            G4D_CUDA(launch_collapse_time_rows(*prm, dcam, cam->time, false, c->trow_ptr, st));
        }
    }
    StageTimer* geom_tm = new StageTimer(c, G4D_STAGE_GEOM, st);
    struct Del { StageTimer*& p; ~Del() { delete p; p = nullptr; } } del{geom_tm};
    if (prm) {
        const bool use_tc = forward_on_tensor_cores(ws, make_desc(ws, prm, c->trow_ptr));
        if (!use_tc && (rc = refresh_packed(ws, prm, st)) != G4D_OK) return rc;
        const DeformDesc d = make_desc(ws, prm, c->trow_ptr);
        if (use_tc && (rc = refresh_tc(ws, prm, st)) != G4D_OK) return rc;
        if (use_tc && (rc = attach_tc_debug(ws, st)) != G4D_OK) return rc;
        c->relu_saved = use_tc && !(cam->debug & G4D_CAM_NO_GRAD);
        if (c->relu_saved) G4D_CUDA(c->relu.ensure(G4D_RELU_BITS_WORDS(n) * 4));
        if ((rc = attach_relu_bits(ws, use_tc, c->relu_saved, c->relu_saved ? c->relu.as<uint32_t>() : nullptr, n, st)) != G4D_OK) return rc;
        if (c->relu_saved) {   // a backward will follow: keep the staged HexPlane features with the context (it re-uses them)
            G4D_CUDA(c->feat.ensure((size_t)(n > 0 ? n : 1) * (size_t)d.F * 4 + 256));
            ws->tcw.feat = c->feat.as<float>();
        }
        G4D_CUDA(launch_deform(d, 1, dcam, cam->time, false, n, g->xyz, g->scaling, g->rotation, g->opacity, shs, dc,
                               g->features_rest, nullptr, nullptr, nullptr, nullptr, nullptr, c->g, fo_arg, out_radii,
                               ws->sm_count, st, use_tc ? &ws->tcw : nullptr));
    } else {
        G4D_CUDA(launch_activate_preprocess(dcam, n, g->xyz, g->scaling, g->rotation, g->opacity, shs, dc, g->features_rest,
                                            c->g, fo_arg, out_radii, st));
    }
    delete geom_tm; geom_tm = nullptr;
    if ((rc = debug_sync(cam, st, "deform+preprocess")) != G4D_OK) return rc;
    rc = bin_and_blend(c, cam, n, out_color, out_depth, st);
    if (rc != G4D_OK) return rc;
    c->is_fused = true; c->deformed = prm != nullptr; c->fused_sh = with_sh;
    return G4D_OK;
}

int g4d_render_backward(G4DContext* c, const G4DCamera* cam, const G4DDeformParams* prm, G4DDeformGrads* pgrads,
                        const G4DGaussians* g, const float* dL_dcolor, G4DGaussianGrads* gg, void* stream) {
    if (!c) return fail(G4D_ERR_ARG, "context is NULL");
    if (!c->has_forward || !c->is_fused || !g || c->n != g->n) return fail(G4D_ERR_STATE, "g4d_render_backward needs the matching g4d_render_forward on this context");
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
    cudaStream_t st = (cudaStream_t)stream;
    G4DWorkspace* ws = c->ws;
    G4D_CUDA(cudaSetDevice(ws->device));
    if ((rc = check_pending(c)) != G4D_OK) return rc;
    if (n == 0) return G4D_OK;
    const size_t N = (size_t)n;
    const bool split = g->features_rest != nullptr;
    RasterInputs in{c->fo.means3D, c->fo.scales, c->fo.rotations, c->fo.opacities,
                    c->fused_sh ? c->fo.shs : (split ? nullptr : g->features_dc), split ? g->features_dc : nullptr,
                    g->features_rest};
    float* sh_fused_sink = split ? nullptr : gg->features_dc;
    float* sh_dc_sink = split ? gg->features_dc : nullptr;
    float* sh_rest_sink = split ? gg->features_rest : nullptr;
    if (!c->deformed) {
        rc = raster_backward_stages(c, cam, n, in, dL_dcolor, gg->xyz, gg->means2D, sh_fused_sink, sh_dc_sink, sh_rest_sink,
                                    gg->opacity, gg->scaling, gg->rotation, st);
        if (rc != G4D_OK) return rc;
        G4D_CUDA(launch_activation_backward(n, c->fo, gg->scaling, gg->rotation, gg->opacity, st));
        return debug_sync(cam, st, "activation_backward");
    }
    // gradients w.r.t. the deformed tensors land in scratch, then flow through the deformation network
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off += align_up(bytes); return o; };
    const size_t o0 = take(N * 12), o1 = take(N * 12), o2 = take(N * 16), o3 = take(N * 4), o4 = take(c->fused_sh ? N * 192 : 16);
    G4D_CUDA(c->gdeform.ensure(off));
    char* base = c->gdeform.as<char>();
    float* gd_xyz = (float*)(base + o0); float* gd_sc = (float*)(base + o1); float* gd_rot = (float*)(base + o2);
    float* gd_op = (float*)(base + o3); float* gd_sh = c->fused_sh ? (float*)(base + o4) : nullptr;
    // SH gradient: identity residual path -> written straight into the caller's sinks; the fused copy (when the SHS
    // head is active) additionally feeds the network's backward
    if (c->fused_sh && !split) { sh_fused_sink = gg->features_dc; }
    rc = raster_backward_stages(c, cam, n, in, dL_dcolor, gd_xyz, gg->means2D, c->fused_sh ? gd_sh : sh_fused_sink, sh_dc_sink,
                                sh_rest_sink, gd_op, gd_sc, gd_rot, st);
    if (rc != G4D_OK) return rc;
    if (c->fused_sh && !split) G4D_CUDA(cudaMemcpyAsync(gg->features_dc, gd_sh, N * 192, cudaMemcpyDeviceToDevice, st));
    G4D_CUDA(launch_activation_backward(n, c->fo, gd_sc, gd_rot, gd_op, st));
    const DeformDesc d = make_desc(ws, prm, c->trow_ptr);
    const float* go[G4D_NUM_HEADS] = {gd_xyz, gd_sc, gd_rot, gd_op, gd_sh};
    float* gi[G4D_NUM_HEADS] = {gg->xyz, gg->scaling, gg->rotation, gg->opacity, nullptr};
    {
        StageTimer tm(c, G4D_STAGE_DEFORM_BWD, st);
        if ((rc = deform_backward_dispatch(ws, d, prm, pgrads, cam->time, n, g->xyz, go, gi, c->relu_saved ? c->relu.as<uint32_t>() : nullptr,
                                           c->relu_saved ? c->feat.as<float>() : nullptr, st)) != G4D_OK) return rc;
    }
    return debug_sync(cam, st, "deform_backward");
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
