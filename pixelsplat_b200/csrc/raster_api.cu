// extern "C" entry points of include/pixelsplat_b200.h: argument validation, workspace layout,
// stage sequencing.  No torch types, no exceptions across the ABI.
#include <cstdarg>
#include <atomic>
#include <cstdio>
#include <cstring>
#include <mutex>

#include "ps_common.cuh"

namespace ps {

static thread_local char g_error[512] = "";

void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_error, sizeof(g_error), fmt, ap);
    va_end(ap);
}

static bool g_timing = false;
static cudaEvent_t g_events[kNumMarks];
static bool g_events_ready = false;
static std::atomic<unsigned long long> g_launches{0};

void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

static std::mutex g_once_mutex;

bool first_use_on_device(unsigned long long &mask) {
    int dev = 0;
    cudaGetDevice(&dev);
    const unsigned long long bit = 1ull << (dev & 63);
    std::lock_guard<std::mutex> lock(g_once_mutex);
    if (mask & bit) return false;
    mask |= bit;
    return true;
}

void mark(int id, cudaStream_t st) {
    if (!g_timing) return;
    if (!g_events_ready) {
        for (int i = 0; i < kNumMarks; ++i) cudaEventCreate(&g_events[i]);
        g_events_ready = true;
    }
    cudaEventRecord(g_events[id], st);
}

// Side stream for work that is independent of the critical path (SH -> RGB overlapping the binning
// in the forward).  Fork/join with events, which also captures cleanly into CUDA graphs.
// The library's side stream and its fork / join events, one set per device ordinal (created on first
// use on that device; a host process may drive several GPUs).
// The fork / join event pair is shared by every call on a device, so the enqueue of one forward
// -- record fork, side-stream work, record join, wait join -- must not interleave with another host thread's on
// the same device: each entry point holds the device's mutex while it enqueues (host-side only; ~tens of us).
struct SideCtx {
    cudaStream_t side = nullptr;
    cudaEvent_t fork = nullptr, join = nullptr;
    cudaEvent_t scanned = nullptr, copied = nullptr;   // the capacity read-back: after the scan, back before return
    std::mutex enqueue;
};
static SideCtx g_side_ctx[64];

static int side_ready(SideCtx *&ctx) {
    int dev = 0;
    PS_CUDA_CHECK(cudaGetDevice(&dev));
    ctx = &g_side_ctx[dev & 63];
    std::lock_guard<std::mutex> lock(g_once_mutex);
    if (ctx->side) return PS_OK;
    PS_CUDA_CHECK(cudaStreamCreateWithFlags(&ctx->side, cudaStreamNonBlocking));
    PS_CUDA_CHECK(cudaEventCreateWithFlags(&ctx->fork, cudaEventDisableTiming));
    PS_CUDA_CHECK(cudaEventCreateWithFlags(&ctx->join, cudaEventDisableTiming));
    PS_CUDA_CHECK(cudaEventCreateWithFlags(&ctx->scanned, cudaEventDisableTiming));
    PS_CUDA_CHECK(cudaEventCreateWithFlags(&ctx->copied, cudaEventDisableTiming));
    return PS_OK;
}

static size_t align_up(size_t x) { return (x + 255) & ~(size_t)255; }

// Deterministic mode (ps_set_option "deterministic"): fixed-order composite backward and loss epilogue.  Read once
// per call, by make_layout.
static int g_deterministic = 0;

struct Layout {
    ps_raster_layout off;
    ps_raster_sizes sizes;
    bool det;                    // deterministic mode: the two arrays below exist
    size_t loss_partials;        // image: f32x2 [S*V*tiles*8] per-task (sse, sse_clipped) of the loss epilogue
    size_t records;              // backward scratch: the composite's block records (d_mean2d, d_conic, d_color)
};

static int validate(const ps_raster_desc *d) {
    if (!d) { set_error("desc is NULL"); return PS_ERR_INVALID_ARGUMENT; }
    if (d->n_scenes < 1 || d->views_per_scene < 1 || d->n_gaussians < 1) {
        set_error("n_scenes, views_per_scene and n_gaussians must be >= 1 (got %d, %d, %d)",
                  d->n_scenes, d->views_per_scene, d->n_gaussians);
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (d->height < 1 || d->width < 1) { set_error("bad image size %dx%d", d->height, d->width); return PS_ERR_INVALID_ARGUMENT; }
    if (d->sh_coeffs < 0 || d->sh_coeffs > 25) { set_error("sh_coeffs must be in [0, 25], got %d", d->sh_coeffs); return PS_ERR_INVALID_ARGUMENT; }
    if (d->sh_degree < 0 || d->sh_degree > 4) { set_error("sh_degree must be in [0, 4], got %d", d->sh_degree); return PS_ERR_INVALID_ARGUMENT; }
    if (d->sh_coeffs > 0 && (d->sh_degree + 1) * (d->sh_degree + 1) > d->sh_coeffs) {
        set_error("sh_degree %d needs %d coefficients, only %d given", d->sh_degree,
                  (d->sh_degree + 1) * (d->sh_degree + 1), d->sh_coeffs);
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (d->sh_layout != PS_SH_M3 && d->sh_layout != PS_SH_3M) { set_error("bad sh_layout %d", d->sh_layout); return PS_ERR_INVALID_ARGUMENT; }
    if (d->sh_basis != PS_SH_BASIS_3DGS && d->sh_basis != PS_SH_BASIS_E3NN) { set_error("bad sh_basis %d", d->sh_basis); return PS_ERR_INVALID_ARGUMENT; }
    if (d->depth_mode < PS_DEPTH_NONE || d->depth_mode > PS_DEPTH_LOG) { set_error("bad depth_mode %d (PS_DEPTH_*: 0..4)", d->depth_mode); return PS_ERR_INVALID_ARGUMENT; }
    if (d->cov_layout != PS_COV_TRIU6 && d->cov_layout != PS_COV_3X3) { set_error("bad cov_layout %d", d->cov_layout); return PS_ERR_INVALID_ARGUMENT; }
    if (d->instance_capacity < 1 || d->instance_capacity > 0x7fffffffll) {
        set_error("instance_capacity must be in [1, 2^31-1], got %lld", (long long)d->instance_capacity);
        return PS_ERR_INVALID_ARGUMENT;
    }
    const long long gx = (d->width + kTile - 1) / kTile, gy = (d->height + kTile - 1) / kTile;
    if (gx > 65535 || gy > 65535) { set_error("image too large for 16-bit tile rectangles"); return PS_ERR_UNSUPPORTED; }
    const long long segs = (long long)d->n_scenes * d->views_per_scene * gx * gy;
    if ((long long)d->n_scenes * d->views_per_scene * d->n_gaussians > 0xffffffffll) {
        set_error("scenes * views * gaussians must fit 32 bits");
        return PS_ERR_UNSUPPORTED;
    }
    if (segs > 0x7fffffffll || (long long)d->n_scenes * d->views_per_scene > 65535) {
        set_error("too many (view, tile) segments: %lld", segs);
        return PS_ERR_UNSUPPORTED;
    }
    return PS_OK;
}

static Dims make_dims(const ps_raster_desc *d) {
    Dims r;
    r.S = d->n_scenes; r.V = d->views_per_scene; r.P = d->n_gaussians; r.M = d->sh_coeffs;
    r.deg = d->sh_degree; r.sh_layout = d->sh_layout; r.cov_layout = d->cov_layout;
    r.H = d->height; r.W = d->width;
    r.gx = (d->width + kTile - 1) / kTile; r.gy = (d->height + kTile - 1) / kTile;
    r.tiles = r.gx * r.gy;
    r.capacity = d->instance_capacity;
    r.sh_basis = d->sh_basis;
    r.segK = composite_segments((long long)r.S * r.V * r.tiles * 8);
    r.hit_lists = composite_hit_lists(r.capacity) ? 1 : 0;
    r.depth_mode = d->depth_mode;
    return r;
}

static Layout make_layout(const ps_raster_desc *d) {
    const Dims m = make_dims(d);
    const size_t vp = (size_t)m.S * m.V * m.P;
    const size_t vt = (size_t)m.S * m.V * m.tiles;
    const size_t px = (size_t)m.S * m.V * m.H * m.W;
    Layout L;
    size_t o = 0;
    auto take = [&](size_t bytes) { const size_t at = o; o = align_up(o + bytes); return at; };
    L.off.depth = take(vp * 4);
    L.off.radii = take(vp * 4);
    L.off.xy = take(vp * 8);
    L.off.conic_opacity = take(vp * 16);
    L.off.rgb = take(vp * 16);
    L.off.rect = take(vp * 8);
    L.off.clamped = take(vp);
    L.off.tile_count = take(vt * 4);
    L.off.tile_start = take(vt * 4);
    L.off.tile_cursor = take(vt * 4);
    L.off.n_instances = take(32);   // [0] instances, [1] longest segment, [2] #visible pairs, [3] unused
    L.off.vis_pairs = take(vp * 4);
    L.off.vis_any = take((size_t)m.S * m.P * 4);   // unused; kept so that the ABI layout does not change
    L.off.cull = take(vp * 16);
    L.sizes.geom_bytes = o;
    o = 0;
    L.off.keys = take((size_t)m.capacity * 8);
    L.off.keys_alt = take((size_t)m.capacity * 8);
    // per-(tile, block, run) hit lists written by the composite forward for its backward (8 x the instances in the
    // worst case: only kept when that stays small; the backward culls for itself otherwise)
    L.off.block_hits = L.off.run_hits = 0;
    if (m.hit_lists) {
        L.off.block_hits = take((size_t)m.capacity * 8 * 8);
        L.off.run_hits = take((size_t)m.S * m.V * m.tiles * 8 * kMaxSegments * 4);
    }
    L.sizes.binning_bytes = o;
    o = 0;
    L.off.final_T = take(px * 4);
    L.off.n_contrib = take(px * 4);
    L.off.color = take(px * 12);
    L.off.run_state = take(px * 16 * (kMaxSegments - 1));
    L.off.depth_image = L.off.run_depth = 0;
    if (m.depth_mode) {
        L.off.depth_image = take(px * 4);
        L.off.run_depth = take(px * 4 * (kMaxSegments - 1));
    }
    L.det = g_deterministic != 0;
    L.loss_partials = L.det ? take(vt * 8 * 8) : 0;
    L.sizes.image_bytes = o;
    // backward scratch: d_mean2d (8) + d_conic (16) + d_color (16) per (view, Gaussian); deterministic mode: the
    // same per (tile block, list position), 8 x instance_capacity of them
    L.sizes.backward_bytes = align_up(vp * 8) + align_up(vp * 16) + align_up(vp * 16);
    L.records = L.sizes.backward_bytes;
    if (L.det) {
        const size_t nr = (size_t)m.capacity * 8;
        L.sizes.backward_bytes += align_up(nr * 8) + align_up(nr * 16) + align_up(nr * 16);
    }
    return L;
}

// ps_raster_camera_workspace_bytes: one partial row per (warp overlapping a scene, view)
static size_t camera_workspace_bytes(const ps_raster_desc *d) {
    return (size_t)d->n_scenes * d->views_per_scene * cam_rows_per_view(d->n_gaussians) * kCamRowFloats * sizeof(float);
}

static Geom make_geom(const Layout &L, void *geom) {
    char *b = static_cast<char *>(geom);
    Geom g;
    g.depth = reinterpret_cast<float *>(b + L.off.depth);
    g.radii = reinterpret_cast<int32_t *>(b + L.off.radii);
    g.xy = reinterpret_cast<float2 *>(b + L.off.xy);
    g.conic_opacity = reinterpret_cast<float4 *>(b + L.off.conic_opacity);
    g.rgb = reinterpret_cast<float4 *>(b + L.off.rgb);
    g.rect = reinterpret_cast<ushort4 *>(b + L.off.rect);
    g.clamped = reinterpret_cast<uint8_t *>(b + L.off.clamped);
    g.tile_count = reinterpret_cast<uint32_t *>(b + L.off.tile_count);
    g.tile_start = reinterpret_cast<uint32_t *>(b + L.off.tile_start);
    g.tile_cursor = reinterpret_cast<uint32_t *>(b + L.off.tile_cursor);
    g.n_instances = reinterpret_cast<long long *>(b + L.off.n_instances);
    g.vis_pairs = reinterpret_cast<uint32_t *>(b + L.off.vis_pairs);
    g.cull = reinterpret_cast<float4 *>(b + L.off.cull);
    return g;
}

static ImageState make_image(const Layout &L, void *image) {
    char *b = static_cast<char *>(image);
    ImageState im;
    im.final_T = reinterpret_cast<float *>(b + L.off.final_T);
    im.n_contrib = reinterpret_cast<uint32_t *>(b + L.off.n_contrib);
    im.color = reinterpret_cast<float *>(b + L.off.color);
    im.run_state = reinterpret_cast<float4 *>(b + L.off.run_state);
    im.depth_image = L.off.depth_image ? reinterpret_cast<float *>(b + L.off.depth_image) : nullptr;
    im.run_depth = L.off.run_depth ? reinterpret_cast<float *>(b + L.off.run_depth) : nullptr;
    return im;
}

// `backward`: the image state needs no room for the loss partials (a forward issued before the option was set
// followed by a backward issued after it is fine).
static int check_common(const ps_raster_desc *desc, const ps_raster_inputs *in, const ps_raster_state *state,
                        const Layout &L, bool backward) {
    const size_t image_bytes = backward && L.det ? L.loss_partials : L.sizes.image_bytes;
    if (!in || !state) { set_error("inputs/state is NULL"); return PS_ERR_INVALID_ARGUMENT; }
    if (!in->means || !in->cov || !in->opacities || !in->sh || !in->viewmatrix || !in->projmatrix ||
        !in->campos || !in->tanfov || !in->background) {
        set_error("a required input pointer is NULL");
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (!state->geom || !state->binning || !state->image) { set_error("a state buffer is NULL"); return PS_ERR_INVALID_ARGUMENT; }
    if (state->geom_bytes < L.sizes.geom_bytes || state->binning_bytes < L.sizes.binning_bytes ||
        state->image_bytes < image_bytes) {
        set_error("state buffers too small: need geom %zu binning %zu image %zu, got %zu %zu %zu",
                  L.sizes.geom_bytes, L.sizes.binning_bytes, image_bytes, state->geom_bytes,
                  state->binning_bytes, state->image_bytes);
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (((uintptr_t)state->geom | (uintptr_t)state->binning | (uintptr_t)state->image) & 15) {
        set_error("state buffers must be 16-byte aligned");
        return PS_ERR_INVALID_ARGUMENT;
    }
    if ((desc->depth_mode == PS_DEPTH_RELATIVE_DISPARITY || desc->depth_mode == PS_DEPTH_LOG) && !in->near_far) {
        set_error("depth_mode %d needs ps_raster_inputs.near_far", desc->depth_mode);
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (desc->depth_mode && composite_impl() == 1) {
        set_error("the legacy compositor (composite_impl = 1) has no depth channel");
        return PS_ERR_UNSUPPORTED;
    }
    if (L.det && composite_impl() == 1) {
        set_error("the legacy compositor (composite_impl = 1) has no fixed-order (deterministic) form");
        return PS_ERR_UNSUPPORTED;
    }
    return PS_OK;
}

static Inputs make_inputs(const ps_raster_inputs *in) {
    Inputs r;
    r.means = in->means; r.cov = in->cov; r.opac = in->opacities; r.sh = in->sh;
    r.view = in->viewmatrix; r.proj = in->projmatrix; r.campos = in->campos; r.tanfov = in->tanfov;
    r.bg = in->background; r.scale = in->scene_scale; r.near_far = in->near_far;
    return r;
}

}  // namespace ps

using namespace ps;

extern "C" {

PS_API int ps_version(void) { return 100; }

PS_API const char *ps_last_error(void) { return g_error; }

PS_API unsigned long long ps_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

PS_API void ps_timing_enable(int on) { g_timing = on != 0; }

// ms[0..6] = preprocess, count-scan+scatter, sort, composite fwd, zero-fill, composite bwd,
// preprocess bwd of the most recent forward+backward pair.  Synchronises on the last event.
PS_API int ps_timing_read(float *ms) {
    if (!g_timing || !g_events_ready) { set_error("timing is not enabled"); return PS_ERR_INVALID_ARGUMENT; }
    static const int pairs[7][2] = {{kMarkFwdStart, kMarkPreprocess}, {kMarkPreprocess, kMarkScatter},
                                    {kMarkScatter, kMarkSort}, {kMarkSort, kMarkCompositeFwd},
                                    {kMarkBwdStart, kMarkBwdZero}, {kMarkBwdZero, kMarkCompositeBwd},
                                    {kMarkCompositeBwd, kMarkPreprocessBwd}};
    PS_CUDA_CHECK(cudaEventSynchronize(g_events[kMarkPreprocessBwd]));
    for (int i = 0; i < 7; ++i) PS_CUDA_CHECK(cudaEventElapsedTime(&ms[i], g_events[pairs[i][0]], g_events[pairs[i][1]]));
    return PS_OK;
}

PS_API int ps_set_option(const char *name, int value) {
    if (!name) { set_error("ps_set_option: name is NULL"); return PS_ERR_INVALID_ARGUMENT; }
    int rc = PS_ERR_INVALID_ARGUMENT;
    if (!strcmp(name, "composite_impl")) rc = set_composite_option(0, value);
    else if (!strcmp(name, "composite_segments")) rc = set_composite_option(1, value);
    else if (!strcmp(name, "composite_hit_lists")) rc = set_composite_option(2, value);
    else if (!strcmp(name, "deterministic") && (value == 0 || value == 1)) { g_deterministic = value; rc = PS_OK; }
    if (rc) set_error("ps_set_option: unknown option or bad value: %s = %d", name, value);
    return rc;
}

PS_API int ps_get_option(const char *name, int *value) {
    if (!name || !value) { set_error("ps_get_option: name / value is NULL"); return PS_ERR_INVALID_ARGUMENT; }
    int which = -1;
    if (!strcmp(name, "composite_impl")) which = 0;
    else if (!strcmp(name, "composite_segments")) which = 1;
    else if (!strcmp(name, "composite_hit_lists")) which = 2;
    else if (!strcmp(name, "deterministic")) { *value = g_deterministic; return PS_OK; }
    if (which < 0) { set_error("ps_get_option: unknown option %s", name); return PS_ERR_INVALID_ARGUMENT; }
    *value = get_composite_option(which);
    return PS_OK;
}

PS_API int ps_raster_sizes_query(const ps_raster_desc *desc, ps_raster_sizes *out) {
    int rc = validate(desc);
    if (rc) return rc;
    if (!out) { set_error("out is NULL"); return PS_ERR_INVALID_ARGUMENT; }
    *out = make_layout(desc).sizes;
    return PS_OK;
}

PS_API int ps_raster_layout_query(const ps_raster_desc *desc, ps_raster_layout *out) {
    int rc = validate(desc);
    if (rc) return rc;
    if (!out) { set_error("out is NULL"); return PS_ERR_INVALID_ARGUMENT; }
    *out = make_layout(desc).off;
    return PS_OK;
}

PS_API int ps_raster_camera_workspace_bytes(const ps_raster_desc *desc, size_t *out) {
    int rc = validate(desc);
    if (rc) return rc;
    if (!out) { set_error("out is NULL"); return PS_ERR_INVALID_ARGUMENT; }
    *out = camera_workspace_bytes(desc);
    return PS_OK;
}

}  // extern "C"

static int raster_forward_impl(const ps_raster_desc *desc, const ps_raster_inputs *in, const ps_raster_state *state,
                               float *out_color, int32_t *out_radii, int64_t *n_instances_host,
                               const ps_raster_loss *loss, void *stream) {
    int rc = validate(desc);
    if (rc) return rc;
    const Layout L = make_layout(desc);
    rc = check_common(desc, in, state, L, false);
    if (rc) return rc;
    LossEpilogue le{nullptr, nullptr, nullptr};
    if (loss) {
        if (!loss->target || !loss->sums) { set_error("ps_raster_loss: target / sums is NULL"); return PS_ERR_INVALID_ARGUMENT; }
        le.target = loss->target; le.sums = loss->sums;
    } else if (!out_color) {
        set_error("out_color is NULL");
        return PS_ERR_INVALID_ARGUMENT;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const Dims d = make_dims(desc);
    const Inputs I = make_inputs(in);
    const Geom g = make_geom(L, state->geom);
    unsigned long long *keys = reinterpret_cast<unsigned long long *>(static_cast<char *>(state->binning) + L.off.keys);
    unsigned long long *keys_alt = reinterpret_cast<unsigned long long *>(static_cast<char *>(state->binning) + L.off.keys_alt);
    const ImageState img = make_image(L, state->image);

    SideCtx *sc = nullptr;
    if ((rc = side_ready(sc))) return rc;
    std::lock_guard<std::mutex> enqueue_lock(sc->enqueue);
    mark(kMarkFwdStart, st);
    if ((rc = launch_preprocess(d, I, g, st))) return rc;
    mark(kMarkPreprocess, st);
    // fork: SH -> RGB of the on-screen Gaussians runs beside the binning (scan / scatter / sort);
    // the two only meet again in the compositor
    PS_CUDA_CHECK(cudaEventRecord(sc->fork, st));
    PS_CUDA_CHECK(cudaStreamWaitEvent(sc->side, sc->fork, 0));
    if ((rc = launch_sh_color(d, I, g, sc->side))) return rc;
    PS_CUDA_CHECK(cudaEventRecord(sc->join, sc->side));
    if ((rc = launch_binning(d, g, keys, keys_alt, desc->sort_impl, desc->sort_segment_hint,
                             n_instances_host ? sc->scanned : nullptr, st)))
        return rc;
    mark(kMarkSort, st);
    PS_CUDA_CHECK(cudaStreamWaitEvent(st, sc->join, 0));   // join
    if (n_instances_host) {
        // capacity read-back on the side stream, once the scan has the counts: a device-to-host copy between the sort
        // and the compositor would sit on the critical path (also of every captured graph); joined back below
        PS_CUDA_CHECK(cudaStreamWaitEvent(sc->side, sc->scanned, 0));
        PS_CUDA_CHECK(cudaMemcpyAsync(n_instances_host, g.n_instances, 2 * sizeof(int64_t), cudaMemcpyDeviceToHost,
                                      sc->side));
        PS_CUDA_CHECK(cudaEventRecord(sc->copied, sc->side));
    }
    // (deterministic mode: the fixed-order finish writes every slot)
    float *loss_partials = L.det ? reinterpret_cast<float *>(static_cast<char *>(state->image) + L.loss_partials) : nullptr;
    if (le.sums && !loss_partials)
        PS_CUDA_CHECK(cudaMemsetAsync(le.sums, 0, sizeof(float) * 2 * kLossSlots * (size_t)d.S * d.V, st));
    HitLists hl{nullptr, nullptr};
    if (d.hit_lists) {
        hl.hits = reinterpret_cast<uint2 *>(static_cast<char *>(state->binning) + L.off.block_hits);
        hl.run_hits = reinterpret_cast<uint32_t *>(static_cast<char *>(state->binning) + L.off.run_hits);
    }
    if ((rc = launch_composite_forward(d, I, g, keys, reinterpret_cast<const uint2 *>(keys_alt), img, out_color, le, hl,
                                       loss_partials, st)))
        return rc;
    if (n_instances_host) PS_CUDA_CHECK(cudaStreamWaitEvent(st, sc->copied, 0));   // join the read-back
    mark(kMarkCompositeFwd, st);
    if (out_radii)
        PS_CUDA_CHECK(cudaMemcpyAsync(out_radii, g.radii, sizeof(int32_t) * (size_t)d.S * d.V * d.P,
                                      cudaMemcpyDeviceToDevice, st));
    return PS_OK;
}

extern "C" {

PS_API int ps_raster_forward(const ps_raster_desc *desc, const ps_raster_inputs *in, const ps_raster_state *state,
                             float *out_color, int32_t *out_radii, int64_t *n_instances_host, void *stream) {
    return raster_forward_impl(desc, in, state, out_color, out_radii, n_instances_host, nullptr, stream);
}

PS_API int ps_raster_forward_loss(const ps_raster_desc *desc, const ps_raster_inputs *in, const ps_raster_state *state,
                                  const ps_raster_loss *loss, float *out_color, int32_t *out_radii,
                                  int64_t *n_instances_host, void *stream) {
    if (!loss) { set_error("ps_raster_forward_loss: loss is NULL"); return PS_ERR_INVALID_ARGUMENT; }
    return raster_forward_impl(desc, in, state, out_color, out_radii, n_instances_host, loss, stream);
}

}  // extern "C"

static int raster_backward_impl(const ps_raster_desc *desc, const ps_raster_inputs *in, const ps_raster_state *state,
                                const float *d_color, const float *target, const float *grad_scale,
                                const float *d_depth, void *scratch, size_t scratch_bytes,
                                const ps_raster_grads *grads, void *stream) {
    int rc = validate(desc);
    if (rc) return rc;
    const Layout L = make_layout(desc);
    rc = check_common(desc, in, state, L, true);
    if (rc) return rc;
    if ((!d_color && !(target && grad_scale)) || !scratch || !grads) {
        set_error("d_color (or target + grad_scale) / scratch / grads is NULL");
        return PS_ERR_INVALID_ARGUMENT;
    }
    const LossEpilogue le{d_color ? nullptr : target, nullptr, d_color ? nullptr : grad_scale};
    if (!grads->d_means || !grads->d_cov || !grads->d_opacities || !grads->d_sh) {
        set_error("a required gradient pointer is NULL");
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (scratch_bytes < L.sizes.backward_bytes || ((uintptr_t)scratch & 15)) {
        set_error("backward scratch too small or misaligned: need %zu, got %zu", L.sizes.backward_bytes, scratch_bytes);
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (const ps_raster_camera_grads *cg = grads->camera) {
        const size_t need = camera_workspace_bytes(desc);
        if (!cg->workspace || cg->workspace_bytes < need || ((uintptr_t)cg->workspace & 15)) {
            set_error("camera-gradient workspace NULL, too small or misaligned: need %zu, got %zu", need,
                      cg->workspace_bytes);
            return PS_ERR_INVALID_ARGUMENT;
        }
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    Dims d = make_dims(desc);
    if (!d_depth) d.depth_mode = 0;     // no depth gradient: the colour-only kernels, dL/dD = 0
    const Inputs I = make_inputs(in);
    const Geom g = make_geom(L, state->geom);
    const unsigned long long *keys = reinterpret_cast<const unsigned long long *>(static_cast<char *>(state->binning) + L.off.keys);
    const uint2 *live = reinterpret_cast<const uint2 *>(static_cast<char *>(state->binning) + L.off.keys_alt);
    const ImageState img = make_image(L, state->image);
    const size_t vp = (size_t)d.S * d.V * d.P;
    char *sb = static_cast<char *>(scratch);
    ViewGrads vg;
    vg.d_mean2d = reinterpret_cast<float2 *>(sb);
    vg.d_conic = reinterpret_cast<float4 *>(sb + align_up(vp * 8));
    vg.d_color = reinterpret_cast<float4 *>(sb + align_up(vp * 8) + align_up(vp * 16));
    ViewGrads rec;                      // deterministic mode: the block records, after the per-(view, Gaussian) arrays
    const size_t nr = (size_t)d.capacity * 8;
    rec.d_mean2d = reinterpret_cast<float2 *>(sb + L.records);
    rec.d_conic = reinterpret_cast<float4 *>(sb + L.records + align_up(nr * 8));
    rec.d_color = reinterpret_cast<float4 *>(sb + L.records + align_up(nr * 8) + align_up(nr * 16));
    mark(kMarkBwdStart, st);
    if ((rc = launch_clear_pair_grads(d, g, vg, st))) return rc;
    // deterministic mode: the gather reads a record for every list position, whether or not a block stored one
    if (L.det) PS_CUDA_CHECK(cudaMemsetAsync(sb + L.records, 0, L.sizes.backward_bytes - L.records, st));
    mark(kMarkBwdZero, st);
    HitLists hl{nullptr, nullptr};
    if (d.hit_lists) {
        hl.hits = reinterpret_cast<uint2 *>(static_cast<char *>(state->binning) + L.off.block_hits);
        hl.run_hits = reinterpret_cast<uint32_t *>(static_cast<char *>(state->binning) + L.off.run_hits);
    }
    if ((rc = launch_composite_backward(d, I, g, keys, live, img, d_color, d_depth, vg, L.det ? &rec : nullptr, le, hl,
                                        st)))
        return rc;
    mark(kMarkCompositeBwd, st);
    if ((rc = launch_preprocess_backward(d, I, g, vg, *grads, st))) return rc;
    mark(kMarkPreprocessBwd, st);
    return PS_OK;
}

extern "C" {

PS_API int ps_raster_backward(const ps_raster_desc *desc, const ps_raster_inputs *in, const ps_raster_state *state,
                              const float *d_color, void *scratch, size_t scratch_bytes,
                              const ps_raster_grads *grads, void *stream) {
    if (!d_color) { set_error("d_color is NULL"); return PS_ERR_INVALID_ARGUMENT; }
    return raster_backward_impl(desc, in, state, d_color, nullptr, nullptr, nullptr, scratch, scratch_bytes, grads,
                                stream);
}

PS_API int ps_raster_backward_loss(const ps_raster_desc *desc, const ps_raster_inputs *in, const ps_raster_state *state,
                                   const float *target, const float *grad_scale, void *scratch, size_t scratch_bytes,
                                   const ps_raster_grads *grads, void *stream) {
    if (!target || !grad_scale) { set_error("target / grad_scale is NULL"); return PS_ERR_INVALID_ARGUMENT; }
    return raster_backward_impl(desc, in, state, nullptr, target, grad_scale, nullptr, scratch, scratch_bytes, grads,
                                stream);
}

PS_API int ps_raster_backward_depth(const ps_raster_desc *desc, const ps_raster_inputs *in, const ps_raster_state *state,
                                    const float *d_color, const float *loss_target, const float *grad_scale,
                                    const float *d_depth, void *scratch, size_t scratch_bytes,
                                    const ps_raster_grads *grads, void *stream) {
    if (!d_depth) { set_error("d_depth is NULL"); return PS_ERR_INVALID_ARGUMENT; }
    if (desc && desc->depth_mode == PS_DEPTH_NONE) {
        set_error("ps_raster_backward_depth needs the depth_mode of a depth forward (got 0)");
        return PS_ERR_INVALID_ARGUMENT;
    }
    if (!d_color && !(loss_target && grad_scale)) { set_error("d_color, or loss_target + grad_scale, is NULL"); return PS_ERR_INVALID_ARGUMENT; }
    return raster_backward_impl(desc, in, state, d_color, d_color ? nullptr : loss_target, d_color ? nullptr : grad_scale,
                                d_depth, scratch, scratch_bytes, grads, stream);
}

}  // extern "C"
