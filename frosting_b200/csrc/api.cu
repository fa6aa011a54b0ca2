// api.cu -- the extern "C" boundary declared in include/frosting_b200.h.
//
// Mirrors, for this path, what DGR/rasterize_points.cu + CudaRasterizer::Rasterizer do for the
// reference: argument checks, workspace carving, kernel sequencing.  Differences by design:
// raw device pointers instead of torch tensors, an explicit stream, no allocation, no host
// synchronisation unless `debug` is set.
#include <atomic>
#include <mutex>
#include <cstdio>
#include <cstring>

#include "common.cuh"

using namespace fb200;

namespace {

thread_local char g_err[512] = "";

int fail(int code, const char* msg) {
    snprintf(g_err, sizeof(g_err), "%s", msg);
    return code;
}

int check(cudaError_t e, const char* what) {
    if (e == cudaSuccess) return FB200_OK;
    snprintf(g_err, sizeof(g_err), "CUDA error in %s: %s", what, cudaGetErrorString(e));
    return FB200_ECUDA;
}

// debug mode: synchronise after every stage like CHECK_CUDA (auxiliary.h:166-173)
int stage(cudaError_t e, const char* what, bool debug, cudaStream_t s) {
    int rc = check(e, what);
    if (rc != FB200_OK) return rc;
    if (debug) return check(cudaStreamSynchronize(s), what);
    return FB200_OK;
}

bool misaligned(const void* p, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) != 0; }

// fb200_frosting_params, for every entry point that reads it.  The alignment is what the kernels' vector accesses need
// (header: fb200_frosting_params): bary logits as float2, quats as float4, and the sh_rest rows moved as float4 blocks of
// a warp's 32 rows (frosting_attr.cu)
int check_frosting(const fb200_frosting_params* fp) {
    if (!fp) return fail(FB200_EINVAL, "frosting_attributes: null params");
    if (fp->P < 0 || fp->sh_rest < 0 || fp->n_verts < 0 || fp->n_faces < 0)
        return fail(FB200_EINVAL, "frosting_attributes: bad extents");
    if (fp->P > 0 && (!fp->d_bary_logits || !fp->d_cells || !fp->d_faces || !fp->d_inner_verts || !fp->d_outer_verts ||
                      !fp->d_opacity_logits || !fp->d_log_scales || !fp->d_quats || !fp->d_sh_dc ||
                      (fp->sh_rest > 0 && !fp->d_sh_rest)))
        return fail(FB200_EINVAL, "frosting_attributes: missing parameter pointer");
    if (fp->P > 0 && (misaligned(fp->d_bary_logits, 8) || misaligned(fp->d_quats, 16) ||
                      (fp->sh_rest > 0 && misaligned(fp->d_sh_rest, 16))))
        return fail(FB200_EINVAL, "frosting_attributes: bary logits must be 8-byte, quats and sh_rest 16-byte aligned");
    // background Gaussians
    if (fp->n_bg < 0) return fail(FB200_EINVAL, "frosting background: n_bg must be >= 0");
    if (fp->n_bg > 0 && (!fp->d_bg_points || !fp->d_bg_opacity_logits || !fp->d_bg_log_scales || !fp->d_bg_quats ||
                         !fp->d_bg_sh_dc || (fp->sh_rest > 0 && !fp->d_bg_sh_rest)))
        return fail(FB200_EINVAL, "frosting background: missing parameter pointer");
    if (fp->n_bg > 0 && misaligned(fp->d_bg_quats, 16))
        return fail(FB200_EINVAL, "frosting background: quats must be 16-byte aligned");
    return FB200_OK;
}

// fb200_frosting_grads over the block fp, for fb200_backward (frosting mode) and fb200_frosting_attributes_backward.
// Mesh rows (fp->P > 0): every parameter gradient, the shell's both or neither, each base 16-byte aligned (the
// attribute backward zero-fills a warp's rows with float4 stores and stores quats as float4).  Background rows: given
// exactly when there are background Gaussians, quats stored as float4.
int check_frosting_grads(const fb200_frosting_params* fp, const fb200_frosting_grads* g) {
    if (!g) return fail(FB200_EINVAL, "frosting gradients: null gradient block");
    if (fp->P > 0 && (!g->d_bary_logits || !g->d_opacity_logits || !g->d_log_scales || !g->d_quats || !g->d_sh_dc ||
                      (fp->sh_rest > 0 && !g->d_sh_rest) || ((g->d_inner_verts == nullptr) != (g->d_outer_verts == nullptr))))
        return fail(FB200_EINVAL, "frosting gradients: parameter-gradient pointers missing");
    if (fp->P > 0 && (misaligned(g->d_bary_logits, 16) || misaligned(g->d_opacity_logits, 16) ||
                      misaligned(g->d_log_scales, 16) || misaligned(g->d_quats, 16) || misaligned(g->d_sh_dc, 16) ||
                      (fp->sh_rest > 0 && misaligned(g->d_sh_rest, 16))))
        return fail(FB200_EINVAL, "frosting gradients: the mesh parameter gradients must be 16-byte aligned");
    const bool any = g->d_bg_points || g->d_bg_opacity_logits || g->d_bg_log_scales || g->d_bg_quats || g->d_bg_sh_dc ||
                     g->d_bg_sh_rest;
    if (any != (fp->n_bg > 0))
        return fail(FB200_EINVAL, "frosting background: give background gradients exactly when there are background "
                                  "Gaussians (n_bg > 0)");
    if (fp->n_bg > 0 && (!g->d_bg_points || !g->d_bg_opacity_logits || !g->d_bg_log_scales || !g->d_bg_quats ||
                         !g->d_bg_sh_dc || (fp->sh_rest > 0 && !g->d_bg_sh_rest)))
        return fail(FB200_EINVAL, "frosting background: gradient pointers missing");
    if (fp->n_bg > 0 && misaligned(g->d_bg_quats, 16))
        return fail(FB200_EINVAL, "frosting background: dL/dquats must be 16-byte aligned");
    return FB200_OK;
}

// frosting mode (fb200_inputs.frosting): the rasterizer's own inputs are derived from the parameter block
int validate_frosting(const fb200_params* prm, const fb200_inputs* in) {
    const fb200_frosting_params* fp = in->frosting;
    int rc = check_frosting(fp);
    if (rc != FB200_OK) return rc;
    if (in->d_means3D || in->d_shs || in->d_colors_precomp || in->d_opacities || in->d_scales || in->d_rotations ||
        in->d_cov3D_precomp || in->d_visibility || in->d_point_cells || in->d_face_visible)
        return fail(FB200_EINVAL, "frosting mode: the attribute / mask pointers of fb200_inputs must be NULL");
    if ((int64_t)fp->P + fp->n_bg != prm->P || prm->sh_coeffs != fp->sh_rest + 1 || fp->sh_rest > 15)
        return fail(FB200_EINVAL, "frosting mode: P / sh_coeffs do not match the parameter block (P = frosting->P + "
                                  "frosting->n_bg, sh_rest <= 15)");
    if (prm->sh_degree < 0 || prm->sh_degree > 3 || (prm->sh_degree + 1) * (prm->sh_degree + 1) > prm->sh_coeffs)
        return fail(FB200_EINVAL, "sh_degree / sh_coeffs inconsistent");
    if (prm->extra) return fail(FB200_EINVAL, "frosting mode: extra feature channels are not supported");
    return FB200_OK;
}

// the fb200_inputs the kernels see in frosting mode: culling inputs taken from the parameter block
fb200_inputs frosting_inputs(const fb200_inputs* in) {
    fb200_inputs r = *in;
    const fb200_frosting_params* fp = in->frosting;
    r.d_visibility = fp->d_mask;
    if (fp->d_face_visible) { r.d_point_cells = fp->d_cells; r.d_face_visible = fp->d_face_visible; r.n_cell_points = fp->P; }
    r.frosting = nullptr;     // a host pointer: never dereferenced on the device
    return r;
}

int validate(const fb200_params* prm, const fb200_inputs* in, const fb200_workspace* ws) {
    if (!prm || !in || !ws) return fail(FB200_EINVAL, "null argument struct");
    if (prm->P < 0 || prm->image_width <= 0 || prm->image_height <= 0)
        return fail(FB200_EINVAL, "bad extents (P >= 0, image dims > 0 required)");
    if (prm->image_width > 65535 * FB200_TILE || prm->image_height > 65535 * FB200_TILE)
        return fail(FB200_EINVAL, "image too large for 16-bit tile coordinates");
    if (prm->debug & ~3)
        return fail(FB200_EINVAL, "debug: only bits 0 (synchronise) and 1 (no sub-tile culling) are defined");
    if (in->frosting) {
        int rc = validate_frosting(prm, in);
        if (rc != FB200_OK) return rc;
    } else if (prm->P > 0) {
        if (!in->d_means3D || !in->d_opacities) return fail(FB200_EINVAL, "means3D / opacities missing");
        const bool has_sh = in->d_shs != nullptr, has_col = in->d_colors_precomp != nullptr;
        if (has_sh == has_col)
            return fail(FB200_EINVAL, "Please provide excatly one of either SHs or precomputed colors!");
        const bool has_sr = in->d_scales != nullptr && in->d_rotations != nullptr;
        const bool any_sr = in->d_scales != nullptr || in->d_rotations != nullptr;
        const bool has_cov = in->d_cov3D_precomp != nullptr;
        if ((!has_sr && !has_cov) || (any_sr && has_cov))
            return fail(FB200_EINVAL,
                        "Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!");
        if (has_sh && (prm->sh_coeffs <= 0 || prm->sh_degree < 0 || prm->sh_degree > 3 ||
                       (prm->sh_degree + 1) * (prm->sh_degree + 1) > prm->sh_coeffs))
            return fail(FB200_EINVAL, "sh_degree / sh_coeffs inconsistent");
        // rows read with 128-bit loads (header: Alignment)
        if (misaligned(in->d_rotations, 16) || (has_sh && (prm->sh_coeffs * 3) % 4 == 0 && misaligned(in->d_shs, 16)))
            return fail(FB200_EINVAL, "rotations / SH rows must be 16-byte aligned");
        if ((in->d_point_cells == nullptr) != (in->d_face_visible == nullptr))
            return fail(FB200_EINVAL, "give both d_point_cells and d_face_visible or neither");
        if (in->d_point_cells && (in->n_cell_points < 0 || in->n_cell_points > prm->P))
            return fail(FB200_EINVAL, "n_cell_points must be within [0, P]");
    }
    if (!in->d_background || !in->d_viewmatrix || !in->d_projmatrix || !in->d_campos)
        return fail(FB200_EINVAL, "camera tensors missing");
    if (!ws->d_geom || !ws->d_image || !ws->d_status) return fail(FB200_EINVAL, "workspace pointers missing");
    if (ws->binning_capacity > 0 && !ws->d_binning) return fail(FB200_EINVAL, "binning buffer missing");
    if (ws->binning_capacity < 0 || ws->binning_capacity > 0x7fffffffLL)
        return fail(FB200_EINVAL, "binning capacity out of range");
    return FB200_OK;
}

inline char* align128(void* p) {
    return reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(p) + 127) & ~uintptr_t(127));
}

// p = the sub-array at byte offset `off` of a 128-byte aligned workspace base; NULL when there is no such workspace
template <typename T>
void carve(T*& p, char* base, size_t off) { p = base ? reinterpret_cast<T*>(base + off) : nullptr; }

// One frame's arguments: checks them and the workspace sizes, then fills the header the kernels read and carves the
// three workspaces into every sub-array pointer (GeomLayout, ImageLayout, BinLayout from 128-byte aligned bases).
// `a` is value-initialised by the caller.
int carve_frame(const fb200_params* prm, const fb200_inputs* in, const fb200_workspace* ws, FrameArgs& a) {
    int rc = validate(prm, in, ws);
    if (rc != FB200_OK) return rc;
    const GeomLayout gl((size_t)prm->P);
    const ImageLayout il(prm->image_width, prm->image_height);
    const BinLayout bl((size_t)ws->binning_capacity);
    if (ws->geom_bytes < gl.total) return fail(FB200_ENOSPC, "geometry workspace too small");
    if (ws->image_bytes < il.total) return fail(FB200_ENOSPC, "image workspace too small");
    if (ws->binning_capacity > 0 && ws->binning_bytes < bl.total)
        return fail(FB200_ENOSPC, "binning workspace too small");
    a.prm = *prm;
    a.in = *in;
    if (in->frosting) { a.frosting = 1; a.fr = *in->frosting; a.in = frosting_inputs(in); }
    // focal lengths exactly as rasterizer_impl.cu:222-223
    a.focal_y = prm->image_height / (2.0f * prm->tanfovy);
    a.focal_x = prm->image_width / (2.0f * prm->tanfovx);
    a.tiles_x = il.tiles_x; a.tiles_y = il.tiles_y;
    char* g = align128(ws->d_geom);
    carve(a.rec, g, gl.rec); carve(a.depth, g, gl.depth); carve(a.rect, g, gl.rect);
    carve(a.clamped, g, gl.clamped); carve(a.acc, g, gl.acc); carve(a.vis_list, g, gl.vis_list);
    char* im = align128(ws->d_image);
    carve(a.final_T, im, il.final_T); carve(a.n_contrib, im, il.n_contrib); carve(a.last_entry, im, il.last_entry);
    carve(a.ranges, im, il.ranges); carve(a.tile_count, im, il.tile_count); carve(a.cursor, im, il.cursor);
    carve(a.list_tiny, im, il.list_tiny); carve(a.list_small, im, il.list_small);
    carve(a.list_large, im, il.list_large); carve(a.list_huge, im, il.list_huge);
    carve(a.tile_order, im, il.tile_order); carve(a.counters, im, il.counters);
    char* bn = align128(ws->d_binning);      // NULL without a binning buffer
    carve(a.point_list, bn, bl.point_list); carve(a.keys, bn, bl.keys); carve(a.keys_scratch, bn, bl.keys_scratch);
    carve(a.sub_hits, bn, bl.sub_hits);
    a.capacity = ws->binning_capacity;
    a.status = ws->d_status;
    return FB200_OK;
}

// row f4: copy the caller's extra-channel block into kernel arguments
int setup_extra(const fb200_params* prm, bool forward, bool backward, ExtraArgs& ex) {
    memset(&ex, 0, sizeof(ex));
    const fb200_extra* e = prm->extra;
    if (!e || prm->P == 0) return FB200_OK;
    if (e->channels < 1 || e->channels > FB200_CHANNELS)
        return fail(FB200_EINVAL, "extra feature channels must be 1..3");
    if (!e->d_features || !e->d_background) return fail(FB200_EINVAL, "extra features / background missing");
    if (forward && !e->d_out) return fail(FB200_EINVAL, "extra output image missing");
    if (backward && (!e->d_dL_dout || !e->d_dL_dfeatures)) return fail(FB200_EINVAL, "extra gradient pointers missing");
    ex.ch = e->channels; ex.feat = e->d_features; ex.bg = e->d_background; ex.out = e->d_out;
    ex.dL_dout = e->d_dL_dout; ex.dL_dfeat = e->d_dL_dfeatures;
    return FB200_OK;
}

// ---- measurement hooks -------------------------------------------------------------------------------
std::atomic<long long> g_launches{0};
std::atomic<int> g_profile{0};
// Process-wide (not thread-local): torch's autograd engine calls fb200_backward from its own thread.
struct StageEvents {
    cudaEvent_t ev[FB200_NUM_STAGES][2];
    bool made = false;
    bool recorded[FB200_NUM_STAGES] = {};
};
StageEvents g_ev;
std::mutex g_ev_mu;

struct StageTimer {
    int stage;
    cudaStream_t s;
    bool on;
    StageTimer(int st, cudaStream_t stream) : stage(st), s(stream), on(g_profile.load() != 0) {
        if (!on) return;
        std::lock_guard<std::mutex> lk(g_ev_mu);
        if (!g_ev.made) {
            for (int i = 0; i < FB200_NUM_STAGES; ++i) { cudaEventCreate(&g_ev.ev[i][0]); cudaEventCreate(&g_ev.ev[i][1]); }
            g_ev.made = true;
        }
        cudaEventRecord(g_ev.ev[stage][0], s);
    }
    ~StageTimer() {
        if (!on) return;
        std::lock_guard<std::mutex> lk(g_ev_mu);
        cudaEventRecord(g_ev.ev[stage][1], s);
        g_ev.recorded[stage] = true;
    }
};

}  // namespace

namespace fb200 {
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int sm_count() {
    static std::atomic<int> cache[64];
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) dev = 0;
    int n = cache[dev].load(std::memory_order_relaxed);
    if (n <= 0) {
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 1;
        cache[dev].store(n, std::memory_order_relaxed);
    }
    return n;
}
}  // namespace fb200

extern "C" {

int fb200_profile_enable(int32_t enable) { g_profile.store(enable ? 1 : 0); return FB200_OK; }

int fb200_profile_read(float* ms_out) {
    if (!ms_out) return fail(FB200_EINVAL, "profile_read: null output");
    std::lock_guard<std::mutex> lk(g_ev_mu);
    for (int i = 0; i < FB200_NUM_STAGES; ++i) {
        ms_out[i] = -1.0f;
        if (g_ev.made && g_ev.recorded[i]) {
            cudaError_t e = cudaEventSynchronize(g_ev.ev[i][1]);
            if (e != cudaSuccess) return check(e, "profile_read");
            e = cudaEventElapsedTime(&ms_out[i], g_ev.ev[i][0], g_ev.ev[i][1]);
            if (e != cudaSuccess) return check(e, "profile_read");
        }
    }
    return FB200_OK;
}

int64_t fb200_kernel_launches(void) { return g_launches.load(); }

int fb200_abi_version(void) { return FB200_ABI_VERSION; }

int fb200_abi_struct_sizes(size_t* out) {
    if (!out) return fail(FB200_EINVAL, "abi_struct_sizes: null output");
    const size_t sizes[FB200_ABI_STRUCTS] = {sizeof(fb200_params), sizeof(fb200_inputs), sizeof(fb200_workspace),
                                             sizeof(fb200_grads), sizeof(fb200_extra), sizeof(fb200_frosting_params),
                                             sizeof(fb200_frosting_grads), sizeof(fb200_adam_args), sizeof(fb200_layout),
                                             sizeof(fb200_frosting_edit), sizeof(fb200_frosting_skin),
                                             sizeof(fb200_texture), sizeof(fb200_sugar_reg)};
    for (int i = 0; i < FB200_ABI_STRUCTS; ++i) out[i] = sizes[i];
    return FB200_OK;
}
const char* fb200_last_error(void) { return g_err; }

size_t fb200_geom_bytes(int32_t P) { return GeomLayout((size_t)(P < 0 ? 0 : P)).total; }
size_t fb200_image_bytes(int32_t W, int32_t H) { return ImageLayout(W < 1 ? 1 : W, H < 1 ? 1 : H).total; }
size_t fb200_binning_bytes(int64_t capacity) { return BinLayout((size_t)(capacity < 0 ? 0 : capacity)).total; }

int fb200_get_layout(int32_t P, int32_t W, int32_t H, int64_t capacity, fb200_layout* out) {
    if (!out || P < 0 || W <= 0 || H <= 0 || capacity < 0) return fail(FB200_EINVAL, "bad layout query");
    const GeomLayout gl((size_t)P);
    const ImageLayout il(W, H);
    const BinLayout bl((size_t)capacity);
    out->geom_rec = gl.rec; out->geom_depth = gl.depth; out->geom_rect = gl.rect; out->geom_clamped = gl.clamped;
    out->img_final_T = il.final_T; out->img_n_contrib = il.n_contrib; out->img_ranges = il.ranges;
    out->img_tile_count = il.tile_count;
    out->bin_point_list = bl.point_list; out->bin_keys = bl.keys;
    out->geom_acc = gl.acc;
    out->img_last_entry = il.last_entry; out->bin_sub_hits = bl.sub_hits;
    return FB200_OK;
}

static int setup_fwd(const fb200_params* prm, const fb200_inputs* in, const fb200_workspace* ws, bool need_binning,
                     float* d_out_color, int32_t* d_radii, FwdArgs& a) {
    int rc = carve_frame(prm, in, ws, a);
    if (rc != FB200_OK) return rc;
    if (prm->P > 0 && !d_radii) return fail(FB200_EINVAL, "output pointers missing");
    if (need_binning && !d_out_color) return fail(FB200_EINVAL, "output pointers missing");
    a.out_color = d_out_color;
    a.radii = d_radii;
    return FB200_OK;
}

int fb200_forward_geometry(const fb200_params* prm, const fb200_inputs* in, const fb200_workspace* ws,
                           int32_t* d_radii, void* stream) {
    FwdArgs a{};
    int rc = setup_fwd(prm, in, ws, false, nullptr, d_radii, a);
    if (rc != FB200_OK) return rc;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const bool debug = (prm->debug & 1) != 0;
    { StageTimer t(FB200_STAGE_PREPROCESS, s);
      if ((rc = stage(launch_preprocess_fwd(a, s), "preprocess", debug, s)) != FB200_OK) return rc;
      if ((rc = stage(launch_tile_scan(a, s), "tile scan", debug, s)) != FB200_OK) return rc; }
    if (ws->acc_zeroed_by_forward && prm->P > 0) {
        // backward's accumulators: cleared here, in the shadow of the host's wait for the instance count
        if ((rc = stage(cudaMemsetAsync(a.acc, 0, sizeof(float) * 12 * (size_t)prm->P, s), "accumulator clear", debug, s)) != FB200_OK)
            return rc;
    }
    return FB200_OK;
}

int fb200_forward_raster(const fb200_params* prm, const fb200_inputs* in, const fb200_workspace* ws,
                         float* d_out_color, int32_t* d_radii, void* stream) {
    FwdArgs a{};
    int rc = setup_fwd(prm, in, ws, true, d_out_color, d_radii, a);
    if (rc != FB200_OK) return rc;
    if ((rc = setup_extra(prm, true, false, a.ex)) != FB200_OK) return rc;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const bool debug = (prm->debug & 1) != 0;
    { StageTimer t(FB200_STAGE_BINNING, s);
      if ((rc = stage(launch_binning(a, s, ws->h_status), "binning", debug, s)) != FB200_OK) return rc; }
    { StageTimer t(FB200_STAGE_RENDER_FWD, s);
      if ((rc = stage(launch_render_fwd(a, s), "render", debug, s)) != FB200_OK) return rc; }
    return FB200_OK;
}

int fb200_forward(const fb200_params* prm, const fb200_inputs* in, const fb200_workspace* ws,
                  float* d_out_color, int32_t* d_radii, void* stream) {
    int rc = fb200_forward_geometry(prm, in, ws, d_radii, stream);
    if (rc != FB200_OK) return rc;
    if (!ws) return fail(FB200_EINVAL, "null argument struct");
    fb200_workspace one_phase = *ws;
    one_phase.h_status = nullptr;      // nobody has synchronised: the host cannot know this frame's status words
    return fb200_forward_raster(prm, in, &one_phase, d_out_color, d_radii, stream);
}

int fb200_backward(const fb200_params* prm, const fb200_inputs* in, const fb200_workspace* ws,
                   const int32_t* d_radii, const float* d_dL_dout_color, const fb200_grads* grads, void* stream) {
    BwdArgs a{};
    int rc = carve_frame(prm, in, ws, a);
    if (rc != FB200_OK) return rc;
    if (!grads || !d_dL_dout_color || (prm->P > 0 && !d_radii)) return fail(FB200_EINVAL, "backward pointers missing");
    // outputs a caller cannot use may be NULL and are then not written: dL/dcolors on the SH path (an intermediate
    // there), dL/dcov3D on the scale/rotation path, dL/dscales + dL/drotations on the precomputed-covariance path
    const fb200_frosting_grads* fg = grads->frosting;
    if (in->frosting) {
        if ((rc = check_frosting_grads(in->frosting, fg)) != FB200_OK) return rc;
    } else if (fg) {
        return fail(FB200_EINVAL, "fb200_grads.frosting given without fb200_inputs.frosting");
    } else if (prm->P > 0 && (!grads->d_dL_dmeans2D || !grads->d_dL_dopacity || !grads->d_dL_dmeans3D ||
                       (in->d_colors_precomp && !grads->d_dL_dcolors) || (in->d_cov3D_precomp && !grads->d_dL_dcov3D) ||
                       (!in->d_cov3D_precomp && (!grads->d_dL_dscales || !grads->d_dL_drotations)) ||
                       (in->d_shs && prm->sh_coeffs > 0 && !grads->d_dL_dsh)))
        return fail(FB200_EINVAL, "gradient output pointers missing");
    if (misaligned(grads->d_dL_drotations, 16) || ((prm->sh_coeffs * 3) % 4 == 0 && misaligned(grads->d_dL_dsh, 16)))
        return fail(FB200_EINVAL, "dL/drotations / dL/dsh rows must be 16-byte aligned");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const bool debug = (prm->debug & 1) != 0;
    if (prm->P == 0) return FB200_OK;

    if (in->frosting) a.fg = *fg;
    a.radii = d_radii;
    a.dL_dpix = d_dL_dout_color;
    a.g = *grads;
    if ((rc = setup_extra(prm, false, true, a.ex)) != FB200_OK) return rc;

    if (!ws->acc_zeroed_by_forward &&
        (rc = stage(launch_render_bwd_clear(a, s), "render backward (clear)", debug, s)) != FB200_OK) return rc;
    { StageTimer t(FB200_STAGE_RENDER_BWD, s);
      if ((rc = stage(launch_render_bwd(a, s), "render backward", debug, s)) != FB200_OK) return rc; }
    { StageTimer t(FB200_STAGE_GEOM_BWD, s);
      if ((rc = stage(launch_geom_bwd(a, s), "geometry backward", debug, s)) != FB200_OK) return rc; }
    if ((rc = stage(launch_extra_grad(a, s), "extra feature gradients", debug, s)) != FB200_OK) return rc;
    return FB200_OK;
}

int fb200_mark_visible(int32_t P, const float* d_means3D, const float* d_viewmatrix, const float* d_projmatrix,
                       uint8_t* d_present, void* stream) {
    (void)d_projmatrix;   // the reference's x/y frustum test is commented out (auxiliary.h:154)
    if (P < 0 || (P > 0 && (!d_means3D || !d_viewmatrix || !d_present)))
        return fail(FB200_EINVAL, "mark_visible: bad arguments");
    return check(launch_mark_visible(P, d_means3D, d_viewmatrix, d_present, static_cast<cudaStream_t>(stream)),
                 "mark_visible");
}

int fb200_mesh_visibility(int32_t V, int32_t F, const float* d_verts, const int32_t* d_faces,
                          const float* d_full_proj, int32_t W, int32_t H, uint64_t* d_zbuf,
                          int32_t* d_pix_to_face, uint8_t* d_face_visible, int32_t mark_last_on_bg,
                          int32_t* d_scratch, void* stream) {
    if (V < 0 || F < 0 || W <= 0 || H <= 0 || !d_full_proj || !d_zbuf || !d_pix_to_face ||
        (F > 0 && (!d_verts || !d_faces)))
        return fail(FB200_EINVAL, "mesh_visibility: bad arguments");
    return check(launch_mesh_visibility(V, F, d_verts, d_faces, d_full_proj, W, H,
                                        reinterpret_cast<unsigned long long*>(d_zbuf), d_pix_to_face,
                                        d_face_visible, mark_last_on_bg, d_scratch, static_cast<cudaStream_t>(stream)),
                 "mesh_visibility");
}

int fb200_gaussian_mask_from_faces(int32_t n_points, const int64_t* d_point_cell_indices, int32_t F,
                                   const uint8_t* d_face_visible, int32_t n_background, uint8_t* d_mask,
                                   void* stream) {
    if (n_points < 0 || n_background < 0 || F < 0 || (n_points > 0 && (!d_point_cell_indices || !d_face_visible)) ||
        (n_points + n_background > 0 && !d_mask))
        return fail(FB200_EINVAL, "gaussian_mask_from_faces: bad arguments");
    return check(launch_mask_from_faces(n_points, reinterpret_cast<const long long*>(d_point_cell_indices), F,
                                        d_face_visible, n_background, d_mask, static_cast<cudaStream_t>(stream)),
                 "gaussian_mask_from_faces");
}

int fb200_frosting_attributes(const fb200_frosting_params* fp, float* d_means3D, float* d_opacities, float* d_scales,
                              float* d_rotations, float* d_shs, void* stream) {
    int rc = check_frosting(fp);
    if (rc != FB200_OK) return rc;
    const bool rows = (int64_t)fp->P + fp->n_bg > 0;
    if (rows && (!d_means3D || !d_opacities || !d_scales || !d_rotations || !d_shs))
        return fail(FB200_EINVAL, "frosting_attributes: missing output pointer");
    // mesh rows of 16 SH coefficients are stored as twelve float4
    if (fp->P > 0 && fp->sh_rest == 15 && misaligned(d_shs, 16))
        return fail(FB200_EINVAL, "frosting_attributes: shs must be 16-byte aligned when sh_rest == 15");
    if (rows && misaligned(d_rotations, 16))
        return fail(FB200_EINVAL, "frosting_attributes: rotations must be 16-byte aligned");
    return check(launch_frosting_attr_fwd(*fp, d_means3D, d_opacities, d_scales, d_rotations, d_shs,
                                          static_cast<cudaStream_t>(stream)), "frosting_attributes");
}

int fb200_frosting_attributes_backward(const fb200_frosting_params* fp, const float* d_g_means3D,
                                       const float* d_g_opacities, const float* d_g_scales,
                                       const float* d_g_rotations, const float* d_g_shs,
                                       const fb200_frosting_grads* grads, void* stream) {
    int rc = check_frosting(fp);
    if (rc != FB200_OK) return rc;
    if ((rc = check_frosting_grads(fp, grads)) != FB200_OK) return rc;
    const bool rows = (int64_t)fp->P + fp->n_bg > 0;
    if (rows && (!d_g_means3D || !d_g_opacities || !d_g_scales || !d_g_rotations || !d_g_shs))
        return fail(FB200_EINVAL, "frosting_attributes_backward: missing upstream gradient pointer");
    // mesh rows of 16 SH coefficients are read as twelve float4
    if (fp->P > 0 && fp->sh_rest == 15 && misaligned(d_g_shs, 16))
        return fail(FB200_EINVAL, "frosting_attributes_backward: dL/dshs must be 16-byte aligned when sh_rest == 15");
    if (rows && misaligned(d_g_rotations, 16))
        return fail(FB200_EINVAL, "frosting_attributes_backward: dL/drotations must be 16-byte aligned");
    return check(launch_frosting_attr_bwd(*fp, d_g_means3D, d_g_opacities, d_g_scales, d_g_rotations, d_g_shs, *grads,
                                          static_cast<cudaStream_t>(stream)), "frosting_attributes_backward");
}

static int check_edit(const fb200_frosting_edit* e) {
    if (!e) return fail(FB200_EINVAL, "frosting_edit: null edit struct");
    if (e->n_verts < 0 || e->n_faces < 0 || e->n_edited < 0 || e->n_edited > e->n_faces)
        return fail(FB200_EINVAL, "frosting_edit: bad extents");
    if (e->rescaling != FB200_RESCALE_MEDIAN && e->rescaling != FB200_RESCALE_TRIANGLE)
        return fail(FB200_EINVAL, "frosting_edit: unknown thickness rescaling method (median = 0, triangle = 1)");
    if (e->n_faces > 0 && (!e->d_base_verts || !e->d_faces || !e->d_edition_mask || !e->d_dists || !e->d_face_normals ||
                           !e->d_rel_quats || !e->d_face_factor || !e->d_face_keep))
        return fail(FB200_EINVAL, "frosting_edit: missing face table pointer");
    if (e->n_verts > 0 && (!e->d_inner_dist || !e->d_outer_dist || !e->d_verts_edition_mask || !e->d_vf_offsets ||
                           !e->d_vf_faces || !e->d_inner_verts || !e->d_outer_verts))
        return fail(FB200_EINVAL, "frosting_edit: missing vertex table pointer");
    if (!e->d_factor || !e->d_select) return fail(FB200_EINVAL, "frosting_edit: missing factor / select scratch");
    const bool capture = !e->d_ref_quats && !e->d_ref_dists && !e->d_ref_median;
    if (!capture && (!e->d_ref_quats || !e->d_ref_dists || (e->rescaling == FB200_RESCALE_MEDIAN && !e->d_ref_median)))
        return fail(FB200_EINVAL, "frosting_edit: give every reference table (or none to capture one)");
    if (misaligned(e->d_rel_quats, 16) || misaligned(e->d_ref_quats, 16))
        return fail(FB200_EINVAL, "frosting_edit: quaternion tables must be 16-byte aligned");
    return FB200_OK;
}

int fb200_frosting_edit_shell(const fb200_frosting_edit* e, void* stream) {
    int rc = check_edit(e);
    if (rc != FB200_OK) return rc;
    if (e->rescaling == FB200_RESCALE_MEDIAN && e->n_edited == 0)
        return fail(FB200_EINVAL, "frosting_edit: median rescaling needs at least one edited face");
    return check(launch_frosting_edit_shell(*e, static_cast<cudaStream_t>(stream)), "frosting_edit_shell");
}

// an edit and the parameter block it adapts: each valid, over the same base mesh
static int check_edit_block(const fb200_frosting_edit* e, const fb200_frosting_params* fp) {
    int rc = check_edit(e);
    if (rc != FB200_OK) return rc;
    if ((rc = check_frosting(fp)) != FB200_OK) return rc;
    if (fp->n_faces != e->n_faces || fp->n_verts != e->n_verts)
        return fail(FB200_EINVAL, "frosting_edit: the parameter block's mesh does not match the edit's");
    return FB200_OK;
}

static int check_edit_attributes(const fb200_frosting_edit* e, const fb200_frosting_params* fp, int32_t sh_degree,
                                 const float* d_campos, const float* d_orig_quats, float* d_means3D,
                                 float* d_opacities, float* d_scales, float* d_rotations, float* d_colors) {
    int rc = check_edit_block(e, fp);
    if (rc != FB200_OK) return rc;
    if (sh_degree < 0 || sh_degree > 3 || (sh_degree + 1) * (sh_degree + 1) > fp->sh_rest + 1)
        return fail(FB200_EINVAL, "frosting_edit: sh_degree needs (sh_degree + 1)^2 <= sh_rest + 1 <= 16");
    const bool rows = (int64_t)fp->P + fp->n_bg > 0;
    if (rows && (!d_campos || !d_means3D || !d_opacities || !d_scales || !d_rotations || !d_colors))
        return fail(FB200_EINVAL, "frosting_edit: missing output pointer");
    if (misaligned(d_rotations, 16) || misaligned(d_orig_quats, 16))
        return fail(FB200_EINVAL, "frosting_edit: rotations / orig quats must be 16-byte aligned");
    return FB200_OK;
}

int fb200_frosting_edit_attributes(const fb200_frosting_edit* e, const fb200_frosting_params* fp, int32_t sh_degree,
                                   const float* d_campos, const float* d_orig_quats, float* d_means3D,
                                   float* d_opacities, float* d_scales, float* d_rotations, float* d_colors,
                                   void* stream) {
    const int rc = check_edit_attributes(e, fp, sh_degree, d_campos, d_orig_quats, d_means3D, d_opacities, d_scales,
                                         d_rotations, d_colors);
    if (rc != FB200_OK) return rc;
    return check(launch_frosting_edit_attr(*e, *fp, sh_degree, d_campos, d_orig_quats, d_means3D, d_opacities, d_scales,
                                           d_rotations, d_colors, static_cast<cudaStream_t>(stream)),
                 "frosting_edit_attributes");
}

// the complex adaptation's tables: [F,9] cell transforms when a face is edited, [P,9] canonical transforms
static int check_edit_complex(const fb200_frosting_edit* e, const fb200_frosting_params* fp, const float* d_cell_T,
                              const float* d_canonical) {
    if (e->n_edited > 0 && !d_cell_T) return fail(FB200_EINVAL, "frosting_edit_complex: missing cell transforms");
    if (fp->P > 0 && !d_canonical) return fail(FB200_EINVAL, "frosting_edit_complex: missing canonical transforms");
    return FB200_OK;
}

int fb200_frosting_edit_complex_capture(const fb200_frosting_edit* e, const fb200_frosting_params* fp, float* d_cell_T,
                                        float* d_canonical, uint32_t* d_n_singular, void* stream) {
    int rc = check_edit_block(e, fp);
    if (rc != FB200_OK) return rc;
    if ((rc = check_edit_complex(e, fp, d_cell_T, d_canonical)) != FB200_OK) return rc;
    if (!d_n_singular) return fail(FB200_EINVAL, "frosting_edit_complex: missing singular-cell counter");
    return check(launch_frosting_edit_complex_capture(*e, *fp, d_cell_T, d_canonical, d_n_singular,
                                                      static_cast<cudaStream_t>(stream)),
                 "frosting_edit_complex_capture");
}

int fb200_frosting_edit_attributes_complex(const fb200_frosting_edit* e, const fb200_frosting_params* fp,
                                           int32_t sh_degree, const float* d_campos, const float* d_orig_quats,
                                           const float* d_canonical, float* d_cell_T, float* d_means3D,
                                           float* d_opacities, float* d_scales, float* d_rotations, float* d_colors,
                                           void* stream) {
    int rc = check_edit_attributes(e, fp, sh_degree, d_campos, d_orig_quats, d_means3D, d_opacities, d_scales,
                                   d_rotations, d_colors);
    if (rc != FB200_OK) return rc;
    if ((rc = check_edit_complex(e, fp, d_cell_T, d_canonical)) != FB200_OK) return rc;
    return check(launch_frosting_edit_attr_complex(*e, *fp, sh_degree, d_campos, d_orig_quats, d_canonical, d_cell_T,
                                                   d_means3D, d_opacities, d_scales, d_rotations, d_colors,
                                                   static_cast<cudaStream_t>(stream)),
                 "frosting_edit_attributes_complex");
}

int fb200_frosting_skin_pose(const fb200_frosting_skin* s, int32_t frame, float* d_base_verts, void* stream) {
    if (!s) return fail(FB200_EINVAL, "frosting_skin: null skin struct");
    if (s->n_rows < 0 || s->n_verts < 0 || s->n_bones < 0 || s->n_frames < 0 || s->n_rows > s->n_verts)
        return fail(FB200_EINVAL, "frosting_skin: bad extents");
    if (frame < 0 || frame >= s->n_frames)
        return fail(FB200_EINVAL, "frosting_skin: frame outside [0, n_frames)");
    if (s->n_rows > 0 && (!s->d_tpose || !s->d_vert_ids || !s->d_offsets || !d_base_verts))
        return fail(FB200_EINVAL, "frosting_skin: missing vertex table pointer");
    if (s->n_rows > 0 && s->n_bones > 0 && (!s->d_bones || !s->d_weights || !s->d_reset || !s->d_pose))
        return fail(FB200_EINVAL, "frosting_skin: missing bone table pointer");
    if (misaligned(s->d_reset, 16) || misaligned(s->d_pose, 16))
        return fail(FB200_EINVAL, "frosting_skin: reset / pose matrices must be 16-byte aligned");
    if (s->n_rows == 0) return FB200_OK;
    return check(launch_frosting_skin(*s, frame, d_base_verts, static_cast<cudaStream_t>(stream)),
                 "frosting_skin_pose");
}

int fb200_mesh_barycentrics(int32_t V, int32_t F, const float* d_verts, const int32_t* d_faces,
                            const float* d_full_proj, int32_t W, int32_t H, const int32_t* d_pix_to_face,
                            float* d_bary, void* stream) {
    if (V < 0 || F < 0 || W <= 0 || H <= 0 || (int64_t)W * H > INT32_MAX || !d_full_proj || !d_pix_to_face ||
        !d_bary || (F > 0 && (!d_verts || !d_faces)))
        return fail(FB200_EINVAL, "mesh_barycentrics: bad arguments");
    return check(launch_mesh_bary(F, d_verts, d_faces, d_full_proj, W, H, d_pix_to_face, d_bary,
                                  static_cast<cudaStream_t>(stream)),
                 "mesh_barycentrics");
}

namespace {

int check_texture(const fb200_texture* t) {
    if (!t) return fail(FB200_EINVAL, "texture: null texture struct");
    const int64_t n = t->n_square_per_axis;
    if (t->n_faces < 1 || t->n_points < 0 || t->square_size < 3 || n < 1 || 2 * n * n < t->n_faces ||
        (int64_t)t->square_size * n != t->texture_size || (int64_t)t->texture_size * t->texture_size > INT32_MAX)
        return fail(FB200_EINVAL, "texture: bad extents (F >= 1, square_size >= 3, 2 n^2 >= F, T = square_size n)");
    if (!t->d_cell_offsets || (t->n_points > 0 && (!t->d_cell_points || !t->d_sh_dc)) || !t->d_face_sh)
        return fail(FB200_EINVAL, "texture: missing face table pointer");
    if (!t->d_face_acc || !t->d_texel_acc || !t->d_face_winner || !t->d_texel_winner)
        return fail(FB200_EINVAL, "texture: missing accumulator / winner pointer");
    if (misaligned(t->d_face_acc, 16) || misaligned(t->d_texel_acc, 16))
        return fail(FB200_EINVAL, "texture: accumulators must be 16-byte aligned");
    return FB200_OK;
}

}  // namespace

int fb200_texture_face_sh_colours(const fb200_texture* t, void* stream) {
    int rc = check_texture(t);
    if (rc != FB200_OK) return rc;
    return check(launch_texture_face_sh(*t, static_cast<cudaStream_t>(stream)), "texture_face_sh_colours");
}

int fb200_texture_add_view(const fb200_texture* t, const float* d_image, const int32_t* d_pix_to_face,
                           const float* d_bary, int32_t W, int32_t H, void* stream) {
    int rc = check_texture(t);
    if (rc != FB200_OK) return rc;
    if (W <= 0 || H <= 0 || (int64_t)W * H > INT32_MAX || !d_image || !d_pix_to_face || !d_bary)
        return fail(FB200_EINVAL, "texture_add_view: bad arguments");
    return check(launch_texture_add_view(*t, d_image, d_pix_to_face, d_bary, W * H, static_cast<cudaStream_t>(stream)),
                 "texture_add_view");
}

int fb200_texture_finish(const fb200_texture* t, float* d_texture, void* stream) {
    int rc = check_texture(t);
    if (rc != FB200_OK) return rc;
    if (!d_texture) return fail(FB200_EINVAL, "texture_finish: missing output");
    return check(launch_texture_fill(*t, d_texture, static_cast<cudaStream_t>(stream)), "texture_finish");
}

size_t fb200_loss_partials(int32_t C, int32_t H, int32_t W) {
    return (C > 0 && H > 0 && W > 0) ? l1_dssim_num_partials(C, H, W) : 0;
}

int fb200_l1_dssim_forward(const float* d_pred, const float* d_gt, int32_t C, int32_t H, int32_t W, float lambda,
                           float* d_maps, float* d_partials, float* d_loss, void* stream) {
    if (C <= 0 || H <= 0 || W <= 0 || !d_pred || !d_gt || !d_maps || !d_partials || !d_loss)
        return fail(FB200_EINVAL, "l1_dssim_forward: bad arguments");
    return check(launch_l1_dssim_fwd(d_pred, d_gt, C, H, W, lambda, d_maps, d_partials, d_loss,
                                     static_cast<cudaStream_t>(stream)), "l1_dssim_forward");
}

int fb200_l1_dssim_backward(const float* d_pred, const float* d_gt, const float* d_maps, int32_t C, int32_t H,
                            int32_t W, float lambda, const float* d_dL_dloss, float* d_dpred, void* stream) {
    if (C <= 0 || H <= 0 || W <= 0 || !d_pred || !d_gt || !d_maps || !d_dL_dloss || !d_dpred)
        return fail(FB200_EINVAL, "l1_dssim_backward: bad arguments");
    return check(launch_l1_dssim_bwd(d_pred, d_gt, d_maps, C, H, W, lambda, d_dL_dloss, d_dpred,
                                     static_cast<cudaStream_t>(stream)), "l1_dssim_backward");
}

size_t fb200_sugar_reg_workspace_bytes(int32_t P, int32_t K, int32_t N, int32_t with_grad) {
    return (P >= 0 && K >= 1 && K <= 32 && N >= 0) ? sugar_reg_workspace_bytes(P, K, N, with_grad != 0) : 0;
}

static int check_sugar_reg(const fb200_sugar_reg* r) {
    if (!r) return fail(FB200_EINVAL, "sugar_reg: null struct");
    if (r->P < 0 || r->N < 0 || (r->N > 0 && r->P == 0))
        return fail(FB200_EINVAL, "sugar_reg: bad extents (P >= 0, N >= 0, P > 0 when N > 0)");
    if (r->K < 1 || r->K > 32) return fail(FB200_EINVAL, "sugar_reg: K must be within [1, 32]");
    if (!r->d_workspace) return fail(FB200_EINVAL, "sugar_reg: missing workspace");
    if (r->P > 0 && (!r->d_points || !r->d_scaling || !r->d_quaternions || !r->d_strengths || !r->d_knn_idx))
        return fail(FB200_EINVAL, "sugar_reg: missing Gaussian pointer");
    if (r->N > 0 && (!r->d_idx || !r->d_eps)) return fail(FB200_EINVAL, "sugar_reg: missing sample pointer");
    if (misaligned(r->d_quaternions, 16) || misaligned(r->d_workspace, 16))
        return fail(FB200_EINVAL, "sugar_reg: quaternions and workspace must be 16-byte aligned");
    return FB200_OK;
}

int fb200_sugar_reg_forward(const fb200_sugar_reg* r, int32_t with_grad, float* d_terms, void* stream) {
    int rc = check_sugar_reg(r);
    if (rc != FB200_OK) return rc;
    if (!d_terms) return fail(FB200_EINVAL, "sugar_reg_forward: missing terms output");
    return check(launch_sugar_reg_fwd(*r, with_grad != 0, d_terms, static_cast<cudaStream_t>(stream)),
                 "sugar_reg_forward");
}

int fb200_sugar_reg_backward(const fb200_sugar_reg* r, const float* d_dL_dterms, float* d_dpoints, float* d_dscaling,
                             float* d_dquaternions, float* d_dstrengths, void* stream) {
    int rc = check_sugar_reg(r);
    if (rc != FB200_OK) return rc;
    if (r->P == 0) return FB200_OK;
    if (!d_dL_dterms || !d_dpoints || !d_dscaling || !d_dquaternions || !d_dstrengths)
        return fail(FB200_EINVAL, "sugar_reg_backward: missing gradient pointer");
    if (misaligned(d_dquaternions, 16))
        return fail(FB200_EINVAL, "sugar_reg_backward: dL/dquaternions must be 16-byte aligned");
    return check(launch_sugar_reg_bwd(*r, d_dL_dterms, d_dpoints, d_dscaling, d_dquaternions, d_dstrengths,
                                      static_cast<cudaStream_t>(stream)),
                 "sugar_reg_backward");
}

static int check_sugar_dn_features(int32_t P, const float* d_points, const float* d_scaling, const float* d_quaternions,
                                   const float* d_viewmatrix, const float* d_campos) {
    if (P < 0) return fail(FB200_EINVAL, "sugar_dn_features: P must be >= 0");
    if (P > 0 && (!d_points || !d_scaling || !d_quaternions || !d_viewmatrix || !d_campos))
        return fail(FB200_EINVAL, "sugar_dn_features: missing input pointer");
    if (misaligned(d_quaternions, 16)) return fail(FB200_EINVAL, "sugar_dn_features: quaternions must be 16-byte aligned");
    return FB200_OK;
}

int fb200_sugar_dn_features(int32_t P, const float* d_points, const float* d_scaling, const float* d_quaternions,
                            const float* d_viewmatrix, const float* d_campos, float* d_features, void* stream) {
    int rc = check_sugar_dn_features(P, d_points, d_scaling, d_quaternions, d_viewmatrix, d_campos);
    if (rc != FB200_OK) return rc;
    if (P > 0 && !d_features) return fail(FB200_EINVAL, "sugar_dn_features: missing features output");
    return check(launch_sugar_dn_features(P, d_points, d_scaling, d_quaternions, d_viewmatrix, d_campos, d_features,
                                          static_cast<cudaStream_t>(stream)), "sugar_dn_features");
}

int fb200_sugar_dn_features_backward(int32_t P, const float* d_points, const float* d_scaling,
                                     const float* d_quaternions, const float* d_viewmatrix, const float* d_campos,
                                     const float* d_dL_dfeatures, float* d_dpoints, float* d_dquaternions,
                                     void* stream) {
    int rc = check_sugar_dn_features(P, d_points, d_scaling, d_quaternions, d_viewmatrix, d_campos);
    if (rc != FB200_OK) return rc;
    if (P > 0 && (!d_dL_dfeatures || !d_dpoints || !d_dquaternions))
        return fail(FB200_EINVAL, "sugar_dn_features_backward: missing gradient pointer");
    if (misaligned(d_dquaternions, 16))
        return fail(FB200_EINVAL, "sugar_dn_features_backward: dL/dquaternions must be 16-byte aligned");
    return check(launch_sugar_dn_features_bwd(P, d_points, d_scaling, d_quaternions, d_viewmatrix, d_campos,
                                              d_dL_dfeatures, d_dpoints, d_dquaternions,
                                              static_cast<cudaStream_t>(stream)),
                 "sugar_dn_features_backward");
}

size_t fb200_sugar_dn_partials(int32_t H, int32_t W) { return (H > 0 && W > 0) ? sugar_dn_num_partials(H, W) : 0; }

static int check_sugar_dn_loss(const float* d_dn, int32_t H, int32_t W, const float* d_viewmatrix,
                               const float* d_projmatrix) {
    if (H <= 0 || W <= 0) return fail(FB200_EINVAL, "sugar_dn_loss: bad image size (H, W > 0)");
    if (!d_dn || !d_viewmatrix || !d_projmatrix) return fail(FB200_EINVAL, "sugar_dn_loss: missing input pointer");
    return FB200_OK;
}

int fb200_sugar_dn_loss_forward(const float* d_dn, int32_t H, int32_t W, const float* d_viewmatrix,
                                const float* d_projmatrix, float* d_partials, float* d_loss, void* stream) {
    int rc = check_sugar_dn_loss(d_dn, H, W, d_viewmatrix, d_projmatrix);
    if (rc != FB200_OK) return rc;
    if (!d_partials || !d_loss) return fail(FB200_EINVAL, "sugar_dn_loss_forward: missing output pointer");
    return check(launch_sugar_dn_loss_fwd(d_dn, H, W, d_viewmatrix, d_projmatrix, d_partials, d_loss,
                                          static_cast<cudaStream_t>(stream)), "sugar_dn_loss_forward");
}

int fb200_sugar_dn_loss_backward(const float* d_dn, int32_t H, int32_t W, const float* d_viewmatrix,
                                 const float* d_projmatrix, const float* d_dL_dloss, float* d_dL_ddn, void* stream) {
    int rc = check_sugar_dn_loss(d_dn, H, W, d_viewmatrix, d_projmatrix);
    if (rc != FB200_OK) return rc;
    if (!d_dL_dloss || !d_dL_ddn) return fail(FB200_EINVAL, "sugar_dn_loss_backward: missing gradient pointer");
    return check(launch_sugar_dn_loss_bwd(d_dn, H, W, d_viewmatrix, d_projmatrix, d_dL_dloss, d_dL_ddn,
                                          static_cast<cudaStream_t>(stream)), "sugar_dn_loss_backward");
}

size_t fb200_knn_workspace_bytes(int32_t P, int32_t Q, int32_t K) {
    return (P >= 1 && Q >= 0 && K >= 1 && K <= 32 && K <= P) ? knn_workspace_bytes(P, Q) : 0;
}

int fb200_knn(const float* d_points, int32_t P, const float* d_queries, int32_t Q, int32_t K, void* d_workspace,
              size_t workspace_bytes, float* d_dists, int64_t* d_idx, void* stream) {
    if (P < 1 || Q < 0 || K < 1 || K > 32 || K > P)
        return fail(FB200_EINVAL, "knn: bad extents (1 <= K <= 32, K <= P, Q >= 0)");
    if (!d_queries && Q != P) return fail(FB200_EINVAL, "knn: self queries (no query pointer) need Q == P");
    if (Q == 0) return FB200_OK;
    if (!d_points || !d_workspace || !d_dists || !d_idx) return fail(FB200_EINVAL, "knn: missing pointer");
    if (misaligned(d_workspace, 256)) return fail(FB200_EINVAL, "knn: the workspace must be 256-byte aligned");
    if (workspace_bytes < knn_workspace_bytes(P, d_queries ? Q : 0)) return fail(FB200_ENOSPC, "knn: workspace too small");
    size_t need, reserved;
    int rc = check(knn_sort_scratch(P, d_queries ? Q : 0, &need, &reserved), "knn: radix-sort scratch query");
    if (rc != FB200_OK) return rc;
    if (need > reserved) {
        char msg[160];
        snprintf(msg, sizeof(msg), "knn: this CUB's radix sort needs %zu bytes of scratch, the workspace reserves %zu",
                 need, reserved);
        return fail(FB200_ENOSPC, msg);
    }
    return check(launch_knn(d_points, P, d_queries, Q, K, d_workspace, d_dists, d_idx, static_cast<cudaStream_t>(stream)),
                 "knn");
}

int fb200_adam_step(const fb200_adam_args* a, void* stream) {
    if (!a) return fail(FB200_EINVAL, "adam_step: null args");
    if (a->world < 1 || a->world > FB200_MAX_PEERS || a->rank < 0 || a->rank >= a->world)
        return fail(FB200_EINVAL, "adam_step: world must be 1..8 and rank inside it");
    if (a->n_groups < 1 || a->n_groups > FB200_ADAM_MAX_GROUPS)
        return fail(FB200_EINVAL, "adam_step: 1..16 parameter groups");
    for (int g = 0; g <= a->n_groups; ++g)
        if ((a->group_start[g] & 3) || (g > 0 && a->group_start[g] < a->group_start[g - 1]))
            return fail(FB200_EINVAL, "adam_step: group starts must be ascending multiples of 4 elements");
    if ((a->shard_lo & 3) || (a->shard_hi & 3) || a->shard_lo < a->group_start[0] || a->shard_hi < a->shard_lo ||
        a->shard_hi > a->group_start[a->n_groups])
        return fail(FB200_EINVAL, "adam_step: shard must be a 4-aligned range inside the slab");
    if (a->shard_hi > a->shard_lo) {
        if (!a->d_exp_avg || !a->d_exp_avg_sq) return fail(FB200_EINVAL, "adam_step: missing moment buffers");
        for (int p = 0; p < a->world; ++p)
            if (!a->peer_params[p] || !a->peer_grads[p]) return fail(FB200_EINVAL, "adam_step: missing slab pointer");
    }
    if ((a->mc_grads == nullptr) != (a->mc_params == nullptr))
        return fail(FB200_EINVAL, "adam_step: give both multicast mappings or neither");
    {
        int given = 0;
        for (int p = 0; p < a->world; ++p) given += a->peer_row_radii[p] != nullptr;
        if (given != 0 && given != a->world) return fail(FB200_EINVAL, "adam_step: give every rank's row radii or none");
        if (given) {
            if (a->row_count < 1) return fail(FB200_EINVAL, "adam_step: row_count must be positive with row radii");
            for (int g = 0; g < a->n_groups; ++g) {
                const int64_t n = a->group_start[g + 1] - a->group_start[g];
                if (a->row_width[g] < 0 || (int64_t)a->row_width[g] * a->row_count > n || n > 0xffffffffLL)
                    return fail(FB200_EINVAL, "adam_step: row_width * row_count exceeds the group");
            }
        }
    }
    if (!(a->bias_correction1 > 0.f) || !(a->bias_correction2_sqrt > 0.f))
        return fail(FB200_EINVAL, "adam_step: bias corrections must be positive (step >= 1)");
    return check(launch_adam_shard(*a, static_cast<cudaStream_t>(stream)), "adam_step");
}

int fb200_peer_alloc(size_t bytes, void** d_ptr) {
    if (!d_ptr || bytes == 0) return fail(FB200_EINVAL, "peer_alloc: bad arguments");
    void* p = nullptr;
    int rc = check(cudaMalloc(&p, bytes), "peer_alloc");
    if (rc != FB200_OK) return rc;
    rc = check(cudaMemset(p, 0, bytes), "peer_alloc (zero-fill)");
    if (rc != FB200_OK) { cudaFree(p); return rc; }
    *d_ptr = p;
    return FB200_OK;
}

int fb200_peer_free(void* d_ptr) { return d_ptr ? check(cudaFree(d_ptr), "peer_free") : FB200_OK; }

int fb200_peer_export(void* d_ptr, unsigned char* handle) {
    static_assert(sizeof(cudaIpcMemHandle_t) == FB200_PEER_HANDLE_BYTES, "handle size");
    if (!d_ptr || !handle) return fail(FB200_EINVAL, "peer_export: bad arguments");
    cudaIpcMemHandle_t h;
    int rc = check(cudaIpcGetMemHandle(&h, d_ptr), "peer_export");
    if (rc == FB200_OK) memcpy(handle, &h, sizeof(h));
    return rc;
}

int fb200_peer_open(const unsigned char* handle, void** d_ptr) {
    if (!d_ptr || !handle) return fail(FB200_EINVAL, "peer_open: bad arguments");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, sizeof(h));
    return check(cudaIpcOpenMemHandle(d_ptr, h, cudaIpcMemLazyEnablePeerAccess), "peer_open");
}

int fb200_peer_close(void* d_ptr) { return d_ptr ? check(cudaIpcCloseMemHandle(d_ptr), "peer_close") : FB200_OK; }

}  // extern "C"
