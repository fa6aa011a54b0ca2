/*
 * frosting_b200.h -- C ABI of the frosting_b200 Gaussian-splatting rasterizer (CUDA, sm_90a).
 *
 * This is the drop-in boundary for Frosting's render path.  Every entry point names the
 * reference interface it replaces (paths relative to the reference repository; DGR =
 * gaussian_splatting/submodules/diff-gaussian-rasterization):
 *
 *   fb200_forward        <- _C.rasterize_gaussians          DGR/ext.cpp:16, DGR/rasterize_points.cu:35-115,
 *                           CudaRasterizer::Rasterizer::forward  DGR/cuda_rasterizer/rasterizer_impl.cu:198-336
 *   fb200_backward       <- _C.rasterize_gaussians_backward DGR/ext.cpp:17, DGR/rasterize_points.cu:117-196,
 *                           Rasterizer::backward            DGR/cuda_rasterizer/rasterizer_impl.cu:340-434
 *   fb200_mark_visible   <- _C.mark_visible                 DGR/ext.cpp:18, DGR/rasterize_points.cu:198-217
 *   fb200_mesh_visibility<- nvdiff_rasterization / MeshRasterizer.forward
 *                           frosting_utils/nvdiffrast.py:8-58, frosting_utils/mesh_rasterization.py:109-156
 *   fb200_*_bytes        <- required<GeometryState|ImageState|BinningState>()
 *                           DGR/cuda_rasterizer/rasterizer_impl.h:66-72
 *
 * Conventions
 *   - plain C: pointers, sizes, ints.  No C++/torch types cross this boundary.
 *   - every pointer named d_* is a DEVICE pointer on the current CUDA device; the library never
 *     allocates, frees or retains device memory (the caller owns every buffer, as the reference's
 *     torch binding does through its resize callbacks, DGR/rasterize_points.cu:27-33).
 *   - `stream` is a cudaStream_t passed as void*; all work is enqueued on it, nothing synchronises
 *     unless `debug` is set (the reference's CHECK_CUDA behaviour, DGR/cuda_rasterizer/auxiliary.h:166-173).
 *   - return value: 0 on success, negative FB200_E* on error; fb200_last_error() gives the
 *     message (thread-local).
 */
#ifndef FROSTING_B200_H_
#define FROSTING_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FB200_ABI_VERSION 9

#define FB200_OK 0
#define FB200_EINVAL (-1)   /* bad argument (shape / null pointer / unsupported channel count) */
#define FB200_ECUDA (-2)    /* CUDA runtime error (message holds cudaGetErrorString) */
#define FB200_ENOSPC (-3)   /* a caller-provided workspace is too small */

#define FB200_TILE 16       /* tile edge in pixels: BLOCK_X/BLOCK_Y, DGR/cuda_rasterizer/config.h:16-17 */
#define FB200_CHANNELS 3    /* NUM_CHANNELS, DGR/cuda_rasterizer/config.h:15 */

/* Extra per-Gaussian feature channels blended with the same weights as the colour, in the same traversal (SURVEY.md
 * row f4).  The reference obtains depth / normal maps by calling the 3-channel rasterizer AGAIN with the features as
 * colors_precomp (frosting_scene/sugar_model.py:2343-2387, coarse_density_and_dn_consistency.py:649,689-714): a second
 * preprocess + sort + blend over the same geometry.  Here: out[c] = sum_i f_i[c] alpha_i T_i + T_final background[c],
 * i.e. exactly what that second pass returns, and the backward adds the features' contribution to dL/dalpha (hence to
 * the geometry gradients) -- the sum of the two passes' gradients. */
typedef struct fb200_extra {
    int32_t channels;             /* 1..3 */
    const float* d_features;      /* [P, channels] */
    const float* d_background;    /* [channels] */
    float* d_out;                 /* [channels, H, W]  written by fb200_forward_raster */
    const float* d_dL_dout;       /* [channels, H, W]  read by fb200_backward */
    float* d_dL_dfeatures;        /* [P, channels]     written by fb200_backward (fully) */
} fb200_extra;

/* Per-call scalars: the non-tensor fields of GaussianRasterizationSettings
 * (DGR/diff_gaussian_rasterization/__init__.py:157-169) plus the tensor extents. */
typedef struct fb200_params {
    int32_t P;               /* number of Gaussians (means3D.size(0)) */
    int32_t sh_degree;       /* D: active SH degree 0..3 */
    int32_t sh_coeffs;       /* M: coefficients stored per Gaussian (sh.size(1)), 0 if colours are precomputed */
    int32_t image_width;
    int32_t image_height;
    float tanfovx;
    float tanfovy;
    float scale_modifier;
    int32_t prefiltered;     /* trap if a Gaussian is near-culled (auxiliary.h:156-160) */
    int32_t debug;           /* bit 0: synchronise + check after every stage.  bit 1: disable sub-tile culling, every
                                tile instance is evaluated in all 8 sub-tiles of its tile (slower; outputs identical).
                                Any other bit set: FB200_EINVAL */
    const fb200_extra* extra; /* NULL: colour only (the reference's surface) */
} fb200_params;

/* Frosting's per-frame attribute construction, fused (frosting_scene/frosting_model.py:713-799): turns the
 * model's learnable parameters into the rasterizer inputs in one kernel (and one backward kernel) instead
 * of the softmax / gather / mul / sum / sigmoid / exp / normalize / cat chain of torch ops.
 *
 * The block describes the whole Frosting model: P mesh-bound Gaussians, then n_bg BACKGROUND Gaussians -- Frosting's
 * free 3DGS Gaussians, concatenated after the mesh-bound ones (frosting_model.py:564-591 parameters, :801-876 bg_*
 * properties, :1415-1418 and :1487-1514 the cat).  A frame is P + n_bg rows, mesh-bound rows first.  A background row
 * skips the occlusion lookup (it is always a candidate, :1571-1576) and maps its parameters like a mesh row, without the
 * prism cell: position = d_bg_points (used as is), opacity = sigmoid, scales = exp, rotation = normalize, SH row =
 * dc | rest.  n_bg == 0: mesh-bound Gaussians only, the d_bg_* pointers are not read.
 *
 * Alignment, checked by every entry point that takes the block (FB200_EINVAL otherwise): with P > 0, d_bary_logits
 * 8-byte, d_quats and (sh_rest > 0) d_sh_rest 16-byte aligned; with n_bg > 0, d_bg_quats 16-byte aligned. */
typedef struct fb200_frosting_params {
    int32_t P;                       /* mesh-bound Gaussians */
    int32_t n_verts, n_faces;        /* shell base mesh */
    int32_t sh_rest;                 /* M - 1: coefficients in _sh_coordinates_rest */
    const float* d_bary_logits;      /* [P,6]  _bary_coords (softmax logits, :713-716) */
    const int64_t* d_cells;          /* [P]    _point_cell_indices */
    const int32_t* d_faces;          /* [F,3]  _shell_base_faces */
    const float* d_inner_verts;      /* [V,3]  inner_verts property (:679-710) */
    const float* d_outer_verts;      /* [V,3]  outer_verts */
    const float* d_opacity_logits;   /* [P]    _opacities */
    const float* d_log_scales;       /* [P,3]  _scales (scale_activation = exp, :32) */
    const float* d_quats;            /* [P,4]  _quaternions (raw) */
    const float* d_sh_dc;            /* [P,1,3] */
    const float* d_sh_rest;          /* [P,M-1,3] */
    const uint8_t* d_mask;           /* optional [P]: 0 = occluded, outputs for it are left untouched */
    const uint8_t* d_face_visible;   /* optional [F]: the same culling as face_visible[d_cells[i]] (no mask tensor) */
    const int32_t* d_radii;          /* optional [P + n_bg], backward only: a Gaussian with radii <= 0 was not rendered,
                                        its upstream gradient rows are zero by definition and are NOT read (they may be
                                        unwritten: fb200_grads.sparse_rows) */
    int32_t n_bg;                    /* background Gaussians (0: none) */
    const float* d_bg_points;        /* [n_bg,3]     _bg_points */
    const float* d_bg_opacity_logits;/* [n_bg]       _bg_opacities */
    const float* d_bg_log_scales;    /* [n_bg,3]     _bg_scales */
    const float* d_bg_quats;         /* [n_bg,4]     _bg_quaternions (raw) */
    const float* d_bg_sh_dc;         /* [n_bg,1,3]   _bg_sh_coordinates_dc */
    const float* d_bg_sh_rest;       /* [n_bg,M-1,3] _bg_sh_coordinates_rest */
} fb200_frosting_params;

typedef struct fb200_frosting_grads {      /* fb200_frosting_attributes_backward: all fully written; frosting mode of
                                            * fb200_backward: rows of rendered Gaussians only.  Inner / outer vertex gradients
                                            * are accumulated (cleared by the call first), both or neither.  The six mesh
                                            * parameter gradients are required when the block's P > 0, each 16-byte
                                            * aligned (d_sh_rest when sh_rest > 0).  The d_bg_* rows are the background
                                            * Gaussians': given exactly when n_bg > 0, d_bg_quats 16-byte aligned */
    float* d_bary_logits; float* d_inner_verts; float* d_outer_verts; float* d_opacity_logits;
    float* d_log_scales; float* d_quats; float* d_sh_dc; float* d_sh_rest;
    float* d_bg_points; float* d_bg_opacity_logits; float* d_bg_log_scales; float* d_bg_quats; float* d_bg_sh_dc;
    float* d_bg_sh_rest;
} fb200_frosting_grads;

/* Device inputs of the forward pass.  Exactly one of (d_shs | d_colors_precomp) and exactly one of
 * (d_scales + d_rotations | d_cov3D_precomp) must be non-null, as GaussianRasterizer.forward
 * requires (__init__.py:191-195). */
typedef struct fb200_inputs {
    const float* d_background;     /* [3] */
    const float* d_means3D;        /* [P,3] */
    const float* d_shs;            /* [P,M,3] or NULL */
    const float* d_colors_precomp; /* [P,3]   or NULL */
    const float* d_opacities;      /* [P]   */
    const float* d_scales;         /* [P,3] or NULL */
    const float* d_rotations;      /* [P,4] (r,x,y,z), NOT normalised (forward.cu:127) or NULL */
    const float* d_cov3D_precomp;  /* [P,6] or NULL */
    const float* d_viewmatrix;     /* [16] as stored by torch: W2C transposed */
    const float* d_projmatrix;     /* [16] */
    const float* d_campos;         /* [3]  */
    const uint8_t* d_visibility;   /* optional [P] mask (0 = drop before tiling): the occlusion-culling
                                      render_mask of frosting_model.py:1564-1586 applied in place instead
                                      of by boolean gathers.  NULL = all Gaussians enter. */
    /* The same occlusion culling WITHOUT a per-Gaussian mask tensor (SURVEY.md row f1): the prepass's visible-face marks
     * and Frosting's _point_cell_indices are looked up inside preprocess, render_mask[i] = face_visible[cells[i]] for
     * i < n_cell_points and 1 for the trailing background Gaussians (frosting_model.py:1564-1576).  Both or neither. */
    const int64_t* d_point_cells;  /* [n_cell_points] or NULL */
    const uint8_t* d_face_visible; /* [F] (0 = occluded) or NULL */
    int64_t n_cell_points;         /* mesh-bound Gaussians (<= P) */
    /* FROSTING MODE (row f1 proper): the rasterizer reads Frosting's learnable parameters directly.  When non-NULL,
     * d_means3D, d_shs, d_colors_precomp, d_opacities, d_scales, d_rotations, d_cov3D_precomp, d_visibility,
     * d_point_cells and d_face_visible above must all be NULL: preprocess builds position (softmax barycentrics over the
     * prism cell), opacity (sigmoid), scales (exp), rotation (normalize) and reads the SH rows from dc | rest IN PLACE --
     * no attribute tensor, in particular no [P,M,3] SH copy, is ever materialised -- and culls with
     * frosting->d_mask / frosting->d_face_visible[d_cells[i]] (mesh-bound rows only: background rows are never culled).
     * prm->P == frosting->P + frosting->n_bg, prm->sh_coeffs == sh_rest + 1.  fb200_backward then needs
     * fb200_grads.frosting and writes the PARAMETER gradients (same chain rule as fb200_frosting_attributes_backward,
     * inside the per-Gaussian backward kernel), row i of the frame being background row i - frosting->P when
     * i >= frosting->P. */
    const fb200_frosting_params* frosting;
} fb200_inputs;

/* Alignment: rows that the kernels read or write with 128-bit accesses must start on 16-byte boundaries -- d_rotations,
 * d_shs when 3*M is a multiple of 4, and the gradient outputs d_dL_drotations / d_dL_dsh likewise.  cudaMalloc'ed and torch
 * tensors are; a contiguous VIEW at an odd element offset is not (the Python shim copies such a view).  Misaligned
 * pointers are rejected with FB200_EINVAL. */

/* Caller-owned workspaces (sizes from the *_bytes queries; 256-byte aligned base pointers). */
typedef struct fb200_workspace {
    void* d_geom;   size_t geom_bytes;     /* per-Gaussian state, kept for backward */
    void* d_image;  size_t image_bytes;    /* per-pixel + per-tile state, kept for backward */
    void* d_binning; size_t binning_bytes; /* per-instance state, kept for backward */
    int64_t binning_capacity;              /* instances the binning buffer was sized for */
    int32_t* d_status;                     /* [FB200_STATUS_WORDS] device words, see below */
    int32_t acc_zeroed_by_forward;         /* backward's per-Gaussian accumulators (48 B each, inside d_geom) must be zero
                                              when fb200_backward starts.  0: fb200_backward clears them itself.
                                              1: fb200_forward_geometry clears them (stream-ordered, while the host
                                              waits for the instance count) and fb200_backward skips its clear; the
                                              caller resets the field to 0 before any further backward over the same
                                              forward state */
    const int32_t* h_status;               /* optional HOST copy of the status words written by fb200_forward_geometry,
                                              read by the caller after synchronising the stream; fb200_forward_raster
                                              then skips launches it can tell are empty.  NULL: launch for the worst case */
} fb200_workspace;

/* d_status words written by fb200_forward (stream-ordered; copy back after the call). */
#define FB200_STATUS_WORDS 8
#define FB200_ST_NUM_RENDERED 0   /* R = total tile instances (reference: point_offsets[P-1]) */
#define FB200_ST_OVERFLOW 1       /* 1 if R > binning_capacity: nothing was rendered, grow and call again */
#define FB200_ST_MAX_TILE 2       /* longest per-tile list */
#define FB200_ST_NUM_VISIBLE 3    /* Gaussians with radii > 0 (V of SURVEY.md 8d) */

size_t fb200_geom_bytes(int32_t P);
size_t fb200_image_bytes(int32_t image_width, int32_t image_height);
size_t fb200_binning_bytes(int64_t capacity);

/* Forward: preprocess + cull, per-tile bin/sort, front-to-back blend.
 *   d_out_color [3,H,W] f32, d_radii [P] i32 -- both fully written (no zero-fill needed).
 * If the instance count exceeds ws->binning_capacity the status word FB200_ST_OVERFLOW is set,
 * d_radii and FB200_ST_NUM_RENDERED are valid, d_out_color is not; the caller re-runs with a larger
 * binning buffer (the reference instead blocks on a D2H copy mid-pipeline, rasterizer_impl.cu:280-281). */
int fb200_forward(const fb200_params* prm, const fb200_inputs* in, const fb200_workspace* ws,
                  float* d_out_color, int32_t* d_radii, void* stream);

/* The same forward in two phases, for callers that want an exactly sized binning buffer and no retry:
 *   fb200_forward_geometry : preprocess + per-tile counts + tile scan.  Needs only the geometry and image
 *                            workspaces; writes d_radii and d_status[FB200_ST_NUM_RENDERED] (stream-ordered).
 *   fb200_forward_raster   : scatter + per-tile sort + blend, with a binning buffer of capacity >= R.
 * This is the reference's own split (it blocks on point_offsets[P-1] between preprocess and binning,
 * rasterizer_impl.cu:280-284); here the wait is the caller's choice and covers ~0.1 ms of GPU work. */
int fb200_forward_geometry(const fb200_params* prm, const fb200_inputs* in, const fb200_workspace* ws,
                           int32_t* d_radii, void* stream);
int fb200_forward_raster(const fb200_params* prm, const fb200_inputs* in, const fb200_workspace* ws,
                         float* d_out_color, int32_t* d_radii, void* stream);

/* Gradient outputs of the backward pass, shapes as DGR/rasterize_points.cu:151-159.
 * All are fully written by the call (invisible Gaussians get zeros) unless sparse_rows / frosting say otherwise; no
 * pre-zeroing needed. */
typedef struct fb200_grads {
    float* d_dL_dmeans2D;     /* [P,3] (z = 0) */
    float* d_dL_dcolors;      /* [P,3]; may be NULL when colours come from SH (then an intermediate, not written) */
    float* d_dL_dopacity;     /* [P,1] */
    float* d_dL_dmeans3D;     /* [P,3] */
    float* d_dL_dcov3D;       /* [P,6]; may be NULL unless d_cov3D_precomp is given */
    float* d_dL_dsh;          /* [P,M,3] (may be NULL when M == 0) */
    float* d_dL_dscales;      /* [P,3]; these two may be NULL when d_cov3D_precomp is given */
    float* d_dL_drotations;   /* [P,4] */
    int32_t sparse_rows;      /* 0: every row is written (zeros for Gaussians with radii == 0) -- the reference's dense
                                 contract.  1 (row f1): rows of Gaussians that were not rendered (radii <= 0) are
                                 SKIPPED: they stay unwritten and must not be read -- for a consumer that has d_radii and
                                 treats radii <= 0 as a zero row (fb200_frosting_attributes_backward with d_radii,
                                 fb200_adam_args.d_row_radii) */
    const fb200_frosting_grads* frosting; /* frosting mode (fb200_inputs.frosting): the parameter-gradient outputs; the
                                 eight pointers above may then be NULL (d_dL_dmeans2D is still written when given) and
                                 the contract is ALWAYS sparse: only rows with radii > 0 are written -- mesh rows into
                                 the block's mesh gradients, background rows into its d_bg_* rows at row i - frosting->P.
                                 The unrendered rows of both are left as they were */
} fb200_grads;

int fb200_backward(const fb200_params* prm, const fb200_inputs* in, const fb200_workspace* ws,
                   const int32_t* d_radii, const float* d_dL_dout_color /* [3,H,W] */,
                   const fb200_grads* grads, void* stream);

/* present[i] = (W2C * p_i).z > 0.2   (checkFrustum, rasterizer_impl.cu:54-66) */
int fb200_mark_visible(int32_t P, const float* d_means3D, const float* d_viewmatrix,
                       const float* d_projmatrix, uint8_t* d_present, void* stream);

/* Occlusion-culling prepass: rasterise a triangle mesh in clip space and report the nearest face per
 * pixel (replaces nvdiffrast's OpenGL rasteriser, frosting_utils/nvdiffrast.py:42-54).
 *   d_verts [V,3], d_faces [F,3] i32, d_full_proj [16] (= full_proj_transform as stored by torch)
 *   d_zbuf  [H*W] u64 scratch
 *   d_pix_to_face [H*W] i32 : face id or -1 (mesh_rasterization.py:146 `rast_out[...,3] - 1`)
 *   d_face_visible [F] u8 (optional) : 1 if the face owns at least one pixel; if `mark_last_on_bg`
 *     the last face is also marked when any pixel is background, reproducing the `_index_mask[-1]`
 *     quirk of frosting_model.py:1565-1570.
 *   d_scratch [2*F + 4] i32 (optional): work lists of the faces that need a warp / a CTA; with it one pass classifies
 *     every face (rasterising the small ones on the spot) and the two larger classes run over their lists only; NULL:
 *     every size class is launched over all F faces. */
int fb200_mesh_visibility(int32_t V, int32_t F, const float* d_verts, const int32_t* d_faces,
                          const float* d_full_proj, int32_t image_width, int32_t image_height,
                          uint64_t* d_zbuf, int32_t* d_pix_to_face, uint8_t* d_face_visible,
                          int32_t mark_last_on_bg, int32_t* d_scratch, void* stream);

/* render_mask[i] = face_visible[cell[i]] for i < n_cells_points, 1 for the trailing background
 * Gaussians (frosting_model.py:1571-1576). */
int fb200_gaussian_mask_from_faces(int32_t n_points, const int64_t* d_point_cell_indices,
                                   int32_t F, const uint8_t* d_face_visible, int32_t n_background,
                                   uint8_t* d_mask, void* stream);

/* Frosting's attribute construction as stand-alone kernels (structs: above, before fb200_inputs), the cross-check of
 * frosting mode.  Outputs and upstream gradients have P + n_bg rows, background rows last; d_rotations and
 * d_g_rotations 16-byte aligned, d_shs and d_g_shs too when sh_rest == 15.  With d_radii the backward writes zeros for
 * a row with radii <= 0 and does not read its upstream rows. */
int fb200_frosting_attributes(const fb200_frosting_params* fp, float* d_means3D /*[P+n_bg,3]*/,
                              float* d_opacities /*[P+n_bg,1]*/, float* d_scales /*[P+n_bg,3]*/,
                              float* d_rotations /*[P+n_bg,4]*/, float* d_shs /*[P+n_bg,M,3]*/, void* stream);
int fb200_frosting_attributes_backward(const fb200_frosting_params* fp, const float* d_g_means3D,
                                       const float* d_g_opacities, const float* d_g_scales,
                                       const float* d_g_rotations, const float* d_g_shs,
                                       const fb200_frosting_grads* grads, void* stream);

/* Edited / animated scenes, simple adaptation (frosting_model.py:1013-1054 make_editable(use_simple_adapt=True), the
 * editable branches of :649-799, blender/frosting_utils.py:519-588 render_composited_image).  Per frame the base
 * vertices move; fb200_frosting_edit_shell rebuilds the shell and the per-face tables from them, and
 * fb200_frosting_edit_attributes turns the parameter block into rasterizer inputs with COLOURS precomputed from SH at
 * view directions rotated by R(q' q_orig^-1) (feed them to fb200_forward as d_colors_precomp).  Forward only.
 *
 * Reference capture: with d_ref_quats, d_ref_dists and d_ref_median all NULL, fb200_frosting_edit_shell writes the
 * face quaternions to d_rel_quats, the distances to d_dists and (median method) their median to d_factor[0], keeps
 * every face and uses factor 1 -- run it once on the reference vertices and keep those three as the references. */
#define FB200_RESCALE_MEDIAN 0      /* one factor: median of the edited faces' centroid distances over the reference's */
#define FB200_RESCALE_TRIANGLE 1    /* per face: median of its three distances over the reference's */
#define FB200_EDIT_SELECT_WORDS 2051
typedef struct fb200_frosting_edit {
    int32_t n_verts, n_faces;
    int32_t rescaling;                    /* FB200_RESCALE_* */
    int32_t n_edited;                     /* faces with d_edition_mask set (median: >= 1) */
    float deformation_threshold;          /* an edited face is dropped when max_k(dist_k / ref_dist_k) > threshold */
    const float* d_base_verts;            /* [V,3] this frame's (deformed) base vertices */
    const int32_t* d_faces;               /* [F,3] */
    const float* d_inner_dist;            /* [V] signed shell offsets along the vertex normal */
    const float* d_outer_dist;            /* [V] */
    const uint8_t* d_edition_mask;        /* [F] edited faces */
    const uint8_t* d_verts_edition_mask;  /* [V] vertices of edited faces */
    const int32_t* d_vf_offsets;          /* [V+1] vertex -> adjacent face CSR (one entry per face corner) */
    const int32_t* d_vf_faces;            /* [3F] */
    const float* d_ref_quats;             /* [F,4] reference face quaternions, 16-byte aligned (NULL: capture) */
    const float* d_ref_dists;             /* [F,3] reference vertex-to-centroid distances */
    const float* d_ref_median;            /* [1]   median of the edited faces' reference distances (median method) */
    /* written by fb200_frosting_edit_shell */
    float* d_dists;                       /* [F,3] */
    float* d_face_normals;                /* [F,3] area-weighted face normals (vertex-normal terms) */
    float* d_rel_quats;                   /* [F,4] face_q * ref_q^-1 on edited faces, identity elsewhere; 16-byte aligned */
    float* d_face_factor;                 /* [F]   triangle factor (1 on unedited faces) */
    uint8_t* d_face_keep;                 /* [F]   deformation keep flag */
    float* d_factor;                      /* [2]   median method: the median, the factor */
    uint32_t* d_select;                   /* [FB200_EDIT_SELECT_WORDS] scratch of the median's radix select */
    float* d_inner_verts;                 /* [V,3] the frame's shell */
    float* d_outer_verts;                 /* [V,3] */
} fb200_frosting_edit;

int fb200_frosting_edit_shell(const fb200_frosting_edit* e, void* stream);
/* fp: the parameter block whose d_inner_verts / d_outer_verts are e's shell (d_mask, d_radii unused; d_face_visible
 * optional: culled rows are not written).  Rows P + n_bg, background rows last: d_rotations 16-byte aligned,
 * d_orig_quats [P+n_bg,4] 16-byte aligned or NULL (directions unrotated), d_colors [P+n_bg,3].
 * sh_degree <= sqrt(sh_rest + 1) - 1. */
int fb200_frosting_edit_attributes(const fb200_frosting_edit* e, const fb200_frosting_params* fp, int32_t sh_degree,
                                   const float* d_campos /*[3]*/, const float* d_orig_quats, float* d_means3D,
                                   float* d_opacities, float* d_scales, float* d_rotations, float* d_colors,
                                   void* stream);

/* Complex adaptation (make_editable(use_simple_adapt=False), frosting_model.py:900-967, :1055-1119, :1149-1183): each
 * edited Gaussian keeps a canonical transform C = T_ref[cell]^-1 R(q) diag(exp(s)), where T maps a canonical cell to
 * the world ([a', b', normalize(n) * d]: two Gram-Schmidt-orthogonalised in-plane axes and the normal scaled by the
 * median distance).  Per frame M = T_frame[cell] C gives the scales (column norms) and the rotation.
 *
 * fb200_frosting_edit_complex_capture: run after the reference capture of fb200_frosting_edit_shell (e's d_dists and,
 * median method, d_factor[0] hold the reference's), with fp the parameter block of that capture.  Writes d_cell_T [F,9]
 * (row-major 3x3, edited faces only; singular cells fixed up as the reference does), d_canonical [P,9] (0 on unedited
 * rows) and d_n_singular [1]: the Gaussians whose cell is still singular (their C is 0; the reference's solve fails).
 * fb200_frosting_edit_attributes_complex: fb200_frosting_edit_attributes with the complex rule for edited rows; run
 * after this frame's fb200_frosting_edit_shell.  Rewrites d_cell_T for the frame's edited faces. */
int fb200_frosting_edit_complex_capture(const fb200_frosting_edit* e, const fb200_frosting_params* fp, float* d_cell_T,
                                        float* d_canonical, uint32_t* d_n_singular, void* stream);
int fb200_frosting_edit_attributes_complex(const fb200_frosting_edit* e, const fb200_frosting_params* fp,
                                           int32_t sh_degree, const float* d_campos /*[3]*/, const float* d_orig_quats,
                                           const float* d_canonical, float* d_cell_T, float* d_means3D,
                                           float* d_opacities, float* d_scales, float* d_rotations, float* d_colors,
                                           void* stream);

/* Linear-blend skinning of a Blender-animated scene's base mesh (blender/frosting_utils.py:474-516
 * apply_poses_to_scene).  Row i of the rigged vertices is base vertex d_vert_ids[i]; its entries
 * [d_offsets[i], d_offsets[i+1]) are (bone, weight) pairs in the armature's bone order.  Per entry:
 *   q = [p, 1] @ d_reset[bone], q = q.xyz / q.w;  r = [q, 1] @ d_pose[bone][frame], r = r.xyz / r.w;
 *   acc = (float)((double)acc + weight * (double)r)
 * starting from acc = 0; the vertex is set to acc (0 without entries).  Base vertices that are no row's are neither
 * read nor written.  Matrices are row-major 4x4 in the row-vector convention (pytorch3d's Transform3d):
 * d_reset = inverse(rest^T), d_pose = the track's matrices transposed; both 16-byte aligned. */
typedef struct fb200_frosting_skin {
    int32_t n_rows;                 /* rigged vertices */
    int32_t n_verts;                /* rows of the base-vertex buffer (d_vert_ids < n_verts) */
    int32_t n_bones;
    int32_t n_frames;               /* frames of every pose track */
    const float* d_tpose;           /* [n_rows,3] T-pose points */
    const int32_t* d_vert_ids;      /* [n_rows] */
    const int32_t* d_offsets;       /* [n_rows+1] CSR into d_bones / d_weights */
    const int32_t* d_bones;         /* [n_entries] bone ids in [0, n_bones) */
    const double* d_weights;        /* [n_entries] normalised weights (float64, as the reference keeps them) */
    const float* d_reset;           /* [n_bones,4,4] */
    const float* d_pose;            /* [n_bones,n_frames,4,4] */
} fb200_frosting_skin;
/* Writes frame `frame` (in [0, n_frames)) into d_base_verts [n_verts,3] in place.  One launch, no allocation. */
int fb200_frosting_skin_pose(const fb200_frosting_skin* s, int32_t frame, float* d_base_verts, void* stream);

/* Texture bake of the base mesh (frosting_utils/texture.py:11-181 compute_textured_mesh_for_frosting_mesh).
 *
 * fb200_mesh_barycentrics: perspective-correct barycentrics d_bary [H,W,3] of the faces d_pix_to_face [H,W] (from
 * fb200_mesh_visibility with the same vertices, faces and d_full_proj [4,4]); (u, v, 1 - (u + v)) on a hit,
 * (0, 0, 1) elsewhere.
 *
 * Face f owns half f % 2 of UV square f / 2 (square s at texels [s / n * sq, +sq) x [s % n * sq, +sq)).  Per view,
 * every touched face and texel receives ONE pixel's colour and a count of 1: the last hit pixel in row-major order
 * (what `acc[idx] = acc[idx] + colors` with duplicate indices does on the CPU).  Accumulation is fp32 in view order.
 * The caller zeroes d_face_acc / d_texel_acc and sets d_face_winner / d_texel_winner to -1 once; every view leaves the
 * winner slots at -1 again.  A face without Gaussians and without a view hit gets NaN, as in the reference. */
typedef struct fb200_texture {
    int32_t n_faces;                /* F >= 1 */
    int32_t n_points;               /* mesh-bound Gaussians */
    int32_t square_size;            /* sq >= 3 */
    int32_t n_square_per_axis;      /* n, with 2 n^2 >= F */
    int32_t texture_size;           /* T = sq * n */
    const int32_t* d_cell_offsets;  /* [F+1] CSR face -> Gaussians */
    const int32_t* d_cell_points;   /* [n_points] Gaussian ids, ascending within each face */
    const float* d_sh_dc;           /* [n_points,3] SH degree-0 coefficients */
    float* d_face_sh;               /* [F,3] written by fb200_texture_face_sh_colours */
    float* d_face_acc;              /* [F,4] colour sum and count, 16-byte aligned */
    float* d_texel_acc;             /* [T*T,4] colour sum and count per texel (row-major, before the flip) */
    int32_t* d_face_winner;         /* [F] */
    int32_t* d_texel_winner;        /* [T*T] */
} fb200_texture;
int fb200_mesh_barycentrics(int32_t V, int32_t F, const float* d_verts, const int32_t* d_faces,
                            const float* d_full_proj, int32_t W, int32_t H, const int32_t* d_pix_to_face,
                            float* d_bary, void* stream);
/* Once per bake, before fb200_texture_finish: mean of clamp(SH2RGB(dc), 0, 1) per face into d_face_sh. */
int fb200_texture_face_sh_colours(const fb200_texture* t, void* stream);
/* One view: d_image [H,W,3] (nan_to_num and clamp(0, 1) are applied here), d_pix_to_face [H,W], d_bary [H,W,3]. */
int fb200_texture_add_view(const fb200_texture* t, const float* d_image, const int32_t* d_pix_to_face,
                           const float* d_bary, int32_t W, int32_t H, void* stream);
/* d_texture [T,T,3]: filled texels sum / count, others their face's colour; rows flipped (row 0 is v = T-1). */
int fb200_texture_finish(const fb200_texture* t, float* d_texture, void* stream);

/* Fused photometric loss (1 - lambda) * mean|x - y| + lambda * (1 - SSIM(x, y)) of Frosting's trainers
 * (frosting_utils/loss_utils.py:17-63 with refine.py:407-409; 11x11 Gaussian window, sigma 1.5, zero padding).
 *   d_pred, d_gt [C,H,W]; d_maps [3,C,H,W] scratch kept for backward; d_partials [fb200_loss_partials(C,H,W)];
 *   d_loss [1].  Backward writes d(loss)/d(pred) scaled by the device scalar d_dL_dloss[0]. */
size_t fb200_loss_partials(int32_t C, int32_t H, int32_t W);
int fb200_l1_dssim_forward(const float* d_pred, const float* d_gt, int32_t C, int32_t H, int32_t W, float lambda,
                           float* d_maps, float* d_partials, float* d_loss, void* stream);
int fb200_l1_dssim_backward(const float* d_pred, const float* d_gt, const float* d_maps, int32_t C, int32_t H,
                            int32_t W, float lambda, const float* d_dL_dloss, float* d_dpred, void* stream);

/* SuGaR's SDF regulariser of the coarse stage (SURVEY.md row a23; frosting_trainers/coarse_density_and_dn_consistency.py
 * :745-833 with frosting_scene/sugar_model.py get_field_values, get_beta 'average', get_smallest_axis; density-mode
 * estimation, gradient through the normals only).  For sample n with owner i = d_idx[n] and neighbours
 * j = d_knn_idx[i,k], k < K:
 *   x = mu_i + q_i ((f s_i) * eps_n) q_i^-1 (pytorch3d quaternion_apply: the conjugate as inverse);
 *   A_j = quaternion_to_matrix(q_j) with column c scaled by 1 / clamp(s_jc, 1e-8);
 *   o_k = sigma_j exp(-clamp(|A_j^T (x - mu_j)|^2, 0, 1e8) / 2), d = sum_k o_k, beta = mean_k min s_j;
 *   nrm = the column of R(q) at the first minimal axis of s; sdf = (x - mu_i) . nrm_i, t = exp(-sdf^2 / (2 beta^2));
 *   m_k = nrm_j sign(nrm_j . nrm_i); w_k = o_k |(x - mu_j) . m_k| / clamp(min s_j, 1e-6)^2 (no gradient);
 *   terms[0] = mean_n |d - t|;  terms[1] = mean_n |nrm_i - sum_k w_k m_k / clamp(sum_k w_k, 1e-6)|^2.
 * The workspace (fb200_sugar_reg_workspace_bytes, 16-byte aligned) holds an 80-byte record per Gaussian and 8 bytes
 * per block of samples, and for with_grad a 128-byte gradient accumulator per Gaussian (replicated to fill 32 MiB when
 * P < 2^18); nothing of size N x K.  A forward without gradient needs only the with_grad = 0 size.
 * fb200_sugar_reg_forward writes d_terms [2]; with `with_grad` it also differentiates both terms at unit upstream
 * into the workspace, and fb200_sugar_reg_backward then writes the dense gradients of terms[0] * d_dL_dterms[0] +
 * terms[1] * d_dL_dterms[1] (a device [2]) with respect to the four inputs, reading the same struct.  A sample whose
 * owner d_idx[n] lies outside [0, P) is skipped and makes both terms NaN (checked on the device, no synchronisation);
 * d_knn_idx is not checked and must lie in [0, P). */
typedef struct fb200_sugar_reg {
    int32_t P;                      /* Gaussians */
    int32_t K;                      /* neighbours per Gaussian, 1..32 */
    int32_t N;                      /* samples; N > 0 needs P > 0 */
    float sampling_scale_factor;    /* f (1.5 in the trainers) */
    const float* d_points;          /* [P,3] */
    const float* d_scaling;         /* [P,3] activated scales */
    const float* d_quaternions;     /* [P,4] (w, x, y, z), 16-byte aligned */
    const float* d_strengths;       /* [P] activated opacities */
    const int32_t* d_knn_idx;       /* [P,K] */
    const int64_t* d_idx;           /* [N] owner Gaussian of each sample */
    const float* d_eps;             /* [N,3] standard normal draws */
    void* d_workspace;              /* fb200_sugar_reg_workspace_bytes(P, K, N, with_grad) bytes */
} fb200_sugar_reg;
size_t fb200_sugar_reg_workspace_bytes(int32_t P, int32_t K, int32_t N, int32_t with_grad);
int fb200_sugar_reg_forward(const fb200_sugar_reg* r, int32_t with_grad, float* d_terms, void* stream);
/* d_dquaternions 16-byte aligned.  Needs a preceding fb200_sugar_reg_forward with_grad on the same workspace. */
int fb200_sugar_reg_backward(const fb200_sugar_reg* r, const float* d_dL_dterms, float* d_dpoints, float* d_dscaling,
                             float* d_dquaternions, float* d_dstrengths, void* stream);

/* SuGaR's depth-normal consistency of the coarse `dn_consistency` trainer (SURVEY.md row 17;
 * frosting_scene/sugar_model.py:2343-2387 render_depth_and_normal, frosting_trainers/coarse_density_and_dn_consistency.py
 * :17-95 depth_normal_consistency_loss).  The camera is the rasterizer's own: d_viewmatrix is world_view_transform and
 * d_projmatrix full_proj_transform (row-major [4,4], row-vector convention), d_campos the camera centre [3]; all stay on
 * the device.
 *
 * Features, one row per Gaussian, to be blended as 3 extra channels (fb200_extra) with background 0:
 *   n = the column of quaternion_to_matrix(q) (raw q, pytorch3d's two_s = 2/|q|^2) at the first minimal axis of s,
 *   n *= sign(n . (campos - p)) (0 gives a zero normal), features = {z, -(V n).x, -(V n).y} with V the COLMAP view
 *   rotation: z and the normal's x, y in pytorch3d's view frame, diag(-1, -1, 1) times the COLMAP one.
 * d_points, d_scaling, d_features [P,3]; d_quaternions [P,4] (w, x, y, z), 16-byte aligned.  The backward writes
 * dL/dpoints (through z only) and dL/dquaternions (16-byte aligned) from dL/dfeatures; dL/dscaling is zero (argmin is
 * discrete) and not written.
 *
 * Loss over the blended image d_dn [3,H,W]: depth dn[0], normal (-dn[1], -dn[2], -sqrt(1 - min(dn[1]^2 + dn[2]^2, 1)));
 * points d ray(x, y) at integer pixel coordinates, ray = c2w[:3,:3] K^-1 (x, y, 1) as depths_to_points derives it;
 * at interior pixels n_d = normalize(cross(P[r+1,c] - P[r-1,c], P[r,c+1] - P[r,c-1])) (eps 1e-12), 0 at border pixels;
 * d_loss[0] = mean over the H W pixels of 1 - normal . (n_d @ V[:3,:3]).  d_partials [fb200_sugar_dn_partials(H, W)].
 * The backward writes d_dL_ddn [3,H,W] (every element), scaled by the device scalar d_dL_dloss[0], without atomics.
 * H < 3 or W < 3: every pixel is a border pixel, the loss is 1 and the gradient 0, and no kernel is launched. */
int fb200_sugar_dn_features(int32_t P, const float* d_points, const float* d_scaling, const float* d_quaternions,
                            const float* d_viewmatrix, const float* d_campos, float* d_features, void* stream);
int fb200_sugar_dn_features_backward(int32_t P, const float* d_points, const float* d_scaling,
                                     const float* d_quaternions, const float* d_viewmatrix, const float* d_campos,
                                     const float* d_dL_dfeatures, float* d_dpoints, float* d_dquaternions,
                                     void* stream);
size_t fb200_sugar_dn_partials(int32_t H, int32_t W);
int fb200_sugar_dn_loss_forward(const float* d_dn, int32_t H, int32_t W, const float* d_viewmatrix,
                                const float* d_projmatrix, float* d_partials, float* d_loss, void* stream);
int fb200_sugar_dn_loss_backward(const float* d_dn, int32_t H, int32_t W, const float* d_viewmatrix,
                                 const float* d_projmatrix, const float* d_dL_dloss, float* d_dL_ddn, void* stream);

/* Exact K nearest neighbours (pytorch3d's knn_points(queries[None], points[None], K).dists[0] / .idx[0] with norm = 2;
 * SuGaR's neighbour table, frosting_scene/sugar_model.py:249, :1044-1061).  For each query q, d_dists [Q,K] and d_idx
 * [Q,K] hold the first K points p in ascending (d, index) order, compared lexicographically, where
 *   d = fmaf(dz, dz, fmaf(dy, dy, dx * dx)),  dx = q.x - p.x rounded to float32 (likewise y, z),
 * so the result is a function of the input bits alone: on distinct points a self query lists the point itself first
 * (d = 0), and ties go to the lower index.  d_queries NULL: the points themselves, Q == P.  Extents 1 <= K <= 32, K <= P,
 * Q >= 0 (Q = 0: nothing is launched); P and Q are int32, so below 2^31.  Point and query rows are [n,3] float32.
 * The inputs are specified for finite coordinates only; given any bits the call still terminates and writes indices in
 * [0, P), and the first int32 of the workspace becomes nonzero (stream-ordered) when a point or query coordinate is not
 * finite.  Stream-ordered on `stream`, no host synchronisation, no allocation.  The workspace is 256-byte aligned and
 * fb200_knn_workspace_bytes(P, Q, K) bytes for Q separate queries, (P, 0, K) for self queries: at most 48 bytes per
 * point plus 48 per separate query plus 72 KiB (0 for bad extents; host only, no CUDA call).  A shorter workspace is
 * FB200_ENOSPC. */
size_t fb200_knn_workspace_bytes(int32_t P, int32_t Q, int32_t K);
int fb200_knn(const float* d_points, int32_t P, const float* d_queries, int32_t Q, int32_t K, void* d_workspace,
              size_t workspace_bytes, float* d_dists, int64_t* d_idx, void* stream);

/* Frosting layer thickness: the level crossings of a Gaussian density field along the base mesh's vertex normals
 * (frosting_model.py compute_level_points_along_normals, :2016-2208, use_last_intersection_as_inner_level_point=True;
 * called twice by Frosting.__init__, :296-369).  One call runs, in order:
 *   normals   (d_faces given) d_normals[v] = the area-weighted normals cross(v2 - v1, v0 - v1) of the faces listed for v
 *             in the CSR d_vf_offsets / d_vf_faces, summed in that order and normalised with eps 1e-6 (pytorch3d's
 *             Meshes.verts_normals); otherwise d_normals is an input;
 *   proposal  (d_std_idx given) s_v = mean over the std_K Gaussians g = d_std_idx[v,k] of
 *             |scaling_g * quaternion_apply(quaternion_invert(q_g), n_v)| (pytorch3d's raw products), then
 *             d_inner_range[v] = std_range s_v and d_outer_range[v] = -std_range s_v; otherwise both are inputs;
 *   levels    t_j = f_j (inner_range - outer_range) + outer_range with f = d_fractions [n_samples] (torch.linspace(0, 1,
 *             n) as computed by the caller), sample x_j = vert + t_j n; over the K Gaussians g = d_knn_idx[v,k] in table
 *             order, d_j = sum_k strength_g exp(-clamp(|A_g^T (x_j - mu_g)|^2, 0, 1e8) / 2) with A_g =
 *             quaternion_to_matrix(q_g) diag(1 / clamp(s_g, 1e-8)), and d_j >= 1 becomes d_j / (d_j + 1e-12).  outer:
 *             linear interpolation of the level before the first sample above it, t_0 when that is sample 0; inner: after
 *             the last sample above it, t_{n-1} when that is sample n-1; a vertex with no sample above the level and
 *             d_0 < level gets (inner_range + outer_range) / 2 for both; then a layer thinner than min_layer is replaced
 *             by (inner_range + outer_range) / 2 -/+ half_layer, then inner = max(inner, d_min_clamp_inner) and outer =
 *             min(outer, d_max_clamp_outer) where given.  Written to d_level_outer / d_level_inner, d_densities [V,n] d_j
 *             where given;
 *   smoothing d_outer_dist[v] = the mean of d_level_outer over the smooth_K vertices d_smooth_idx[v,:] (smooth_K = 0:
 *             the value itself), likewise inner; d_outer_verts / d_inner_verts [V,3] = vert + dist n.
 * Extents: V >= 0, P >= 1, 1 <= K <= 32, K <= P, 1 <= n_samples <= 32, 0 <= smooth_K <= 32, 0 <= std_K <= 32 (>= 1 with
 * d_std_idx).  The neighbour tables are not checked and must lie in [0, P) (Gaussians) or [0, V) (vertices).  Every
 * array is float32 row-major unless marked; quaternions (w, x, y, z) raw, strengths [P] or [P,1].  Stream-ordered, no
 * host synchronisation, no allocation, no atomics: the outputs depend on the input bits alone. */
typedef struct fb200_frosting_init {
    int32_t n_verts, n_faces, P, K, n_samples, smooth_K, std_K;
    float level;
    float std_range;
    float min_layer;                    /* min_layer_size * spatial_extent rounded to float32, 0: none */
    float half_layer;                   /* 0.5 * min_layer_size * spatial_extent rounded to float32 */
    const float* d_verts;               /* [V,3] */
    const int32_t* d_faces;             /* [F,3] or NULL: d_normals is an input */
    const int32_t* d_vf_offsets;        /* [V+1] with d_faces */
    const int32_t* d_vf_faces;          /* [3F] with d_faces */
    float* d_normals;                   /* [V,3] */
    const float* d_points;              /* [P,3] */
    const float* d_scaling;             /* [P,3] activated */
    const float* d_quaternions;         /* [P,4] */
    const float* d_strengths;           /* [P] activated */
    const int64_t* d_knn_idx;           /* [V,K] */
    const int64_t* d_std_idx;           /* [V,std_K] or NULL: the ranges are inputs */
    float* d_inner_range;               /* [V] */
    float* d_outer_range;               /* [V] */
    const float* d_min_clamp_inner;     /* [V] or NULL */
    const float* d_max_clamp_outer;     /* [V] or NULL */
    const float* d_fractions;           /* [n_samples] */
    const int64_t* d_smooth_idx;        /* [V,smooth_K], NULL when smooth_K = 0 */
    float* d_level_outer;               /* [V] */
    float* d_level_inner;               /* [V] */
    float* d_outer_dist;                /* [V] */
    float* d_inner_dist;                /* [V] */
    float* d_outer_verts;               /* [V,3] */
    float* d_inner_verts;               /* [V,3] */
    float* d_densities;                 /* [V,n_samples] or NULL */
} fb200_frosting_init;
int fb200_level_points(const fb200_frosting_init* lp, void* stream);

/* Creating a Frosting layer from its thickness (frosting_model.py Frosting.__init__, :398-554, with
 * avoid_self_intersections, contract_points and use_softmax_for_bary_coords).  Four calls over one struct, in order:
 *   fb200_frosting_trim     the self-intersection trimming, n_iterations times: with d = 0 at first, every still active
 *                           vertex side tries d + step * init (a float32 multiply, then an add); the trial shell vertex is
 *                           vert + d n (multiply, then add) into d_shell [2V,3] (inner rows, then outer), each face's cell
 *                           centre is the left-to-right sum of its 6 shell vertices (inner corners, then outer) over 6
 *                           into d_centres; fb200_knn gives each of the 2V shell vertices its FB200_TRIM_K nearest
 *                           centres (d_knn_*, workspace as fb200_knn_workspace_bytes(F, 2V, 8)); a vertex is inside a
 *                           cell when all five projections (x - p_j) . n_j of is_inside_frosting (:1675-1737, n_j
 *                           F.normalize(cross(...)) with eps 1e-12) exceed inside_th.  Inside any of its 8 cells: the side
 *                           keeps its previous distance and stops (d_*_stop = the iteration); otherwise it takes the trial.
 *                           Never stopped: d_*_stop = n_iterations.  Needs F >= 8;
 *   fb200_frosting_volumes  d_volumes [F]: Heron's area of the face on contract(verts, camera centre, extent) times the
 *                           mean over its vertices of max(|d_inner_dist - d_outer_dist|, min_height), times (extent / |vert
 *                           - centre|)^2 beyond extent (contract = 0: plain vertices and heights);
 *   fb200_frosting_sample   per Gaussian i in cell d_cells[i]: u = d_u[i] with u_5 = 1, sorted; b_0 = u_0, b_k = u_k -
 *                           u_{k-1}; d_bary_logits = log(max(b, 1e-8)); d_points = sum_k b_k cell_k over the cell of
 *                           d_inner_verts / d_outer_verts (inner corners, then outer); d_max_scales the longest of the
 *                           cell's 3 sides and 6 base edges;
 *   fb200_frosting_finish   d_dist2 = distCUDA2's ((b_0 + b_1) + b_2) / 3 over the neighbours d_nn_idx[i, 1..3] (a K = 4
 *                           table over d_points, column 0 the point itself), each distance as simple-knn computes it for
 *                           sm_90a, fmaf(dz, dz, fmaf(dx, dx, dy * dy)), ascending; d_log_scales [N,3] = log(sqrt(max(min(
 *                           dist2, max_scale^2), 1e-7))); d_quats (1, 0, 0, 0); d_opacity_logits inverse_sigmoid(0.1);
 *                           d_sh_dc / d_sh_rest the rows d_sh_idx[i] of d_gs_sh_dc [n_gs,3] / d_gs_sh_rest [n_gs,sh_rest,3].
 * Tables are not checked and must lie in range.  Stream-ordered, no host synchronisation, no allocation, no atomics:
 * the outputs depend on the input bits alone. */
#define FB200_TRIM_K 8
typedef struct fb200_frosting_create {
    int32_t n_verts, n_faces, n_iterations, n_gaussians, n_gs, sh_rest, contract;
    float step;                         /* 1 / n_iterations rounded to float32 */
    float inside_th;                    /* spatial_extent * proj_th rounded to float32 */
    float extent;                       /* spatial_extent rounded to float32 */
    float min_height;                   /* min_frosting_size * spatial_extent rounded to float32 */
    const float* d_verts;               /* [V,3] base mesh */
    const int32_t* d_faces;             /* [F,3] */
    const float* d_normals;             /* [V,3] */
    const float* d_inner_init;          /* [V] the untrimmed distances */
    const float* d_outer_init;          /* [V] */
    const float* d_inner_verts;         /* [V,3] the untrimmed shell */
    const float* d_outer_verts;         /* [V,3] */
    float* d_inner_dist;                /* [V] trimmed (trim writes, volumes reads) */
    float* d_outer_dist;                /* [V] */
    int32_t* d_inner_stop;              /* [V] */
    int32_t* d_outer_stop;              /* [V] */
    float* d_shell;                     /* [2V,3] */
    float* d_centres;                   /* [F,3] */
    void* d_knn_workspace;
    size_t knn_workspace_bytes;
    float* d_knn_dists;                 /* [2V,8] */
    int64_t* d_knn_idx;                 /* [2V,8] */
    const float* d_camera_center;       /* [3] */
    float* d_volumes;                   /* [F] */
    const int64_t* d_cells;             /* [N] */
    const float* d_u;                   /* [N,6] */
    float* d_bary_logits;               /* [N,6] */
    float* d_points;                    /* [N,3] */
    float* d_max_scales;                /* [N] */
    const int64_t* d_nn_idx;            /* [N,4] */
    const int64_t* d_sh_idx;            /* [N] */
    const float* d_gs_sh_dc;            /* [n_gs,3] */
    const float* d_gs_sh_rest;          /* [n_gs,sh_rest,3] */
    float* d_dist2;                     /* [N] */
    float* d_log_scales;                /* [N,3] */
    float* d_quats;                     /* [N,4] */
    float* d_opacity_logits;            /* [N] */
    float* d_sh_dc;                     /* [N,3] */
    float* d_sh_rest;                   /* [N,sh_rest,3] */
} fb200_frosting_create;
int fb200_frosting_trim(const fb200_frosting_create* c, void* stream);
int fb200_frosting_volumes(const fb200_frosting_create* c, void* stream);
int fb200_frosting_sample(const fb200_frosting_create* c, void* stream);
int fb200_frosting_finish(const fb200_frosting_create* c, void* stream);

/* Data-parallel gradient reduction fused with the Adam update (SURVEY.md row f3).  Replaces "all-reduce every
 * .grad, then torch.optim.Adam(l, lr=0.0, eps=1e-15).step()" (frosting_scene/frosting_optimizer.py:101,116-118) for
 * camera-sharded training.  All learnable tensors of a rank live in ONE flat fp32 parameter slab and their gradients
 * in ONE gradient slab of the same indexing; group g owns elements [group_start[g], group_start[g+1]) (starts are
 * multiples of 4 elements) and has its own learning rate.  Rank `rank` owns elements [shard_lo, shard_hi) (multiples
 * of 4): it sums that range of all `world` gradient slabs in rank order, scales by grad_scale, updates ITS moments
 * (arrays of shard_hi - shard_lo elements) and stores the new parameters into all `world` parameter slabs.
 * peer_params / peer_grads hold device pointers valid on THIS device (fb200_peer_open for the other ranks' slabs;
 * entry `rank` is the local slab).  The caller orders the step after every rank's backward and orders the next
 * forward after every rank's step (two stream-ordered rendezvous, e.g. 4-byte NCCL all-reduces).  world == 1: plain
 * fused multi-group Adam.  bias_correction1 = 1 - beta1^t, bias_correction2_sqrt = sqrt(1 - beta2^t). */
#define FB200_ADAM_MAX_GROUPS 16
#define FB200_MAX_PEERS 8
typedef struct fb200_adam_args {
    int32_t world, rank;
    float* peer_params[FB200_MAX_PEERS];
    const float* peer_grads[FB200_MAX_PEERS];
    float* d_exp_avg;
    float* d_exp_avg_sq;
    int64_t shard_lo, shard_hi;
    int32_t n_groups;
    int64_t group_start[FB200_ADAM_MAX_GROUPS + 1];
    float lr[FB200_ADAM_MAX_GROUPS];   /* learning rate per group; NEGATIVE = skip the group this step (no gradient: its
                                        * moments and parameters stay untouched, like torch's `.grad is None`) */
    double beta1, beta2;   /* double: 1 - beta is formed in double like torch does, then rounded to fp32 */
    float eps;
    float bias_correction1, bias_correction2_sqrt;
    float grad_scale;
    /* Optional NVSwitch multicast mappings of the SAME slabs (NVLS; e.g. torch symmetric memory's multicast_ptr), both
     * or neither.  When given (and world > 1) the gradient shard is summed IN THE SWITCH (multimem.ld_reduce) and the
     * new parameters are broadcast by the switch (multimem.st): 1/world of the wire bytes of the peer-pointer path. */
    const float* mc_grads;
    float* mc_params;
    /* Sparse gradient rows (the producers' contract: fb200_grads.sparse_rows, frosting mode).  Optional, for all ranks or
     * none: peer_row_radii[r] is rank r's [row_count] radii of the frame that produced its gradient slab, mapped on THIS
     * device like peer_grads[r].  In a group with row_width[g] > 0, element j belongs to row j / row_width[g]; a row whose
     * radii is <= 0 on rank r is a ZERO row of r's gradient and its slab elements are NOT READ (they may be unwritten) --
     * ~90 % of a frosting layer per camera, so the step reads a tenth of the gradient bytes, locally and over NVLink.
     * The in-switch sum cannot skip rows: with row radii the gradients go through peer_grads and only the parameter
     * broadcast uses the multicast mapping. */
    const int32_t* peer_row_radii[FB200_MAX_PEERS];
    int32_t row_width[FB200_ADAM_MAX_GROUPS];   /* 0: the group has no row structure (always read) */
    int32_t row_count;
} fb200_adam_args;
int fb200_adam_step(const fb200_adam_args* args, void* stream);

/* Peer-mapped slabs for fb200_adam_step (cudaMalloc + cudaIpc*; the only device allocations this library makes, and
 * only on request).  fb200_peer_alloc zero-fills.  A handle is FB200_PEER_HANDLE_BYTES opaque bytes to be sent to the
 * other ranks of the box (any host transport); fb200_peer_open maps that slab into the calling process. */
#define FB200_PEER_HANDLE_BYTES 64
int fb200_peer_alloc(size_t bytes, void** d_ptr);
int fb200_peer_free(void* d_ptr);
int fb200_peer_export(void* d_ptr, unsigned char* handle /* [FB200_PEER_HANDLE_BYTES] */);
int fb200_peer_open(const unsigned char* handle, void** d_ptr);
int fb200_peer_close(void* d_ptr);

/* Introspection for parity tests: byte offsets of the internal arrays inside the caller's buffers,
 * so tests can compare depth bits / rects / records / ranges / point_list with the reference's
 * geomBuffer / binningBuffer / imgBuffer one-to-one (SURVEY.md section 8c). */
typedef struct fb200_layout {
    size_t geom_rec;       /* float4[3P]: {x,y,conic.x,conic.y},{conic.z,opacity,r,g},{b,ext_x,ext_y,depth} */
    size_t geom_depth;     /* f32[P]  view-space z (sort key bits) */
    size_t geom_rect;      /* u32[2P] (min.x | min.y<<16, max.x | max.y<<16) in tiles */
    size_t geom_clamped;   /* u8[P]   bit c = colour channel c was clamped */
    size_t img_final_T;    /* f32[H*W] */
    size_t img_n_contrib;  /* u32[H*W] */
    size_t img_ranges;     /* u32[2T]  (start,end) per tile, (0,0) for empty tiles */
    size_t img_tile_count; /* u32[T] */
    size_t bin_point_list; /* u32[capacity] sorted Gaussian index per instance */
    size_t bin_keys;       /* u64[capacity] (depth_bits<<32 | gaussian idx), sorted within each tile */
    size_t geom_acc;       /* f32[12P] the blend backward's per-Gaussian accumulators, the per-Gaussian backward's input:
                              {dmean2D.x, dmean2D.y, dconic.x, dconic.y}, {dconic.w, dopacity, dr, dg}, {db, e0, e1, e2}
                              (e*: extra feature channels).  Valid after fb200_backward until the next forward or
                              backward on the workspace */
    size_t img_last_entry; /* u32[H*W] per pixel: entries of its sub-tile's hit list up to and including its last
                              contributor (0: none), written by the forward blend */
    size_t bin_sub_hits;   /* u32[8*capacity] the hit lists of the 8 sub-tiles (8x4 pixels, row-major: w = 2 * row + col)
                              of every tile: Gaussian ids that passed the forward's sub-tile test, in tile-list order.
                              Sub-tile w of a tile with range [s, e) owns entries [8 s + w (e - s), + (e - s)); the first
                              max(last_entry) of them are valid */
} fb200_layout;

int fb200_get_layout(int32_t P, int32_t image_width, int32_t image_height, int64_t capacity,
                     fb200_layout* out);

/* Measurement hooks (bench.py's roofline block).  When enabled, every kernel stage of
 * fb200_forward / fb200_backward is bracketed by cudaEvents on the caller's stream (the stream the
 * kernels are launched on); fb200_profile_read() synchronises those events and returns the device
 * time of each stage of the most recent forward/backward pair.  Off by default: no events are recorded
 * and the hot path pays nothing. */
#define FB200_STAGE_PREPROCESS 0
#define FB200_STAGE_BINNING 1      /* tile scan + scatter + per-tile sort */
#define FB200_STAGE_RENDER_FWD 2   /* alpha-blend forward kernel alone */
#define FB200_STAGE_RENDER_BWD 3   /* alpha-blend backward kernel alone (accumulator memset excluded) */
#define FB200_STAGE_GEOM_BWD 4
#define FB200_NUM_STAGES 5
int fb200_profile_enable(int32_t enable);
int fb200_profile_read(float* ms_out /* [FB200_NUM_STAGES] */);
/* Number of kernels this library has launched in this process (all threads). */
int64_t fb200_kernel_launches(void);

const char* fb200_last_error(void);
int fb200_abi_version(void);
/* sizeof() of the ABI structs, in this order: {params, inputs, workspace, grads, extra, frosting_params,
 * frosting_grads, adam_args, layout, frosting_edit, frosting_skin, texture, sugar_reg, frosting_init,
 * frosting_create}: lets a
 * foreign-language binding verify its struct mirrors at load time.  `out` holds FB200_ABI_STRUCTS entries of this
 * header; structs are only ever appended to the list. */
#define FB200_ABI_STRUCTS 15
int fb200_abi_struct_sizes(size_t* out /* [FB200_ABI_STRUCTS] */);

#ifdef __cplusplus
}
#endif
#endif /* FROSTING_B200_H_ */
