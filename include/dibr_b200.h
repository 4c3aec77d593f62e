/*
 * dibr_b200.h — C ABI of libdibr_b200.so: H100 (sm_90a) kernels for Kaolin's
 * DIB-R hot path (rasterize + dibr_soft_mask, forward and backward).
 *
 * Plain pointers and sizes only; no torch / ATen types.  All pointers are DEVICE
 * pointers on the current CUDA device unless stated otherwise; all tensors are
 * dense row-major ("contiguous") fp32 / int64 / uint8 exactly as the reference
 * operators take them.  Nothing is allocated by the library: the caller passes
 * the outputs and a scratch `workspace` of at least dibr_b200_workspace_bytes().
 * Every output is fully written (no pre-zeroing needed).  Calls are asynchronous
 * on `stream` and never synchronise; they are re-entrant (no global state).
 *
 * Return value: 0 on success; DIBR_B200_E* (<0) for argument errors detected on
 * the host; a positive cudaError_t if a launch failed (cudaGetLastError()).
 * The fused entry points (dibr_b200_forward*, dibr_b200_backward*) check every
 * argument before they enqueue anything: an argument error leaves the outputs
 * untouched.
 *
 * Alignment: every non-NULL tensor pointer passed to dibr_b200_forward, _bf16,
 * _f64, dibr_b200_backward, _bf16, _views, _f64 (and so dibr_b200_rasterize_backward,
 * which calls dibr_b200_backward) must be 16-byte aligned; otherwise the call
 * returns DIBR_B200_EINVAL.  The kernels make 16-byte vector accesses on them.
 * A fresh allocation is aligned; a contiguous view at an element offset may not be
 * (the Python layer copies such inputs).  The workspace needs no alignment.
 *
 * The four "operator" entry points replace, one for one, the functions the
 * reference registers in kaolin/csrc/bindings.cpp:111-115; the two "fused"
 * entry points implement the same mathematics directly on the public-API
 * tensors (kaolin/render/mesh/dibr.py:119-209) without the packed temporaries.
 */
#ifndef DIBR_B200_H_
#define DIBR_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DIBR_B200_OK 0
#define DIBR_B200_EINVAL (-1)      /* null pointer / non-positive size / bad flag */
#define DIBR_B200_EWORKSPACE (-3)  /* workspace_bytes too small */
#define DIBR_B200_ESIZE (-4)       /* image larger than 16384 px or index overflow */

#define DIBR_B200_MAX_IMAGE_DIM 16384

/* forward `mode` bits */
#define DIBR_B200_RASTER 1     /* compute face_idx / weights / features */
#define DIBR_B200_SOFT_MASK 2  /* compute soft_mask */

/* backward `flags` bits */
#define DIBR_B200_BINS_VALID 1  /* workspace still holds forward's bins / hit cache for the same inputs */
#define DIBR_B200_ACCUMULATE 2  /* add into grad_face_vertices_image instead of overwriting it */

typedef struct CUstream_st* dibr_b200_stream_t; /* == cudaStream_t */

int dibr_b200_version(void);

/* Diagnostics: per-kernel device time of every launch made by the CALLING THREAD between
 * _begin and _end (thread-local: concurrent callers do not interact; no global state).
 * _end synchronises the recorded events, writes up to `capacity` durations (ms, launch
 * order) and the '\n'-separated kernel names, and returns the number of launches. */
int dibr_b200_trace_begin(void);
int dibr_b200_trace_end(char* names, size_t names_bytes, float* ms, int capacity);

/* Scratch needed by any entry point for `batch` views with `total_faces` faces
 * in all views together on a height x width image. */
size_t dibr_b200_workspace_bytes(int batch, int64_t total_faces, int height, int width);

/* Minimum scratch + a soft-mask hit cache for `cache_tiles` 16x16 screen tiles
 * (3072*knum + 16 bytes each).  Any workspace larger than the minimum is used by
 * dibr_b200_forward (mode & SOFT_MASK) to record, per tile that has any, the
 * (pixel, face, probability, distance type) hits — what the reference stores as
 * 13*knum bytes for EVERY pixel (dibr.py:49-54) — so that dibr_b200_backward with
 * bins_valid = 1 streams over them instead of recomputing the neighbour walk.
 * Tiles that do not fit are recomputed in backward; results are identical. */
size_t dibr_b200_workspace_bytes_cached(int batch, int64_t total_faces, int height, int width,
                                        int knum, int64_t cache_tiles);

/*
 * Fused forward on the public-API tensors.
 * Replaces: kaolin/render/mesh/rasterization.py:273-352 (RasterizeCuda.forward:
 * valid-face packing, x multiplier, bboxes, op call, index remap) and
 * kaolin/render/mesh/dibr.py:29-55 (DibrSoftMaskCuda.forward) in one pass.
 *
 *  face_vertices_z      (B,F,3)   f32
 *  face_vertices_image  (B,F,3,2) f32, NOT multiplied
 *  face_features        (B,F,3,D) f32 (may be NULL when D == 0)
 *  face_normals_z       (B,F) f32 or NULL: faces with value >= 0 are rasterized
 *  valid_faces          (B,F) u8  or NULL: faces with non-zero are rasterized
 *  boxlen_m             = (float)(boxlen * multiplier)   (dibr.py:36-37)
 *  mode                 DIBR_B200_RASTER | DIBR_B200_SOFT_MASK
 *  face_idx             (B,H,W) i64: output if RASTER, else INPUT (dibr_soft_mask alone)
 *  interpolated_features(B,H,W,D) f32: output if RASTER
 *  output_weights       (B,H,W,3) f32: output if RASTER, or NULL: the weights are not
 *                       written (dibr_b200_backward can recompute them, bit for bit)
 *  soft_mask            (B,H,W) f32: output if SOFT_MASK
 * The workspace keeps the face bins; pass it unchanged to dibr_b200_backward
 * with bins_valid = 1 to skip rebuilding them.
 */
int dibr_b200_forward(
    int batch, int num_faces, int height, int width, int feat_dim,
    const float* face_vertices_z, const float* face_vertices_image,
    const float* face_features, const float* face_normals_z, const uint8_t* valid_faces,
    float multiplier, float eps, int mode, float sigmainv, float boxlen_m, int knum,
    float* interpolated_features, int64_t* face_idx, float* output_weights, float* soft_mask,
    void* workspace, size_t workspace_bytes, dibr_b200_stream_t stream);

/*
 * Fused backward: grad wrt face_vertices_image (sum of the rasterize and the
 * soft-mask branches, as autograd would add them) and wrt face_features.
 * Replaces rasterization.py:355-371 + dibr.py:58-73 and the kernels behind them.
 *  grad_features  (B,H,W,D) f32 or NULL (skips the rasterize branch; grad_face_features is zeroed)
 *  grad_soft_mask (B,H,W)   f32 or NULL (skips the soft-mask branch)
 *  output_weights forward's output, or NULL: the rasterize branch recomputes each covered
 *                 pixel's weights from face_idx, face_vertices_image * multiplier and eps with
 *                 the forward's arithmetic (the same bits), so multiplier and eps MUST then be
 *                 the values the forward was called with
 *  soft_mask      forward's output (needed only with grad_soft_mask)
 *  flags          DIBR_B200_BINS_VALID: workspace still holds forward's bins for the same
 *                 inputs.  DIBR_B200_ACCUMULATE: grad_face_vertices_image is added to, not
 *                 zeroed first - lets a caller run the two branches as two calls (e.g. to
 *                 start sending grad_face_features while the soft-mask branch still runs);
 *                 grad_face_features is only touched when grad_features is given.
 *  workspace      may be NULL when grad_soft_mask is NULL.  When it is at least
 *                 dibr_b200_workspace_bytes() the rasterize branch (fp32 features, D <= 4,
 *                 width a multiple of 4) runs the row-walk kernel, which scatters into padded
 *                 per-face records in the workspace with 16-byte vector reductions; otherwise
 *                 the warp-reduction kernel scatters straight into the outputs.
 */
int dibr_b200_backward(
    int batch, int num_faces, int height, int width, int feat_dim,
    const float* grad_features, const float* grad_soft_mask,
    const int64_t* face_idx, const float* output_weights, const float* soft_mask,
    const float* face_vertices_image, const float* face_features,
    float multiplier, float eps, float sigmainv, float boxlen_m, int knum,
    float* grad_face_vertices_image, float* grad_face_features,
    void* workspace, size_t workspace_bytes, int flags, dibr_b200_stream_t stream);

/*
 * dibr_b200_backward restricted to the views [view_begin, view_end) of the batch.  ALL pointers are
 * the full-batch tensors and the forward's workspace (exactly what dibr_b200_backward takes;
 * grad_features / face_features hold bfloat16 bit patterns when features_bf16 != 0); only the rows
 * of grad_face_vertices_image / grad_face_features that belong to those views are written.  Lets a
 * caller pipeline the backward of one view chunk with the exchange (all-gather) of the previous
 * chunk's gradients: kaolin_b200.multi_gpu.pipelined_backward_all_gather.
 */
int dibr_b200_backward_views(
    int batch, int num_faces, int height, int width, int feat_dim,
    const void* grad_features, const float* grad_soft_mask,
    const int64_t* face_idx, const float* output_weights, const float* soft_mask,
    const float* face_vertices_image, const void* face_features, int features_bf16,
    float multiplier, float eps, float sigmainv, float boxlen_m, int knum,
    float* grad_face_vertices_image, float* grad_face_features,
    void* workspace, size_t workspace_bytes, int flags, int view_begin, int view_end,
    dibr_b200_stream_t stream);

/*
 * float64 instantiation of the fused entry points (the reference dispatches float and double:
 * rasterization_cuda.cu:218/427, dibr_soft_mask_cuda.cu:205/376; its tests parametrise the dtype).
 * Same contract as dibr_b200_forward / dibr_b200_backward with double tensors (face_idx stays i64).
 * multiplier is a double: the vertices are scaled by it in double, as the reference's wrappers do in
 * torch (rasterization.py:320, dibr.py:32); its float rounding is what the reference's kernels get, so
 * it places the pixel centres and is the multiplier of 4*m*m, the probability and the gradient
 * division.  eps / sigmainv are C floats as in the reference kernels' signatures; the enlarged-bbox
 * margin boxlen * multiplier is a double as in dibr.py:33-39.  Every per-pixel decision is taken with
 * the reference's <double> arithmetic, and face_idx, the weights, the features and the forward soft
 * mask are bit-identical to the reference's <double> kernels (tests/test_f64_matrix_gpu.py); the
 * gradients differ only in the order of the double atomics.  Built for exactness, not speed (one
 * thread per pixel walks its tile's bins; double atomics in the backward).  workspace >= dibr_b200_workspace_bytes_f64(); pass it unchanged to the backward with
 * DIBR_B200_BINS_VALID to reuse the forward's bins.
 */
size_t dibr_b200_workspace_bytes_f64(int batch, int64_t total_faces, int height, int width);
int dibr_b200_forward_f64(
    int batch, int num_faces, int height, int width, int feat_dim,
    const double* face_vertices_z, const double* face_vertices_image,
    const double* face_features, const double* face_normals_z, const uint8_t* valid_faces,
    double multiplier, float eps, int mode, float sigmainv, double boxlen_m, int knum,
    double* interpolated_features, int64_t* face_idx, double* output_weights, double* soft_mask,
    void* workspace, size_t workspace_bytes, dibr_b200_stream_t stream);
int dibr_b200_backward_f64(
    int batch, int num_faces, int height, int width, int feat_dim,
    const double* grad_features, const double* grad_soft_mask,
    const int64_t* face_idx, const double* output_weights, const double* soft_mask,
    const double* face_vertices_image, const double* face_features,
    double multiplier, float eps, float sigmainv, double boxlen_m, int knum,
    double* grad_face_vertices_image, double* grad_face_features,
    void* workspace, size_t workspace_bytes, int flags, dibr_b200_stream_t stream);

/*
 * bf16 feature storage (BASELINE.json configs[3], "bf16 features"; an extension - the
 * reference dispatches float/double only, rasterization_cuda.cu:218): same as
 * dibr_b200_forward / dibr_b200_backward except that face_features (B,F,3,D),
 * interpolated_features (B,H,W,D) and grad_features (B,H,W,D) hold bfloat16 bit patterns.
 * Arithmetic is the fp32 arithmetic of the fp32 entry points on the upcast values; the
 * interpolated feature is rounded to nearest-even once, on store, so it equals the fp32
 * entry point's output converted to bf16.  Geometry, weights, soft mask and BOTH output
 * gradients (fp32 accumulation) stay fp32.
 */
int dibr_b200_forward_bf16(
    int batch, int num_faces, int height, int width, int feat_dim,
    const float* face_vertices_z, const float* face_vertices_image,
    const uint16_t* face_features, const float* face_normals_z, const uint8_t* valid_faces,
    float multiplier, float eps, int mode, float sigmainv, float boxlen_m, int knum,
    uint16_t* interpolated_features, int64_t* face_idx, float* output_weights, float* soft_mask,
    void* workspace, size_t workspace_bytes, dibr_b200_stream_t stream);

int dibr_b200_backward_bf16(
    int batch, int num_faces, int height, int width, int feat_dim,
    const uint16_t* grad_features, const float* grad_soft_mask,
    const int64_t* face_idx, const float* output_weights, const float* soft_mask,
    const float* face_vertices_image, const uint16_t* face_features,
    float multiplier, float eps, float sigmainv, float boxlen_m, int knum,
    float* grad_face_vertices_image, float* grad_face_features,
    void* workspace, size_t workspace_bytes, int flags, dibr_b200_stream_t stream);

/*
 * Operator: kaolin::packed_rasterize_forward_cuda
 * (kaolin/csrc/render/mesh/rasterization.h:23-32, rasterization.cpp:49-104).
 * Packed valid faces of all meshes; coordinates already multiplied; tight bboxes
 * [xmin,ymin,xmax,ymax]; first_idx_face_per_mesh is a DEVICE int64 array (B+1).
 * selected_face_idx is relative to the mesh's first face, -1 = background.
 */
int dibr_b200_packed_rasterize_forward(
    int batch, int64_t total_faces, int height, int width, int feat_dim,
    const float* face_vertices_z, const float* face_vertices_image,
    const float* face_bboxes, const float* face_features,
    const int64_t* first_idx_face_per_mesh, float multiplier, float eps,
    float* interpolated_features, int64_t* selected_face_idx, float* output_weights,
    void* workspace, size_t workspace_bytes, dibr_b200_stream_t stream);

/*
 * Operator: kaolin::rasterize_backward_cuda
 * (rasterization.h:34-41, rasterization.cpp:106-168).  face_vertices_image is the
 * UNSCALED (B,F,3,2) tensor; selected_face_idx holds original face ids.
 * (The reference's `interpolated_features` argument is never read by its kernel
 * and is therefore not part of this ABI.)  output_weights is required (not NULL).
 */
int dibr_b200_rasterize_backward(
    int batch, int num_faces, int height, int width, int feat_dim,
    const float* grad_interpolated_features, const int64_t* selected_face_idx,
    const float* output_weights, const float* face_vertices_image,
    const float* face_features, float eps,
    float* grad_face_vertices_image, float* grad_face_features,
    dibr_b200_stream_t stream);

/*
 * Operator: kaolin::dibr_soft_mask_forward_cuda
 * (kaolin/csrc/render/mesh/dibr_soft_mask.h:23-30, dibr_soft_mask.cpp:48-108).
 * face_vertices_image already multiplied; face_large_bboxes (B,F,4).
 * close_face_prob (B,H,W,K) f32, close_face_idx (B,H,W,K) i64 (-1 padded),
 * close_face_dist_type (B,H,W,K) u8 (0 padded; 1-3 edge, 4-6 vertex).
 */
int dibr_b200_soft_mask_forward(
    int batch, int num_faces, int height, int width, int knum,
    const float* face_vertices_image, const float* face_large_bboxes,
    const int64_t* selected_face_idx, float sigmainv, float multiplier,
    float* soft_mask, float* close_face_prob, int64_t* close_face_idx,
    uint8_t* close_face_dist_type,
    void* workspace, size_t workspace_bytes, dibr_b200_stream_t stream);

/*
 * Operator: kaolin::dibr_soft_mask_backward_cuda
 * (dibr_soft_mask.h:32-42, dibr_soft_mask.cpp:110-183).
 */
int dibr_b200_soft_mask_backward(
    int batch, int num_faces, int height, int width, int knum,
    const float* grad_soft_mask, const float* soft_mask, const int64_t* selected_face_idx,
    const float* close_face_prob, const int64_t* close_face_idx,
    const uint8_t* close_face_dist_type, const float* face_vertices_image,
    float sigmainv, float multiplier, float* grad_face_vertices_image,
    dibr_b200_stream_t stream);

/* =========================================================================
 * The steps either side of the rasterizer in every DIB-R caller (SURVEY.md 8f rank 1, 2);
 * kaolin_b200/csrc/mesh_pipeline.cu.  The reference has no native interface for them: they
 * are chains of PyTorch ops (cited per entry point); the signatures below are what a
 * binding for a fused version would take.  No workspace; asynchronous on `stream`.
 * ========================================================================= */

/*
 * prepare_vertices (kaolin/render/mesh/utils.py:129-175): camera transform
 * (camera/legacy.py:22-37 with camera_rot (B,3,3) + camera_trans (B,3), or
 * [p,1] @ camera_transform (B,4,3); pass exactly one of the two), perspective divide
 * (camera/legacy.py:120-138; camera_proj_host = 3 floats on the HOST), gather by `faces`
 * (F,3) i64 (ops/mesh/mesh.py:54-76) and unit face normals (ops/mesh/trianglemesh.py:314-338).
 * Outputs: face_vertices_camera (B,F,3,3), face_vertices_image (B,F,3,2), face_normals (B,F,3).
 */
int dibr_b200_prepare_vertices_forward(
    int batch, int num_vertices, int num_faces, const float* vertices, const int64_t* faces,
    const float* camera_transform, const float* camera_rot, const float* camera_trans,
    const float* camera_proj_host, float* face_vertices_camera, float* face_vertices_image,
    float* face_normals, dibr_b200_stream_t stream);

/* Gradient wrt the CAMERA-SPACE vertices (B,V,3) (zeroed inside, scattered with float
 * atomics); any of the three upstream gradients may be NULL.  The linear map back to
 * world-space vertices / camera parameters is a (B,V,3)x(3,3) product left to the caller. */
int dibr_b200_prepare_vertices_backward(
    int batch, int num_vertices, int num_faces, const float* vertices, const int64_t* faces,
    const float* camera_transform, const float* camera_rot, const float* camera_trans,
    const float* camera_proj_host, const float* grad_face_vertices_camera,
    const float* grad_face_vertices_image, const float* grad_face_normals,
    float* grad_vertices_camera, dibr_b200_stream_t stream);

/*
 * texture_mapping (kaolin/render/mesh/utils.py:22-79): texture_coordinates (B,N,2) in [0,1]
 * (OpenGL convention), texture_maps (B,C,Ht,Wt); clamp, y flip,
 * grid_sample(align_corners=False, padding_mode='border'), mode nearest (1) or bilinear (0).
 * out (B,N,C).  Backward: grad_texture_maps (B,C,Ht,Wt) (zeroed inside) and/or
 * grad_texture_coordinates (B,N,2); either may be NULL.
 */
int dibr_b200_texture_mapping_forward(
    int batch, int64_t num_points, int channels, int tex_height, int tex_width,
    const float* texture_coordinates, const float* texture_maps, int nearest, float* out,
    dibr_b200_stream_t stream);
int dibr_b200_texture_mapping_backward(
    int batch, int64_t num_points, int channels, int tex_height, int tex_width,
    const float* texture_coordinates, const float* texture_maps, int nearest,
    const float* grad_out, float* grad_texture_maps, float* grad_texture_coordinates,
    dibr_b200_stream_t stream);

/*
 * mask_iou (kaolin/metrics/render.py:18-41): loss = 1 - mean_b(sum(l*r) / (sum(l+r-l*r) + 1e-10)).
 * sums (B,2) f32 scratch/output {sum(l*r), sum(l+r-l*r)} kept for the backward; loss: 1 f32.
 */
int dibr_b200_mask_iou_forward(
    int batch, int64_t pixels_per_view, const float* lhs_mask, const float* rhs_mask,
    float* sums, float* loss, dibr_b200_stream_t stream);
int dibr_b200_mask_iou_backward(
    int batch, int64_t pixels_per_view, const float* lhs_mask, const float* rhs_mask,
    const float* sums, const float* grad_loss, float* grad_lhs, float* grad_rhs,
    dibr_b200_stream_t stream);

/*
 * DefTet volumetric renderer operators (SURVEY.md 8f rank 3; kaolin_b200/csrc/deftet.cu).
 * Operator: kaolin::deftet_sparse_render_forward_cuda (kaolin/csrc/render/mesh/deftet.h,
 * deftet.cpp:48-113, kernel deftet_cuda.cu:31-194; registered at bindings.cpp next to the four
 * DIB-R operators).  For every query point the first `knum` faces IN INDEX ORDER whose half-open
 * bbox holds the point, whose eps-normalised barycentric weights are all >= 0 and whose
 * interpolated depth lies in [render_ranges[...,0], render_ranges[...,1]).
 *  face_vertices_z (B,F,3), face_vertices_image (B,F,3,2), face_bboxes (B,F,4) [xmin,ymin,xmax,ymax],
 *  pixel_coords (B,P,2), render_ranges (B,P,2)  f32
 *  outputs (B,P,K): face_idx i64 (-1 padded), pixel_depth f32 (-inf padded), w0, w1 f32 (0 padded),
 *  fully written.  workspace >= dibr_b200_deftet_workspace_bytes(batch, num_faces).
 */
size_t dibr_b200_deftet_workspace_bytes(int batch, int num_faces);
int dibr_b200_deftet_sparse_render_forward(
    int batch, int num_faces, int num_pixels, int knum,
    const float* face_vertices_z, const float* face_vertices_image, const float* face_bboxes,
    const float* pixel_coords, const float* render_ranges, float eps,
    int64_t* face_idx, float* pixel_depth, float* w0, float* w1,
    void* workspace, size_t workspace_bytes, dibr_b200_stream_t stream);

/*
 * Operator: kaolin::deftet_sparse_render_backward_cuda (deftet.cpp:115-170, kernel
 * deftet_cuda.cu:238-430).  grad_interpolated_features (B,P,K,D), face_idx (B,P,K) i64,
 * weights (B,P,K,3), face_vertices_image (B,F,3,2), face_features (B,F,3,D);
 * outputs grad_face_vertices_image (B,F,3,2), grad_face_features (B,F,3,D), zeroed inside.
 */
int dibr_b200_deftet_sparse_render_backward(
    int batch, int num_faces, int num_pixels, int knum, int feat_dim,
    const float* grad_interpolated_features, const int64_t* face_idx, const float* weights,
    const float* face_vertices_image, const float* face_features, float eps,
    float* grad_face_vertices_image, float* grad_face_features, dibr_b200_stream_t stream);

/*
 * Diffuse lighting (kaolin/render/lighting/sg.py, sh.py; kaolin_b200/csrc/lighting.cu).
 *
 * General reduced SG inner product, the operator kaolin::unbatched_reduced_sg_inner_product_
 * {forward,backward}_cuda: sg side amplitude (N,3), direction (N,3), sharpness (N); "other" side
 * (M,3), (M,3), (M); out (N,3) = sum_m <sg_n, other_m> with, per pair, v = lambda d + Lambda D,
 * um = |v|, <.,.> = 2 pi a A exp(um - lambda - Lambda) (1 - exp(-2 um)) / um.  The backward writes
 * any subset of the six gradients; a NULL gradient is not computed.  The "other"-side gradients
 * need workspace >= dibr_b200_sg_inner_product_workspace_bytes(M) (NULL when none is requested).
 *
 * Diffuse shading of N points lit by L lights, `model` one of:
 *  SG_INNER_PRODUCT  sg_diffuse_inner_product / sg_irradiance_inner_product: the cosine lobe
 *                    (amplitude 1.17, direction = normal, sharpness 2.133) against each light,
 *                    summed over lights, clamp(min=0), x albedo/pi.
 *  SG_FITTED         sg_diffuse_fitted: Stephen Hill's fitted irradiance per (point, light), MEAN over
 *                    lights, clamp(min=0), x albedo/pi.  L = 0 gives zeros (the reference's mean of an
 *                    empty set is NaN).
 *  SH9               sh9_diffuse / sh9_irradiance: sum_k band_k(normal) c_k lights_k, x albedo, no
 *                    clamp; light_amplitude holds the 9 coefficients and num_lights must be 1.
 * light_amplitude (L,3), light_direction (L,3), light_sharpness (L); normal (N,3) (not normalised);
 * albedo (N,3) or NULL.  out (N,3); with albedo == NULL the irradiance alone: (N,3) for the SG
 * models, (N,) for SH9.  The backward writes grad_normal, grad_albedo (both optional, per point)
 * and the light gradients (optional; SG: amplitude, direction, sharpness; SH9: the 9 coefficients
 * in grad_light_amplitude), which need workspace >= dibr_b200_diffuse_workspace_bytes(model, L).
 *
 * Light gradients are bit-reproducible: no float atomics; per-CTA partials summed in a fixed order
 * in fp64.  The workspace does not depend on N: 264 CTA slots x 7 floats per light (SH9: 9 floats)
 * = 7.4 KB per light.  Per-point data is read once for any L (kept in registers while the lights
 * are streamed through shared memory); with only light gradients requested the backward reads
 * grad_out, normal and albedo and writes nothing per point.  Clamp gradients pass where the input is
 * >= 0, as torch.clamp's do.
 * The formulas are the reference's, literally, in fp32.  Where the reference itself produces inf or
 * NaN the result is unspecified: um = 0 (opposite directions of equal sharpness), sharpness 0, and
 * sharpness so small that sqrt(1 - scale) is 0 in the fitted model.
 */
#define DIBR_B200_LIGHT_SG_INNER_PRODUCT 0
#define DIBR_B200_LIGHT_SG_FITTED 1
#define DIBR_B200_LIGHT_SH9 2

size_t dibr_b200_sg_inner_product_workspace_bytes(int num_other);
int dibr_b200_sg_inner_product_forward(
    int64_t num_sg, int num_other, const float* amplitude, const float* direction, const float* sharpness,
    const float* other_amplitude, const float* other_direction, const float* other_sharpness, float* out,
    dibr_b200_stream_t stream);
int dibr_b200_sg_inner_product_backward(
    int64_t num_sg, int num_other, const float* grad_out, const float* amplitude, const float* direction,
    const float* sharpness, const float* other_amplitude, const float* other_direction,
    const float* other_sharpness, float* grad_amplitude, float* grad_direction, float* grad_sharpness,
    float* grad_other_amplitude, float* grad_other_direction, float* grad_other_sharpness,
    void* workspace, size_t workspace_bytes, dibr_b200_stream_t stream);

size_t dibr_b200_diffuse_workspace_bytes(int model, int num_lights);
int dibr_b200_diffuse_forward(
    int model, int64_t num_points, int num_lights, const float* light_amplitude, const float* light_direction,
    const float* light_sharpness, const float* normal, const float* albedo, float* out,
    dibr_b200_stream_t stream);
int dibr_b200_diffuse_backward(
    int model, int64_t num_points, int num_lights, const float* light_amplitude, const float* light_direction,
    const float* light_sharpness, const float* normal, const float* albedo, const float* grad_out,
    float* grad_normal, float* grad_albedo, float* grad_light_amplitude, float* grad_light_direction,
    float* grad_light_sharpness, void* workspace, size_t workspace_bytes, dibr_b200_stream_t stream);

/*
 * Specular lighting (kaolin/render/lighting/sg.py sg_warp_specular_term; kaolin_b200/csrc/lighting.cu):
 * the Cook-Torrance SG specular term of DIB-R++ for N points lit by L spherical-Gaussian lights
 * light_amplitude (L,3), light_direction (L,3), light_sharpness (L).  Per point: normal n (N,3), not
 * normalised; roughness r (N); view v (N,3), the direction towards the camera; spec_albedo s (N,3).
 *   m2 = r^2; lobe amplitude a = 1 / (pi m2) in all three channels;
 *   w  = -v - 2 ((-v).n) n;  ws = (2 / m2) / (4 max(n.v, 1e-4))
 *   acc = sum_l <(a, w, ws), light_l>   (the SG inner product of the general operator above)
 *   ndl = clamp(n.w, 0, 1), ndv = clamp(n.v, 0, 1), h = (w + v) / sqrt((w + v).(w + v)),
 *   ldh = clamp(w.h, 0, 1), V(x) = 1 / (x + sqrt(m2 + (1 - m2) x^2))
 *   out (N,3) = clamp(acc V(ndl) V(ndv) (s + (1 - s) (1 - ldh)^5) ndl, min=0)
 * in fp32, with the reference's formulas and nothing normalised that the reference does not
 * normalise.  The backward writes any subset of grad_normal (N,3), grad_roughness (N), grad_view
 * (N,3), grad_spec_albedo (N,3) and the light gradients; a NULL gradient is not computed, and with
 * only light gradients requested nothing is written per point.  Clamp gradients pass where
 * min <= x <= max, as torch.clamp's do.  Light gradients need workspace >=
 * dibr_b200_specular_workspace_bytes(L) = 264 CTA slots x 7 floats = 7.4 KB per light, independent
 * of N; they are bit-reproducible, as the diffuse models' are.  L = 0 gives zero output and zero
 * per-point gradients (the reference's empty sum); N = 0 does nothing per point.
 * Unspecified, as the reference itself gives inf or NaN there: roughness 0, and w + v = 0 (a unit
 * normal exactly perpendicular to the view).
 */
size_t dibr_b200_specular_workspace_bytes(int num_lights);
int dibr_b200_specular_forward(
    int64_t num_points, int num_lights, const float* light_amplitude, const float* light_direction,
    const float* light_sharpness, const float* normal, const float* roughness, const float* view,
    const float* spec_albedo, float* out, dibr_b200_stream_t stream);
int dibr_b200_specular_backward(
    int64_t num_points, int num_lights, const float* light_amplitude, const float* light_direction,
    const float* light_sharpness, const float* normal, const float* roughness, const float* view,
    const float* spec_albedo, const float* grad_out, float* grad_normal, float* grad_roughness,
    float* grad_view, float* grad_spec_albedo, float* grad_light_amplitude, float* grad_light_direction,
    float* grad_light_sharpness, void* workspace, size_t workspace_bytes, dibr_b200_stream_t stream);

/*
 * Deferred shading (kaolin/render/easy_render/mesh.py:427-464 sg_shade; kaolin_b200/csrc/lighting.cu):
 * the diffuse and specular terms above for every pixel of a (B, H, W) G-buffer, in one pass per
 * pixel.  Per view b (camera, B x 16 floats): R (3x3 row-major, world to camera), tan_x =
 * (camera width / 2) / focal_x, tan_y likewise, x0, y0, camera width, camera height, one unused float.
 * Per pixel (i, j): face_idx (B,H,W) int64; albedo, spec_albedo, normals (B,H,W,3); roughness (B,H,W).
 *   face_idx < 0 (background): diffuse = specular = img = 0, every per-pixel gradient 0, and the
 *     pixel adds nothing to the light gradients;
 *   n = normals / max(|normals|, 1e-12)                                (F.normalize)
 *   pixel = ((j + 1/2) cw / W - x0, (i + 1/2) ch / H + y0), ndc = 2 pixel / (cw, ch) - 1,
 *   d = (ndc_x tan_x, -ndc_y tan_y, -1), v = -R^T d / |R^T d|          (kaolin/render/camera/raygen.py,
 *     the custom-resolution pixel grid; fp32, in the reference's order of operations)
 *   diffuse  = dibr_b200_diffuse_forward(SG_INNER_PRODUCT) of (n, albedo)
 *   specular = dibr_b200_specular_forward of (n, roughness, v, spec_albedo)
 *   img      = diffuse + specular                                       all (B,H,W,3) float32
 * Every output element is written.  The backward takes any subset of grad_diffuse, grad_specular and
 * grad_img (NULL counts as zero); the diffuse term sees grad_diffuse + grad_img and the specular term
 * grad_specular + grad_img.  It writes any subset of grad_albedo, grad_spec_albedo, grad_roughness,
 * grad_normals (through the normalisation) and the light gradients; a NULL gradient is not
 * computed, and with only light gradients requested nothing is written per pixel.  The camera gets
 * no gradient.  Light gradients need workspace >= dibr_b200_sg_shade_workspace_bytes(L) = 7.4 KB per
 * light, independent of the pixel count, and are bit-reproducible.  H or W above 16384 gives
 * DIBR_B200_ESIZE; negative sizes or a NULL input that is read give DIBR_B200_EINVAL, before any
 * CUDA call.  Unspecified, where the reference itself gives inf or NaN: a covered pixel of roughness 0,
 * or whose unit normal is exactly perpendicular to its view (w + v = 0).
 */
size_t dibr_b200_sg_shade_workspace_bytes(int num_lights);
int dibr_b200_sg_shade_forward(
    int batch, int height, int width, int num_lights, const float* camera, const int64_t* face_idx,
    const float* albedo, const float* spec_albedo, const float* roughness, const float* normals,
    const float* light_amplitude, const float* light_direction, const float* light_sharpness, float* diffuse,
    float* specular, float* img, dibr_b200_stream_t stream);
int dibr_b200_sg_shade_backward(
    int batch, int height, int width, int num_lights, const float* camera, const int64_t* face_idx,
    const float* albedo, const float* spec_albedo, const float* roughness, const float* normals,
    const float* light_amplitude, const float* light_direction, const float* light_sharpness,
    const float* grad_diffuse, const float* grad_specular, const float* grad_img, float* grad_albedo,
    float* grad_spec_albedo, float* grad_roughness, float* grad_normals, float* grad_light_amplitude,
    float* grad_light_direction, float* grad_light_sharpness, void* workspace, size_t workspace_bytes,
    dibr_b200_stream_t stream);

/*
 * Mesh topology, uniform Laplacian and vertex averaging (kaolin_b200/csrc/mesh_topology.cu) for one
 * mesh of V vertices and F faces of S >= 3 vertices, `faces` (F, S) int64.  The reference builds dense
 * V x V matrices; these entry points work on two CSR structures built once by
 * dibr_b200_mesh_topology_build, in caller-owned int32 buffers:
 *   corner_ptr (V+1), corners (F*S)  for vertex i, the corners f*S + k with faces[f, k] == i, in the
 *                                    order of the key k*F + f (that of the reference's per-corner
 *                                    scatter_add_ loop, kaolin/ops/mesh/mesh.py:202-204)
 *   adj_ptr (V+1), adj (2*F*S)       for vertex i, its unique neighbours faces[f, (k +- 1) mod S] in
 *                                    ascending order (the unique `roll` pairs of mesh.py:100-103); the
 *                                    first adj_ptr[V] entries are used.  A degenerate face gives a
 *                                    self-loop i -> i.  Quads give their four cyclic edges.
 *   degree (V) int32, weight (V) f32 the number of neighbours (self-loop included) and 1.0f / degree
 *                                    as an IEEE division (0 for degree 0)
 *   status (2) int32                 {adj_ptr[V], error}: error is non-zero when a face index lies
 *                                    outside [0, V).  Such a corner is counted and written nowhere;
 *                                    the topology is then not usable.  (Deliberate deviation: the
 *                                    reference does not check; on the CPU it drops an index >= V from
 *                                    its sparse matrix, and a negative index writes out of bounds.)
 * The build needs V < 2^31 - 1 and 2*F*S < 2^31 (else DIBR_B200_ESIZE) and workspace >=
 * dibr_b200_mesh_topology_workspace_bytes(); it is deterministic and never needs O(V^2) memory.
 * Read status to know the edge count; nothing else has to come back to the host.
 */
size_t dibr_b200_mesh_topology_workspace_bytes(int num_vertices, int64_t num_faces, int face_size);
int dibr_b200_mesh_topology_build(int num_vertices, int64_t num_faces, int face_size, const int64_t* faces,
                                  int32_t* corner_ptr, int32_t* corners, int32_t* adj_ptr, int32_t* adj,
                                  int32_t* degree, float* weight, int32_t* status, void* workspace,
                                  size_t workspace_bytes, dibr_b200_stream_t stream);

/*
 * uniform_laplacian (kaolin/ops/mesh/mesh.py:116-151) applied without the matrix: L[i, i] = -1,
 * L[i, j] = weight[i] for the neighbours j != i, 0 elsewhere; x and y (batch, V, channels) f32.
 *   transpose = 0: y = L x      y_i = weight_i sum_{j in N(i), j != i} x_j - x_i
 *   transpose = 1: y = L^T x    y_j = sum_{i in N(j), i != j} weight_i x_i - x_j   (the backward)
 *   smooth = 1:    without the -x term, i.e. (L + I) x: uniform_laplacian_smoothing
 *                  (kaolin/metrics/trianglemesh.py:318-350)
 * A gather per output element (no atomics: bit-reproducible), sums in adjacency order, in fp32.
 */
int dibr_b200_laplacian_apply(int batch, int num_vertices, int channels, const int32_t* adj_ptr, const int32_t* adj,
                              const float* weight, const float* x, int transpose, int smooth, float* y,
                              dibr_b200_stream_t stream);

/*
 * average_face_vertex_features / compute_vertex_normals (kaolin/ops/mesh/mesh.py:154-208):
 * face_features (batch, F, S, channels) f32 -> out (batch, V, channels): per vertex the sum over its
 * corners in key order, divided by max(count, 1).  Backward: grad_face_features[b, f, k, c] =
 * grad_out[b, faces[f, k], c] / max(count, 1).
 */
int dibr_b200_vertex_average_forward(int batch, int num_vertices, int64_t num_faces, int face_size, int channels,
                                     const int32_t* corner_ptr, const int32_t* corners, const float* face_features,
                                     float* out, dibr_b200_stream_t stream);
int dibr_b200_vertex_average_backward(int batch, int num_vertices, int64_t num_faces, int face_size, int channels,
                                      const int64_t* faces, const int32_t* corner_ptr, const float* grad_out,
                                      float* grad_face_features, dibr_b200_stream_t stream);

/*
 * Dense (V, V) f32 from the adjacency CSR, every element written: laplacian = 1 gives
 * uniform_laplacian (mesh.py:116-151), laplacian = 0 adjacency_matrix(sparse=False) (mesh.py:78-114).
 * dibr_b200_adjacency_coo writes the (2, num_edges) int64 indices of adjacency_matrix(sparse=True):
 * rows and columns in CSR (lexicographic) order, which is the order of the reference's unique(dim=0).
 */
int dibr_b200_mesh_dense(int num_vertices, int laplacian, const int32_t* adj_ptr, const int32_t* adj,
                         const float* weight, float* out, dibr_b200_stream_t stream);
int dibr_b200_adjacency_coo(int num_vertices, int64_t num_edges, const int32_t* adj_ptr, const int32_t* adj,
                            int64_t* indices, dibr_b200_stream_t stream);

/*
 * One level of Loop subdivision (kaolin/ops/mesh/trianglemesh.py:482-612, subdivide_trianglemesh) for
 * a triangle mesh of V vertices and F faces (F, 3) int64, on top of its topology
 * (dibr_b200_mesh_topology_build with face_size 3).  The reference's unique edges in lexicographic
 * order are the adjacency entries (i, j) with j >= i, in CSR order; edge e becomes vertex V + e.
 * dibr_b200_loop_subdivision_build writes, in caller-owned buffers:
 *   edge_ptr (V+1) int32          exclusive scan over rows of the number of neighbours j >= i;
 *                                 edge_ptr[V] = E, the edge count (E <= 3F)
 *   adj_edge (2*F*3) int32        the edge id of every adjacency entry (first adj_ptr[V] used)
 *   face_edge (F, 3) int32        the ids of edges (f0,f1), (f1,f2), (f2,f0) of each face (the
 *                                 reference's inverse_indices)
 *   edges (3F, 4) int32           first E rows: {a, b, f0, f1}, a <= b the endpoints; f0 <= f1 the
 *                                 faces of its two face edges when it has exactly two, else -1, -1
 *   new_faces (4F, 3) int64       the next level's faces: for each face, in face order,
 *                                 (v0, v1, v2, V+e01, V+e12, V+e20)[[1,4,3], [0,3,5], [2,5,4], [5,3,4]]
 *   status (1) int32              E.  Read it to size the next level; nothing else has to come back.
 * Needs workspace >= dibr_b200_loop_subdivision_workspace_bytes(); no atomics, deterministic.  When the
 * topology build reported an index outside [0, V), the outputs are not usable.
 *
 * dibr_b200_loop_subdivision_forward: vertices (batch, V, 3) f32 -> out (batch, V + E, 3), one thread
 * per output vertex, reading vertices only (the odd vertices use the input, not the updated ones):
 *   even i   (1 - a_i) x_i + (a_i / n_i) sum_{j in N(i)} x_j      n_i = the degree, self-loop included
 *   odd e    two faces: (both faces' 3 vertices + both endpoints) / 8; otherwise (x_a + x_b) / 2
 * alpha NULL: a_i = the reference's default weight _get_alpha(n_i) * n_i in fp32 (NaN for n_i = 0).
 * alpha (batch, V) f32: a_i = alpha[b, i]; alpha_out (batch, V + E) or NULL gets the next level's
 * alpha: alpha[b, i] for even rows, the odd stencils over alpha for odd rows.
 *
 * dibr_b200_loop_subdivision_backward: the transpose, one thread per input vertex, as gathers over the
 * same structures (adjacency entries: neighbours and edge endpoints; corners -> face_edge: the 1/8 face
 * terms of two-face edges).  grad_out (batch, V + E, 3); grad_alpha_out (batch, V + E) or NULL (zero);
 * grad_vertices (batch, V, 3) or NULL; grad_alpha (batch, V) or NULL, which needs alpha and vertices:
 *   grad_alpha_i = (g_i . sum_{j in N(i)} x_j) / n_i - g_i . x_i + the gradient through alpha_out,
 *   the first two terms in fp64 (they nearly cancel on a smooth surface).
 * No atomics: every output is bit-reproducible.
 */
size_t dibr_b200_loop_subdivision_workspace_bytes(int num_vertices, int64_t num_faces);
int dibr_b200_loop_subdivision_build(int num_vertices, int64_t num_faces, const int64_t* faces,
                                     const int32_t* corner_ptr, const int32_t* corners, const int32_t* adj_ptr,
                                     const int32_t* adj, int32_t* edge_ptr, int32_t* adj_edge, int32_t* face_edge,
                                     int32_t* edges, int64_t* new_faces, int32_t* status, void* workspace,
                                     size_t workspace_bytes, dibr_b200_stream_t stream);
int dibr_b200_loop_subdivision_forward(int batch, int num_vertices, int num_edges, const int32_t* adj_ptr,
                                       const int32_t* adj, const int32_t* edges, const int64_t* faces,
                                       const float* vertices, const float* alpha, float* out, float* alpha_out,
                                       dibr_b200_stream_t stream);
int dibr_b200_loop_subdivision_backward(int batch, int num_vertices, int num_edges, const int32_t* corner_ptr,
                                        const int32_t* corners, const int32_t* adj_ptr, const int32_t* adj,
                                        const int32_t* adj_edge, const int32_t* face_edge, const int32_t* edges,
                                        const float* vertices, const float* alpha, const float* grad_out,
                                        const float* grad_alpha_out, float* grad_vertices, float* grad_alpha,
                                        dibr_b200_stream_t stream);

/*
 * Tet-mesh topology for `tets` (T, 4) int64 over V vertices (csrc/mesh_topology.cu): the adjacency of
 * dibr_b200_mesh_topology_build, but with all three other corners of a tet as each corner's
 * neighbours, so every tet contributes its six edges (faces keep their cyclic edges).  Edges are
 * numbered as for Loop subdivision: the adjacency entries (i, j) with j >= i in CSR order, which is
 * the lexicographic order of the reference's unique(dim=0) over the tets' sorted edges; a degenerate
 * tet's self-loop (i, i) is an edge.  dibr_b200_tet_topology_build writes, in caller-owned buffers:
 *   adj_ptr (V+1), adj (12T) int32   the adjacency CSR (first adj_ptr[V] entries used)
 *   edges (6T, 2) int32              first E rows: {a, b}, a <= b
 *   adj_edge (12T) int32             the edge id of every adjacency entry, in both directions
 *   tet_edge (T, 6) int32            the edge ids of corner pairs 01, 02, 03, 12, 13, 23 of each tet
 *   status (3) int32                 {E, error, adj_ptr[V]}: error is non-zero when a tet index lies
 *                                    outside [0, V); the outputs are then not usable.
 * Needs 12T < 2^31 and V < 2^31 - 1 (else DIBR_B200_ESIZE) and workspace >=
 * dibr_b200_tet_topology_workspace_bytes(); deterministic.  Read status; nothing else comes back.
 */
size_t dibr_b200_tet_topology_workspace_bytes(int num_vertices, int64_t num_tets);
int dibr_b200_tet_topology_build(int num_vertices, int64_t num_tets, const int64_t* tets, int32_t* adj_ptr,
                                 int32_t* adj, int32_t* edges, int32_t* adj_edge, int32_t* tet_edge, int32_t* status,
                                 void* workspace, size_t workspace_bytes, dibr_b200_stream_t stream);

/*
 * Marching tetrahedra (kaolin/ops/conversions/tetmesh.py:57-168) for B views of one tet grid, on its
 * topology (above).  occ = sdf > 0 (0 and NaN are outside).  Each view's output vertices are its
 * sign-change edges (occ(a) != occ(b)) in edge order, at (x_a (-s_b) + x_b s_a) / (s_a + (-s_b)),
 * each step rounded as the reference's element-wise ops.  A tet's case is sum_k occ(corner k) 2^k;
 * its faces follow the case table (dibr_b200_marching_tets_case_table), those of one-triangle tets
 * first, in tet order, then both of each two-triangle tet, in tet order.
 *   dibr_b200_marching_tets_count: flags every (view, edge) and classifies every (view, tet), and
 *     writes scan (B*(E + 2T) + 1) int32, the exclusive scan of [edge flags | one-triangle | two-
 *     triangle flags], and counts (B, 3) int32 {vertices, one-triangle tets, two-triangle tets}: the
 *     one value to read back to size the outputs.  Workspace >= dibr_b200_marching_tets_workspace_bytes.
 *   dibr_b200_marching_tets_emit: writes, all views in one array each, view after view,
 *     out_vertices (sum nv, 3) f32, out_faces (sum nf, 3) int64 (vertex ids per view, nf = n1 + 2 n2),
 *     out_tet_idx (sum nf) int64 or NULL, and vid (B, E) int32: the row of each (view, edge) in
 *     out_vertices, -1 where the edge has no sign change.
 *   dibr_b200_marching_tets_backward: grad_out (sum nv, 3) -> grad_vertices (B, V, 3) and grad_sdf
 *     (B, V), either NULL: one thread per (view, vertex) over its adjacency row, no atomics.
 * B*(E + 2T) must be < 2^31 - 1 (else DIBR_B200_ESIZE).
 * dibr_b200_marching_tets_case_table (host): pairs (16, 2, 3, 2) int32, the corners (i, j) of the edge
 * of each vertex of each triangle of each case, -1 where the case has fewer triangles.
 */
int dibr_b200_marching_tets_case_table(int32_t* pairs);
size_t dibr_b200_marching_tets_workspace_bytes(int batch, int num_edges, int64_t num_tets);
int dibr_b200_marching_tets_count(int batch, int num_vertices, int num_edges, int64_t num_tets, const int32_t* edges,
                                  const int64_t* tets, const float* sdf, int32_t* scan, int32_t* counts,
                                  void* workspace, size_t workspace_bytes, dibr_b200_stream_t stream);
int dibr_b200_marching_tets_emit(int batch, int num_vertices, int num_edges, int64_t num_tets, const int32_t* edges,
                                 const int64_t* tets, const int32_t* tet_edge, const float* vertices, const float* sdf,
                                 const int32_t* scan, int32_t* vid, float* out_vertices, int64_t* out_faces,
                                 int64_t* out_tet_idx, dibr_b200_stream_t stream);
int dibr_b200_marching_tets_backward(int batch, int num_vertices, int num_edges, const int32_t* adj_ptr,
                                     const int32_t* adj, const int32_t* adj_edge, const float* vertices,
                                     const float* sdf, const int32_t* vid, const float* grad_out,
                                     float* grad_vertices, float* grad_sdf, dibr_b200_stream_t stream);

/*
 * subdivide_tetmesh (kaolin/ops/mesh/tetmesh.py:85-181) on the tet topology: vertices (B, V, 3) and
 * features (B, V, channels) or NULL -> out_vertices (B, V + E, 3), out_features: rows < V copied, row
 * V + e the midpoint (y_a + y_b) * 0.5 of edge e; out_tets (8T, 4) int64 or NULL: child k of tet t at
 * row k*T + t, over (v0, v1, v2, v3, V+e01, V+e02, V+e03, V+e12, V+e13, V+e23):
 *   [0,4,5,6] [1,7,4,8] [2,5,7,9] [3,6,9,8] [4,5,6,8] [4,5,8,7] [9,5,8,6] [9,5,7,8].
 * Backward: one thread per input vertex, its row's gradient plus half of each of its edges' rows.
 * V + E >= 2^31 - 1 or 12T >= 2^31 gives DIBR_B200_ESIZE; negative sizes or a NULL buffer that is
 * used give DIBR_B200_EINVAL.
 */
int dibr_b200_tet_subdivide_forward(int batch, int num_vertices, int num_edges, int64_t num_tets, int channels,
                                    const int32_t* edges, const int64_t* tets, const int32_t* tet_edge,
                                    const float* vertices, const float* features, float* out_vertices,
                                    float* out_features, int64_t* out_tets, dibr_b200_stream_t stream);
int dibr_b200_tet_subdivide_backward(int batch, int num_vertices, int num_edges, int channels, const int32_t* adj_ptr,
                                     const int32_t* adj, const int32_t* adj_edge, const float* grad_out_vertices,
                                     const float* grad_out_features, float* grad_vertices, float* grad_features,
                                     dibr_b200_stream_t stream);

/*
 * Exchange step of the view-sharded path (SURVEY.md 8e; kaolin_b200/csrc/peer_push.cu): the
 * reference has no multi-GPU code - its callers all-gather the per-view gradients with
 * torch.distributed.  All-gather by STORES over NVLink: copies `bytes` (multiple of 16) from the
 * local device buffer `src` to dst[i] + dst_offset_bytes for i < n_dst (<= 16), where dst[i] are
 * device pointers valid in this process (local memory or peer memory mapped through CUDA
 * symmetric / IPC memory; host array of pointers).  `ctas` bounds the grid (<= 0: 32) so that the
 * kernel can run underneath compute.  Asynchronous on `stream`; a cross-rank barrier after it is
 * the caller's (kaolin_b200/multi_gpu.py:PeerGradAllGather).
 */
int dibr_b200_peer_push(const void* src, size_t bytes, void* const* dst, int n_dst, size_t dst_offset_bytes,
                        int ctas, dibr_b200_stream_t stream);
/*
 * The same through an NVSwitch MULTICAST address (multimem.st): `multicast_dst` is the multicast
 * mapping of the symmetric landing buffer; one store per 16 bytes lands at multicast_dst +
 * dst_offset_bytes in EVERY GPU bound to the multicast object, this one included - a rank's
 * egress is its shard once, not once per peer.
 */
int dibr_b200_peer_push_multicast(const void* src, size_t bytes, void* multicast_dst, size_t dst_offset_bytes,
                                  int ctas, dibr_b200_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* DIBR_B200_H_ */
