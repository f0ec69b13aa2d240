/*
 * lgrast.h -- C-ABI of liblgrast.so, the H100 (sm_90a) rasterizer for LightGaussian's hot path.
 *
 * Drop-in boundary.  The four work entry points replace, one for one, the static C++ API the
 * reference's torch binding calls (RAST = submodules/compress-diff-gaussian-rasterization):
 *
 *   lgr_forward        <- CudaRasterizer::Rasterizer::forward       RAST/cuda_rasterizer/rasterizer.h:35-57
 *   lgr_forward_count  <- CudaRasterizer::Rasterizer::forwardCount  RAST/cuda_rasterizer/rasterizer.h:60-84
 *   lgr_backward       <- CudaRasterizer::Rasterizer::backward      RAST/cuda_rasterizer/rasterizer.h:86-112
 *   lgr_mark_visible   <- CudaRasterizer::Rasterizer::markVisible   RAST/cuda_rasterizer/rasterizer.h:28-33
 *
 * Conventions kept from the reference: every data pointer is a DEVICE pointer to contiguous float32 /
 * int32 memory owned by the caller; a NULL pointer means "input absent" (shs / colors_precomp /
 * scales / rotations / cov3D_precomp); viewmatrix and projmatrix are the TRANSPOSED 4x4 matrices
 * (scene/cameras.py:70-84); out_color is planar [3,H,W]; the three opaque state blobs are obtained
 * through caller-supplied allocators in the order geometry -> image -> binning (the last one only
 * after the instance count is known) and are handed back unchanged to lgr_backward.
 *
 * Differences (all additive): plain function-pointer allocators instead of std::function, an explicit
 * cudaStream_t (the reference launches on the legacy default stream), an int status return with
 * lgr_last_error(), and gradient outputs that need NOT be zero-initialised by the caller.
 *
 * No torch / C++ types cross this boundary.
 */
#ifndef LGRAST_H_INCLUDED
#define LGRAST_H_INCLUDED

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LGR_ABI_VERSION 2

/* status codes */
#define LGR_OK 0
#define LGR_ERR_INVALID_ARG 1 /* bad sizes / required pointer missing */
#define LGR_ERR_CUDA 2        /* a CUDA runtime call or kernel failed; see lgr_last_error() */
#define LGR_ERR_ALLOC 3       /* an allocator callback returned NULL */

/* Replaces std::function<char*(size_t)> (RAST/cuda_rasterizer/rasterizer.h:36-38): must return a device
 * pointer to at least `bytes` bytes, aligned to 256 B, that stays valid until the matching backward call. */
typedef char* (*lgr_alloc_fn)(void* user, size_t bytes);

/* Per-view constants: the numeric fields of GaussianRasterizationSettings
 * (RAST/diff_gaussian_rasterization/__init__.py:248-261). */
typedef struct lgr_view {
    int32_t image_width;
    int32_t image_height;
    float tan_fovx;
    float tan_fovy;
    float scale_modifier;
    int32_t sh_degree;       /* active degree D (0..3) */
    int32_t prefiltered;     /* as the reference: a culled point traps the kernel when set */
    int32_t debug;           /* synchronise and check after every stage */
    const float* viewmatrix; /* device, 16 floats, transposed W2C */
    const float* projmatrix; /* device, 16 floats, transposed Proj*W2C */
    const float* campos;     /* device, 3 floats */
    const float* background; /* device, 3 floats */
} lgr_view;

/* Forward render.  P Gaussians, M stored SH coefficients per channel (0 when shs == NULL).
 * Writes out_color[3*H*W], radii[P]; *num_rendered receives the reference's instance count
 * (sum over Gaussians of the tile-rectangle area, rasterizer_impl.cu:278-282). */
int lgr_forward(const lgr_view* view, int P, int M,
                const float* means3D, const float* shs, const float* colors_precomp, const float* opacities,
                const float* scales, const float* rotations, const float* cov3D_precomp,
                lgr_alloc_fn geometry_alloc, void* geometry_user,
                lgr_alloc_fn binning_alloc, void* binning_user,
                lgr_alloc_fn image_alloc, void* image_user,
                float* out_color, int32_t* radii, int32_t* num_rendered, void* cuda_stream);

/* Forward render + Global Significance accumulation (RAST/cuda_rasterizer/forward.cu:378-501).
 * gaussians_count[P] and important_score[P] are fully written (no zero-init needed):
 *   gaussians_count[i] = number of (pixel, i) pairs that were blended in this view (exact, deterministic),
 *   important_score[i] = opacity[i] * gaussians_count[i]. */
int lgr_forward_count(const lgr_view* view, int P, int M,
                      const float* means3D, const float* shs, const float* colors_precomp, const float* opacities,
                      const float* scales, const float* rotations, const float* cov3D_precomp,
                      lgr_alloc_fn geometry_alloc, void* geometry_user,
                      lgr_alloc_fn binning_alloc, void* binning_user,
                      lgr_alloc_fn image_alloc, void* image_user,
                      float* out_color, int32_t* gaussians_count, float* important_score, int32_t* radii,
                      int32_t* num_rendered, void* cuda_stream);

/* Backward.  The three blobs and num_rendered come from the matching lgr_forward call.
 * Outputs (all fully written): dL_dmeans2D[P,3], dL_dcolors[P,3], dL_dopacity[P], dL_dmeans3D[P,3],
 * dL_dcov3D[P,6], dL_dsh[P,M,3] (may be NULL when M == 0), dL_dscales[P,3], dL_drotations[P,4]
 * -- the tuple RAST/rasterize_points.cu:298 returns. */
int lgr_backward(const lgr_view* view, int P, int M, int num_rendered,
                 const float* means3D, const float* shs, const float* colors_precomp,
                 const float* scales, const float* rotations, const float* cov3D_precomp,
                 const int32_t* radii, char* geometry_blob, char* binning_blob, char* image_blob,
                 const float* dL_dout_color,
                 float* dL_dmeans2D, float* dL_dcolors, float* dL_dopacity, float* dL_dmeans3D,
                 float* dL_dcov3D, float* dL_dsh, float* dL_dscales, float* dL_drotations, void* cuda_stream);

/* ---- fused-activation variants (SURVEY.md section 8f row N1; used inside gaussian_renderer.render()) ----
 * The six parameter leaves of GaussianModel (scene/gaussian_model.py:46-56) are read directly and the activations of
 * its getters (:98-118: exp, normalize, sigmoid, cat) are applied in-kernel, bit-identically to the torch CUDA ops, so
 * the result equals lgr_forward on the activated tensors.  M counts ALL SH coefficients per channel
 * (features_dc holds 1, features_rest M-1).  features_* and rotation must be 16-byte aligned. */
typedef struct lgr_raw_params {
    const float* xyz;           /* [P,3]      */
    const float* features_dc;   /* [P,1,3]    */
    const float* features_rest; /* [P,M-1,3]  */
    const float* scaling;       /* [P,3] log-scale         -> exp        */
    const float* rotation;      /* [P,4] raw quaternion    -> normalize  */
    const float* opacity;       /* [P,1] logit             -> sigmoid    */
    int32_t features_rest_row_stride; /* floats between consecutive rows of features_rest; 0 = dense, i.e. (M-1)*3.
                                       * A larger value describes a row-strided view such as the distillation student's
                                       * _features_rest[:, :8, :] of a [P,15,3] tensor (scene/gaussian_model.py:129-136):
                                       * stride 45, 24 floats used.  The storage must hold P*stride floats from the pointer. */
} lgr_raw_params;

typedef struct lgr_raw_grads { /* dL/d(leaf), same shapes, fully written */
    float* xyz;
    float* features_dc;
    float* features_rest;
    float* scaling;
    float* rotation;
    float* opacity;
    float* rgb; /* optional [P,3]: clamp-masked dL/dRGB of this view.  When rgb != NULL and features_rest == NULL ("compact
                   mode") features_dc / features_rest are not written: see lgr_sh_grad_from_views. */
} lgr_raw_grads;

/* gaussians_count / important_score may both be NULL (plain forward) or both non-NULL (significance mode). */
int lgr_forward_raw(const lgr_view* view, int P, int M, const lgr_raw_params* params,
                    lgr_alloc_fn geometry_alloc, void* geometry_user,
                    lgr_alloc_fn binning_alloc, void* binning_user,
                    lgr_alloc_fn image_alloc, void* image_user,
                    float* out_color, int32_t* gaussians_count, float* important_score, int32_t* radii,
                    int32_t* num_rendered, void* cuda_stream);

/* ---- rendering a VecTree-compressed model in place (render.py / render_video.py --load_vq) ----
 * The arrays of extreme_saving/ (vectree/vectree.py:107-155) as they stay resident on the GPU; no [P,dim] table is built.  The
 * forward reads them instead of the six float32 leaves GaussianModel.load_vq (scene/gaussian_model.py:420-461) would inflate them
 * to, with the same activations, so the image, radii and significance outputs are bit-identical to lgr_forward_raw on those leaves.
 * All arrays are device memory, 16-byte aligned. */
typedef struct lgr_vq_resident_params {
    const float* xyz;      /* [P,3] float32 */
    const void* attr;      /* [P,8] raw opacity | scale x3 | rotation x4 (other_attribute.npz order): fp16 if attr_half, else float32 */
    const int32_t* slot;   /* [P]: >= 0 a codebook row; < 0 the row -(slot) - 1 of nonvq */
    const void* codebook;  /* [K,Dp] fp16 */
    const void* nonvq;     /* [Pn,Dp] fp16 if nonvq_half, else float32; may be NULL when no slot is negative */
    int32_t attr_half;
    int32_t nonvq_half;
    int32_t D;  /* colour values per row, 3*(max_degree+1)^2: f_dc_0..2, then f_rest channel-major (row[3 + c*(M-1) + j]) */
    int32_t Dp; /* row pitch of codebook and nonvq in elements: a multiple of 8, >= D */
    int32_t K;  /* codebook rows */
} lgr_vq_resident_params;

/* Forward of a resident VQ model: the allocator, output and stream contract of lgr_forward_raw (M = D/3).  gaussians_count /
 * important_score are both NULL or both set.  There is no backward: a model that is trained gets its leaves materialised. */
int lgr_forward_vq(const lgr_view* view, int P, const lgr_vq_resident_params* params,
                   lgr_alloc_fn geometry_alloc, void* geometry_user,
                   lgr_alloc_fn binning_alloc, void* binning_user,
                   lgr_alloc_fn image_alloc, void* image_user,
                   float* out_color, int32_t* gaussians_count, float* important_score, int32_t* radii,
                   int32_t* num_rendered, void* cuda_stream);

/* ---- blending-weight significance (DESIGN.md section 3, "Blending-weight significance") ----
 * The count forwards above with one more output, blend_weight[P] (int64, device, fully written: no zero-init needed):
 *   blend_weight[i] = sum over the pixels p that blend Gaussian i in this view of rint(fl(alpha * T) * 2^32),
 * alpha and T being the float32 alpha and pre-blend transmittance the colour uses, fl one rounding.  Resolution 2^-32; the sum is
 * exact, so it does not depend on launch order, stream, binning mode, deterministic mode or tile culling.  Every other output is
 * bit-identical to the sibling.  blend_weight is required when P > 0; the raw / VQ variants need count mode (gaussians_count and
 * important_score set).  The round-1 blend kernels (lgr_set_blend_mode(1)) have no weight output: LGR_ERR_INVALID_ARG, nothing
 * launched. */
int lgr_forward_count_weight(const lgr_view* view, int P, int M,
                             const float* means3D, const float* shs, const float* colors_precomp, const float* opacities,
                             const float* scales, const float* rotations, const float* cov3D_precomp,
                             lgr_alloc_fn geometry_alloc, void* geometry_user,
                             lgr_alloc_fn binning_alloc, void* binning_user,
                             lgr_alloc_fn image_alloc, void* image_user,
                             float* out_color, int32_t* gaussians_count, float* important_score, int64_t* blend_weight,
                             int32_t* radii, int32_t* num_rendered, void* cuda_stream);
int lgr_forward_raw_weight(const lgr_view* view, int P, int M, const lgr_raw_params* params,
                           lgr_alloc_fn geometry_alloc, void* geometry_user,
                           lgr_alloc_fn binning_alloc, void* binning_user,
                           lgr_alloc_fn image_alloc, void* image_user,
                           float* out_color, int32_t* gaussians_count, float* important_score, int64_t* blend_weight,
                           int32_t* radii, int32_t* num_rendered, void* cuda_stream);
int lgr_forward_vq_weight(const lgr_view* view, int P, const lgr_vq_resident_params* params,
                          lgr_alloc_fn geometry_alloc, void* geometry_user,
                          lgr_alloc_fn binning_alloc, void* binning_user,
                          lgr_alloc_fn image_alloc, void* image_user,
                          float* out_color, int32_t* gaussians_count, float* important_score, int64_t* blend_weight,
                          int32_t* radii, int32_t* num_rendered, void* cuda_stream);

int lgr_backward_raw(const lgr_view* view, int P, int M, int num_rendered, const lgr_raw_params* params,
                     const int32_t* radii, char* geometry_blob, char* binning_blob, char* image_blob,
                     const float* dL_dout_color, const lgr_raw_grads* grads, float* dL_dmeans2D, void* cuda_stream);

/* The same backward in two stages, so a caller can start exchanging this view's dL/dRGB (written to d_rgb[P,3] when non-NULL)
 * while the per-Gaussian stage runs:  begin = accumulator clear + blend backward (+ dRGB extraction),  end = K7+K8.
 * lgr_backward_raw == begin(d_rgb = NULL) followed by end.  In lgr_backward_raw_end, grads->features_rest == NULL selects the
 * compact mode (SH leaves not written). */
int lgr_backward_raw_begin(const lgr_view* view, int P, int num_rendered, const int32_t* radii, char* geometry_blob, char* binning_blob,
                           char* image_blob, const float* dL_dout_color, float* d_rgb, void* cuda_stream);
int lgr_backward_raw_end(const lgr_view* view, int P, int M, const lgr_raw_params* params, const int32_t* radii, char* geometry_blob,
                         const lgr_raw_grads* grads, float* dL_dmeans2D, void* cuda_stream);
/* stage 2 for Gaussians [first, first+count) only (first a multiple of 256): lets a view-parallel caller exchange one range's
 * gradients while the next range is computed */
int lgr_backward_raw_end_range(const lgr_view* v, int P, int M, const lgr_raw_params* params, const int32_t* radii, char* geometry_blob,
                               const lgr_raw_grads* grads, float* dL_dmeans2D, int first, int count, void* cuda_stream);

/* ---- depth and alpha planes (DESIGN.md section 7, "Depth and alpha maps") ----
 * For pixel p let w_i = alpha_i * T_i be the weight the colour blend gives Gaussian i, in the colour's float32 operations and order
 * (fma(T, alpha * c, acc)), and z_i the view-space depth of the geometry blob.
 *   depth_mode 1 ("z"):       out_depth[p] = sum_i w_i * z_i         (background 0, not divided by alpha)
 *   depth_mode 2 ("inverse"): out_depth[p] = sum_i w_i * (1/z_i)     (1/z_i correctly rounded: torch's 1 / z in float32)
 *   out_alpha[p] = fl(1 - final_T[p])
 * Both planes are [H,W] float32 on the device and fully written (0 in empty tiles).
 * lgr_forward_raw_depth: the lgr_forward_raw contract plus depth_mode (0 = none, 1 = z, 2 = inverse), out_depth and out_alpha.
 * Either output may be NULL; out_depth needs depth_mode 1 or 2; with both NULL the call is lgr_forward_raw.  Every other output is
 * bit-identical to lgr_forward_raw's.  Count mode, deterministic mode and the round-1 blend kernels have no depth or alpha output:
 * LGR_ERR_INVALID_ARG, nothing launched.  The forward records its depth mode in the geometry blob.
 * lgr_backward_raw_depth: the lgr_backward_raw contract plus the forward's depth_mode and dL_ddepth / dL_dalpha ([H,W], either may
 * be NULL, meaning zero; with both NULL the call is lgr_backward_raw).  When the geometry blob comes from a forward that ran
 * without depth or alpha, or in another depth_mode, every gradient of a visible Gaussian is NaN. */
int lgr_forward_raw_depth(const lgr_view* view, int P, int M, const lgr_raw_params* params,
                          lgr_alloc_fn geometry_alloc, void* geometry_user,
                          lgr_alloc_fn binning_alloc, void* binning_user,
                          lgr_alloc_fn image_alloc, void* image_user,
                          float* out_color, int32_t* gaussians_count, float* important_score,
                          int depth_mode, float* out_depth, float* out_alpha,
                          int32_t* radii, int32_t* num_rendered, void* cuda_stream);
int lgr_backward_raw_depth(const lgr_view* view, int P, int M, int num_rendered, const lgr_raw_params* params,
                           const int32_t* radii, char* geometry_blob, char* binning_blob, char* image_blob,
                           const float* dL_dout_color, int depth_mode, const float* dL_ddepth, const float* dL_dalpha,
                           const lgr_raw_grads* grads, float* dL_dmeans2D, void* cuda_stream);

/* ---- absolute-gradient densification statistic (DESIGN.md section 7, "Absolute-gradient densification statistics") ----
 * lgr_backward_raw_absgrad: the lgr_backward_raw contract (every other output is computed exactly as there) plus
 * dL_dmeans2D_abs ([P,2] float32 on the device, 8-byte aligned, fully written), the AbsGS / gsplat "absgrad" statistic:
 *   dL_dmeans2D_abs[i] = (sum_p |dL_p/dmean2D_x(i)|, sum_p |dL_p/dmean2D_y(i)|)
 * over exactly the pixels p that blend Gaussian i, dL_p/dmean2D being pixel p's term of dL/dmeans2D (the backward run with dL/dpix
 * zero everywhere except at p), in the units of dL_dmeans2D; 0 for a Gaussian that no pixel blends.  Deterministic mode and the
 * round-1 blend kernels (lgr_set_blend_mode(1)) have no absgrad: LGR_ERR_INVALID_ARG, nothing launched.  The depth / alpha forward
 * is recorded on the device only, so a geometry blob from lgr_forward_raw_depth is refused there: every gradient of a visible
 * Gaussian and every absgrad row is NaN. */
int lgr_backward_raw_absgrad(const lgr_view* view, int P, int M, int num_rendered, const lgr_raw_params* params,
                             const int32_t* radii, char* geometry_blob, char* binning_blob, char* image_blob,
                             const float* dL_dout_color, const lgr_raw_grads* grads, float* dL_dmeans2D,
                             float* dL_dmeans2D_abs, void* cuda_stream);

/* ---- camera gradients (DESIGN.md section 7, "Camera gradients") ----
 * lgr_backward_raw_camera: the lgr_backward_raw_depth contract (depth_mode 0 with dL_ddepth and dL_dalpha NULL is lgr_backward_raw;
 * every other output is computed exactly as there) plus the loss gradient with respect to the three camera arrays of `view`:
 *   dL_dviewmatrix [16], dL_dprojmatrix [16], dL_dcampos [3]: float32 device arrays, fully written.
 * With V = viewmatrix, Pm = projmatrix, c = campos and p = (x, y, z, 1) a Gaussian's world mean, summed over every Gaussian the
 * per-Gaussian backward differentiates:
 *   dL/dV[4r+k]  = p_r dL/dt_k (t_k = sum_r p_r V[4r+k], k < 3: the camera-space mean, through the J path of the 2D covariance with the
 *                  forward's 1.3 tan(fov) clamp, and the depth plane) plus, for r, k < 3, (J^T dL/dT)[k][r] (T = J W, W[a][k] = V[4k+a])
 *   dL/dPm[4r+k] = p_r dL/dh_k, k in {0, 1, 3} (h_k = sum_r p_r Pm[4r+k]; ndc = (h_0, h_1) / (h_3 + 1e-7))
 *   dL/dc        = minus the sum of the view-direction terms of the SH backward
 * V[4r+3] and Pm[4r+2] are never read: those eight entries are 0.  The intrinsics (tan_fovx / tan_fovy) get no gradient.  All three
 * outputs are 0 when P == 0 or nothing is differentiated.  Deterministic mode runs the dense per-Gaussian kernel, whose partial sums
 * have a fixed order: two calls on one forward return bit-identical camera gradients.  Otherwise the compacted kernel's list is in
 * block-arrival order and the camera gradients may differ between runs in the last bits.  `workspace`: device memory of at least
 * lgr_camera_grad_workspace_bytes(P) bytes, 4-byte aligned.  With a depth or alpha plane, deterministic mode and the round-1 blend
 * kernels are refused as by lgr_backward_raw_depth (LGR_ERR_INVALID_ARG, nothing launched); a geometry blob from a forward in another
 * depth mode gives NaN camera gradients along with the NaN leaf gradients. */
size_t lgr_camera_grad_workspace_bytes(int P);
int lgr_backward_raw_camera(const lgr_view* view, int P, int M, int num_rendered, const lgr_raw_params* params,
                            const int32_t* radii, char* geometry_blob, char* binning_blob, char* image_blob,
                            const float* dL_dout_color, int depth_mode, const float* dL_ddepth, const float* dL_dalpha,
                            const lgr_raw_grads* grads, float* dL_dmeans2D, float* dL_dviewmatrix, float* dL_dprojmatrix,
                            float* dL_dcampos, void* workspace, size_t workspace_bytes, void* cuda_stream);

/* View-parallel training: for one view dL/dSH[k][c] = basis_k(dir) * dRGB[c] is rank-1 per Gaussian
 * (RAST/cuda_rasterizer/backward.cu:44-97), so ranks exchange dRGB (12 B/Gaussian/view, all-gather) instead of the
 * dense 12*M B/Gaussian gradient, and each rank rebuilds the SUM over views here:
 *   d_features_dc/rest[i] = sum_v basis(normalize(xyz[i] - campos[v])) (x) d_rgb[v][i]       (rows k >= (D+1)^2 are zero)
 * campos: [n_views,3] device; d_rgb: [n_views,P,3] device. */
int lgr_sh_grad_from_views(int P, int M, int sh_degree, int n_views, const float* xyz, const float* campos, const float* d_rgb,
                           float* d_features_dc, float* d_features_rest, void* cuda_stream);

/* All-reduce (sum) of n_floats floats over NVLink peer memory, for the view-parallel gradient exchange.
 * peer_buffers[r] (HOST array of `world` DEVICE pointers) is rank r's buffer as mapped into THIS process (symmetric /
 * IPC memory, 16-byte aligned); n_floats must be a multiple of 4.  This rank reduces slice `rank` from all peers with P2P
 * loads (fixed rank order: every rank obtains bit-identical sums) and stores it into all peers.  The caller must place a
 * cross-GPU barrier on the stream BEFORE (all ranks' data written) and AFTER (all peers' stores landed) this call. */
int lgr_peer_allreduce(float* const* peer_buffers, int rank, int world, size_t n_floats, void* cuda_stream);

/* Same contract as lgr_peer_allreduce, with the sum formed inside the NVSwitch: multicast_ptr is the NVLS multicast mapping
 * of the symmetric buffer (multimem.ld_reduce / multimem.st).  Barriers before and after are the caller's. */
int lgr_multimem_allreduce(float* multicast_ptr, int rank, int world, size_t n_floats, void* cuda_stream);

/* ---- fused image loss of the training loops (SURVEY.md section 8f row N2; utils/loss_utils.py:18-85) ----
 * forward: out2[0] = mean|img - target| (l1_loss), out2[1] = ssim(img, target) (11x11 Gaussian window, sigma 1.5, zero padding,
 * C1 = 0.01^2, C2 = 0.03^2, mean over C*H*W).  dmaps (optional, [3,C,H,W]) receives what the backward needs.  All device
 * pointers; planar [C,H,W] float32.  workspace: lgr_image_loss_workspace_bytes() bytes, 8-byte aligned.
 * backward: d_img = s * d/d img ( g_l1 * l1 + g_ssim * ssim ),  s = *grad_scale (device scalar) or 1 when NULL.
 * The reference's training loss (1-l)*l1 + l*(1-ssim) (prune_finetune.py:160-164) is g_l1 = 1-l, g_ssim = -l. */
size_t lgr_image_loss_workspace_bytes(int C, int H, int W);
int lgr_image_loss_forward(const float* img, const float* target, int C, int H, int W, float* out2, float* dmaps, void* workspace,
                           void* cuda_stream);
/* L1 only: out2[0] = mean|img - target|, out2[1] = 0 (no SSIM filtering); same workspace; backward = lgr_image_loss_backward with g_ssim = 0 */
int lgr_image_l1_forward(const float* img, const float* target, int C, int H, int W, float* out2, void* workspace, void* cuda_stream);
int lgr_image_loss_backward(const float* img, const float* target, const float* dmaps, int C, int H, int W, float g_l1, float g_ssim,
                            const float* grad_scale, float* d_img, void* cuda_stream);

/* Push variant of lgr_backward_raw_sparse_pack for N ranks (N <= 8): every rank owns ONE exchange buffer of N slots of
 * lgr_sparse_exchange_bytes(P) bytes each, mapped into all peers; slot_of_this_rank[r] is the address of slot `self` inside the buffer
 * of rank r.  The packed view is written to all of them (plain stores over NVLink from inside the kernels), so after one cross-GPU
 * barrier lgr_backward_raw_sparse_accumulate runs on the N slots of the rank's OWN buffer: no remote load is on its critical path. */
int lgr_backward_raw_sparse_pack_push(const lgr_view* view, int P, int M, const lgr_raw_params* params, const int32_t* radii, char* geometry_blob,
                                      void* const* slot_of_this_rank, int world, int self, void* workspace, float* dL_dmeans2D,
                                      void* cuda_stream);

/* ---- sparse view-parallel gradient exchange over peer memory (DESIGN.md section 6) ----
 * Only ~13 % of the Gaussians get a non-zero gradient from one view.  lgr_backward_raw_sparse_pack (after lgr_backward_raw_begin) runs the
 * per-Gaussian backward on those only and publishes, in `exchange_buffer` (lgr_sparse_exchange_bytes(P) bytes, 256-byte aligned, mapped into
 * every peer): the view's camera position, a bitmap + prefix counts of the non-zero Gaussians and their 64-byte gradient rows.  After a
 * cross-GPU barrier, lgr_backward_raw_sparse_accumulate reads the rows of all `world` buffers (peer_buffers[r] = rank r's buffer as mapped
 * here; P2P loads) in rank order and writes the six dense leaf gradients, summed over the views, bit-identically on every rank.
 * workspace: lgr_sparse_workspace_bytes(P) bytes of local scratch.  dL_dmeans2D (local view only) is written dense. */
size_t lgr_sparse_exchange_bytes(int P);
size_t lgr_sparse_workspace_bytes(int P);
int lgr_backward_raw_sparse_pack(const lgr_view* v, int P, int M, const lgr_raw_params* params, const int32_t* radii, char* geometry_blob,
                                 void* exchange_buffer, void* workspace, float* dL_dmeans2D, void* cuda_stream);
int lgr_backward_raw_sparse_accumulate(int P, int M, int sh_degree, int world, const void* const* peer_buffers, const float* xyz,
                                       const lgr_raw_grads* grads, void* cuda_stream);

/* ---- view-parallel densification statistics (DESIGN.md section 6) ----
 * lgr_backward_raw_sparse_pack_push_ex: lgr_backward_raw_sparse_pack_push with stats == NULL; with stats, every slot is
 *   lgr_sparse_exchange_bytes_stats(P) bytes and also carries this view's densification statistics: |dL/dmeans2D[i, 0:2]| in word 14
 *   of every row, a bitmap of radii > 0 after the rows, and header words 4-6 = 0x53544154, stats->serial, P.
 * lgr_densify_stats_exchanged: after the barrier of such a step, adds every rank's view in rank order 0..world-1 to accum / denom,
 *   bit-identical on every rank and to lgr_densify_stats called once per view in that order.  peer_buffers: view v's slot as the
 *   accumulate kernel reads it.  It also checks the caller's own slot `self` against grad / update_filter (this rank's
 *   add_densification_stats arguments) and ORs into *error_word: 1 = a slot without statistics, of another serial or another P (those
 *   32-Gaussian groups are left unchanged), 2 = update_filter != radii > 0, 4 = |grad[i, 0:2]| != the published norm.
 * lgr_densify_stats_encode / lgr_densify_stats_add_views: the same sum without the sparse exchange.  encode writes one float per
 *   Gaussian (the norm where update_filter is set, -1.0f elsewhere); add_views adds `world` such rows ([world, P], rank order). */
typedef struct lgr_sparse_stats {
    uint32_t serial;
} lgr_sparse_stats;
size_t lgr_sparse_exchange_bytes_stats(int P);
int lgr_backward_raw_sparse_pack_push_ex(const lgr_view* view, int P, int M, const lgr_raw_params* params, const int32_t* radii,
                                         char* geometry_blob, void* const* slot_of_this_rank, int world, int self, void* workspace,
                                         float* dL_dmeans2D, const lgr_sparse_stats* stats, void* cuda_stream);
int lgr_densify_stats_exchanged(int P, int world, int self, const void* const* peer_buffers, uint32_t serial, const float* grad,
                                int grad_row_stride, const uint8_t* update_filter, float* accum, float* denom, uint32_t* error_word,
                                void* cuda_stream);
int lgr_densify_stats_encode(int P, const float* grad, int grad_row_stride, const uint8_t* update_filter, float* out, void* cuda_stream);
int lgr_densify_stats_add_views(int P, int world, const float* views, float* accum, float* denom, void* cuda_stream);

/* ---- optimizer side of the training loops (SURVEY.md 8f row N3) ----
 * lgr_adamw_step: torch.optim.AdamW's default (foreach) update, amsgrad off, for up to 8 tensors in ONE launch; replaces
 * `gaussians.optimizer.step()` (prune_finetune.py:287, optimizer built at scene/gaussian_model.py:184-217).  `step` is the
 * tensor's step count AFTER the increment (t >= 1); lr is per tensor (one per param group), the rest is shared.  The host
 * scalars are formed in double precision exactly as torch/optim/adam.py does and rounded to fp32 at the kernel boundary. */
typedef struct lgr_adamw_tensor {
    float* param;
    const float* grad;
    float* exp_avg;
    float* exp_avg_sq;
    int64_t numel;
    double lr;
    double step;
    int64_t row_elems;        /* 0: param is contiguous.  Otherwise param is a row-strided view: element e lives at     */
    int64_t param_row_stride; /* param[(e / row_elems) * param_row_stride + e % row_elems]; grad and moments stay dense */
} lgr_adamw_tensor;
int lgr_adamw_step(int n_tensors, const lgr_adamw_tensor* tensors, double beta1, double beta2, double eps, double weight_decay,
                   void* cuda_stream);

/* lgr_adamw_step_selective: the same update, restricted to the ACTIVE rows.  All tensors share `rows` in dim 0 (one row per
 * Gaussian); row i is active when any element of row i of any tensor's gradient compares unequal to zero (+0 and -0 do not, NaN
 * does).  Every element of an active row is updated bit-identically to lgr_adamw_step; the parameter and both moments of an inactive
 * row are neither read nor written.  Each array is a [rows, width] view: element (r, c) lives at base[r * row_stride + c * col_stride]
 * (dense [P, ...]: (width, 1); a row-strided view: (its row stride, 1); the permuted dense _xyz of create_from_pcd: (1, P)).  At most
 * 8 tensors whose widths add up to at most 400 floats per row; width 0 = the tensor takes no part; rows == 0 launches nothing. */
typedef struct lgr_adamw_row_tensor {
    float* param;
    const float* grad;
    float* exp_avg;
    float* exp_avg_sq;
    int64_t width;                  /* elements per row */
    int64_t param_row_stride, param_col_stride;
    int64_t grad_row_stride, grad_col_stride;
    int64_t exp_avg_row_stride, exp_avg_col_stride;
    int64_t exp_avg_sq_row_stride, exp_avg_sq_col_stride;
    double lr;
    double step;                    /* step count AFTER the increment, as lgr_adamw_tensor.step */
} lgr_adamw_row_tensor;
int lgr_adamw_step_selective(int n_tensors, const lgr_adamw_row_tensor* tensors, long long rows, double beta1, double beta2, double eps,
                             double weight_decay, void* cuda_stream);

/* Row compaction of GaussianModel._prune_optimizer / prune_points (scene/gaussian_model.py:564-600): `keep` is a device byte
 * mask over P rows.  lgr_compact_plan writes the indices of the kept rows, ascending, to src_row[0..rows_out) and returns
 * rows_out through a host pointer (one stream synchronisation); lgr_compact_rows then gathers up to 24 row-major tensors
 * (row_words 4-byte words per row: parameters and both Adam moments of all groups) in ONE launch. */
typedef struct lgr_compact_tensor {
    const void* src;
    void* dst;
    int32_t row_words;
} lgr_compact_tensor;
size_t lgr_compact_workspace_bytes(int P);
int lgr_compact_plan(int P, const uint8_t* keep, int32_t* src_row, void* workspace, size_t workspace_bytes, int32_t* rows_out_host,
                     void* cuda_stream);
int lgr_compact_rows(int rows_out, const int32_t* src_row, int n_tensors, const lgr_compact_tensor* tensors, void* cuda_stream);

/* ---- VecTree vector quantisation of the SH features (SURVEY.md 8f row N4; vectree/vq.py:262-306, vectree/vectree.py:86-125,166-207) ----
 * All pointers are device pointers; x is [n,d] row-major float32, embed [K,d], d <= 64.
 * lgr_vq_assign: idx[i] = argmin_c |x_i - e_c|^2 (evaluated as |e_c|^2 - 2 x_i.e_c like torch.cdist's expansion; smallest index wins
 *   ties).  When cluster_batch / embed_sum are given they receive sum_i w_i [idx_i = c] and sum_i w_i x_i [idx_i = c], with
 *   w_i = weight_i * n / *weight_sum (the reference's normalisation), or 1 when weight is NULL: the quantities EuclideanCodebook.forward
 *   forms with F.one_hot and einsum.  workspace: lgr_vq_workspace_bytes(n) bytes, 8-byte aligned.  The size is the same in every mode:
 *   it includes the deterministic mode's sort buffers (4 uint32 per sample plus the radix sort's temporary storage, which the function
 *   queries from CUB on the host), so a workspace stays valid when the mode changes; the default mode uses only the first 8n bytes.
 * lgr_vq_ema_update: cluster_size <- decay*cluster_size + (1-decay)*cluster_batch; embed <- decay*embed + (1-decay)*embed_sum/smoothed,
 *   smoothed = (cluster_size+eps)/(sum+K*eps)*sum (vq.py:286-300).  scratch: one float.
 * lgr_vq_gather: out[i,:] = embed[idx[i],:] (batched_embedding, vq.py:161-165).
 * lgr_vq_pack_indices / lgr_vq_unpack_indices: `bits` bits per index, most significant first, bytes filled from the high bit
 *   (dec2bin + np.packbits, vectree.py:120-125; np.unpackbits + bin2dec, vectree/utils.py:33-39); out has (n*bits+7)/8 bytes. */
size_t lgr_vq_workspace_bytes(int64_t n);
/* lgr_vq_assign for d <= 32 and n*K >= 2^20 runs the scores on the tensor cores (csrc/lgr_vq_tc.cuh: bf16 hi/lo split operands, wgmma,
 * FP32 accumulators in registers) and re-scores in exact FP32 only the rows whose two best codes are closer than the split's error bound; indices are
 * the same as the FP32 kernel's.  lgr_set_vq_mode(1) forces the FP32 kernel (A/B measurements).  The tensor-core path keeps a grow-only
 * device scratch (operand tiles) inside the library. */
int lgr_set_vq_mode(int mode);
int lgr_vq_assign(int n, int d, int K, const float* x, const float* embed, const float* weight, const float* weight_sum, int32_t* idx,
                  float* cluster_batch, float* embed_sum, void* workspace, void* cuda_stream);
int lgr_vq_ema_update(int K, int d, double decay, double eps, float* cluster_size, float* embed, const float* cluster_batch,
                      const float* embed_sum, float* scratch, void* cuda_stream);
int lgr_vq_gather(int n, int d, const int32_t* idx, const float* embed, float* out, void* cuda_stream);
int lgr_vq_pack_indices(int64_t n, int bits, const int32_t* idx, uint8_t* out, void* cuda_stream);
int lgr_vq_unpack_indices(int64_t n, int bits, const uint8_t* in, int32_t* idx, void* cuda_stream);

/* ---- initial scales from a point cloud: distCUDA2 of submodules/simple-knn (spatial.cu:15-26, simple_knn.cu:147-221) ----
 * out[i] = mean of the squared distances from points[i] to its three nearest OTHER points (by index: a duplicate counts, at 0),
 * bit-identical to the reference's extension on sm_90a (csrc/lgr_knn.cuh).  With fewer than three other points the missing ones
 * count as FLT_MAX, as in the reference.  points: device [P,3] contiguous float32; out: device [P] float32.
 * workspace: lgr_knn_workspace_bytes(P) bytes, 256-byte aligned.  No host synchronisation; P == 0 does nothing. */
size_t lgr_knn_workspace_bytes(int P);
int lgr_knn_mean_dist3(int P, const float* points, float* out, void* workspace, size_t workspace_bytes, void* cuda_stream);

/* ---- densification: GaussianModel.add_densification_stats / densify_and_prune (scene/gaussian_model.py:602-788) ----
 * Bit-identical to the reference's torch code (csrc/lgr_densify.cuh).  All pointers are device pointers to contiguous float32.
 * lgr_densify_stats: for rows with update_filter[i] != 0, accum[i] += |grad[i, 0:2]| and denom[i] += 1; grad rows are
 *   grad_row_stride floats apart.  No host synchronisation.
 * lgr_densify_plan: classifies every row (clone, split, prune) from accum, denom, the raw scaling [P,3] and the raw opacity [P].
 *   Thresholds are float32, as torch compares a float tensor with a Python scalar: max_grad, dense_scale = percent_dense*extent,
 *   min_opacity, big_scale = 0.1*extent.  prune_all removes every row (the reference's big_points_vs on its just-zeroed radii, when
 *   0 > max_screen_size); prune_big enables the big_scale test.  Returns counts_host[4] = {kept original rows, kept clones, kept
 *   split children per copy, split rows S} after one stream synchronisation.  workspace: lgr_densify_workspace_bytes(P) bytes,
 *   256-byte aligned; lgr_densify_rows reads it, so it must stay untouched in between.
 * lgr_densify_split_inputs: the operands of the split's product bmm(build_rotation(q), samples) for the 2S children, rows r and
 *   S + r for the split row of rank r, as the reference's .repeat(2, 1) lays them out: rotations_out [2S,3,3] and samples_out [2S,3] =
 *   normals * exp(scaling) + 0.  normals: [2S,3] standard normals drawn by the caller through torch's generator.  No fixed operation
 *   order of that 3x3 . 3x1 product matches torch.bmm on every sample, so the caller forms it with torch.bmm.
 * lgr_densify_rows: writes the rows_out = counts[0] + counts[1] + 2*counts[2] output rows of up to 24 tensors in one launch, in the
 *   order unsplit rows, clones, first children, second children.  child_offsets: [2S,3] product of lgr_densify_split_inputs' operands,
 *   added to the parents' xyz.  Roles: COPY = raw copy to every destination; XYZ / SCALING = copied, computed for the children
 *   (row_words 3); MOMENT = copied to the kept original row, zero for new rows; ZERO = zero everywhere (src may be NULL).  Tensors
 *   with row_words == 0 are skipped, their pointers are not read. */
enum { LGR_DENSIFY_COPY = 0, LGR_DENSIFY_XYZ = 1, LGR_DENSIFY_SCALING = 2, LGR_DENSIFY_MOMENT = 3, LGR_DENSIFY_ZERO = 4 };
typedef struct lgr_densify_tensor {
    const void* src;
    void* dst;
    int32_t row_words;
    int32_t role;
} lgr_densify_tensor;
int lgr_densify_stats(int P, const float* grad, int grad_row_stride, const uint8_t* update_filter, float* accum, float* denom,
                      void* cuda_stream);
size_t lgr_densify_workspace_bytes(int P);
int lgr_densify_plan(int P, const float* accum, const float* denom, const float* scaling, const float* opacity, float max_grad,
                     float dense_scale, float min_opacity, float big_scale, int prune_all, int prune_big, void* workspace,
                     size_t workspace_bytes, int32_t* counts_host, void* cuda_stream);
int lgr_densify_split_inputs(int P, const void* workspace, const int32_t* counts, const float* scaling, const float* rotation,
                             const float* normals, float* rotations_out, float* samples_out, void* cuda_stream);
int lgr_densify_rows(int P, const void* workspace, const int32_t* counts, const float* xyz, const float* child_offsets, int n_tensors,
                     const lgr_densify_tensor* tensors, void* cuda_stream);

/* present[i] = (view-space z of point i) > 0.2   (RAST/cuda_rasterizer/rasterizer_impl.cu:54-66, auxiliary.h:139-164) */
int lgr_mark_visible(int P, const float* means3D, const float* viewmatrix, const float* projmatrix, uint8_t* present,
                     void* cuda_stream);

/* ---- introspection (tests, diagnostics) ---- */
int lgr_abi_version(void);
const char* lgr_last_error(void); /* thread-local, valid until the next failing call on this thread */

/* Byte offsets of the per-Gaussian arrays inside a geometry blob for P points, so tests can read the
 * intermediates the way RAST/cuda_rasterizer/rasterizer_impl.cu:155-170 lays them out for the reference.
 * out[0]=depth(f32) out[1]=means2D(float2) out[2]=conic_opacity(float4) out[3]=rgb(float4, w unused)
 * out[4]=cov3D(6 f32) out[5]=clamped(u8 bitmask r=1,g=2,b=4) out[6]=tiles_touched(u32) out[7]=depth-sorted ids(u32)
 * Returns the total geometry blob size. */
size_t lgr_geometry_layout(int P, size_t* out, int n_out);
/* out[0]=final_T(f32[N]) out[1]=n_contrib(u32[N]) out[2]=ranges(uint2[tiles]).  Returns image blob size. */
size_t lgr_image_layout(int width, int height, size_t* out, int n_out);
/* out[0]=point_list(u32[R]) -- per-tile, depth-sorted Gaussian ids.  Returns binning blob size for R instances. */
size_t lgr_binning_layout(int num_rendered, int width, int height, size_t* out, int n_out);
/* Kernel launches issued by this library since load (for bench.py's gpu_launches). */
uint64_t lgr_launch_count(void);

/* Diagnostics / A-B measurements: which blend kernels forward and backward launch.  0 (default) = the shared-ring kernels
 * (csrc/lgr_blend.cuh: producer warp + TMA-staged per-instance records), 1 = the round-1 per-warp kernels.  Process-wide; a
 * backward must run in the mode its forward ran in (the ring backward streams the records the ring forward stored). */
int lgr_set_blend_mode(int mode);

/* Binning (per-tile depth-ordered instance lists; replaces the scan + 64-bit radix sort of RAST/cuda_rasterizer/rasterizer_impl.cu:278-319
 * and its blocking device-to-host copy of num_rendered at :282).  2 (default) = depth sort of the P Gaussians + stable tile bucketing with the
 * CUDA toolkit's radix sort / scan, no GPU idle on the host: the binning allocator is called BEFORE the instance count is known, with a size
 * from a running estimate (25 % above the previous view); emit, tile sort and ranges run over that capacity (the slots past the count hold a
 * pad key that sorts after every tile), the host reads the count while the blend kernel is already queued and repeats emit, sort, ranges and
 * blend with an exactly sized blob (a second binning_alloc call) when the estimate was too small.  Deterministic mode, or the environment
 * variable LGR_BINNING_SYNC=1, sizes the blob exactly after one stream synchronisation instead (one binning_alloc call, the reference's
 * behaviour).  0 = hand-written kernels (csrc/lgr_bin.cuh), no library, the same estimate and repeat.  1 = the same kernels, blob sized
 * exactly after a stream synchronisation.  All three produce bit-identical lists (tests/test_gpu_binning.py); 2 is the default because it is
 * the fastest measured (DESIGN.md section 9); it is also used automatically above 32 768 tiles.  Process-wide.
 * lgr_binning_overflows() = views that took the repeat; lgr_forward_stream_syncs() = forwards that synchronised the stream for the count. */
int lgr_set_binning_mode(int mode);
uint64_t lgr_binning_overflows(void);
uint64_t lgr_forward_stream_syncs(void);
void lgr_set_binning_estimate(uint64_t instances);   /* overwrite the running estimate of modes 0 and 2 (tests; 0 = forget) */

/* Deterministic mode (default off).  On: every output is a function of the inputs alone, whatever the block scheduling, the stream or
 * other work on the GPU.  The blend backward writes one partial row per (tile, Gaussian) instance, summing the 8 warps of a tile in warp
 * order, and one pass per Gaussian adds its rows in ascending instance order into the accumulator record (no float atomics, no memset);
 * lgr_vq_assign's weighted sums come from a stable radix sort of (code, sample) pairs and per-code sums in ascending sample order.
 * Forward outputs (image, radii, final_T, n_contrib, lists, counts, scores) are bit-identical to the default mode's.  The binning blob
 * of a forward in this mode is larger: [R][9] floats of partial rows and an R-bit bitmap.  Needs library binning (lgr_set_binning_mode(2))
 * and the ring blend kernels (lgr_set_blend_mode(0)); any other combination fails with LGR_ERR_INVALID_ARG before any launch.
 * Process-wide, like the other switches; a backward must run in the mode its forward ran in (the deterministic backward reads the
 * permutation the deterministic forward stored in its records).  The forward records its mode in geometry header word [10]; a
 * deterministic backward of a forward that did not run in deterministic mode reads no record and writes NaN into every accumulator,
 * so all its gradients are NaN (a default backward of a deterministic forward is valid: it ignores the permutation). */
int lgr_set_deterministic(int on);

/* Diagnostics / A-B: the fused K7+K8 of lgr_backward_raw for a whole view with dense outputs.  0 (default) = one pass zero-fills all
 * output rows (TMA bulk stores) and lists the Gaussians whose accumulators are non-zero, a second kernel runs K7+K8 on that list;
 * 1 = the dense one-warp-per-32-Gaussians kernel. */
int lgr_set_kback_mode(int mode);

/* Exact tile-level culling at binning time (default on): (tile, Gaussian) instances in which no pixel can reach
 * alpha >= 1/255 are not listed.  Images, gradients and significance are unchanged; only the internal lists shrink.
 * Turn it off to obtain per-tile lists identical to the reference's (tests).  num_rendered always reports the
 * reference's value.  The geometry blob starts with int32 words: [0] instances listed, [1] the reference's num_rendered,
 * [2] instances the binning blob was sized for, [3] capacity overflow flag (0 once a forward call has returned). */
int lgr_set_tile_culling(int on);

/* Optional per-stage device timing: when enabled every launch is bracketed by CUDA events on its stream.
 * lgr_profile_collect() synchronises the device, writes the accumulated milliseconds and launch counts of each
 * stage (index < lgr_profile_stage_count()) and resets them.  Timing mode adds event overhead; do not use it
 * inside a throughput measurement. */
int lgr_profile_enable(int on);
int lgr_profile_stage_count(void);
const char* lgr_profile_stage_name(int stage);
int lgr_profile_collect(double* ms_out, uint64_t* launches_out, int n);

#ifdef __cplusplus
}
#endif
#endif /* LGRAST_H_INCLUDED */
