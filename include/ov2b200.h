/* ov2b200.h - C ABI of the H100 OV2SLAM hot paths (libov2b200.so).
 *
 * This is the drop-in boundary (SURVEY.md section 8b).  The reference has no FFI of its own: its
 * callers (visual_front_end.cpp, map_manager.cpp, estimator.cpp) call three C++ classes
 * directly.  The C++ shim classes in ov2slam_b200/host/ keep those class declarations
 * unchanged and forward to the entry points below; every entry point names the reference
 * interface it replaces.
 *
 * Conventions
 *   - Plain C types only.  All functions return an ov2_status (0 = OK); none throws or exits.
 *   - There is no CPU fallback: without a CUDA device ov2_create() fails with
 *     OV2_ERR_NO_DEVICE and every other call needs a context.
 *   - Array arguments may point to HOST memory (pageable or pinned) or to DEVICE memory of the
 *     context's device; the library detects which (cudaPointerGetAttributes).  Host inputs are
 *     copied H2D on the context's stream, host outputs are copied D2H and the call returns after
 *     they have landed.  With device pointers only, a call just enqueues work on the stream
 *     (use ov2_sync()).
 *   - A context is not re-entrant; use one per host thread (the reference calls
 *     fbKltTracking concurrently from the front-end and mapper threads, map_manager.cpp:510).
 *   - Batches are either "fixed stride" (frame_idx == NULL: element i belongs to frame slot
 *     first_frame + i / per_frame) or "ragged" (frame_idx[i] gives the frame slot).
 */
#ifndef OV2B200_H
#define OV2B200_H

#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#define OV2_API __attribute__((visibility("default")))
#else
#define OV2_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
    OV2_OK = 0,
    OV2_ERR_NO_DEVICE = 1,   /* no CUDA device / driver: there is no CPU path */
    OV2_ERR_CUDA = 2,        /* a CUDA call failed; see ov2_last_error() */
    OV2_ERR_INVALID = 3,     /* bad argument */
    OV2_ERR_CAPACITY = 4,    /* a fixed-capacity device buffer overflowed (reported, never silent) */
    OV2_ERR_NOMEM = 5,
    OV2_ERR_NUMERIC = 6      /* BA: non-finite cost / failed factorisation */
} ov2_status;

typedef struct ov2_ctx ov2_ctx;   /* device + stream + scratch arenas */
typedef struct ov2_pyr ov2_pyr;   /* device-resident image pyramids for a batch of frames */

/* ------------------------------------------------------------------ context */
OV2_API ov2_status ov2_create(int device, ov2_ctx** out);
OV2_API void       ov2_destroy(ov2_ctx* ctx);
OV2_API const char* ov2_last_error(const ov2_ctx* ctx);      /* valid until the next call on ctx */
OV2_API const char* ov2_version(void);
/* Run the context's work on an existing stream (e.g. torch's current stream). NULL = own stream. */
OV2_API ov2_status ov2_set_stream(ov2_ctx* ctx, void* cuda_stream);
OV2_API ov2_status ov2_sync(ov2_ctx* ctx);
/* Batch mode: between ov2_batch_begin and ov2_batch_end every call on the context only ENQUEUES
 * (H2D of host inputs, kernels); host outputs are copied back and the stream is synchronised once,
 * in ov2_batch_end.  A host buffer written by one call of the batch and read by a later one (e.g.
 * the tracked positions fbKltTracking returns and describeBRIEF consumes) is served from its device
 * staging copy, so operator chains keep host-pointer semantics without round trips.  Host outputs
 * must not be read before ov2_batch_end.  (ov2_grid_fast's capacity check is skipped in a batch.) */
OV2_API ov2_status ov2_batch_begin(ov2_ctx* ctx);
OV2_API ov2_status ov2_batch_end(ov2_ctx* ctx);
/* Pinned host memory helpers (for callers that want true async H2D/D2H). */
OV2_API ov2_status ov2_host_alloc(ov2_ctx* ctx, size_t bytes, void** out);
OV2_API ov2_status ov2_host_free(ov2_ctx* ctx, void* p);
/* Number of kernels this context has launched since creation (bench.py's gpu_launches). */
OV2_API uint64_t   ov2_launch_count(const ov2_ctx* ctx);

/* Per-kernel timing with CUDA events on the launching stream (serialises launches; for
 * bench.py's roofline pass, never on during the timed benchmark region).
 * ov2_profile_query: idx-th kernel class -> name, accumulated ms, launch count; returns 0 past the end. */
OV2_API ov2_status ov2_profile_enable(ov2_ctx* ctx, int on);
OV2_API int        ov2_profile_query(const ov2_ctx* ctx, int idx, char* name_out, int name_cap, double* total_ms,
                             uint64_t* launches);

/* ------------------------------------------------------------------ P: pyramid
 * Replaces cv::buildOpticalFlowPyramid(img, pyr, Size(9,9), 3) as called by
 * VisualFrontEnd::preprocessImage (/root/reference/src/visual_front_end.cpp:1172, also :53 and
 * src/mapper.cpp:81).  The Scharr derivative planes are not materialised; the tracker
 * recomputes them on the fly from the 8-bit levels (identical values). */
OV2_API ov2_status ov2_pyr_create(ov2_ctx* ctx, int batch, int width, int height, int nlevels_extra, ov2_pyr** out);
OV2_API void       ov2_pyr_destroy(ov2_pyr* pyr);
/* Load `count` 8-bit images into frame slots [first, first+count) and build their levels.
 * `images` = host or device pointer; row r of image k starts at images + k*frame_stride + r*row_stride.
 * Device images are used in place as level 0 (they must stay alive and unchanged while the
 * pyramid is used); host images are copied into the pyramid's own level-0 storage. */
OV2_API ov2_status ov2_pyr_build(ov2_ctx* ctx, ov2_pyr* pyr, const uint8_t* images, size_t row_stride,
                         size_t frame_stride, int first, int count);
/* Copy one level of one frame slot back to host (tests). `out` holds level_w*level_h bytes, packed. */
OV2_API ov2_status ov2_pyr_download(ov2_ctx* ctx, const ov2_pyr* pyr, int frame, int level, uint8_t* out,
                            int* level_w, int* level_h);

/* ------------------------------------------------------------------ C: CLAHE
 * Replaces pclahe_->apply(img, img) with cv::createCLAHE(fclahe_val, Size(W/50, H/50))
 * (/root/reference/src/ov2slam.cpp:85-89; src/visual_front_end.cpp:1158-1160; src/mapper.cpp:75-76;
 * `use_clahe: 1`, the accurate/ configurations).  `count` 8-bit images, host or device; dst may
 * alias src only for host buffers (the device path reads src while writing dst). */
OV2_API ov2_status ov2_clahe(ov2_ctx* ctx, const uint8_t* src, uint8_t* dst, int width, int height, size_t row_stride,
                     size_t frame_stride, int count, double clip_limit, int tiles_x, int tiles_y);

/* preprocessImage as one call: VisualFrontEnd::preprocessImage (/root/reference/src/visual_front_end.cpp:1143-1177:
 * optional pclahe_->apply, prev/cur swap, cv::buildOpticalFlowPyramid) and the right-image path of Mapper::run
 * (src/mapper.cpp:75-81).  `raw` holds the untouched images (loaded with ov2_pyr_build; describeBRIEF reads the
 * raw image, src/map_manager.cpp:301-303,326-329); frames [first, first+count) of `out` receive the equalised level 0
 * (own storage) and levels 1.. built from it.  use_clahe = 0 (fast/ and average/ configurations): `out` aliases the raw
 * level 0.  The image is uploaded once however many operators read it. */
OV2_API ov2_status ov2_preprocess(ov2_ctx* ctx, const ov2_pyr* raw, ov2_pyr* out, int first, int count, int use_clahe,
                          double clip_limit, int tiles_x, int tiles_y);

/* ------------------------------------------------------------------ R: rectification / undistortion
 * Replaces CameraCalibration::rectifyImage(img, rect) (/root/reference/src/camera_calibration.cpp:233-241), i.e.
 * cv::remap(img, rect, undist_map_x_, undist_map_y_, cv::INTER_LINEAR) with the default BORDER_CONSTANT 0, which the
 * reference runs on every incoming image when `bdo_stereo_rect` or `bdo_undist` is set (src/ov2slam.cpp:239-243, 252-257).
 * 8-bit single-channel images, bit-exact with cv::remap.  A map is built once per camera (its maps come from
 * CameraCalibration::setUndistStereoMap, CV_16SC2 + CV_16UC1, src/camera_calibration.cpp:141, or setUndistMap, two CV_32FC1,
 * :92; fisheye maps are the same data) and has the image's size.
 *   map_type OV2_MAP_16SC2: map1 = int16 (x, y) pairs, map2 = uint16 interpolation-table indices (cv::convertMaps' layout);
 *            OV2_MAP_32FC1: map1 = float x, map2 = float y.  The values equal OpenCV's type codes (CV_16SC2, CV_32FC1).
 *   Strides in bytes; maps host or device (copied and converted at creation, then no longer needed).
 *   width or height above 2046 -> OV2_ERR_CAPACITY.
 * A map belongs to the device of the creating context and may be used by every context on that device; destroy it after
 * their last use. */
#define OV2_MAP_16SC2 11
#define OV2_MAP_32FC1 5
typedef struct ov2_remap_map ov2_remap_map;
OV2_API ov2_status ov2_remap_create(ov2_ctx* ctx, int map_type, int width, int height, const void* map1, size_t map1_stride,
                                    const void* map2, size_t map2_stride, ov2_remap_map** out);
OV2_API void       ov2_remap_destroy(ov2_remap_map* map);
/* `count` images of the map's size, frame k at src + k*src_frame_stride (likewise dst), host or device.  A host dst may alias
 * the host src (the reference calls rectifyImage(im0, im0), src/ov2slam.cpp:255-256); a device dst may not. */
OV2_API ov2_status ov2_remap(ov2_ctx* ctx, const ov2_remap_map* map, const uint8_t* src, size_t src_row_stride, size_t src_frame_stride,
                             uint8_t* dst, size_t dst_row_stride, size_t dst_frame_stride, int count);
/* ov2_pyr_build with the rectification fused in: the unrectified images (host: uploaded once; device: read in place) are
 * remapped into the pyramid's OWN level 0 of frame slots [first, first+count), then its levels are built.  ov2_preprocess, the
 * detectors, ov2_describe and ov2_fb_klt run on that pyramid unchanged.  The map must have the pyramid's level-0 size. */
OV2_API ov2_status ov2_pyr_build_remap(ov2_ctx* ctx, ov2_pyr* pyr, const ov2_remap_map* map, const uint8_t* images, size_t row_stride,
                                       size_t frame_stride, int first, int count);

/* ------------------------------------------------------------------ K: forward/backward KLT
 * Replaces FeatureTracker::fbKltTracking(vprevpyr, vcurpyr, nwinsize, nbpyrlvl, ferr,
 * fmax_fbklt_dist, vkps, vpriorkps, vkpstatus) (/root/reference/src/feature_tracker.cpp:35-137;
 * declaration include/feature_tracker.hpp:44-47), i.e. forward cv::calcOpticalFlowPyrLK with
 * USE_INITIAL_FLOW|LK_GET_MIN_EIGENVALS, the status/err/inBorder filter, the level-0 backward
 * pass and the forward-backward distance test, fused per keypoint. */
typedef struct {
    int   win;        /* nwinsize: any size from 3 to 31, even sizes included (Size(win, win)); OV2_ERR_INVALID outside
                         that range.  9 (every shipped configuration) runs its own kernel, every other size a general one */
    int   max_iter;   /* klt_convg_crit_.maxCount (30) */
    float eps;        /* klt_convg_crit_.epsilon (0.01f) */
    float ferr;       /* nklt_err (30) */
    float fb_dist;    /* fmax_fbklt_dist (0.5) */
} ov2_klt_params;

/* n keypoints.  nbpyrlvl: per-keypoint pyramid depth (the reference's two calls, nbpyrlvl 1 for
 * keypoints with a 3D prior and 3 for the rest, visual_front_end.cpp:196,242, become one launch),
 * or NULL to use nbpyrlvl_all for every keypoint.  kps = vkps (n x 2 float), priors_inout =
 * vpriorkps (in: initial guess, out: forward result), status_out = vkpstatus (n bytes, 0/1).
 * Keypoints with x < 0 are empty-slot markers of fixed-stride batches (the detectors pad with (-1, -1)):
 * status 0, prior untouched.
 * Depths are clamped as the reference clamps nbpyrlvl (feature_tracker.cpp:50-52): to the depth
 * cv::buildOpticalFlowPyramid(img, pyr, Size(win, win), levels - 1) reaches, i.e. never to a level
 * whose width or height is <= win.  On small images that is shallower than the pyramid's levels
 * (96x72 and 64x48: 2, 40x30: 1, 17x16: 0); the levels themselves stay exact pyrDown images. */
OV2_API ov2_status ov2_fb_klt(ov2_ctx* ctx, const ov2_pyr* prev, const ov2_pyr* cur, const ov2_klt_params* prm,
                      int n, const int32_t* frame_idx, int first_frame, int per_frame,
                      const uint8_t* nbpyrlvl, int nbpyrlvl_all,
                      const float* kps, float* priors_inout, uint8_t* status_out);

/* Measurement hook: ov2_fb_klt with the same arguments and results, plus counts_out (2 n int32): level set-ups (template
 * built) at 2 i and Lucas-Kanade iterations at 2 i + 1, forward and backward tracks of keypoint i together.  A second
 * instantiation of the kernel; ov2_fb_klt carries no counter. */
OV2_API ov2_status ov2_debug_klt_counts(ov2_ctx* ctx, const ov2_pyr* prev, const ov2_pyr* cur, const ov2_klt_params* prm,
                      int n, const int32_t* frame_idx, int first_frame, int per_frame,
                      const uint8_t* nbpyrlvl, int nbpyrlvl_all,
                      const float* kps, float* priors_inout, uint8_t* status_out, int32_t* counts_out);

/* ------------------------------------------------------------------ K2: the front-end's frame tracking
 * Replaces VisualFrontEnd::kltTracking() (/root/reference/src/visual_front_end.cpp:132-275) for frames [first, first+count)
 * of two pyramids.  Frame k owns keypoints [offsets[k], offsets[k+1]) of px ([n][2] float, kp.px_), wpt ([n][3] double, the
 * keypoint's map point; read only where is3d) and is3d ([n] bytes, kp.is3d_); n = offsets[count].  Per frame: Tcw[k] = 12
 * doubles (row-major rotation, then translation, as ov2_match_problem), K[k] = fx, fy, cx, cy, dist[k] = k1, k2, p1, p2, k3 of
 * the radial-tangential model (dist NULL: no distortion in any frame), img_wh[k] = the calibration's image width, height.
 *   prior    Frame::projWorldToImageDist (src/frame.cpp:825-828, src/camera_calibration.cpp:254-281): Tcw * X in double,
 *            invz = 1 / z, x * invz, y * invz; without distortion fx * x + cx in double rounded to float, with it
 *            cv::projectPoints on Point3f(x, y, 1) as ov2_match_to_map evaluates it.  z is not tested (the reference does not):
 *            a point behind the camera whose projection lands in the image gets a prior.
 *   in image Frame::isInImage (src/frame.cpp:840-843): x >= 0 && y >= 0 && x < img_w && y < img_h, float against int.
 *   pass 1   the 3-D keypoints whose prior is in the image, tracked from the prior at depth 1 (fbKltTracking, nbpyrlvl 1).
 *            Skipped when use_prior == 0 or the frame has no such keypoint.
 *   rule     p3p_req = nbgood < 0.33 * nbkps in double, on the frame's pass-1 counts (0 when pass 1 is skipped).
 *   pass 2   the 2-D keypoints, the 3-D keypoints without an in-image prior (prior = px) and the failed pass-1 keypoints,
 *            at depth nklt_pyr_lvl; a failed pass-1 keypoint starts from its pass-1 forward result, or from px when p3p_req.
 * Outputs: tracked_out ([n][2]: the pass-1 result of a pass-1 track, else the pass-2 forward result, the position the
 * reference's updateKeypoint receives for a tracked keypoint), status_out ([n] 0/1), pass_out ([n]: 0 none, 1 pass 1,
 * 2 pass 2); per frame p3p_req_out, nbgood_out and nbkps_out (pass-1 counts).  A keypoint with px.x < 0 is an empty slot:
 * pass 0, status 0, tracked = px, not counted.
 * Both passes are ov2_fb_klt over all n slots (non-members are empty slots): status and positions equal to fbKltTracking
 * on each pass's keypoints.  offsets must be a HOST pointer that starts at 0 and never decreases (OV2_ERR_INVALID
 * otherwise, nothing staged or written); every other array may be host or device memory.  There is no host
 * synchronisation between the passes; with device arrays the call only enqueues. */
OV2_API ov2_status ov2_klt_tracking(ov2_ctx* ctx, const ov2_pyr* prev, const ov2_pyr* cur, const ov2_klt_params* prm, int first,
                                    int count, const int32_t* offsets, const double* Tcw, const double* K, const double* dist,
                                    const int32_t* img_wh, const float* px, const double* wpt, const uint8_t* is3d,
                                    int nklt_pyr_lvl, int use_prior, float* tracked_out, uint8_t* status_out, uint8_t* pass_out,
                                    uint8_t* p3p_req_out, int32_t* nbgood_out, int32_t* nbkps_out);

/* ------------------------------------------------------------------ F + S: grid FAST + cornerSubPix
 * Replaces FeatureExtractor::detectGridFAST(im, ncellsize, vcurkps, roi)
 * (/root/reference/src/feature_extractor.cpp:443-570; include/feature_extractor.hpp:41-42) with
 * the sequential ascending cell order as the defined semantics, including the CV_32F-mask byte
 * aliasing, libstdc++ std::sort tie resolution, the response >= 20 rule, disc painting, the
 * adaptive nfast_th_ update (:546-552) and cv::cornerSubPix((3,3),(-1,-1),{30,0.01}) (:556-565).
 *
 * Frames [first, first+count) of `pyr` (level 0).  Existing keypoints of frame k are
 * curkps[2*curkp_offsets[k] .. 2*curkp_offsets[k+1]) (curkp_offsets has count+1 entries; NULL =
 * no existing keypoints).  fast_th_inout[k] is the per-stream nfast_th_ state (in: threshold to
 * use, out: adapted threshold).  out_pts holds count * max_per_frame points (x, y float; unused
 * slots are set to (-1, -1)), in the reference's cell order; out_counts[k] = number found;
 * max_per_frame >= (H/cellsize)*(W/cellsize).  out_pts_int (optional, may be NULL) receives the
 * integer pixel positions before sub-pixel refinement (int32 x, y). */
OV2_API ov2_status ov2_grid_fast(ov2_ctx* ctx, const ov2_pyr* pyr, int first, int count, int cellsize,
                         const int32_t* curkp_offsets, const float* curkps,
                         int32_t* fast_th_inout, int max_per_frame,
                         float* out_pts, int32_t* out_counts, int32_t* out_pts_int, int do_subpix);

/* ------------------------------------------------------------------ D + S: single-scale detector + cornerSubPix
 * ("next" row, SURVEY.md 8f-1; the detector of the accurate/ and average/ configurations)
 * Replaces FeatureExtractor::detectSingleScale(im, ncellsize, vcurkps, roi)
 * (/root/reference/src/feature_extractor.cpp:288-440; include/feature_extractor.hpp:38-39): per cell
 * cv::GaussianBlur(3x3) + cv::cornerMinEigenVal(3, 3), first maximum of response * mask twice with the
 * disc mask, second detections admitted while cells stayed empty (:400-412), the adaptive dmaxquality_
 * update (:418-423) and cv::cornerSubPix (:424-436); sequential ascending cell order as the defined
 * semantics.  Arguments as ov2_grid_fast; roi_xywh = {x, y, width, height} on the HOST (NULL = whole
 * image); quality_inout[k] is the per-stream dmaxquality_ state (double, in/out); cellsize in [8, 64]. */
OV2_API ov2_status ov2_detect_single_scale(ov2_ctx* ctx, const ov2_pyr* pyr, int first, int count, int cellsize,
                         const int32_t* curkp_offsets, const float* curkps, const int32_t* roi_xywh,
                         double* quality_inout, int max_per_frame,
                         float* out_pts, int32_t* out_counts, int32_t* out_pts_int, int do_subpix);

/* Largest number of FAST candidates (strict 3x3 maxima at cell-local x % 4 in {2, 3}) a cell of `cellsize` can hold:
 * ((cellsize - 6) / 4 + 1) * ((cellsize - 5) / 2), e.g. 264 at 50 and 1891 at 128; 0 outside [8, 128].  ov2_grid_fast
 * keeps that many per cell, so no input is refused for its content. */
OV2_API int ov2_fast_cell_capacity(int cellsize);

/* Test hook: stage F1 alone (per-cell FAST-9/16 + NMS candidates of one frame, pre-filtered by the
 * mask byte rule), for cell-by-cell parity against cv::FastFeatureDetector.  cap_in >= ov2_fast_cell_capacity(cellsize)
 * words per cell. */
OV2_API ov2_status ov2_debug_fast_cells(ov2_ctx* ctx, const ov2_pyr* pyr, int frame, int cellsize, int fast_th,
                                uint32_t* cand_out, int32_t* cand_n_out, int cap_in, int* cap_out);

/* Measurement hook: cornerSubPix alone on count * max_per_frame integer points (x < 0: empty slot) of frames
 * [first, first + count), as ov2_grid_fast runs it.  out_pts: the refined points; iters_out: iterations run per slot
 * (1 .. 30; -1 for an empty slot).  Host or device pointers. */
OV2_API ov2_status ov2_debug_subpix_iters(ov2_ctx* ctx, const ov2_pyr* pyr, int first, int count, int max_per_frame,
                                  const int32_t* pts_int, float* out_pts, int32_t* iters_out);

/* ------------------------------------------------------------------ ceresPnP (motion-only BA), "next" row 2
 * Replaces MultiViewGeometry::ceresPnP(vunkps, vwpts, vscales, Twc, nmaxiter, chi2th, buse_robust,
 * bapply_l2_after_robust, fx, fy, cx, cy, voutliersidx)
 * (/root/reference/src/multi_view_geometry.cpp:492-588; called per frame at src/visual_front_end.cpp:791-801),
 * batched: problem k owns points [offsets[k], offsets[k+1]) of unpx ([N][2] undistorted pixels), wpts ([N][3]
 * world points) and scales (pyramid level per point or NULL), calibration K[k] = fx, fy, cx, cy and pose
 * Twc[k] = tx,ty,tz,qx,qy,qz,qw (in: initial guess, out: refined; unchanged when every block is rejected).
 * ReprojectionErrorSE3 residuals with SE3LeftParameterization, HuberLoss(sqrt(chi2th)), Ceres' Levenberg-
 * Marquardt loop (DENSE_QR in the reference; 6x6 damped normal equations here), max nmaxiter iterations,
 * function tolerance 1e-3; blocks with chi2 > chi2th or non-positive depth after the first solve are flagged
 * in outlier_flags (and removed before an L2 re-solve when apply_l2_after_robust).  success_out[k] = the
 * reference's return value.  The 5 ms wall-clock cap of the reference (:538) is not modelled.
 * offsets must be a HOST pointer, start at 0 and never decrease (else OV2_ERR_INVALID, nothing staged or
 * written); the other arrays may be host or device memory.  An empty problem returns success 0 and its pose as
 * given.  The start quaternion is normalised as Sophus' SE3d(q, t) would.  iterations_out (optional, NULL
 * accepted) = LM iterations of the last solve of each problem: every iteration started, so a solve that a
 * tolerance ends inside an iteration counts it, where Ceres' Summary::iterations.size() (which also counts
 * iteration 0) does not.
 * Known deviation: when a solve is unusable (five consecutive invalid steps, Ceres' FAILURE), Ceres restores the
 * parameters it started from; this kernel writes its best iterate (success_out is 0 either way).
 * Tested: the solve code compiled for the host against the oracle and against the real Ceres; the kernel by
 * tests/test_pnp_gpu.py and tests/test_pnp_paths_gpu.py on 1 to 20 000 points per problem, per-problem K, levels
 * 0-3 and NULL, every option the callers vary, points behind the camera, batches of > 1 000 problems, device
 * buffers and refused offsets: success, outlier flags and iterations exact, pose to 1e-9 of the oracle. */
OV2_API ov2_status ov2_pnp_solve(ov2_ctx* ctx, int nprob, const int32_t* offsets, const double* unpx, const double* wpts,
                         const int32_t* scales, const double* K, double* pose_inout, int nmaxiter, float chi2th,
                         int use_robust, int apply_l2_after_robust, uint8_t* outlier_flags, uint8_t* success_out,
                         int32_t* iterations_out);

/* ------------------------------------------------------------------ B: descriptors
 * Replaces FeatureExtractor::describeBRIEF(im, vpts)
 * (/root/reference/src/feature_extractor.cpp:224-285), non-contrib branch
 * cv::ORB::create(500, 1., 0) (:245): 256 tests of the ORB pattern on the float32-Gaussian
 * smoothed image, centre = cvRound(pt), points whose rounded centre is closer than 31 px to the
 * border (and points with x < 0, used as "empty slot" markers) get valid = 0 and a zero
 * descriptor, mirroring the empty cv::Mat the reference returns for them. */
OV2_API ov2_status ov2_describe(ov2_ctx* ctx, const ov2_pyr* pyr, int n, const int32_t* frame_idx, int first_frame, int per_frame,
                        const float* pts, uint8_t* desc32_out, uint8_t* valid_out);

/* Descriptor selection for ov2_describe on this context (the reference selects it at compile time,
 * /root/reference/CMakeLists.txt:12,35-39 and src/feature_extractor.cpp:69-70,242-246):
 *   OV2_DESC_ORB_FALLBACK (default, pairs = NULL): the non-contrib branch described above.
 *   OV2_DESC_BRIEF32: cv::xfeatures2d::BriefDescriptorExtractor::create() (32 bytes, no orientation):
 *     256 tests SMOOTHED(y0, x0) < SMOOTHED(y1, x1) of 9 x 9 box sums around (int)(pt + 0.5), first test of a
 *     byte in bit 7, border 28 px.  `pairs` = int8[256][4] = (y0, x0, y1, x1) in the order of opencv_contrib's
 *     modules/xfeatures2d/src/generated_32.i (that table is not redistributed here; |offset| <= 24 is checked). */
#define OV2_DESC_ORB_FALLBACK 0
#define OV2_DESC_BRIEF32 1
OV2_API ov2_status ov2_describe_config(ov2_ctx* ctx, int mode, const int8_t* pairs);

/* ------------------------------------------------------------------ 8f-3: stereo prior by a row search
 * Replaces the per-keypoint loop over FeatureTracker::getLineMinSAD(iml, imr, pt, nwinsize, xprior, l1err, bgoleft)
 * (/root/reference/src/feature_tracker.cpp:138-204) that MapManager::stereoMatching runs for every 2-D keypoint of a
 * keyframe on the coarsest pyramid level when `bdo_stereo_rect` is set (/root/reference/src/map_manager.cpp:417-431):
 * for each point (coordinates of pyramid level `level`) the column of the right image, scanned in unit steps from the
 * point's own column (downwards when goleft), whose nwinsize x nwinsize window has the smallest mean absolute
 * difference to the sub-pixel patch of the left image.  xprior_out = that column (float, same fractional part as the
 * input) or -1 when the window shrinks to nothing at the border / no candidate is below 255; l1err_out = the minimum
 * (255 when xprior is -1; the reference leaves it unset there).  nwinsize must be odd (OV2_ERR_INVALID otherwise, the
 * reference prints a message and returns) and <= 15.  Frame addressing as ov2_fb_klt. */
OV2_API ov2_status ov2_line_min_sad(ov2_ctx* ctx, const ov2_pyr* left, const ov2_pyr* right, int level, int n,
                            const int32_t* frame_idx, int first_frame, int per_frame, const float* pts, int nwinsize,
                            int goleft, float* xprior_out, float* l1err_out);

/* ------------------------------------------------------------------ 8f-4: local-map matching
 * The data-parallel core of Mapper::matchToMap(frame, fmaxprojerr, fdistratio, set_local_lmids)
 * (/root/reference/src/mapper.cpp:576-774): for every candidate map point of the local map (cand_mp, in the caller's
 * iteration order) projection into the frame, culling, the keypoints of the four surrounding grid cells
 * (Frame::getSurroundingKeypoints, src/frame.cpp:624-650), pixel distance, "never observed together", mean co-projection
 * error, minimal descriptor distance (MapPoint::computeMinDescDist, src/map_point.cpp:236-252), best / second with the
 * 0.9 ratio test -> best_kp_out[ncand] (keypoint index or -1), best_dist_out[ncand]; then per keypoint the candidate with
 * the smallest distance (later candidates win ties) -> kp_match_out[nkps] (index INTO cand_mp or -1), kp_dist_out[nkps]
 * (1024 when unmatched).  The caller (the Mapper shim) flattens the map and applies the merges (mapper.cpp:559-570).
 * Map-point table = the candidates AND the map points of the frame's keypoints.  Rotations are 3x3 matrices (row major)
 * followed by the translation: Tcw[12], kf_Tcw[nkfs][12].  dist = (k1, k2, p1, p2, k3) of the pinhole model or NULL
 * (fisheye calibrations are not built: keep the reference's matchToMap for them).  dmaxpxdist = fmaxprojerr, doubled by
 * the caller when the frame has fewer than 30 3-D keypoints (:597-600); view_th = cos(max half field of view) (:586-596). */
typedef struct {
    double Tcw[12]; double K[4]; const double* dist;
    int img_w, img_h, ncellsize, nbwcells, ncells;
    const int32_t* cell_ptr;      /* [ncells + 1] keypoints per grid cell (Frame::vgridkps_), CSR */
    const int32_t* cell_kp;       /* [nkps] keypoint indices, cell by cell, in the cell lists' order */
    int nkps; const float* kp_px; /* [nkps][2] kp.px_ */
    const int32_t* kp_lm;         /* [nkps] map-point table index of the keypoint's map point, -1: none */
    int nmps; const double* mp_xyz;                                   /* [nmps][3] */
    const int32_t* mp_desc_ptr; int ndesc; const uint8_t* desc;       /* [nmps + 1], [ndesc][32] */
    const uint64_t* mp_kfmask;    /* [nmps][4] bit k: observed by local keyframe k (k < 256) */
    const int32_t* mp_obs_ptr; int nobs; const int32_t* obs_kf; const float* obs_px;   /* [nmps + 1], [nobs], [nobs][2] */
    int nkfs; const double* kf_Tcw;                                   /* [nkfs][12] */
    int ncand; const int32_t* cand_mp;
    float dmaxpxdist, fdistratio, view_th;
} ov2_match_problem;
OV2_API ov2_status ov2_match_to_map(ov2_ctx* ctx, const ov2_match_problem* p, int32_t* best_kp_out, float* best_dist_out,
                            int32_t* kp_match_out, float* kp_dist_out);

/* ------------------------------------------------------------------ composite: one front-end step
 * P(prev), P(cur), K, F+S on cur (no existing keypoints), B(tracked), B(new) for `count` frame pairs in
 * ONE call (batch mode inside): what VisualFrontEnd::trackMono + MapManager::extractKeypoints do per
 * frame (/root/reference/src/visual_front_end.cpp:65-128, src/map_manager.cpp:286-341).  Pointers
 * host or device as everywhere; n_kps = count * kps_per_frame; cellsize <= 0 skips F/B(new).
 * The step is captured into a CUDA graph per distinct argument block (at most 16 are kept per context): zero the struct
 * before filling it (its padding bytes are part of the cache key), and reuse argument blocks - a block that changes every
 * call runs eagerly. */
typedef struct {
    const uint8_t* prev_images; const uint8_t* cur_images; size_t row_stride, frame_stride; int count;
    ov2_klt_params klt; int n_kps, kps_per_frame; const uint8_t* nbpyrlvl; int nbpyrlvl_all;
    const float* kps; float* priors_inout; uint8_t* status_out;
    int cellsize; int32_t* fast_th_inout; int max_per_frame; float* new_pts; int32_t* new_counts;
    uint8_t* desc_tracked; uint8_t* valid_tracked; uint8_t* desc_new; uint8_t* valid_new;
} ov2_frontend_step_args;
OV2_API ov2_status ov2_frontend_step(ov2_ctx* ctx, ov2_pyr* prev, ov2_pyr* cur, const ov2_frontend_step_args* args);

/* ------------------------------------------------------------------ L: local bundle adjustment
 * Replaces the solve sections of Optimizer::localBA(Frame&, bool)
 * (/root/reference/src/optimizer.cpp:436-479 robust solve, :492-594 outlier scan,
 *  :603-627 refinement, :637-735 second scan), i.e. Ceres 2.0 TrustRegionMinimizer +
 * LevenbergMarquardtStrategy + SCHUR linear solver on ReprojectionErrorKSE3AnchInvDepth
 * residuals (src/ceres_parametrization.cpp:361-473) with SE3LeftParameterization.
 * The flat problem description is what localBA's setup (:43-430) builds from the map. */
typedef struct {
    int32_t  ncam, npts, nobs;
    const double*  K;              /* [4] fx, fy, cx, cy (constant block) */
    double*        pose;           /* [ncam][7] Twc = tx,ty,tz,qx,qy,qz,qw ; in/out */
    const uint8_t* pose_const;     /* [ncam] 1 = SetParameterBlockConstant */
    const int32_t* lm_anchor_cam;  /* [npts] */
    const double*  lm_anchor_px;   /* [npts][2] undistorted anchor pixel */
    double*        lm_invdepth;    /* [npts] in/out */
    const int32_t* obs_cam;        /* [nobs] observing camera (non-anchor observations) */
    const int32_t* obs_lm;         /* [nobs] landmark index, sorted ascending (CSR by landmark) */
    const double*  obs_px;         /* [nobs][2] */
    /* stereo windows (NULL / ignored for mono): residual type per observation -
     *   0 left camera, other keyframe    ReprojectionErrorKSE3AnchInvDepth             (ceres_parametrization.cpp:361-473)
     *   1 right camera, other keyframe   ReprojectionErrorRightCamKSE3AnchInvDepth     (:579-712)
     *   2 right camera, anchor keyframe  ReprojectionErrorRightAnchCamKSE3AnchInvDepth (:476-577; obs_cam = anchor)
     * Kr = right calibration [4], Trl = constant right-from-left extrinsic [7] (tx..tz, qx..qw). */
    const uint8_t* obs_type;       /* [nobs] or NULL */
    const double*  Kr;             /* [4] or NULL */
    const double*  Trl;            /* [7] or NULL */
} ov2_ba_problem;

typedef struct {
    int    max_iters_robust;   /* 5  (optimizer.cpp:462) */
    int    max_iters_refine;   /* 10 (optimizer.cpp:610) */
    double huber_th;           /* robust_mono_th = 5.9915 (loss = HuberLoss(sqrt(th)), :49) */
    double function_tolerance; /* 1e-3 (:463) */
    int    use_robust;         /* buse_robust_cost */
    int    apply_l2_after_robust; /* (:603) */
    int    refine_loss;        /* refinement loss: -1 = as the reference decides (trivial loss iff left-camera AND
                                * other-frame right-camera residuals both survive the first scan, :606-608; i.e.
                                * mono windows keep Huber), 0 = keep the robust loss, 1 = trivial loss */
} ov2_ba_opts;

typedef struct {
    int    iters_robust, iters_refine;  /* LM iterations executed (successful + unsuccessful) */
    double initial_cost, final_cost;    /* of the last solve that ran */
    int    n_outliers_first, n_outliers_second;
    int    termination;                 /* 0 convergence, 1 max iterations, 2 failure */
} ov2_ba_result;

/* outlier_out (optional): [nobs] bytes, bit0 = flagged after solve #1, bit1 = after solve #2.
 * The whole two-stage solve (both Ceres solves, every LM iteration, both outlier scans) is ONE kernel launch with the
 * trust-region controller on the device (csrc/ba_lm.cu).  At most 64 optimised keyframes per window (OV2_ERR_CAPACITY
 * beyond): non-constant keyframes that no residual touches (or only right-camera residuals in their own anchor frame,
 * obs_type 2) drop out of the problem as in Ceres and do not count, except in a multi-GPU window, where every declared
 * non-constant keyframe counts.  No limit on the total keyframe count (constant keyframes included).
 * Residency of a window's arrays is decided on `pose`: host poses = every array of the window (and outlier_out) is host
 * memory, the reference's flow; device poses = each array is inspected and may be either. */
OV2_API ov2_status ov2_localba_solve(ov2_ctx* ctx, const ov2_ba_problem* pb, const ov2_ba_opts* opts,
                             ov2_ba_result* res, uint8_t* outlier_out);

/* K independent windows in ONE launch (the solves/s metric; SURVEY.md 7 "hard parts" (ii)): window k is pbs[k] with results[k]
 * and outlier_outs[k] (NULL entries / NULL array allowed); the same options for every window.  Groups of thread blocks pull
 * windows round-robin, every group runs the whole two-stage solve of its window on the device. */
OV2_API ov2_status ov2_localba_solve_batch(ov2_ctx* ctx, int nprob, const ov2_ba_problem* pbs, const ov2_ba_opts* opts,
                                   ov2_ba_result* results, uint8_t* const* outlier_outs);

/* Optimizer::signalStopLocalBA / stopLocalBA (/root/reference/src/optimizer.cpp:2334-2343, raised by Estimator::addNewKf,
 * src/estimator.cpp:228-232): stop = 1 asks the solve running (or about to run) on `ctx` to skip the L2 refinement; the
 * solve kernel polls the flag where the reference does (optimizer.cpp:603-604).  May be called from another host thread
 * while ov2_localba_solve runs; the caller clears it (stop = 0) as optimizer.cpp:896 does. */
OV2_API ov2_status ov2_localba_request_stop(ov2_ctx* ctx, int stop);

/* Multi-GPU localBA over PEER MEMORY (BASELINE.json configs[4], SURVEY.md 8e).  One process per GPU (or several contexts in one
 * process): every rank creates a communicator (it allocates the rank's exchange buffer), the 64-byte CUDA IPC handles are
 * exchanged by the caller (torch.distributed.all_gather, MPI, a pipe ...) and handed to ov2_ba_comm_connect.  The solve is
 * collective: every rank calls ov2_localba_solve_p2p with ITS shard (landmarks with all their observations partitioned over
 * the ranks, every rank holds all keyframe poses; a shard may be empty).  Inside the solve kernel every LM iteration sums
 * the ranks' partial reduced camera systems [cost, rhs, F'r, column norms, S] straight out of peer memory over NVLink
 * (rank order, so every rank holds bit-identical sums, solves the same system and takes the same decisions): no NCCL call
 * and no host round trip between iterations.  Poses come back identical on all ranks, inverse depths / flags / outlier
 * counts are the shard's own.  A window of more than 256 keyframes (constant ones included) is refused with
 * OV2_ERR_CAPACITY when world > 1; every rank refuses it on the host before anything is launched, so no rank waits for a
 * peer that never started.  With world == 1 the window is solved as ov2_localba_solve would. */
typedef struct ov2_ba_comm ov2_ba_comm;
OV2_API ov2_status ov2_ba_comm_create(ov2_ctx* ctx, int rank, int world, ov2_ba_comm** out);       /* world <= 8 */
OV2_API ov2_status ov2_ba_comm_handle(ov2_ba_comm* comm, void* handle_out, size_t handle_bytes);    /* >= 64 bytes */
OV2_API ov2_status ov2_ba_comm_connect(ov2_ba_comm* comm, const void* handles, size_t handle_stride);   /* world handles, rank order */
OV2_API ov2_status ov2_ba_comm_connect_local(ov2_ba_comm* comm, ov2_ba_comm* const* all);            /* all ranks in this process */
OV2_API void       ov2_ba_comm_destroy(ov2_ba_comm* comm);
OV2_API ov2_status ov2_localba_solve_p2p(ov2_ctx* ctx, ov2_ba_comm* comm, const ov2_ba_problem* pb, const ov2_ba_opts* opts,
                                 ov2_ba_result* res, uint8_t* outlier_out);

#ifdef __cplusplus
}
#endif
#endif /* OV2B200_H */
