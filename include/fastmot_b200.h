/*
 * fastmot_b200 — C-ABI of the H100-native FastMOT hot path (libfastmot_b200.so, sm_90a).
 *
 * The reference (GeekAlexis/FastMOT) is Python; its only native boundary is the TensorRT plugin
 * "YoloLayer_TRT" (fastmot/plugins/yolo_layer.h:44-147) loaded with ctypes
 * (fastmot/utils/inference.py:49-53).  This header is what the reference's Python stages bind instead
 * (ctypes stubs in INTEGRATION.md).  Each entry point cites the reference code it replaces.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name starts with `h_` (host) or says so;
 *   - the caller owns all memory; kernels never allocate, never synchronise;
 *   - `stream` is a cudaStream_t passed as void*;
 *   - return 0 on success, non-zero error code otherwise (text via fm_last_error());
 *   - boxes are inclusive-pixel tlbr doubles [x1,y1,x2,y2] as in fastmot/utils/rect.py.
 */
#ifndef FASTMOT_B200_H
#define FASTMOT_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---------------------------------------------------------------- library ---------------------------------- */
const char* fm_last_error(void);
int fm_version(void);
/* 1 if a CUDA device with compute capability 9.x is present and usable, else 0 (no kernels are run). */
int fm_device_ok(void);
/* cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, stream) — lets the Python host move small blocks without
 * another CUDA binding. */
int fm_memcpy_async(void* dst, const void* src, long long bytes, void* stream);
/* kernels launched through this library so far in the process (bench.py `gpu_launches`). */
long long fm_launch_count(void);
/* 1 if the HOST pointer is page-locked (cudaHostAlloc / cudaHostRegister), else 0. */
int fm_host_is_pinned(const void* h_ptr);

/* ---------------------------------------------------------------- Kalman filter ----------------------------- */
/* Mirrors fastmot/kalman_filter.py:14-24 (ctor params) + :294-306 (_init_mat). */
typedef struct FmKalmanParams {
    double trans_mat[64];     /* A, row-major 8x8 */
    double acc_cov[64];       /* Q0, row-major 8x8 */
    double std_factor_acc, std_offset_acc;
    double std_factor_det[2], std_factor_klt[2];
    double min_std_det[2], min_std_klt[2];
    double init_pos_weight, init_vel_weight;
} FmKalmanParams;

#define FM_KF_WARP 1      /* kalman_filter.py:227-292 */
#define FM_KF_PREDICT 2   /* kalman_filter.py:128-147, 308-319 */
#define FM_KF_UPDATE 4    /* kalman_filter.py:180-204, 321-345 */
#define FM_KF_MEAS_DET 8  /* measurement noise of MeasType.DETECTOR, else MeasType.FLOW */
#define FM_KF_MEAS_BY_SLOT 16 /* meas / has_meas are slot-indexed pools instead of per-item arrays */

/* One launch for the whole track set; replaces the per-track loop of tracker.py:164-183 (flags
 * WARP|PREDICT|UPDATE, FLOW noise, multiplier = mult_num[i] / mult_den_pool[slot]) and of tracker.py:262-274
 * (flags UPDATE|MEAS_DET).  State lives in slot-indexed pools mean_pool[cap][8], cov_pool[cap][64].
 * slots[n] selects the tracks; meas[n][4], has_meas[n] (NULL = all), mult_num[n] (NULL = 1).
 * h_ok: optional device flag; if *h_ok == 0 the launch is a no-op (flow failed, tracker.py:160-162).
 * hold: optional device flag; if *hold != 0 the launch is a no-op as well (the per-track KLT rounds that were enqueued
 * ahead did not reach their fixed point; the caller runs more rounds and launches again).
 * out_tlbr[n][4] = round-half-even(mean[:4]) (rect.py:5-12), also stored to tlbr_pool[slot] when non-NULL;
 * out_lost[n] = ios(box, frame) < 0.5 (tracker.py:179). */
int fm_kalman_step_batched(double* mean_pool, double* cov_pool, double* tlbr_pool, const int* slots, int n, int flags,
                           const double* homography, const int* h_ok, const int* hold, const double* meas,
                           const unsigned char* has_meas, const double* mult_num, const double* mult_den_pool,
                           const FmKalmanParams* h_params, double frame_w, double frame_h, double* out_tlbr,
                           unsigned char* out_lost, void* stream);

/* kalman_filter.py:96-126 for n detections at once; box i is tlbr[tlbr_idx ? tlbr_idx[i] : i]. */
int fm_kalman_create_batched(double* mean_pool, double* cov_pool, double* tlbr_pool, const int* slots,
                             const double* tlbr, const int* tlbr_idx, int n, const FmKalmanParams* h_params,
                             void* stream);

/* kalman_filter.py:206-225: out[n_trk][n_det] squared Mahalanobis distances (slots NULL = identity). */
int fm_motion_distance(const double* mean_pool, const double* cov_pool, const int* slots, int n_trk,
                       const double* det_tlbr, int n_det, const FmKalmanParams* h_params, double* out, void* stream);

/* ---------------------------------------------------------------- association ------------------------------ */
#define FM_METRIC_EUCLIDEAN 0 /* fastmot/utils/distance.py:11-13 */
#define FM_METRIC_COSINE 1
#define FM_INF_COST 1e5       /* fastmot/utils/matching.py:7 */
#define FM_CHI_SQ_INV_95 9.4877

/* Fused replacement of MultiTracker._matching_cost (tracker.py:314-341):
 *   cdist(features, embeddings, metric, empty_mask, fill) (distance.py:16-87)
 *   + per-row Mahalanobis gating (kalman_filter.py:206-225, 347-353)
 *   + fuse_motion (matching.py:100-106) + gate_cost (matching.py:109-116).
 * feat_pool[cap][dim] f32 running-average features, feat_valid_pool[cap] (count > 0);
 * trk_slots[n_trk], trk_labels[n_trk]; det_* arrays have n_det rows, det_sel[n_det] (NULL = identity) selects
 * the rows of the full detection arrays that are still unmatched.  cost[n_trk][n_det] f64 row-major.
 * The label gate applies only when both trk_labels and det_labels are non-NULL (as in fm_iou_cost).
 * motion_weight < 0 disables the motion term; max_cost < 0 disables the cost gate (tracker.py:355-366 re-ID). */
int fm_matching_cost(const float* feat_pool, const unsigned char* feat_valid_pool, const double* mean_pool,
                     const double* cov_pool, const int* trk_slots, const long long* trk_labels, int n_trk,
                     const float* det_emb, const double* det_tlbr, const long long* det_labels,
                     const unsigned char* det_occluded, const int* det_sel, int n_det, int dim, int metric,
                     double fill_val, double motion_weight, double max_cost, const FmKalmanParams* h_params,
                     double* cost, void* stream);

/* AverageFeature.update / merge (fastmot/track.py:100-126) for n tracks at once.
 * vec[.][dim] rows selected by vec_idx[n] (NULL = identity); counts[n] = the NEW count of each track
 * (count == 1: sum = avg = vec; else sum += vec, avg = normalise(sum / count)).  Sets valid_pool[slot] = 1. */
int fm_feature_update(float* sum_pool, float* avg_pool, float* last_pool, unsigned char* valid_pool, const int* slots,
                      const float* vec, const int* vec_idx, const int* counts, int n, int dim, void* stream);

/* iou_dist (distance.py:90-108) + gate_cost (matching.py:109-116); boxes gathered by index lists.
 * trk_tlbr_pool[cap][4]; the label gate applies only when both label arrays are non-NULL, max_cost < 0 disables the
 * cost gate. */
int fm_iou_cost(const double* trk_tlbr_pool, const int* trk_slots, const long long* trk_labels, int n_trk,
                const double* det_tlbr, const long long* det_labels, const int* det_sel, int n_det,
                double max_cost, double* cost, void* stream);

/* find_occluded (rect.py:142-157): out[i] = any j != i with inter(i,j)/area(i) >= thresh. */
int fm_find_occluded(const double* tlbr, int n, double thresh, unsigned char* out, void* stream);

/* scipy.optimize.linear_sum_assignment (SciPy 1.18.1 rectangular_lsap.cpp, shortest augmenting path;
 * call site matching.py:27) — bit-exact replay of its scan order and tie rules, one warp.
 * cost[nr][nc] f64 row-major.  col4row[nr]: assigned column, -1 if the row is unassigned, and
 * (-2 - col) if assigned but cost >= FM_INF_COST (demoted by matching.py:64-69).  Returns FM_ERR_ARG via
 * status[0] = 1 if the matrix is infeasible.  workspace: >= fm_lsa_workspace_bytes(nr, nc). */
long long fm_lsa_workspace_bytes(int nr, int nc);
int fm_lsa(const double* cost, int nr, int nc, int* col4row, int* status, void* workspace, void* stream);

/* _greedy_match (matching.py:73-97): repeated global argmin <= max_cost with row/column removal.
 * col4row[nr] = matched column or -1; match_order[nr] = rank of the match in discovery order or -1. */
int fm_greedy_match(const double* cost, int nr, int nc, double max_cost, int* col4row, int* match_order,
                    void* stream);

/* The whole association cascade of MultiTracker.update (fastmot/tracker.py:185-247) in one launch, id lists on the
 * device (csrc/assoc_cascade.cu).  The caller computes the three cost matrices once for ALL rows x ALL detections
 * (fm_matching_cost / fm_iou_cost with identity selections; an entry depends only on its pair):
 *   feat_cost [n_conf x n_det]             confirmed tracks, concatenated by age-depth group (goff[n_groups + 1])
 *   iou_cost  [(n_conf + n_unconf) x n_det] the same rows followed by the unconfirmed tracks
 *   reid_cost [n_hist x n_det]             lost-track history
 * Stages: LSA per depth group -> LSA of the still-active leftovers on IoU -> LSA of the unconfirmed tracks on IoU ->
 * greedy re-identification of the confident, non-occluded leftovers.  Unmatched lists follow the reference's Numba
 * typed-set order (matching.py:57-70).  Every dimension <= 256.
 * out (ints, fm_assoc_cascade_out_ints(cap) of them): hdr[16] = {status (1 = infeasible LSA), n_m1, n_m2, n_m3, n_u1
 * (inactive leftovers of stage 1), n_u2, n_u3, n_reid, n_invalid, n_reid_u}, then arrays of `cap` ints each:
 * m1_row, m1_det, m2_row, m2_det, m3_row, m3_det, u1, u2, u3, reid_row, reid_det, invalid_det, reid_u_det, occluded.
 * Rows are indices into the concatenated (confirmed | unconfirmed) order / the history order. */
typedef struct FmCascadeDesc {
    int n_det, n_conf, n_groups, n_unconf, n_hist, cap;
    const int* goff;
    const unsigned char* conf_active;   /* [n_conf] Track.active */
    const double* feat_cost;
    const double* iou_cost;
    const double* reid_cost;
    const double* det_conf;             /* [n_det] */
    const unsigned char* det_occluded;  /* [n_det] fm_find_occluded */
    double* sub;                        /* scratch, >= 256 * 256 doubles */
    int* out;
    double conf_thresh, max_reid_cost;
} FmCascadeDesc;
int fm_assoc_cascade(const FmCascadeDesc* h_desc, void* stream);
long long fm_assoc_cascade_out_ints(int cap);

/* ---------------------------------------------------------------- detector pre/post-processing --------------- */
#define FM_MAX_ANCHORS 6 /* fastmot/plugins/yolo_layer.h:11 */
typedef struct FmYoloHead {
    float anchors[2 * FM_MAX_ANCHORS]; /* (w,h) pairs in input pixels, fastmot/models/yolo.py:154-299 */
    float scale_x_y;
} FmYoloHead;

/* Pixel formats of the frames the letterbox, crop, KLT gray and frame-resize kernels read, read in place:
 *   NV12 (hardware video decoders, CSI cameras): a Y plane of h rows and a UV plane of h / 2 rows, both w bytes wide
 *        (U, V interleaved at half resolution);
 *   I420 (software decoders, PyAV / FFmpeg yuv420p): a Y plane of h rows, then a U and a V plane of h / 2 rows of
 *        w / 2 bytes;
 *   YUY2 (USB / V4L2 cameras): one packed plane of h rows of 2w bytes, Y0 U Y1 V per pixel pair;
 *   BGRX (nvvidconv's BGRx): one packed plane of h rows of 4w bytes, B G R x per pixel (x is not read).
 * Every entry gives on such a frame bit for bit what it gives on the BGR frame cv2.cvtColor(frame, code), code =
 * COLOR_YUV2BGR_NV12, _I420, _YUY2 or COLOR_BGRA2BGR (OpenCV 4.13: BT.601 limited range, 20-bit fixed point,
 * nearest-neighbour chroma); the pixels are converted inline, no BGR frame is written. */
#define FM_PIX_BGR 0
#define FM_PIX_NV12 1
#define FM_PIX_I420 2
#define FM_PIX_YUY2 3
#define FM_PIX_BGRX 4

/* One camera frame in device memory, as every entry that reads camera pixels takes it.  Row pitches are in bytes.
 *   FM_PIX_BGR : y is the tight u8 HWC frame (w * 3 bytes per row); uv, v, pitch and uv_pitch are ignored.
 *   FM_PIX_NV12: y and uv are the two planes, pitch and uv_pitch their row pitches (0 = w, else >= w); w, h even.
 *   FM_PIX_I420: y is the Y plane with row pitch `pitch` (0 = w, else >= w), uv the U plane and v the V plane, which
 *                share the row pitch uv_pitch (0 = w / 2, else >= w / 2); w, h even.
 *   FM_PIX_YUY2: y is the packed plane, pitch its row pitch (0 = 2w, else >= 2w); w even; uv, v, uv_pitch ignored.
 *   FM_PIX_BGRX: y is the packed plane, pitch its row pitch (0 = 4w, else >= 4w); uv, v, uv_pitch ignored.
 * The one-frame entries take a host pointer to it and reject a NULL y, an empty frame, an unknown format and a frame
 * that breaks the rules above.  v was appended last, so the other fields keep their offsets. */
typedef struct FmFrame {
    const unsigned char* y;
    const unsigned char* uv;
    int w, h;
    int pitch, uv_pitch;
    int format;
    const unsigned char* v;
} FmFrame;

/* One frame of a batch whose frames may differ in size: the device frame, its letterbox ROI in the network input, and
 * the pixel scale (size_w, size_h = upscaled_sz) and offset (off_x, off_y = bbox_offset) the head decode maps its boxes
 * back with -- the values a one-frame detector of that size passes as scalars. */
typedef struct FmFrameGeom {
    FmFrame frame;
    int roi_x, roi_y, roi_w, roi_h;
    float size_w, size_h, off_x, off_y;
} FmFrameGeom;

/* YOLODetector._preprocess + _create_letterbox (fastmot/detector.py:289-320): bilinear resize of the frame into the
 * ROI [roi_x, roi_y, roi_w, roi_h] of a dst_w x dst_h network input (half-pixel centres, edge replicate, rounded to u8
 * like the reference's CuPy zoom), BGR->RGB, x/255; everything outside the ROI = 0.5.  An NV12 frame's four bilinear
 * taps (of any YUV format) are each converted to BGR with their own chroma sample before they are interpolated.
 * layout 0: fp32 planar CHW (the reference's TensorRT input); layout 1: fp16 NHWC, C padded to 8 (16 bytes per pixel). */
int fm_letterbox_preproc(const FmFrame* frame, int dst_w, int dst_h, int roi_x, int roi_y, int roi_w, int roi_h,
                         int layout, void* out, void* stream);
/* fm_letterbox_preproc (layout 1) of `batch` frames of any sizes and formats in one launch: geom is a DEVICE array of
 * batch rows (frame and roi_* are read; every roi_w, roi_h > 0); out is fp16 [batch][dst_h][dst_w][8], image b
 * bit-identical to the one-frame call on geom[b]'s frame and ROI. */
int fm_letterbox_preproc_geom(const FmFrameGeom* geom, int batch, int dst_w, int dst_h, void* out, void* stream);

/* FeatureExtractor.extract_async preprocessing (fastmot/feature_extractor.py:48-60, 84-98; rect.py:92-97) for all
 * crops in one launch: integer-truncated clamp crop, OpenCV INTER_LINEAR 8-bit fixed-point resize to
 * out_w x out_h, BGR->RGB, (x/255 - mean)/std (a YUV frame's taps are converted to BGR before they are
 * interpolated).  n = min(*n_dev, n_max) if n_dev != NULL else n_max.
 * layout as above; output is [n][3][out_h][out_w] f32 or [n][out_h][out_w][8] f16; layout 2: fp16
 * [n][out_h + 8][out_w + 8][4] with the crop at (+4, +4) inside a border the CALLER zeroed once (the zero padding of
 * the OSNet 7x7 stem, fm_osnet_stem). */
int fm_roi_resize_norm(const FmFrame* frame, const double* tlbrs, const int* n_dev, int n_max, int out_w, int out_h,
                       int layout, void* out, void* stream);
/* fm_roi_resize_norm over several frames of any sizes and formats in one launch: crop i (tlbrs[i]) is cut from
 * geom[frame_idx[i]]'s frame, clamped to and addressed with that frame's w and h (geom: DEVICE FmFrameGeom array, the
 * ROI and scale fields are not read; frame_idx: device int32 [n]); each crop is bit-identical to the one-frame call on
 * its own frame and box. */
int fm_roi_resize_norm_geom(const FmFrameGeom* geom, const int* frame_idx, const double* tlbrs, int n, int out_w,
                            int out_h, int layout, void* out, void* stream);

/* cv2.resize(bgr(src), (dw, dh)) with the default INTER_LINEAR into a tight dh x dw x 3 u8 BGR frame.  bgr(src) is
 * src itself for FM_PIX_BGR, cv2.cvtColor(src, code) for the other formats, code as listed at FM_PIX_BGR (read in
 * place, as the letterbox / crop / gray kernels read it).  dst must not overlap src.  Bit-identical to OpenCV 4.13: an exact 2x downscale in
 * both axes is the 2x2 rounded mean, every other size pair the 11-bit fixed-point generic path.  Any size pair is
 * accepted (dh <= 65535); capture frames tracked at another size go through it (a camera's stream_cfg.resolution ->
 * resize_to). */
int fm_frame_resize(const FmFrame* src, unsigned char* dst, int dw, int dh, void* stream);

/* CalDetection / CalDetection_NewCoords (fastmot/plugins/yolo_layer.cu:127-230) fused with the class mask +
 * score threshold + pixel scaling of YOLODetector._filter_dets (fastmot/detector.py:331-341).  One call per
 * head; head_out is [(5+C)*A, H, W] (nhwc = 0, the plugin's layout) or [H, W, (5+C)*A] (nhwc = 1), fp32 or fp16.  Survivors write their 7-float record to
 * dense[cand_base + idx][8] and append a sort key to keys[] (counter is incremented atomically; the caller zeroes
 * it before the first head). */
int fm_yolo_decode_filter(const void* head_out, int is_fp16, int nhwc, int yolo_w, int yolo_h, int num_anchors,
                          const FmYoloHead* h_head, int num_classes, int input_w, int input_h, int new_coords,
                          int cand_base, const unsigned char* label_mask, double conf_thresh, float size_w,
                          float size_h, float off_x, float off_y, float* dense, unsigned long long* keys,
                          int* counter, int key_cap, void* stream);
/* fm_yolo_decode_filter for one head of `batch` images in one launch, with image b's size_w, size_h, off_x, off_y read
 * from geom[b] (DEVICE FmFrameGeom array of batch rows).  Image b reads head_out + b * head_stride elements and owns
 * dense rows [b * cand_stride, (b + 1) * cand_stride) (its candidate cand_base + idx at row
 * b * cand_stride + cand_base + idx), keys[b * key_cap .. + key_cap) and counters[b]: its keys and rows are the
 * one-image call's on its head slice with its own geometry. */
int fm_yolo_decode_filter_geom(const void* head_out, int batch, long long head_stride, int is_fp16, int nhwc,
                               int yolo_w, int yolo_h, int num_anchors, const FmYoloHead* h_head, int num_classes,
                               int input_w, int input_h, int new_coords, int cand_base, int cand_stride,
                               const unsigned char* label_mask, double conf_thresh, const FmFrameGeom* geom,
                               float* dense, unsigned long long* keys, int* counters, int key_cap, void* stream);

/* Rest of _filter_dets (detector.py:343-365) + diou_nms (rect.py:198-244): sort by (class, objectness desc),
 * per-class DIoU-NMS, to_tlbr rounding, area / aspect-ratio filters.  mask: >= fm_nms_mask_bytes(key_cap) bytes.
 * Outputs (device): out_tlbr[max_out][4] f64, out_label[max_out] i64, out_conf[max_out] f64, out_count[1];
 * status[0] = 1 if more than key_cap candidates passed the threshold, 2 if more than max_out boxes survived (only
 * the first max_out are written); the caller must raise on either.  key_cap <= 16384 (shared-memory sort). */
long long fm_nms_mask_bytes(int key_cap);
int fm_diou_nms_filter(unsigned long long* keys, const float* dense, const int* counter, int key_cap,
                       double nms_thresh, double max_area, double min_aspect_ratio, unsigned long long* mask,
                       int max_out, double* out_tlbr, long long* out_label, double* out_conf, int* out_count,
                       int* status, void* stream);
/* fm_diou_nms_filter for `batch` images in one call, on the segments fm_yolo_decode_filter_geom wrote: a box only
 * suppresses boxes of its own image and class.  mask: batch x fm_nms_mask_bytes(key_cap) bytes (image b's rows at
 * b x that size; only its first counters[b] rows are written).  Outputs: image b's detections at rows
 * [b * max_out, b * max_out + out_count[b]) of out_tlbr / out_label / out_conf; status[b] as above. */
int fm_diou_nms_filter_batch(int batch, unsigned long long* keys, const float* dense, int cand_stride,
                             const int* counters, int key_cap, double nms_thresh, double max_area,
                             double min_aspect_ratio, unsigned long long* mask, int max_out, double* out_tlbr,
                             long long* out_label, double* out_conf, int* out_count, int* status, void* stream);

/* ---------------------------------------------------------------- conv stacks (replace the TensorRT engines) -- */
/* The reference runs YOLO / OSNet as TensorRT engines (fastmot/utils/inference.py:39-125, built by
 * fastmot/models/yolo.py:106-151 and reid.py:48-92).  Here the same graphs run layer by layer on NHWC fp16
 * tensors; layer semantics follow scripts/yolo2onnx.py:558-870.  BN is folded into weight + bias by the host. */
#define FM_ACT_LINEAR 0
#define FM_ACT_LEAKY 1    /* alpha 0.1, yolo2onnx.py:421 */
#define FM_ACT_MISH 2
#define FM_ACT_SWISH 3
#define FM_ACT_LOGISTIC 4
#define FM_ACT_RELU 5
#define FM_ACT_AFTER_RESIDUAL 0x100 /* OR-ed into `act`: out = act(conv + bias + residual) (OSNet block tail) instead of
                                       act(conv + bias) + residual (Darknet shortcut after a conv) */

typedef struct FmConvDesc {
    int n, hi, wi, cin, cin_stride, cin_offset;     /* input  [n][hi][wi][cin_stride], channels [off, off+cin) */
    int ho, wo, cout, cout_stride, cout_offset;     /* output [n][ho][wo][cout_stride], channels [off, off+cout) */
    int kh, kw, stride, pad, act;
    int res_stride, res_offset;                     /* optional residual added after the activation */
    void* ws;                                       /* fp32 split-K scratch owned by the caller (one per engine /
                                                       stream: convs that may run concurrently must not share it), or
                                                       NULL = never split K.  Used when the 128 x BN output tiling
                                                       alone cannot fill the 132 SMs (e.g. 20x20 layers at batch 1). */
    long long ws_bytes;
} FmConvDesc;

/* weights: [cout][kh][kw][cin] fp16 (K-major), bias fp32[cout] or NULL, residual fp16 or NULL. */
int fm_conv2d_simt(const FmConvDesc* h_desc, const void* in, const void* wgt, const float* bias, const void* residual,
                   void* out, void* stream);
/* wgmma implicit-GEMM path (csrc/conv_tc.cu); requires cin % 16 == 0, 16-byte aligned channel slices. */
int fm_conv2d_tc(const FmConvDesc* h_desc, const void* in, const void* wgt, const float* bias, const void* residual,
                 void* out, void* stream);
int fm_conv2d_tc_supported(const FmConvDesc* h_desc);
/* Warp-specialised TMA + wgmma path with the split-K reduction inside a thread-block cluster (csrc/conv_tma.cu):
 * 1x1 / 3x3, stride 1, "same" padding, cin % 64 == 0, 8-channel aligned views; batch 1 for 3x3.  Needs no workspace
 * (FmConvDesc.ws is ignored).  Same role as fm_conv2d_tc: the TensorRT conv tactics behind
 * fastmot/utils/inference.py:106-117. */
int fm_conv2d_tma(const FmConvDesc* h_desc, const void* in, const void* wgt, const float* bias, const void* residual,
                  void* out, void* stream);
int fm_conv2d_tma_supported(const FmConvDesc* h_desc);
/* Darknet maxpool (SAME_UPPER, yolo2onnx.py:838-863) with channel-slice in/out; PyTorch-style padded maxpool. */
int fm_maxpool(const void* in, void* out, int n, int hi, int wi, int c, int cin_stride, int cin_off, int k, int stride,
               int cout_stride, int cout_off, void* stream);
int fm_maxpool_pad(const void* in, void* out, int n, int hi, int wi, int c, int k, int stride, int pad, void* stream);
int fm_avgpool2(const void* in, void* out, int n, int hi, int wi, int c, void* stream);
/* nearest upsample (yolo2onnx.py:806-836) and/or route copy (:743-804): channel slice in -> channel slice out. */
int fm_upsample_copy(const void* in, void* out, int n, int hi, int wi, int c, int cin_stride, int cin_off, int scale,
                     int cout_stride, int cout_off, void* stream);
int fm_add_act(const void* a, const void* b, void* out, long long n, int act, void* stream);
/* shortcut :707-731 */
int fm_add_act_strided(const void* a, int a_stride, int a_off, const void* b, int b_stride, int b_off, void* out,
                       int o_stride, int o_off, long long pixels, int c, int act, void* stream);
int fm_dwconv3(const void* in, const void* w, const float* bias, void* out, int n, int h, int wd, int c, int act,
               void* stream);
int fm_global_avgpool(const void* in, float* out, int n, int hw, int c, void* stream);
/* OSNet channel gate: acc (+)= x * sigmoid(W2 relu(W1 GAP(x) + b1) + b2) */
int fm_channel_gate(const void* x, float* pooled, float* gate, const float* w1, const float* b1, const float* w2,
                    const float* b2, void* acc, int n, int hw, int c, int cr, int accumulate, void* stream);
/* The four streams of an OSBlock share one gate: acc = sum_s x_s * gate(x_s) in one fused pass.
 * pooled / gate: scratch of 4*n*c floats each. */
int fm_channel_gate4(const void* x0, const void* x1, const void* x2, const void* x3, float* pooled, float* gate,
                     const float* w1, const float* b1, const float* w2, const float* b2, void* acc, int n, int hw, int c,
                     int cr, void* stream);
/* Same aggregation fed by fm_osb_streams: x0..x3 are its chunk-planar tails [n][c / 8][hw][8], gap_part
 * [n][strips][4][c] holds their channel SUMS; acc is NHWC.  hw % 64 == 0. */
int fm_channel_gate4_pooled(const void* x0, const void* x1, const void* x2, const void* x3, const float* gap_part,
                            int strips, float* gate, const float* w1, const float* b1, const float* w2, const float* b2,
                            void* acc, int n, int hw, int c, int cr, void* stream);
/* FC (+ReLU) and the row L2 normalisation of FeatureExtractor.postprocess (feature_extractor.py:73). */
int fm_fc_norm(const float* in, const float* w, const float* bias, float* out, int n, int cin, int cout, int relu,
               int normalize, void* stream);

/* ---------------------------------------------------------------- KLT optical flow (fastmot/flow.py) ---------- */
#define FM_NO_OWNER 0x7fffffff
#define FM_MAX_PYR_LEVELS 8

typedef struct FmPyramid {       /* one image pyramid: u8 levels + int16x2 Scharr derivatives per level */
    int n_levels;
    int w[FM_MAX_PYR_LEVELS], h[FM_MAX_PYR_LEVELS];
    const unsigned char* img[FM_MAX_PYR_LEVELS];
    const short* deriv[FM_MAX_PYR_LEVELS];
} FmPyramid;

typedef struct FmTrackJob {      /* per-track record produced by fm_flow_keypoints (device) */
    int slot, x0, y0, cw, ch, area, n_keep, redetect, min_dist, scratch_off;
    float eig_max;
    int pad;
} FmTrackJob;

/* cv2.cvtColor(BGR2GRAY) + cv2.resize(0.5x) of flow.py:153-154 / :129-131 in one pass (w, h even); gray is
 * frame->w x h.  On an NV12 frame a thread's 2x2 block is one chroma sample (one UV load). */
int fm_gray_half(const FmFrame* frame, unsigned char* gray, unsigned char* small, void* stream);
/* cv2.cvtColor(BGR2GRAY) + cv2.resize(gray, (sw, sh)) INTER_LINEAR at any optical-flow size 0 < sw <= w,
 * 0 < sh <= h (odd frame sizes, anisotropic scales, scale 1). */
int fm_gray_resize(const FmFrame* frame, unsigned char* gray, unsigned char* small, int sw, int sh, void* stream);
/* one pyrDown step ((sw+1)/2 x (sh+1)/2) and the Scharr derivative image of a level — what
 * cv2.calcOpticalFlowPyrLK builds internally (flow.py:203-207). */
int fm_pyr_level(const unsigned char* src, int sw, int sh, unsigned char* dst, void* stream);
int fm_scharr(const unsigned char* src, int w, int h, short* deriv, void* stream);
/* flow.py:187-189: background-scale image (cv2.resize INTER_LINEAR) and nearest-neighbour mask from the owner map. */
int fm_bg_small(const unsigned char* gray, const int* owner, int w, int h, unsigned char* bg, unsigned char* bg_mask,
                int bw, int bh, void* stream);

/* flow.py:156-184 for all active tracks (slots[] in nearest-first order, boxes from tlbr_pool): occlusion/owner
 * map, keypoint filtering (_rect_filter), Shi-Tomasi re-detection (cv2.goodFeaturesToTrack, blockSize 3, gradient
 * aperture 3, 0 < max_corners <= 1024) where len(kp) < feat_density * area, ellipse filter.  Keypoints live in
 * kp_pool[cap][max_kp][2] / kp_count[cap].  scratch: scratch_cap floats for the eigenvalue maps and, for a box with
 * more than 4096 candidate corners (local maxima above the quality threshold), 4 floats per candidate, 2 per accepted
 * corner and one per minDistance cell of the box; status[0] != 0 reports scratch (2) or keypoint (4, more kept corners in one box than
 * max_kp) overflow. */
int fm_flow_keypoints(const unsigned char* prev_gray, int w, int h, const double* tlbr_pool, const int* slots,
                      int n_trk, int* owner, float* kp_pool, int* kp_count, int max_kp, double feat_density,
                      double feat_dist_factor, double quality, int max_corners, FmTrackJob* jobs, float* scratch,
                      int scratch_cap, int* scratch_counter, int* status, void* stream);
/* The same for every cv2.goodFeaturesToTrack setting: block_size >= 1 (unnormalised box window anchored at
 * block_size / 2), gradient_size (Sobel aperture) 1 / 3 / 5 / 7, the minimum-eigenvalue response or, with use_harris,
 * a*c - b^2 - harris_k*(a+c)^2; max_corners <= 0 keeps every corner.  max_kp must hold min(max_corners, 4096) corners
 * (4096 when max_corners <= 0); a box that keeps more sets status 4.  The default setting runs fm_flow_keypoints; the
 * others use four scratch floats per crop pixel, plus 4 per candidate, 2 per accepted corner and one per minDistance
 * cell for a box with more than 4096 candidates. */
int fm_flow_keypoints_cfg(const unsigned char* prev_gray, int w, int h, const double* tlbr_pool, const int* slots,
                          int n_trk, int* owner, float* kp_pool, int* kp_count, int max_kp, double feat_density,
                          double feat_dist_factor, double quality, int max_corners, int block_size, int gradient_size,
                          int use_harris, double harris_k, FmTrackJob* jobs, float* scratch, int scratch_cap,
                          int* scratch_counter, int* status, void* stream);

/* cv2.FastFeatureDetector(threshold, nonmaxSuppression=True, TYPE_9_16).detect(img, mask) (flow.py:190) followed
 * by _unscale_pts (flow.py:335-344); output points in row-major order, any image size, 0 <= threshold <= 255.
 * score: w*h scratch bytes.
 * At most max_pts points are written; no two corners touch, so max_pts >= ceil((w-6)/2) * ceil((h-6)/2) keeps all. */
int fm_fast_detect(const unsigned char* img, const unsigned char* mask, int w, int h, int threshold, float unscale_x,
                   float unscale_y, unsigned char* score, float* out_pts, int* out_count, int max_pts, void* stream);

/* flow.py:182-186, 199-200: all_prev_pts = concat(track keypoints) ++ background points.
 * trk_begin[n_trk + 1]; meta[0] = bg_begin, meta[1] = total points, meta[2] = #bg, meta[3] = overflow flag (more
 * than max_pts points: the list is cut at max_pts and every trk_begin is clamped to max_pts). */
int fm_gather_points(const float* kp_pool, const int* kp_count, int max_kp, const int* slots, int n_trk,
                     const float* bg_pts, const int* bg_count, float* all_pts, int* trk_begin, int* meta,
                     int max_pts, void* stream);

/* cv2.calcOpticalFlowPyrLK (flow.py:203-209) incl. _scale_pts / _get_status / _unscale_pts: points are given and
 * returned in full-resolution coordinates; out_status = status & (err < max_error). n = meta[1]. */
int fm_lk_track(const FmPyramid* h_prev, const FmPyramid* h_cur, const float* pts_full, const int* meta,
                float pt_scale_x, float pt_scale_y, int win_w, int win_h, int max_count, float epsilon,
                float min_eig_thr, float max_error, float* out_pts, unsigned char* out_status, float* out_err,
                void* stream);

/* cv2.findHomography(RANSAC, 3.0, maxIters, confidence) on the background matches + the failure tests of
 * flow.py:215-232.  H_out[9] f64 (H[8] = 1), h_ok[0] = 1 on success; inlier points go to bg_kp / bg_kp_prev. */
int fm_ransac_homography(const float* all_prev, const float* all_cur, const unsigned char* status, const int* meta,
                         int max_iters, double confidence, double thresh, int inlier_thresh, int* good_idx,
                         int* inl_idx, double* H_out, int* h_ok, float* bg_kp, float* bg_kp_prev, int* bg_kp_count,
                         int max_bg, void* stream);

/* cv2.estimateAffinePartial2D(RANSAC, 3.0, maxIters, confidence, refineIters) per track + _estimate_bbox + the
 * acceptance tests and mask painting of flow.py:234-264.  The serial "paint predicted box, filter the next
 * track's points" dependency is resolved by rounds: round r filters with the boxes of round r-1 and recomputes
 * only tracks whose filtered point set changed; round_flags[r & 15] = 1 if anything changed (fixed point when 0).
 * est_boxes: 2*n_trk*5 ints, sig: n_trk u64.  Results: klt_tlbr / klt_ok / inlier_ratio (slot-indexed pools),
 * kp_pool <- inlier matched points, kp_prev_pool <- inlier previous points. */
int fm_ransac_affine_partial_batch(const float* all_prev, const float* all_cur, const unsigned char* status,
                                   const int* trk_begin, const int* slots, int n_trk, int n_rounds, int* round_flags,
                                   const int* h_ok, int* est_boxes, unsigned long long* sig, double* tlbr_pool,
                                   double* klt_tlbr, unsigned char* klt_ok, double* inlier_ratio, float* kp_pool,
                                   float* kp_prev_pool, int* kp_count, int max_kp, int frame_w, int frame_h,
                                   int max_iters, double confidence, double thresh, int inlier_thresh,
                                   int refine_iters, int first_round, void* stream);

/* ---- KLT stage runner: Flow.predict (flow.py:135-264) as ONE call -------------------------------------------
 * fm_flow_plan_create copies the plan (all pointers are caller-owned device buffers that stay fixed between frames;
 * the fields are the arguments of the per-call functions above, named alike) and creates two private events;
 * fm_flow_predict enqueues, on s_main: gray + optical-flow image (fm_gray_half when pyr[k].w[0] x h[0] is exactly half
 * the frame, fm_gray_resize otherwise) + pyramid + Scharr of `frame` into buffer 1 - prev, klt_ok clear,
 * fm_flow_keypoints_cfg / fm_bg_small / fm_fast_detect / fm_gather_points on buffer prev, fm_lk_track prev -> cur, then
 * fm_ransac_homography on s_side (forked / joined with the private events) next to rounds_ahead (a multiple of 4)
 * rounds of fm_ransac_affine_partial_batch on s_main.  Identical launches to the per-call sequence; no allocation,
 * no synchronisation.  flags: int[32] = {scratch counter, keypoint status, -, .., [8..23] round flags}. */
typedef struct FmFlowPlan {
    int frame_w, frame_h;
    unsigned char* gray[2];
    FmPyramid pyr[2];
    const double* tlbr_pool;
    const int* slots;
    int* owner;
    float* kp_pool;
    float* kp_prev_pool;
    int* kp_count;
    int max_kp;
    double feat_density, feat_dist_factor, quality;
    int max_corners;
    FmTrackJob* jobs;
    float* scratch;
    int scratch_cap;
    int* flags;
    unsigned char* bg;
    unsigned char* bg_mask;
    unsigned char* bg_score;
    int bg_w, bg_h, bg_thresh;
    float unscale_x, unscale_y;
    float* bg_pts;
    int* bg_count;
    int max_bg;
    float* all_prev;
    float* all_cur;
    unsigned char* status;
    float* err;
    int* trk_begin;
    int* meta;
    int max_points;
    float pt_scale_x, pt_scale_y;
    int win_w, win_h, lk_max_count;
    float lk_epsilon, lk_min_eig, max_error;
    int ransac_max_iter;
    double ransac_conf, ransac_thresh;
    int inlier_thresh, refine_iters;
    int* good_idx;
    int* inl_idx;
    float* bg_kp;
    float* bg_kp_prev;
    int* bg_kp_count;
    int* est_boxes;
    unsigned long long* sig;
    double* klt_tlbr;
    unsigned char* klt_ok;
    long long klt_ok_bytes;
    double* inlier_ratio;
    int rounds_ahead;
    /* goodFeaturesToTrack settings of fm_flow_keypoints_cfg (the default: 3, 3, 0, any k) */
    int block_size, gradient_size, use_harris;
    double harris_k;
} FmFlowPlan;
void* fm_flow_plan_create(const FmFlowPlan* plan);      /* NULL on error (fm_last_error) */
void fm_flow_plan_destroy(void* handle);
/* frame: the plan's frame_w x frame_h (anything else is rejected) */
int fm_flow_predict(void* handle, const FmFrame* frame, int prev, int n_trk, double* H_out, int* h_ok, void* s_main,
                    void* s_side);

/* ---------------------------------------------------------------- tensor-core primitive self-test ----------- */
/* One CTA exercises the building blocks of the fused kernels (csrc/tc_common.cuh): TMA tensor-map load of a
 * [128 x 64] fp16 tile (rows row0.. of a [rows][64] matrix; rows past the end read as zero) into 128-byte-swizzled
 * shared memory, cp.async.bulk of the packed weight images, wgmma with both operands in shared memory
 * (out0 = A * B1^T, fp32 [128][n1]), and wgmma with the fp16-rounded result as A operand in registers
 * (out1 = fp16(out0) * B2^T, fp32 [128][n2]).  b1 / b2: K-slice images made by
 * fastmot_b200.packing.pack_b_sw128 ([n][k] -> slices of 64 k, rows of 128 bytes, 16-byte chunks XOR-swizzled). */
int fm_probe_umma(const void* a, int rows, int row0, const void* b1, const void* b2, int n1, int n2, float* out0,
                  float* out1, void* stream);

/* ---------------------------------------------------------------- fused OSNet OSBlock kernels --------------- */
/* Kernel S (csrc/osnet_fused.cu): conv1 (1x1, cin -> mid, ReLU) and the four Lite-3x3 streams of one OSBlock
 * (torchreid OSBlock.conv1 / conv2a..d; role of the TensorRT OSNet engine, fastmot/utils/inference.py:106-117) in a
 * single launch.  x: [n][h][w][cin] fp16 NHWC; tails[s]: chunk-planar [n][mid / 8][h][w][8] fp16 (output of stream s);
 * gap_part: fp32 [n][strips][4][mid], the per-strip channel sums of the tails (strips = fm_osb_streams_strips()).
 * w1: fm pack_b_sw128 image of the conv1 weights [mid][cin]; pw: ten pack_b_sw128 images [mid][mid] in the order
 * a.0, b.0, b.1, c.0, c.1, c.2, d.0 .. d.3; dw: ten blobs { fp16 [9][mid] depthwise taps, fp32 [mid] pointwise bias,
 * fp32 [mid] depthwise bias }.  Supported (w, mid, h): (32, 64, multiple of 8), (16, 96, 32), (8, 128, 16). */
typedef struct FmOsbStreams {
    const void* x;
    int n, h, w, cin, mid;
    const void* w1;
    const float* b1;
    const void* pw;
    const void* dw;
    void* tails[4];
    float* gap_part;
} FmOsbStreams;
int fm_osb_streams(const FmOsbStreams* h_desc, void* stream);
/* number of strips per crop kernel S uses for this geometry (0 = unsupported) */
int fm_osb_streams_strips(int h, int w, int mid);

/* OSNet stem in one launch (csrc/osnet_stem.cu): conv 7x7 / 2 (3 -> 64) + bias + ReLU + max-pool 3x3 / 2.
 * x: fp16 [n][264][136][4] (fm_roi_resize_norm layout 2: 256 x 128 crop at (+4, +4), zero border); wimg:
 * pack_b_sw64 image of W[64][224], W[o][r * 32 + j * 4 + c] = w[o][r][j - 1][c] (zero for j = 0 and c = 3);
 * bias fp32 [64]; out: fp16 [n][64][32][64] NHWC. */
int fm_osnet_stem(const void* x, int n, const void* wimg, const float* bias, void* out, void* stream);

/* Kernel G: the rest of the OSBlock in one launch (torchreid OSBlock: gate, conv3, downsample, residual, ReLU):
 *   out = relu(conv3(sum_s gate(tail_s) * tail_s) + b3 + identity),  identity = res (cin == cout) or downsample(x).
 * tails / gap_part: outputs of fm_osb_streams; gw1 [cr][mid], gb1 [cr], gw2 [mid][cr], gb2 [mid]: gate FCs (fp32);
 * wimg: for every range of fm_osb_merge_ncta(mid, cout) output channels, the pack_b_sw128 image of the rows of
 * [W_down | W_3] (K = cin, then mid rounded up to 64; W_down only when x != NULL); bias [cout] = b3 (+ b_down);
 * exactly one of x ([n][hw][cin], downsample input) and res ([n][hw][cout], identity) is non-NULL; out [n][hw][cout].
 * hw % 128 == 0, cr <= 8. */
typedef struct FmOsbMerge {
    int n, hw, cin, cout, mid, cr, strips;
    const void* tails[4];
    const float* gap_part;
    const float* gw1; const float* gb1; const float* gw2; const float* gb2;
    const void* wimg;
    const float* bias;
    const void* x;
    const void* res;
    void* out;
    float* gate_scratch;        /* 4 * n * mid floats: the gates, written by a small FC kernel launched first */
} FmOsbMerge;
int fm_osb_merge(const FmOsbMerge* h_desc, void* stream);
int fm_osb_merge_ncta(int mid, int cout);

#ifdef __cplusplus
}
#endif
#endif /* FASTMOT_B200_H */
