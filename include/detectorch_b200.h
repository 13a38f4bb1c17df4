/*
 * detectorch_b200 -- C ABI of the H100-native two-stage-detector inference hot path.
 *
 * Plain pointers and sizes only (no torch types).  Every pointer is a DEVICE pointer unless
 * stated otherwise; every call is asynchronous on `stream` (a cudaStream_t passed as void*),
 * never synchronises, and returns 1 on success / 0 on failure (the reference's launcher
 * convention, lib/cppcuda_cffi/src/cuda/roi_align_forward_cuda_kernel.cu:161-199), printing the
 * reason to stderr.  Layouts are fp32 throughout.
 *
 * Each entry point names the reference interface it replaces (paths relative to the reference
 * repository root).  INTEGRATION.md shows the reference-side binding for each.
 */
#ifndef DETECTORCH_B200_H
#define DETECTORCH_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* dt_stream_t; /* cudaStream_t */

/* ---------------------------------------------------------------------------------------------
 * RoIAlign forward.
 * Replaces: lib/cppcuda_cffi/src/cuda/roi_align_forward_cuda_kernel.h:7-19 (exact signature kept:
 * this symbol is what lib/cppcuda_cffi/src/roi_align_forward_cuda.c:35-47 calls), and through it
 * lib/cppcuda/roi_align_cuda.h:4-11 / lib/model/roi_align.py:32-89.
 * bottom_data NCHW [B,C,H,W]; bottom_rois [R,5] (batch,x1,y1,x2,y2); top_data [R,C,ph,pw];
 * outputElements = R*C*ph*pw (int, as in the reference: < 2^31).
 */
int launch_roi_align_forward_cuda(const int outputElements, const float* bottom_data, const float* bottom_rois,
                                  const float spatial_scale, const int channels, const int height, const int width,
                                  const int pooled_height, const int pooled_width, const int sampling_ratio, float* top_data,
                                  dt_stream_t stream);

/* RoIAlign backward (gradient w.r.t. the features), the training-side caller of the same boundary.
 * Replaces: lib/cppcuda_cffi/src/cuda/roi_align_backward_cuda_kernel.h:7-21 (exact signature kept; called by
 * lib/cppcuda_cffi/src/roi_align_backward_cuda.c and lib/model/roi_align.py:91-147).  top_diff [R,C,ph,pw];
 * bottom_diff [B,C,H,W] is ACCUMULATED into (the caller zeroes it, roi_align.py:117); atomic fp32 scatter like the reference,
 * so the last bits depend on the summation order exactly as they do there. */
int launch_roi_align_backward_cuda(const int nthreads, const float* top_diff, const int num_rois, const float spatial_scale,
                                   const int channels, const int height, const int width, const int pooled_height,
                                   const int pooled_width, const int sampling_ratio, float* bottom_diff, const float* bottom_rois,
                                   int roi_cols, dt_stream_t stream);

/* Deterministic (atomics-free) backward: the contributions to every feature-map cell are summed in exactly the order of the reference's
 * single-threaded CPU loop (lib/cppcuda/roi_align_backward_cpu.cpp:79-186) => bit-identical to it and bit-reproducible run to run
 * (the atomic scatter above is neither).  Two calls: _plan writes the number of (sample, corner) contributions of the RoI set to *total_dev
 * (device int64; the grid is adaptive when sampling_ratio == 0, so only the device knows it); the caller reads it, allocates
 * dt_roi_align_backward_det_workspace_bytes(num_rois, total) bytes and calls _deterministic.  bottom_diff is accumulated into. */
int64_t dt_roi_align_backward_det_workspace_bytes(int64_t num_rois, int64_t total_contributions);
int dt_roi_align_backward_plan(const float* rois, int64_t num_rois, int roi_cols, float spatial_scale, int pooled_height, int pooled_width,
                               int sampling_ratio, void* scratch, int64_t* total_dev, dt_stream_t stream);
int dt_roi_align_backward_deterministic(const float* top_diff, const float* rois, int64_t num_rois, int roi_cols, int batch, int channels,
                                        int height, int width, int pooled_height, int pooled_width, float spatial_scale, int sampling_ratio,
                                        int64_t total_contributions, float* bottom_diff, void* workspace, dt_stream_t stream);

/* 64-bit-safe variant (R*C*ph*pw may exceed 2^31, e.g. 100k RoIs x 256 ch x 14 x 14); roi_cols is 4 or 5
 * like the reference CPU loop (lib/cppcuda_cffi/src/cpp/roi_align_cpu_loop.h:5-17). */
int dt_roi_align_forward_nchw(const float* features, const float* rois, int64_t num_rois, int roi_cols, int channels, int height,
                              int width, int pooled_height, int pooled_width, float spatial_scale, int sampling_ratio, float* out,
                              dt_stream_t stream);

/* Fast variant for sampling_ratio == 2 (the FPN configurations and the RoIAlign microbench): separable bilinear weights with
 * merged duplicate taps, fused multiply-adds, output tile assembled in shared memory and written by one bulk async copy per
 * RoI.  Same contract as dt_roi_align_forward_nchw (any other configuration is forwarded to it); results agree with the
 * exact kernel to fp32 re-association (~1e-7 relative).  Maps small enough for an 8-channel slab of the whole map to live in
 * shared memory (H*W <= ~3600 cells, 7x7 or 14x14 bins) take the shared-memory-resident variant: the gathers never leave
 * the SM.  workspace: dt_roi_align_fast_workspace_bytes() (an NHWC copy of the feature map + the per-RoI tap tables). */
int64_t dt_roi_align_fast_workspace_bytes(int batch, int channels, int height, int width, int64_t num_rois, int pooled_height,
                                          int pooled_width);
int dt_roi_align_forward_nchw_fast(const float* features, int batch, const float* rois, int64_t num_rois, int roi_cols, int channels, int height,
                                   int width, int pooled_height, int pooled_width, float spatial_scale, int sampling_ratio, float* out,
                                   void* workspace, dt_stream_t stream);

/* Multi-level NHWC variant used inside the fused detector (replaces the 4 per-level RoIAlign calls + cat +
 * index-restore of lib/model/detector.py:259-270 and :100-106).  feats[l] is an NHWC map [B,H[l],W[l],C];
 * rois [max_rois,5]; level[max_rois] (index into feats, NULL = all level 0); num_rois_dev: optional device int
 * (rows >= *num_rois_dev are written as zeros); out [max_rois, ph, pw, C]. */
int dt_roi_align_forward_nhwc(const float* const* feats_host_array, const int* heights, const int* widths, const float* scales,
                              int num_levels, const float* rois, const int* level, const int* num_rois_dev, int max_rois,
                              int channels, int pooled_height, int pooled_width, int sampling_ratio, float* out, dt_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Greedy hard NMS with the reference's exact fp32 semantics ("+1" widths, ovr >= thresh).
 * Replaces: lib/utils/boxes.py:332-336 -> lib/utils_cython/cython_nms.pyx:37-87.
 * dets [n,5] (x1,y1,x2,y2,score).  keep_out [n] int64 receives the ASCENDING ORIGINAL indices of the
 * survivors, *num_keep_out (device int) their count.  workspace: dt_nms_workspace_bytes(n) bytes.
 */
int64_t dt_nms_workspace_bytes(int64_t n);
int dt_nms(const float* dets, int n, float thresh, int64_t* keep_out, int* num_keep_out, void* workspace, dt_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Mask paste + COCO run-length encoding (the step right after the path, SURVEY.md 8f rank 1).
 * Replaces: lib/utils/result_utils.py:170-228 (segm_results): per detection zero-pad the MxM mask by one cell, expand the
 * reference box by (M+2)/M (lib/utils/boxes.py:245-261), truncate to int32, cv2.resize(float32, INTER_LINEAR) to the box,
 * threshold, paste into an im_h x im_w image, pycocotools rleEncode + rleToString -- without ever materialising the image.
 *   masks          [max_dets, num_mask_classes, M, M] with classes[d] selecting the plane, or [max_dets, M, M] (classes NULL)
 *   ref_boxes      [max_dets,4] fp32 image-space boxes (expanded on the device), or expanded_boxes [max_dets,4] int32
 *                  (already expanded and truncated by the caller); one of the two must be non-NULL
 *   num_dets_dev   optional device int: detections >= *num_dets_dev produce empty results
 *   counts         [max_dets, runs_cap] uint32 run lengths (column-major, zeros run first), num_counts[max_dets]
 *   strings        dt_segm_strings_bytes() bytes: the compressed RLE strings back to back; str_offsets[max_dets+1]
 *   overflow       device int: 0, or the number of runs a detection needed when runs_cap (or its string staging) was too small
 * dt_segm_paste writes the pasted binary masks themselves, uint8 [max_dets, im_h, im_w].
 */
int64_t dt_segm_workspace_bytes(int max_dets, int runs_cap);
int64_t dt_segm_strings_bytes(int max_dets, int runs_cap);
int dt_segm_rle(const float* masks, const int* classes, int num_mask_classes, int mask_size, const float* ref_boxes,
                const int* expanded_boxes, const int* num_dets_dev, int max_dets, int im_h, int im_w, float thresh_binarize,
                uint32_t* counts, int* num_counts, int runs_cap, uint8_t* strings, int64_t* str_offsets, int* overflow, void* workspace,
                dt_stream_t stream);
int dt_segm_paste(const float* masks, const int* classes, int num_mask_classes, int mask_size, const float* ref_boxes,
                  const int* expanded_boxes, const int* num_dets_dev, int max_dets, int im_h, int im_w, float thresh_binarize,
                  uint8_t* out, dt_stream_t stream);

/* The same paste + RLE for a whole batch of images, each with its own canvas size and detection count: the padded outputs of the
 * fused engine (det_boxes, det_classes, det_counts, masks / masks_full) go in as they are, one launch covers every (image, slot).
 * dt_segm_rle is the one-image case of this code.
 *   masks          [batch, cap, M, M] (the detected class), or [batch, cap, num_mask_classes, M, M] with classes [batch, cap] selecting
 *                  the plane (classes NULL for the first layout)
 *   boxes          [batch, cap, 4] fp32 image-space boxes (expanded by (M+2)/M and truncated on the device)
 *   num_dets_dev   int32 [batch]: live slots of each image; slots at or past it produce empty strings
 *   im_sizes       int32 [batch, 2]: (im_h, im_w) of each image's RLE canvas, each within max_im_h x max_im_w (the host-known maxima
 *                  size the shared-memory tables; an entry outside [1, max] gives that image empty strings)
 *   strings        dt_segm_batch_strings_bytes() bytes: the strings of slot s = b * cap + d back to back; str_offsets [batch*cap+1] int64
 *   overflow       device int: 0, or the number of runs a slot needed when runs_cap (or its string staging) was too small: grow and redo
 * Run lengths and their counts stay in the workspace (dt_segm_batch_workspace_bytes()).  Returns 0 for a mask size outside [1, 126],
 * max_im_h * max_im_w >= 2^32, tables beyond the shared-memory limit, batch > 65535, runs_cap < 2 or a NULL pointer. */
int64_t dt_segm_batch_workspace_bytes(int batch, int cap, int runs_cap);
int64_t dt_segm_batch_strings_bytes(int batch, int cap, int runs_cap);
int dt_segm_rle_batch(const float* masks, const int* classes, int num_mask_classes, int mask_size, const float* boxes, const int* num_dets_dev,
                      const int* im_sizes, int batch, int cap, int max_im_h, int max_im_w, float thresh_binarize, int runs_cap,
                      uint8_t* strings, int64_t* str_offsets, int* overflow, void* workspace, dt_stream_t stream);

/* dt_segm_rle_batch for a caller that must not wait for the device (utils.coco_eval.DeviceResults.add, a captured CUDA graph): the
 * same strings, byte for byte, appended to a caller-owned char arena at a device-side cursor, with every outcome left in device flags.
 * The call issues stream operations only (no host read, no allocation), so it can be captured and replayed with new table contents.
 *   masks, classes, num_mask_classes, boxes, num_dets_dev, thresh_binarize, runs_cap, workspace: as for dt_segm_rle_batch (the workspace
 *                  is dt_segm_batch_workspace_bytes(batch, cap, runs_cap))
 *   im_sizes       int32 [batch, 2]: (im_h, im_w) of each image's RLE canvas, read on the device only.  The shared-memory tables are
 *                  sized for images of up to DT_SEGM_APPEND_MAX_SIDE x DT_SEGM_APPEND_MAX_SIDE, which with the 200 KB shared-memory
 *                  limit allows masks of up to 98 x 98
 *   arena          arena_capacity bytes; cursor int64 [1]: its used length.  The batch's B*cap strings go to arena[*cursor ..], slot
 *                  s = b * cap + d after slot s - 1, and *cursor advances by their total; str_offsets [batch*cap+1] int64 are arena
 *                  offsets (str_offsets[s + 1] - str_offsets[s] is slot s's length)
 *   flags          int32 [3], zeroed by the call: [0] 0, or the most runs a slot needed when runs_cap (or its string staging) was too
 *                  small; [1] 1 if an image's size is outside [1, DT_SEGM_APPEND_MAX_SIDE]; [2] 1 if the strings did not fit: cursor +
 *                  total > arena_capacity (then str_offsets[batch*cap] - str_offsets[0] is the total needed).
 *                  With any flag raised nothing is written to the arena and the cursor is left as it was: grow, then redo the batch.
 * Returns 0 for a mask size beyond the table limit, batch > 65535, runs_cap < 2 or a NULL pointer. */
#define DT_SEGM_APPEND_MAX_SIDE 8192
int dt_segm_rle_batch_append(const float* masks, const int* classes, int num_mask_classes, int mask_size, const float* boxes,
                             const int* num_dets_dev, const int* im_sizes, int batch, int cap, float thresh_binarize, int runs_cap,
                             uint8_t* arena, int64_t arena_capacity, int64_t* cursor, int64_t* str_offsets, int* flags, void* workspace,
                             dt_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Image pre-processing (the step right before the path, SURVEY.md 8f rank 3).
 * Replaces: lib/utils/blob.py:57-87 prep_im_for_blob (float32, minus pixel_means, cv2.resize(fx=fy=im_scale, INTER_LINEAR)) fused
 * with blob.py:27-55 im_list_to_blob (zero-pad to a multiple of the coarsest FPN stride, HWC -> CHW).
 *   image_hwc    device uint8 [height, width, 3] (BGR, as cv2.imread returns it)
 *   pixel_means  HOST double[3]; im_scale: the factor prep_im_for_blob computes (target_size / min side, capped by max_size)
 *   out_height/out_width = cvRound(height * im_scale), cvRound(width * im_scale)  (the size cv2.resize produces)
 *   blob_chw     device fp32 [3, blob_height, blob_width], zero outside the resized image
 */
int dt_prep_image(const uint8_t* image_hwc, int height, int width, const double* pixel_means, double im_scale, int out_height, int out_width,
                  float* blob_chw, int blob_height, int blob_width, dt_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Convolution / GEMM on wgmma tensor cores (3xTF32 or 3xFP16, fp32-accurate), NHWC activations.
 * Replaces the torch.nn.Conv2d / Linear / ConvTranspose2d calls of lib/model/detector.py
 * (:17-27 FPN, :58-59 FC6/FC7, :71-74 mask convs, :89-90 deconv + mask logits, :119-121 RPN, :170-183 trunk).
 *   x        [N,H,W,Cin]   (Cin % 32 == 0), x_pix_stride floats between pixels
 *   w        [Cout][kh][kw][Cin] fp32, w_lo = w - trunc_tf32(w) (dt_tf32_residual)
 *   y        [N,Ho,Wo,Cout] (Cout % 4 == 0), y = act( conv(x,w)*scale[c] + shift[c] (+ residual) )
 *   res_mode 0 none | 1 residual [N,Ho,Wo,Cout] | 2 nearest-2x-upsampled up_src [N,up_h,up_w,Cout]
 *   relu     0/1 ; sigmoid_ch: channels [0,sigmoid_ch) get a sigmoid ; passes 3 (3xTF32) or 1 (TF32)
 *   force_block_n 0 = auto | 64 | 128 (256 runs as 128-wide tiles) | -1 = 64 with 3 rotating accumulators (shortest truncating-accumulate chains)
 * dt_conv2d_nhwc_f16x3 is the same product with fp16 MMAs (twice the tf32 rate): w_hi16 / w_lo16 are the fp16 halves of
 * w * multiplier from dt_fp16_split (multiplier a power of two that keeps the low half a normal fp16 number; the caller folds
 * 1/multiplier into `scale`); the fp32 activations are split in shared memory.  *range_flag (device int, may be NULL) is set
 * to 1 if an activation does not fit fp16 (|x| >= 65504); the result is then not meaningful and the tf32 entry must be used.
 */
int dt_tf32_residual(const float* w, float* w_lo, int64_t n, dt_stream_t stream);
int dt_fp16_split(const float* w, int64_t n, float multiplier, void* w_hi16, void* w_lo16, dt_stream_t stream);
int dt_conv2d_nhwc_f16x3(const float* x, int N, int H, int W, int Cin, int x_pix_stride, const void* w_hi16, const void* w_lo16, int Cout,
                         int kh, int kw, int pad, int stride, const float* scale, const float* shift, const float* residual, int res_mode,
                         const float* up_src, int up_h, int up_w, int relu, int sigmoid_ch, int passes, int force_block_n, int* range_flag,
                         float* y, int y_pix_stride, dt_stream_t stream);
int dt_conv2d_nhwc(const float* x, int N, int H, int W, int Cin, int x_pix_stride, const float* w, const float* w_lo, int Cout,
                   int kh, int kw, int pad, int stride, const float* scale, const float* shift, const float* residual,
                   int res_mode, const float* up_src, int up_h, int up_w, int relu, int sigmoid_ch, int passes, int force_block_n,
                   float* y, int y_pix_stride, dt_stream_t stream);

/* One operand of dt_conv2d_nhwc_two_phase: conv(x, w) over filter taps [tap0, tap0 + ntaps) (ntaps 0: all kh*kw), * scale + shift.
 * x [N,H,W,Cin] fp32, dense; w_hi / w_lo as for dt_conv2d_nhwc (kind 0) or dt_conv2d_nhwc_f16x3 (kind 1). */
typedef struct dt_conv_operand {
    const float* x;
    int H, W, Cin;
    const void* w_hi;
    const void* w_lo;
    int kh, kw, pad, stride, tap0, ntaps;
    const float* scale;
    const float* shift;
} dt_conv_operand;
/* y [N,Ho,Wo,Cout] = act( phase2 + phase1 ), with phase 1's fp32 result kept on chip as the residual of phase 2 (both GEMMs run in one
 * launch, tile by tile; what the engine runs for a bottleneck's downsample + conv3 and for the two K-split halves of a mask-head conv).
 * The sum is rounded exactly as phase 1 written to a buffer and then phase 2 with that buffer as its residual.  The phases must give
 * the same output extents and tile shape.  phase1 NULL: phase 2 alone, plus `residual` [N,Ho,Wo,Cout] when given.
 * kind 0 = 3xTF32, 1 = 3xFP16.  im_info [N,5] (may be NULL): output pixels outside image n (its network size at im_stride) are zero. */
int dt_conv2d_nhwc_two_phase(int kind, const dt_conv_operand* phase1, const dt_conv_operand* phase2, const float* residual, int N, int Cout,
                             int relu, int passes, int force_block_n, int* range_flag, const float* im_info, int im_stride, float* y,
                             dt_stream_t stream);


/* ---------------------------------------------------------------------------------------------
 * Fused Mask R-CNN (ResNet-50/101 + FPN) inference engine: the whole of
 *   lib/model/detector.py:233-286 (detector.forward), lib/utils/result_utils.py:76-168
 *   (postprocess_output) and lib/model/detector.py:99-112 (mask_head.forward)
 * as one static, sync-free program of sm_90a kernels.  The caller owns two flat device buffers
 * (weights, workspace); named intermediate / output tensors are exposed as (offset, shape) into the
 * workspace so the host language wraps them without copies.
 */
typedef struct dt_engine_config {
    int arch_blocks[4];          /* bottlenecks per stage: {3,4,6,3} = ResNet-50, {3,4,23,3} = ResNet-101 */
    int batch, height, width;    /* network input [batch,3,height,width], height/width multiples of 32 */
    int pre_nms_top_n;           /* per-level RPN top-k before NMS (1000, detector.py:206)  */
    int post_nms_top_n;          /* per-level and collected RoI count (1000, detector.py:207) */
    float rpn_nms_thresh;        /* 0.7 (generate_proposals.py:28) */
    float rpn_min_size;          /* 0   (generate_proposals.py:17) */
    int num_classes;             /* 81 */
    float score_thresh;          /* 0.05 (result_utils.py:98) */
    float det_nms_thresh;        /* 0.5  (result_utils.py:99) */
    int max_dets;                /* 100  (result_utils.py:106) */
    int det_cap;                 /* padded detections per image in the fused outputs (>= max_dets) */
    int use_mask;                /* build the '1up4convs' mask head */
    int output_prob;             /* softmax / sigmoid on the outputs (detector.py:147) */
    int emit_full_masks;         /* also materialise masks_full [D,num_classes,28,28] (the public layout) */
    int passes;                  /* 3 = 3xTF32 (fp32-accurate, default), 1 = single-pass TF32 */
    int exact_roialign;          /* 1 = RoIAlign in the reference's exact fp32 operation order (bit-identical to its CPU loop);
                                    0 = separable / FMA fast path (fp32 re-association only, ~1e-7 relative) */
    int model_type;              /* 0 = R-50/101-FPN + RPN (+ '1up4convs' mask head); 1 = R-50/101-C4 (res5 head, 'upshare' mask head) */
    int use_rpn;                 /* 1 = Faster/Mask R-CNN (RPN head + proposal generation on the device), 0 = Fast R-CNN with pre-computed
                                    proposals (eval_fast.ipynb / eval_fast_FPN.ipynb): the caller fills `rois` (+ `roi_levels` for FPN), `roi_counts`.
                                    FPN engines without the RPN can instead take the raw proposals: float32 "fast_props" [batch,
                                    post_nms_top_n, 4] (original-image coordinates) and int32 "fast_prop_counts" [batch]; stage 4 then
                                    scales them by each image's scaling factor, drops the duplicates of preprocess_sample.remove_dup_prop
                                    (spatial scale 1/16) and writes the survivors in its order, with their FPN levels, to `rois` /
                                    `roi_levels` / `roi_counts`.  The host must keep |box * scale / 16| below 8990 (exact hash). */
    int conv_kind;               /* 0 = three-term product on the kind::f16 pipe (fp16 hi/lo halves, default: twice the tf32 issue rate; an
                                    activation >= 65504 raises the int32 buffer "range_flag", which every run that starts at the first stage clears
                                    before it launches anything), 1 = 3xTF32 (no range limit).  An FPN engine of kind 0 hands activations
                                    over as two fp16 planes (hi, lo) from conv1 to conv2 to conv3 of every trunk bottleneck and from the packed
                                    image to the stem, so the consumer loads its operand tiles without re-converting them */
} dt_engine_config;

typedef void* dt_engine_t;

dt_engine_t dt_engine_create(const dt_engine_config* cfg);
void dt_engine_destroy(dt_engine_t e);
int64_t dt_engine_weight_bytes(dt_engine_t e);
int64_t dt_engine_workspace_bytes(dt_engine_t e);
/* attach caller-owned device memory and build the launch program (TMA descriptors) */
int dt_engine_bind(dt_engine_t e, void* weights, void* workspace, dt_stream_t stream);
/* same, on a weight buffer that another engine with the same model configuration (all of dt_engine_config but batch/height/width)
 * has already loaded and finalised: packed weights are shape-independent, so engines for different image sizes share one copy */
int dt_engine_attach(dt_engine_t e, void* loaded_weights, void* workspace, dt_stream_t stream);
/* load one parameter by its reference state_dict name (torch layout, e.g. conv [Cout,Cin,kh,kw]); BN gains are
 * folded as g/sqrt(1+1e-5) (detector.py:231,301).  returns 1 loaded, 2 ignored (not on the hot path), 0 error */
int dt_engine_load_param(dt_engine_t e, const char* name, const float* src_dev, int64_t numel, dt_stream_t stream);
int dt_engine_finalize_weights(dt_engine_t e, dt_stream_t stream);
/* named buffer -> byte offset into the workspace, shape (<=5 dims), dtype (0 f32, 1 i32, 2 u8) */
int dt_engine_buffer(dt_engine_t e, const char* name, int64_t* byte_offset, int* ndim, int* dims5, int* dtype);
int dt_engine_num_stages(void);
/* the hot-path parameter table: reference state_dict names and element counts */
int dt_engine_param_count(dt_engine_t e);
int dt_engine_param_info(dt_engine_t e, int i, char* name_out, int name_cap, int64_t* numel);
/* original (un-scaled) image size used by the detection clip (result_utils.py:86); 0,0 = network size / scaling_factor */
int dt_engine_set_original_size(dt_engine_t e, float orig_h, float orig_w);
/* Batches of differently-sized images (FPN engine; returns 0 for C4).  The network input [batch,3,height,width] is then a canvas:
 * image b occupies the top-left net_h x net_w of its slot (its own im_list_to_blob size, a multiple of 32 <= the canvas) and has its
 * own scaling factor and original size.  The caller writes them into the engine buffer "im_info", float32 [batch, 5] =
 * (net_h, net_w, scaling_factor, orig_h, orig_w), orig <= 0 meaning net / scaling_factor; what the canvas holds outside the images
 * is ignored (NaN included).  Kernels read the table when they run, not when they are launched: a CUDA graph captured with the table
 * on replays for any size mix; write it on the stream of the run, before the run.  Each image's outputs are bit-identical to a
 * batch-1 run of that image at its own size; the scaling_factor argument of dt_engine_run is ignored while the table is on.
 * enabled = 0 returns to whole-canvas images and the scalar scaling factor / dt_engine_set_original_size. */
int dt_engine_use_image_info(dt_engine_t e, int enabled);
/* stages: 0 trunk, 1 FPN, 2 RPN convs, 3 proposals, 4 collect (FPN Fast R-CNN: pre-computed proposals -> RoIs), 5 RoIAlign(box), 6 box head, 7 detect (decode+NMS+limit),
 *         8 mask RoIs, 9 RoIAlign(mask), 10 mask convs, 11 mask output */
int dt_engine_run(dt_engine_t e, const float* image_nchw, float scaling_factor, int first_stage, int last_stage, dt_stream_t stream);
int dt_engine_count_launches(dt_engine_t e, int first_stage, int last_stage);
/* the RPN proposals of the last run through stage 4 (FPN engine with the RPN; 0 otherwise): boxes [batch, post_nms_top_n, 4] float32
 * = the collected RoIs / each image's scaling factor (fp32 division, original-image coordinates), scores [batch, post_nms_top_n] float32
 * = their RPN objectness, in the collect's order; rows past roi_counts are zero.  boxes 16-byte aligned.  Launched on `stream`, not
 * part of the engine program (a run to the detections never pays for it). */
int dt_engine_proposals(dt_engine_t e, float* boxes, float* scores, dt_stream_t stream);
/* measurement aid: one pass with a CUDA-event pair around every launch on `stream` (synchronises at the end);
 * per-op milliseconds, algorithmic FLOPs (0 for non-GEMM ops), stage id, BLOCK_N (0 for non-GEMM ops) */
int dt_engine_profile(dt_engine_t e, const float* image_nchw, float scaling_factor, int first_stage, int last_stage, dt_stream_t stream,
                      float* ms_out, double* flops_out, int* stage_out, int* block_n_out, int cap);

/* ---------------------------------------------------------------------------------------------
 * COCO box / mask evaluation (pycocotools COCOeval, iouType 'bbox' or 'segm'; the default thresholds, area ranges and maxDets), bit for bit.
 * Table layouts are the constants at the top of detectorch_b200/csrc/coco_eval.cuh.
 * dt_coco_gt_build: ground-truth masks -> RLE, one CTA per annotation.
 *   anns [num_anns, 6] int64      kind (0 polygon parts, 1 uncompressed counts, 2 compressed string), h, w, first part, parts, output offset
 *   parts [.., 4] int64           first element of xy (point pairs) / ucounts / chars, its element count, int32 workspace offset, and for a
 *                                 polygon the number of upsampled boundary points (k points, m of them: k + 4 m + 3 ints of workspace)
 *   out_counts / tmp_counts       uint32 run lengths at each annotation's offset (capacity: up to the next annotation's offset)
 *   out_len [num_anns] int64, out_box [num_anns, 4] double (rleToBbox)
 * dt_coco_eval: one evaluation of a detection set against a built ground truth, grouped by (category, image) pair in
 *   category-major order.  iou_type 0 bbox, 1 segm.
 *   pairs [num_active, 7]         pair index, first detection, D, first gt, G, first kept slot (min(D, 100) per pair), first IoU (min(D,100) G)
 *   cat_gt / cat_kept [K+1]       each category's gt range / kept-slot range; order_off [3, K+1] each category's list for maxDets 1, 10, 100
 *   det_f [num_dets, 5] double    score, x, y, w, h;  det_i [num_dets, 4] int64: char offset, char count, h, w (segm strings in det_chars)
 *   gt_f [num_gts, 9] double      bbox x y w h, area, RLE box;  gt_i [num_gts, 6] int64: RLE offset, length, h, w, iscrowd, id != 0
 *   params [119] double           area ranges [4][2], IoU thresholds min(t, 1 - 1e-10) [10], recall thresholds [101]
 *   precision / scores [10, 101, K, 4, 3], recall [10, K, 4, 3] double
 *   ious                          optional [num_ious] double: each pair's IoU matrix [min(D, 100), G] (detections in score order, gts in
 *                                 annotation order) at its first IoU; NULL keeps them in the workspace
 *   det_area                      optional [num_dets] double: each detection's area for the area ranges (loadRes's 'area' of a results
 *                                 file); NULL: w h of its box for bbox, its RLE area for segm
 * dt_coco_det_check: bad [num_dets] uint8, 1 where a segm detection's string (det_i / det_chars as for dt_coco_eval) decodes to
 *   counts that do not sum to h * w.  rleIou never ends on such a mask, so dt_coco_eval must not be given one.
 * dt_coco_results_append / _count / _write: detect() batches kept on the device as records (utils.coco_eval.DeviceResults) and
 *   flattened into dt_coco_eval's tables.  Record: rec_f [n, 5] float x1, y1, x2, y2, score; rec_i [n, 7] int64 image ordinal (-1 for a
 *   dead slot), class, rank inside its class in the image, char offset, char count, h, w.
 *   append: boxes [B, cap, 4], scores [B, cap] float, classes [B, cap], counts [B] int; images [B, 3] int64 ordinal, h, w; str_offs
 *   [B cap + 1] the batch's string offsets (NULL without masks) placed at char_base; writes B cap records; err int [2] (err[1] set to
 *   INT_MAX by the caller): err[0] |= 1 and err[1] = min ordinal of an image with a live class outside 1..num_classes-1 or out of order.
 *   count: cls_k [num_classes] category slot of each class (-1: none), ord_i [ordinals] image index (-1: none); num_images x num_cats
 *   pairs of cats_per_pair slots each (1, or num_cats = 1 for a class-agnostic evaluation whose slots are the categories in the order
 *   their detections are concatenated; coco_eval.cuh has the fine bin layout); bin_cnt int [K I cats_per_pair] zeroed by the caller;
 *   scan_in [5, K I] int64 gets D, D > 0, min(D, 10), min(D, 100), min(D, 100) G per pair, to be scanned (inclusive, along the pairs)
 *   into write's scan; gt_keys: the evaluated gts' pair indices (sorted); nonfinite (zeroed) |= 1 for a non-finite value in a counted record.
 *   write: det_key [N] int64 (each row's fine bin), det_f [N, 5], det_i [N, 4], pairs [num_active, 7], cat_kept [K+1], order_off [3, K+1]
 *   as dt_coco_eval takes them.
 * All return 0 on bad sizes or a NULL pointer. */
int dt_coco_results_append(int batch, int cap, int num_classes, const float* boxes, const float* scores, const int* classes, const int* counts,
                           const int64_t* images, const int64_t* str_offs, int64_t char_base, float* rec_f, int64_t* rec_i, int* err,
                           dt_stream_t stream);
int dt_coco_results_count(int64_t num_records, const float* rec_f, const int64_t* rec_i, int num_classes, const int* cls_k, const int* ord_i,
                          int num_images, int num_cats, int cats_per_pair, const int64_t* gt_keys, int64_t num_gts, int* bin_cnt, int64_t* scan_in,
                          int* nonfinite, dt_stream_t stream);
int dt_coco_results_write(int64_t num_records, const float* rec_f, const int64_t* rec_i, int num_classes, const int* cls_k, const int* ord_i,
                          int num_images, int num_cats, int cats_per_pair, const int* bin_cnt, const int64_t* scan, const int64_t* gt_keys,
                          int64_t num_gts, int64_t* det_key, double* det_f, int64_t* det_i, int64_t* pairs, int64_t* cat_kept, int64_t* order_off,
                          dt_stream_t stream);
int dt_coco_det_check(int64_t num_dets, const int64_t* det_i, const char* det_chars, uint8_t* bad, dt_stream_t stream);
int64_t dt_coco_gt_workspace_bytes(int64_t num_parts, int64_t num_points, int64_t num_upsampled);
int dt_coco_gt_build(int num_anns, const int64_t* anns, const int64_t* parts, const double* xy, const uint32_t* ucounts, const char* chars,
                     void* workspace, uint32_t* out_counts, uint32_t* tmp_counts, int64_t* out_len, double* out_box, dt_stream_t stream);
int64_t dt_coco_eval_workspace_bytes(int64_t num_dets, int64_t num_chars, int64_t kept, int64_t num_ious, int64_t num_gts, int64_t num_order,
                                     int num_cats);
int dt_coco_eval(int iou_type, int num_images, int num_cats, int num_active, const int64_t* pairs, const int64_t* cat_gt, const int64_t* cat_kept,
                 const int64_t* order_off, int64_t num_dets, const double* det_f, const int64_t* det_i, const char* det_chars, int64_t num_chars,
                 int64_t kept, int64_t num_ious, int64_t num_gts, int64_t num_order, const double* gt_f, const int64_t* gt_i,
                 const uint32_t* gt_counts, const double* params, double* precision, double* recall, double* scores, double* ious, void* workspace,
                 dt_stream_t stream, const double* det_area);
/* dt_coco_eval_imgs: COCOeval's per-image records (evalImgs) of the evaluation dt_coco_eval has just enqueued, from its workspace and
 * IoU matrices (every size argument and table as given to it; ious must not be NULL there).  union_keys [num_union] int64: the sorted
 * pair indices of the pairs with detections or gts; gt_keys [num_gts] each gt's pair index (sorted).  Outputs, state c = area * 10 +
 * threshold:  slot_det [kept] int: detection index of each kept slot;  dt_gt [kept, 40] int: index in its pair of the gt a kept detection
 * matched, -1 none;  dt_ig [kept, 40] uint8: dtIgnore;  gt_dt [num_gts, 40] int: rank in its pair of the last kept detection that matched
 * the gt, -1 none;  gt_pos [num_gts, 4] int: position in the area's ignore-last gt order;  gt_ig [num_gts, 4] uint8: gtIgnore.
 * det_area: the one given to dt_coco_eval. */
int dt_coco_eval_imgs(int iou_type, int num_union, const int64_t* union_keys, int num_active, const int64_t* pairs, int64_t num_dets,
                      const double* det_f, int64_t num_chars, int64_t kept, int64_t num_ious, int64_t num_gts, int64_t num_order,
                      const int64_t* gt_keys, const double* gt_f, const int64_t* gt_i, const double* params, const double* ious,
                      const void* workspace, int* slot_det, int* dt_gt, uint8_t* dt_ig, int* gt_dt, int* gt_pos, uint8_t* gt_ig,
                      dt_stream_t stream, const double* det_area);

/* dt_coco_json: the COCO results json of the reference's results writers + json.dump, byte for byte, in two passes over the
 * flattened results (iou_type 0 bbox, 1 segm; det_f / det_i / det_chars as dt_coco_eval takes them, rows in any order).
 *   det_key [num_dets] int64        category index * num_images + image index; img_ids [num_images], cat_ids json ids of those indexes
 *   file_pos [num_dets] int64       each row's record in the file (a permutation of 0..num_dets-1)
 *   counts_first [num_dets] uint8   segm, by file position: 1 where the RLE dict is written 'counts' first (NULL: 'size' first everywhere)
 *   offsets == NULL                 length pass: lens [num_dets] int64 = each record's bytes at its file position ("[" / ", " before it,
 *                                   "]" after the last)
 *   offsets != NULL                 write pass: offsets [num_dets] the inclusive scan of lens; text [offsets[num_dets - 1]] bytes
 * bbox runs one thread per record, segm one warp.  Returns 0 on bad sizes or a NULL pointer. */
int dt_coco_json(int iou_type, int64_t num_dets, const double* det_f, const int64_t* det_key, const int64_t* file_pos, int num_images,
                 const int64_t* img_ids, const int64_t* cat_ids, const int64_t* det_i, const char* det_chars, const uint8_t* counts_first,
                 const int64_t* offsets, int64_t* lens, char* text, dt_stream_t stream);

/* COCO results json read on the device (COCO.loadRes of a results file; detectorch_b200/csrc/coco_results_file.cuh), in four calls:
 * dt_coco_file_struct: the structural pass over text [num_bytes] with a workspace of dt_coco_file_struct_workspace_bytes, kept for
 *   dt_coco_file_separators.  info [8] int64 (zeroed, info[4] = INT64_MAX by the caller): separators, error bits, summary bits, records of
 *   unknown categories, first record with an error, top-level '[' count, 1 for an empty array.
 * dt_coco_file_separators: separators [info[0]] int64, the top-level '[', the ',' between records and the closing ']'.
 * dt_coco_file_records: num_records = separators - 1; img_ids [num_images] / cat_ids [num_cats] the ground truth's sorted json ids;
 *   rec_f [R, 5] double score, bbox x y w h (rec_open [R, 5] int64 scratch for the numbers decided exactly); rec_i [R, 6] int64 image index, category index (-1: not in the ground truth), raw span of
 *   'counts' in text, h, w; rec_n [R] int64 decoded counts length; rec_b [R] uint8 flags (coco_results_file.cuh).
 * dt_coco_file_finish: offsets = the inclusive scan of rec_n, num_chars its total; chars [num_chars + 1]; segm 1 for loadRes's segm
 *   branch; workspace of dt_coco_file_finish_workspace_bytes.  det_key [num_records] int64: the keys (category index * num_images + image
 *   index) sorted; the first num_kept rows (the records of known categories) of det_f [.., 5], det_i [.., 4] (dt_coco_eval's layout),
 *   det_area (loadRes's area) and det_id (1 + the record's index in the file), in key order, stable.
 * All return 0 on bad sizes or a NULL pointer. */
int64_t dt_coco_file_struct_workspace_bytes(int64_t num_bytes);
int dt_coco_file_struct(int64_t num_bytes, const uint8_t* text, void* workspace, int64_t* info, dt_stream_t stream);
int dt_coco_file_separators(int64_t num_bytes, void* workspace, int64_t* separators, dt_stream_t stream);
int dt_coco_file_records(int64_t num_records, int64_t num_bytes, const uint8_t* text, const int64_t* separators, int num_images,
                         const int64_t* img_ids, int num_cats, const int64_t* cat_ids, double* rec_f, int64_t* rec_open, int64_t* rec_i,
                         int64_t* rec_n, uint8_t* rec_b, int64_t* info, dt_stream_t stream);
int64_t dt_coco_file_finish_workspace_bytes(int64_t num_records, int64_t num_chars, int segm);
int dt_coco_file_finish(int64_t num_records, int segm, const uint8_t* text, const int64_t* rec_i, const int64_t* rec_n, const int64_t* offsets,
                        const uint8_t* rec_b, double* rec_f, int num_images, int num_cats, int64_t num_chars, char* chars, void* workspace,
                        int64_t num_kept, int64_t* det_key, double* det_f, int64_t* det_i, double* det_area, int64_t* det_id, int64_t* info,
                        dt_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Proposal recall (Detectron's evaluate_box_proposals), bit for bit.  One CTA per (image, combination); every combination of
 * (area range, proposal limit) in one launch.
 *   prop_off / gt_off [I+1] int64  each image's range in props [NP, 4] / gts [NG, 4] (float32 x1 y1 x2 y2; gts: gt_classes > 0, not crowd)
 *   gt_area [NG] double            seg_areas
 *   area_rng [C, 2] double         inclusive range; limits [C] int64 (< 0: no limit)
 *   out_off [C, I] int64           first output of (combination, image): the image's GTs in the range when it has proposals, else none
 *   max_gts / max_props            the largest gt / proposal count of one image (shared-memory sizing)
 *   out double                     each GT's recorded overlap, in assignment order, 0 past the last round
 *   flag int (zeroed by the caller) bit 0: a chosen overlap < 0 (the reference asserts), bit 1: a union of 0 (it divides by zero)
 * dt_proposal_recall_smem_bytes: the dynamic shared memory one CTA needs (the launch refuses more than 227 KB). */
int64_t dt_proposal_recall_smem_bytes(int max_gts, int64_t max_props);
int dt_proposal_recall(int num_images, int num_combos, const int64_t* prop_off, const float* props, const int64_t* gt_off, const float* gts,
                       const double* gt_area, const double* area_rng, const int64_t* limits, const int64_t* out_off, int max_gts,
                       int64_t max_props, double* out, int* flag, dt_stream_t stream);

/* library / build info */
const char* dt_version(void);

#ifdef __cplusplus
}
#endif
#endif
