/*
 * ssdk.h -- C-ABI of the H100-native SSD hot path (libssdk.so).
 *
 * The reference (pierluigiferrari/ssd_keras) is pure Python: it has no FFI / plugin
 * interface of its own, so the drop-in boundary is its public Python surface (SURVEY.md
 * section 8b).  Each entry point below names the reference interface it replaces
 * (file:line relative to the reference root).  The Python package `ssd_keras_b200`
 * re-creates those reference names on top of this library through ctypes; see
 * INTEGRATION.md for the binding a reference maintainer would add.
 *
 * Conventions
 *   - extern "C", plain pointers and sizes, no C++/torch types.
 *   - every function returns 0 on success or a negative ssdk_status; it never throws.
 *     ssdk_last_error() returns a thread-local, human readable message for the last failure.
 *   - "dev" pointers are CUDA device pointers on the context's device; "host" pointers are
 *     ordinary host memory.  Outputs are caller-allocated.
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).  Calls are
 *     asynchronous with respect to the host unless stated otherwise.
 *   - a context (and the objects created from it) may be used by one host thread at a time.
 *   - there is NO CPU fallback: without a CUDA device every compute call fails with
 *     SSDK_ERR_CUDA.
 */
#ifndef SSDK_H_
#define SSDK_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SSDK_VERSION 100

typedef enum {
  SSDK_OK = 0,
  SSDK_ERR_INVALID = -1,     /* bad argument (the Python layer raises ValueError)          */
  SSDK_ERR_CUDA = -2,        /* CUDA runtime/driver failure, message has the cuda error    */
  SSDK_ERR_UNSUPPORTED = -3, /* valid in the reference but not implemented here            */
  SSDK_ERR_NOMEM = -4,
  SSDK_ERR_DEGENERATE = -5   /* degenerate ground-truth box (reference: DegenerateBoxError) */
} ssdk_status;

typedef enum { SSDK_COORDS_CENTROIDS = 0, SSDK_COORDS_CORNERS = 1, SSDK_COORDS_MINMAX = 2 } ssdk_coords;

typedef struct ssdk_ctx ssdk_ctx;
typedef struct ssdk_encoder ssdk_encoder;
typedef struct ssdk_model ssdk_model;

int ssdk_version(void);
const char* ssdk_last_error(void);

/* One context per (device, host thread).  Owns scratch workspaces. */
int ssdk_ctx_create(int device, ssdk_ctx** out);
int ssdk_ctx_destroy(ssdk_ctx* ctx);
/* Number of kernels this library launched through `ctx` since creation (bench.py's gpu_launches). */
int64_t ssdk_ctx_launch_count(const ssdk_ctx* ctx);

/* ------------------------------------------------------------------------------------------
 * Anchor boxes.  Replaces SSDInputEncoder.generate_anchor_boxes_for_layer
 * (ssd_encoder_decoder/ssd_input_encoder.py:420-548) and AnchorBoxes.call
 * (keras_layers/keras_layer_AnchorBoxes.py:133-255).  Host-side float64 arithmetic, bit-exact
 * with the reference; `out_f32` is the float32 cast the Keras layer emits (:252).
 * steps_* / offsets_* entries that are NaN mean "None" (derive step from the feature map,
 * offset 0.5).  Prior order: layers in order, ((y*W + x)*n_boxes + b) within a layer.
 * ------------------------------------------------------------------------------------------ */
typedef struct {
  int img_height, img_width;
  int n_layers;
  const int* fm_height;          /* [n_layers] predictor feature-map sizes */
  const int* fm_width;           /* [n_layers] */
  const double* scales;          /* [n_layers + 1] */
  const int* n_aspect_ratios;    /* [n_layers] */
  const double* aspect_ratios;   /* concatenated, sum(n_aspect_ratios) entries */
  int two_boxes_for_ar1;
  const double* steps_h;         /* [n_layers] or NULL; NaN = None */
  const double* steps_w;
  const double* offsets_h;       /* [n_layers] or NULL; NaN = None */
  const double* offsets_w;
  int clip_boxes;
  int coords;                    /* ssdk_coords */
  int normalize_coords;
} ssdk_anchor_cfg;

int ssdk_anchors_count(const ssdk_anchor_cfg* cfg, int* out_P, int* out_n_boxes /* [n_layers] or NULL */);
int ssdk_anchors_generate(const ssdk_anchor_cfg* cfg, double* out_f64 /* host [P*4] */, float* out_f32 /* host [P*4] or NULL */);

/* ------------------------------------------------------------------------------------------
 * Ground-truth encoder.  Replaces SSDInputEncoder.__call__
 * (ssd_encoder_decoder/ssd_input_encoder.py:277-418) together with iou
 * (bounding_box_utils/bounding_box_utils.py:283-383), match_bipartite_greedy and match_multi
 * (ssd_encoder_decoder/matching_utils.py:22-116) and generate_encoding_template (:550-611).
 * IoU and matching decisions are taken in float64 like the reference; the target tensor is
 * written as float32 (what Keras feeds the loss).  One kernel launch per batch; an encoder object owns
 * scratch memory and must not be used from two streams at the same time.
 * ------------------------------------------------------------------------------------------ */
typedef struct {
  int img_height, img_width;
  int n_classes_total;       /* including background */
  int P;                     /* number of anchors */
  int background_id;
  int coords;                /* ssdk_coords: format of `anchors` and of the encoded targets */
  int matching_multi;        /* 1 = 'multi', 0 = 'bipartite' */
  double pos_iou_threshold;
  double neg_iou_limit;
  int border_d;              /* 0 'half', 1 'include', -1 'exclude' */
  int normalize_coords;
  double variances[4];
  /* Optional predictor-layer geometry (prior index = layer offset + (y*fm_width + x)*n_boxes + box): lets the encoder
   * group priors into compact blocks of feature-map cells, so that fewer ground-truth boxes touch a block.  n_layers = 0
   * (or NULL arrays): consecutive groups of 256 priors only.  The arrays are read during ssdk_encoder_create. */
  int n_layers;
  const int* fm_height;      /* [n_layers] */
  const int* fm_width;       /* [n_layers] */
  const int* n_boxes;        /* [n_layers] */
} ssdk_encode_cfg;

int ssdk_encoder_create(ssdk_ctx* ctx, const ssdk_encode_cfg* cfg, const double* anchors_host /* [P*4], in cfg->coords */,
                        ssdk_encoder** out);
int ssdk_encoder_destroy(ssdk_encoder* enc);
/* gt_boxes_dev: [sum(G_i) * 5] float32 rows (class_id, xmin, ymin, xmax, ymax) in pixels, images concatenated;
 * gt_offsets_host: [B+1] row offsets (host; the ragged shape is host knowledge in the reference too);
 * out_y_dev: [B * P * (C+12)] float32;  out_match_dev (optional): [B * P] int32, matched gt index within the
 * image, -1 = background, -2 = neutral.  status_dev (optional): one int32 that is set to the 1-based index of
 * a batch item with a degenerate box (xmax<=xmin or ymax<=ymin), else left 0 (reference raises :333-336). */
int ssdk_encode(ssdk_encoder* enc, const float* gt_boxes_dev, const int* gt_offsets_host, int B,
                float* out_y_dev, int* out_match_dev, int* status_dev, void* stream);
/* Same with float64 ground-truth rows: the reference converts whatever it is given to float64 (:330), so labels that are
 * not representable in float32 (sub-pixel coordinates after augmentation) need this entry to stay bit-exact. */
int ssdk_encode_f64(ssdk_encoder* enc, const double* gt_boxes_dev, const int* gt_offsets_host, int B,
                    float* out_y_dev, int* out_match_dev, int* status_dev, void* stream);
/* Same with the row offsets already on the device (the batch was assembled there, see ssdk_assemble_batch): nothing
 * is read from the host; total_g = gt_offsets[B] and max_g = the largest per-image box count (or an upper bound of it). */
int ssdk_encode_dev(ssdk_encoder* enc, const float* gt_boxes_dev, const int* gt_offsets_dev, int B, int total_g, int max_g,
                    float* out_y_dev, int* out_match_dev, int* status_dev, void* stream);
/* Standalone pieces, used by tests and the micro-benchmark: IoU matrix (G x P, float64, row-major). */
int ssdk_iou_matrix(ssdk_encoder* enc, const float* gt_boxes_dev, int G, double* out_dev, void* stream);
/* General IoU, replaces iou() (bounding_box_utils/bounding_box_utils.py:283-383): boxes1 [m*4], boxes2 [n*4] float64 in
 * `coords` format; elementwise=0 -> out [m*n] ('outer_product'), elementwise=1 -> out [max(m,n)] with broadcasting of a
 * single box ('element-wise').  Keeps the reference quirk: the intersection ignores border_d, the areas use it. */
int ssdk_iou(ssdk_ctx* ctx, const double* boxes1_dev, int m, const double* boxes2_dev, int n, int coords, int border_d,
             int elementwise, double* out_dev, void* stream);

/* ------------------------------------------------------------------------------------------
 * Batch assembly (the hand-off DataGenerator.generate -> label_encoder, data_generator/object_detection_2d_data_generator.py:
 * 1095-1151) and the box half of the reference's geometric augmentation ops on the device: per image a list of operations
 * with the parameters the caller's (host-side, random) augmentation logic decided, applied to every box in float64 like
 * NumPy does, boxes that fail a filter are dropped, the survivors are packed into the encoder's ragged format.
 *   CROP_PAD  a0=patch_ymin a1=patch_xmin a2=patch_height a3=patch_width; flags bit0: BoxFilter 'center_point' against the
 *             patch, bit1: clip to the patch      (CropPad.__call__, object_detection_2d_patch_sampling_ops.py:312-330;
 *             SSDExpand = negative patch origin without filter / clip, SSDRandomCrop = filter + clip)
 *   FLIP_H    a0=image width   FLIP_V  a0=image height                  (object_detection_2d_geometric_ops.py:186,194)
 *   RESIZE    a0=in_height a1=in_width a2=out_height a3=out_width; flags bit0: drop degenerate boxes afterwards (:88-100)
 *   FILTER    flags bit0: drop degenerate boxes (xmax <= xmin or ymax <= ymin), bit1: drop boxes with area < a0
 *             (BoxFilter, object_detection_2d_image_boxes_validation_utils.py:155-165; also DataGenerator's
 *             degenerate_box_handling='remove')
 *   TRANSLATE a0=dy_abs a1=dx_abs (integers, Translate's int(round(h*dy)) / int(round(w*dx))) a2=image height a3=image width;
 *             boxes += dx_abs / dy_abs                                  (Translate.__call__, object_detection_2d_geometric_ops.py:276-317)
 *   SCALE     a0=factor a1=image height a2=image width: both corners through M = getRotationMatrix2D((w/2, h/2), 0, factor)
 *             as np.dot computes it, (m0*x + m1*y) + m2 with every step rounded, then np.round      (Scale.__call__, :487-532)
 *             stored as an integer (astype(int)): a corner that rounds to -0 is +0.  Both clips are np.clip: a NaN passes
 *             through and a coordinate equal to a bound keeps its sign (-0.0 stays -0.0)
 *   ROTATE    a0=angle (90, 180 or 270; other values leave the boxes alone) a1=image height a2=image width: Rotate's adjusted
 *             matrix, the same corner arithmetic, then its ymin/ymax and xmin/xmax swaps             (Rotate.__call__, :681-737)
 *   OVERLAP   BoxFilter's overlap test against an a2 x a3 (height x width) image, bounds (a0, a1] / [a0, a1]: flags bits 0-1
 *             criterion 0 'center_point', 1 'area' (lower == 0 compares with >), 2 'iou' (the intersection ignores
 *             border_pixels, as bounding_box_utils.iou does); bits 2-3 border_pixels 0 'half', 1 'include', 2 'exclude'
 *             (object_detection_2d_image_boxes_validation_utils.py:186-230)
 *   CLIP      a0=image height a1=image width: clip to [0, h-1] x [0, w-1] (the clip_boxes step of Translate / Scale / CropPad)
 * Codes the kernel does not know are skipped.
 * ------------------------------------------------------------------------------------------ */
typedef enum { SSDK_BOXOP_END = 0, SSDK_BOXOP_CROP_PAD = 1, SSDK_BOXOP_FLIP_H = 2, SSDK_BOXOP_FLIP_V = 3, SSDK_BOXOP_RESIZE = 4,
               SSDK_BOXOP_FILTER = 5, SSDK_BOXOP_TRANSLATE = 6, SSDK_BOXOP_SCALE = 7, SSDK_BOXOP_ROTATE = 8,
               SSDK_BOXOP_OVERLAP = 9, SSDK_BOXOP_CLIP = 10,
               /* photometric ops, from 16 on (11-15 are unassigned: ssdk_assemble_images rejects them as unknown): images only; the
                * box kernel skips them */
               SSDK_BOXOP_TO_FLOAT32 = 16, SSDK_BOXOP_TO_UINT8 = 17, SSDK_BOXOP_BRIGHTNESS = 18, SSDK_BOXOP_CONTRAST = 19,
               SSDK_BOXOP_SATURATION = 20, SSDK_BOXOP_HUE = 21, SSDK_BOXOP_RGB2HSV = 22, SSDK_BOXOP_HSV2RGB = 23,
               SSDK_BOXOP_CHANNEL_SWAP = 24 } ssdk_box_op_kind;
typedef struct { int op; int flags; double a0, a1, a2, a3; } ssdk_box_op;
/* gt_in_dev [total_in*5] float32 (gt_in_f64 = 0) or float64 (1) rows (class, xmin, ymin, xmax, ymax), offsets_in_dev [B+1]; ops_dev [B*max_ops] (a list ends at
 * SSDK_BOXOP_END or after max_ops entries; max_ops = 0: pack only).  Outputs: gt_out_dev [<= total_in*5], offsets_out_dev [B+1],
 * out_stats_dev (optional) [2] = total number of boxes left, largest per-image count.  Everything stays on the device: feed
 * the result to ssdk_encode_dev with total_in / the input's largest count as upper bounds. */
int ssdk_assemble_batch(ssdk_ctx* ctx, const void* gt_in_dev, int gt_in_f64, const int* offsets_in_dev, int B, int total_in,
                        const ssdk_box_op* ops_dev, int max_ops, float* gt_out_dev, int* offsets_out_dev, int* out_stats_dev,
                        void* stream);
/* The image half of the same op lists: ConvertTo3Channels (object_detection_2d_photometric_ops.py:88-108; gray is replicated,
 * RGBA drops alpha, applied first), the image arithmetic of CropPad (:266-313) and Flip, uint8 cv2.resize, and uint8
 * cv2.warpAffine (INTER_LINEAR, BORDER_CONSTANT) of Translate / Scale / Rotate, into a float32 NHWC batch of [0,255] integers
 * (what ssdk_model_forward takes).  The image fields live in flag bits the box kernel never reads:
 *   CROP_PAD  flags bits 8-31: background R, G, B bytes (0 = black, as CropPad's default; SSDExpand uses 123,117,104)
 *   RESIZE    flags bits 8-15: cv2 interpolation code, INTER_NEAREST = 0 or INTER_LINEAR = 1 (an exact 2x linear downscale
 *             takes INTER_AREA's fast path, as cv2 does); any other code is an error
 *   TRANSLATE flags bits 8-31: background; an integer shift, composed like a pad / crop
 *   SCALE     flags bits 8-31: background; the bilinear warp, cv2's fixed-point scheme bit for bit
 *   ROTATE    an exact signed axis permutation (cv2's fixed-point map is checked on the host to have fraction 0 everywhere),
 *             black where the inverse map leaves the source
 *   FILTER, OVERLAP, CLIP   nothing to do for images
 * The photometric ops (object_detection_2d_photometric_ops.py) form a prefix of the list, run by one launch of
 * photometric_kernel in front of the assembly kernel, uint8 in and uint8 h x w x 3 out, bit for bit what NumPy and OpenCV 4.13
 * compute (oracle/photoops.py):
 *   TO_FLOAT32 / TO_UINT8    ConvertDataType: astype(float32) / np.round(x, 0).astype(uint8) (round half to even)
 *   BRIGHTNESS a0=delta      np.clip(image + delta, 0, 255); a0 is rounded to float32, as NumPy does with a Python float
 *   CONTRAST   a0=factor     np.clip(127.5 + factor * (image - 127.5), 0, 255), every step rounded to float32
 *   SATURATION a0=factor     channel 1: np.clip(s * factor, 0, 255)
 *   HUE        a0=delta      channel 0: (h + delta) % 180.0, NumPy's float32 remainder
 *   RGB2HSV / HSV2RGB        uint8 cv2.cvtColor.  HSV2RGB is cv2's float32 code on a CPU with AVX2, which truncates in its
 *                            32-pixel vector loop and rounds in the scalar loop that finishes each row: columns >= w / 32 * 32
 *                            round, the others truncate
 *   CHANNEL_SWAP a0..a2=order  image[:, :, order]
 * Gamma, histogram equalisation and conversions to GRAY are not covered; the random draws stay with the caller (an op that a
 * draw skipped is absent from the list).
 * src_dev: the B uint8 images packed back to back, image b at bytes src_offsets_host[b] .. src_offsets_host[b+1] (host, [B+1]),
 * of shape src_hwc_host[3b..3b+2] = h, w, c with c in {1, 3, 4}.  ops_host: [B*max_ops] on the HOST (a list ends at
 * SSDK_BOXOP_END or after max_ops entries).  out_dev: [B*out_h*out_w*3] float32.
 * Checked on the host before anything is enqueued (SSDK_ERR_INVALID, nothing written): sizes positive, B <= 65535, offsets
 * consistent with the shapes; each CROP_PAD integer with a positive size and overlapping its input (CropPad's own test, :270-271);
 * each flip's a0, and each TRANSLATE's, SCALE's and ROTATE's image height / width, equal to the canvas size at that point;
 * TRANSLATE integer, ROTATE by 90 / 180 / 270, SCALE by a positive factor whose fixed-point coordinates fit cv2's int32 / int16
 * ranges (canvas below 32767); at most one resampling step (RESIZE or SCALE); no crop / pad / flip / translate / rotate after
 * a RESIZE (after a SCALE they are applied to its output); the final size out_h x out_w; a supported interpolation code; and one
 * background colour per list: every pad or translate that brings in background, every SCALE, and a ROTATE whose map leaves
 * the source (black) must agree (bands of different colours are not represented).  Photometric ops: all of them before the
 * first op that changes the image geometry; at most 16; BRIGHTNESS / CONTRAST / SATURATION / HUE only between a TO_FLOAT32 and
 * the next TO_UINT8, the colour conversions and the end of the prefix only in the uint8 state; factors > 0, -180 <= hue delta
 * <= 180 (the reference's own ValueErrors), brightness delta finite, the swap order a permutation of (0, 1, 2).
 * Images with photometric ops are written, converted to 3 channels, to a scratch buffer owned by the context (grown when needed,
 * freed with the context) and assembled from there; the others are read from src_dev as before, and a call without photometric
 * ops launches and allocates nothing more than it did.
 * The integer ops before the resampling step are composed on the host into one signed-permutation map per image, those after a
 * SCALE into a second one; one kernel launch evaluates the whole list without an intermediate image.  The descriptors go to the
 * device with one asynchronous copy from pinned staging owned by the context (a ring of four buffers: the call waits only if the
 * upload of the call four calls earlier has not run yet); like the encoder, one context must not run this on two streams at the
 * same time. */
int ssdk_assemble_images(ssdk_ctx* ctx, const uint8_t* src_dev, const long long* src_offsets_host, const int* src_hwc_host, int B,
                         const ssdk_box_op* ops_host, int max_ops, int out_h, int out_w, float* out_dev, void* stream);

/* ------------------------------------------------------------------------------------------
 * Evaluation.  Replaces the per-prediction Python loop of Evaluator.match_predictions
 * (eval_utils/average_precision_evaluator.py:538-736, element-wise iou at :679) and the cumulative sums of :726-727.
 * The caller sorts the predictions twice (stable): by (class, confidence desc) -- the order of the outputs -- and by
 * (class, image, confidence desc) -- the order of the pred_* inputs, whose (class, image) runs are given by seg_offsets.
 *   pred_rank[i]   position of input prediction i in the (class, confidence desc) order
 *   gt_rows        float64 (class, xmin, ymin, xmax, ymax, area) rows of all images, gt_offsets [n_images+1]; area is the
 *                  reference's (xmax - xmin + d) * (ymax - ymin + d) computed in the labels' own dtype (an int16 area wraps)
 *   gt_f32         uint8 [n_images]: 1 when result_type(labels dtype, float32) is float32 (float32 / float16 / int16 / uint8
 *                  labels), 0 when it is float64 (int32 / int64 / float64 labels)
 *   gt_neutral     optional uint8 flags (eval_neutral, :684), gt_matched uint8 scratch zeroed by the caller
 *   tp / fp        int32 [n_pred], zeroed by the caller, in (class, confidence desc) order
 * The overlaps follow NumPy's types: the predicted area is float32 arithmetic (the reference's 'f4' structured array), the
 * intersection, union and quotient run in the image's type, NaN-propagating minimum / maximum, and on the float32 path the
 * threshold is rounded to float32.  Class ids are compared as float64 (a label class of 1.5 is no class).  The arg-max is
 * np.argmax's: first maximum, the first NaN wins, and NaN < threshold is False.
 * Two deliberate departures from the reference: every prediction is matched (its verbose=False loop matches only the first of
 * each class), and a class without predictions has empty outputs (the reference's cumulative lists skip it).
 * ssdk_eval_cumsum: inclusive scans of tp / fp inside each of the n_segments ranges class_offsets[c] .. class_offsets[c+1].
 * ------------------------------------------------------------------------------------------ */
int ssdk_eval_match(ssdk_ctx* ctx, int n_pred, const int* seg_offsets_dev, int n_seg, const int* pred_image_dev,
                    const int* pred_class_dev, const float* pred_box_dev, const int* pred_rank_dev, const double* gt_rows_dev,
                    const int* gt_offsets_dev, const unsigned char* gt_f32_dev, const unsigned char* gt_neutral_dev,
                    unsigned char* gt_matched_dev, double matching_iou_threshold, int border_d, int* tp_dev, int* fp_dev, void* stream);
int ssdk_eval_cumsum(ssdk_ctx* ctx, const int* tp_dev, const int* fp_dev, const int* class_offsets_dev, int n_segments,
                     int* ctp_dev, int* cfp_dev, void* stream);

/* ssdk_eval_collect: the per-box loop of Evaluator.predict_on_dataset (:374-419) and predict_all_to_json for one batch of
 * decoded rows_dev (B, max_out, 6) float32.  A row is kept when its column 0 is not 0 (y_pred[i][y_pred[i,:,0] != 0]) and, if
 * counts_dev is given, when it lies below counts_dev[b].  Each kept row goes through its image's inverters in the generator's
 * (reversed) order: Resize's (geometric_ops.py:74-79), v = rint(v * ratio) on the y and x columns, then, when a pad offset is
 * set (pad = 1, 'pad' mode), CropPad's (patch_sampling_ops.py:315-320), v += offset.  inv_dev holds four doubles per image:
 * ratio_y = canvas_h / out_h, ratio_x = canvas_w / out_w, offset_y, offset_x.  Then the confidence is rounded to conf_decimals
 * (0: not rounded) and the four box coordinates to one decimal, as round(numpy_scalar, n) does: rint(v * 10^n) / 10^n.
 * f64 = 0: every step in float32 (the layer path: NumPy computes float32_array * python_float in float32, the ratio rounded to
 * float32 first); f64 = 1: every step in float64 (the rows of decode_detections).
 * cols[10] (host): the pred_format columns class, conf, xmin, ymin, xmax, ymax, then the inverter columns ymin, ymax, xmin, xmax
 * (gt_format + 1).  The kept rows are appended in (image, row) order at *count_dev (device counter, not read by the host) to
 * out_image (image_base + b), out_class (the class truncated to int), out_conf and out_box (4 per row), float64; rows past
 * capacity are counted but not written, so that the caller can detect the overflow after the last batch.  One launch, no host
 * synchronisation. */
int ssdk_eval_collect(ssdk_ctx* ctx, const float* rows_dev, int B, int max_out, const int* counts_dev, const double* inv_dev,
                      const int* cols_host, int f64, int pad, int conf_decimals, int image_base, int capacity, int* count_dev, int* out_image_dev,
                      int* out_class_dev, double* out_conf_dev, double* out_box_dev, void* stream);

/* ------------------------------------------------------------------------------------------
 * Decoders.
 *   mode PER_CLASS + layer_semantics=1: DecodeDetections.call   (keras_layers/keras_layer_DecodeDetections.py:109-265)
 *   mode FAST      + layer_semantics=1: DecodeDetectionsFast.call (keras_layers/keras_layer_DecodeDetectionsFast.py:111-248)
 *   mode PER_CLASS + layer_semantics=0: decode_detections        (ssd_encoder_decoder/ssd_output_decoder.py:111-226)
 *   mode FAST      + layer_semantics=0: decode_detections_fast   (ssd_encoder_decoder/ssd_output_decoder.py:228-333)
 * layer_semantics=1: float32 arithmetic, tf.image.non_max_suppression IoU rule, at most nms_max_output
 *   survivors per class, output sorted by confidence (ties: lower row), zero padded to top_k rows.
 * layer_semantics=0: float32 decode stored in float64 like NumPy, float64 IoU with the border_pixels
 *   quirk, no per-class cap, strict '>' (per-class) / '>=' (fast) confidence test; out rows are the
 *   top_k set (order: confidence desc, then class-major NMS order); out_counts gives the valid rows.
 * ------------------------------------------------------------------------------------------ */
typedef enum { SSDK_DECODE_PER_CLASS = 0, SSDK_DECODE_FAST = 1 } ssdk_decode_mode;

typedef struct {
  int mode;                 /* ssdk_decode_mode */
  int layer_semantics;
  int n_classes_total;
  int P;
  double confidence_thresh; /* compared in float32 (layer) or float64 (NumPy API), like the reference */
  double iou_threshold;     /* <= 0 with layer_semantics=0 and mode FAST: skip NMS (reference :326) */
  int top_k;                /* <= 0: 'all' (NumPy API only; out must hold max_out rows) */
  int nms_max_output;       /* layer only */
  int coords;               /* input_coords */
  int normalize_coords;
  int img_height, img_width;
  int border_d;
  int max_out;              /* rows per image in `out`; layer: == top_k */
} ssdk_decode_cfg;

/* y_pred_dev [B*P*(C+12)] float32 -> out_dev [B*max_out*6] float32 rows (class, conf, xmin, ymin, xmax, ymax),
 * out_counts_dev [B] int32 valid rows, out_index_dev (optional) [B*max_out] int32 prior index of each row (-1 pad). */
int ssdk_decode(ssdk_ctx* ctx, const ssdk_decode_cfg* cfg, const float* y_pred_dev, int B,
                float* out_dev, int* out_counts_dev, int* out_index_dev, void* stream);
/* Single-class NMS micro-benchmark entry (SURVEY 8d config 5): boxes [B*n*4] corners, scores [B*n]. */
int ssdk_nms(ssdk_ctx* ctx, const float* boxes_dev, const float* scores_dev, int B, int n,
             double confidence_thresh, double iou_threshold, int nms_max_output, int top_k,
             float* out_dev /* [B*top_k*6] */, int* out_counts_dev, int* out_index_dev, void* stream);

/* ------------------------------------------------------------------------------------------
 * SSD loss.  Replaces SSDLoss.compute_loss (keras_loss_function/keras_ssd_loss.py:98-211).
 * out_loss_dev [B] float32.  bwd writes d(sum_b upstream[b]*loss[b])/d y_pred with the hard-negative
 * mask held constant (upstream_dev NULL = 1/B each, the Keras batch mean).  One cooperative kernel launch per call
 * (csrc/loss.cu): per-box losses, batch-global top-k by a two-level histogram select, masked sums / gradient.
 * ------------------------------------------------------------------------------------------ */
int ssdk_ssd_loss_fwd(ssdk_ctx* ctx, const float* y_true_dev, const float* y_pred_dev, int B, int P, int n_classes_total,
                      int neg_pos_ratio, int n_neg_min, float alpha, float* out_loss_dev,
                      int* out_stats_dev /* optional [4]: n_positive, n_neg_losses, k, ties_taken */, void* stream);
int ssdk_ssd_loss_bwd(ssdk_ctx* ctx, const float* y_true_dev, const float* y_pred_dev, int B, int P, int n_classes_total,
                      int neg_pos_ratio, int n_neg_min, float alpha, const float* upstream_dev,
                      float* out_grad_dev /* [B*P*(C+12)] */, void* stream);
/* Loss and gradient from ONE launch of the same kernel (what a training step needs). */
int ssdk_ssd_loss_fwd_bwd(ssdk_ctx* ctx, const float* y_true_dev, const float* y_pred_dev, int B, int P, int n_classes_total,
                          int neg_pos_ratio, int n_neg_min, float alpha, const float* upstream_dev, float* out_loss_dev,
                          int* out_stats_dev, float* out_grad_dev, void* stream);

/* Multi-GPU, global-batch-exact loss.  The reference's n_positive (:143) and hard-negative top-k (:179-183) run over the
 * WHOLE batch; when the batch is sharded over ranks the kernel's phases are launched one by one on a caller-provided
 * workspace and the integer counts / histograms inside it are summed over the ranks (NCCL all-reduce) in between:
 *   zero the workspace; phase 0; all-reduce(sum) counts + hist1; phase 1; all-reduce(sum) hist2; phase 2; phase 3;
 *   all-gather the int32 at ties_offset (one per rank, rank order = global image order) -> ties_all_dev; phase 4.
 * Phase 4 writes the (B,) losses of this rank's images (normalised by the global n_positive and multiplied by global_B
 * like :204-209) and / or the gradient with respect to this rank's y_pred.  Boxes whose loss equals the k-th largest are
 * taken in global flat-index order, like tf.nn.top_k on the single-process batch. */
typedef struct {
  long long bytes;            /* size of the workspace */
  long long counts_offset;    /* int64[counts_n] */
  long long counts_n;
  long long hist1_offset;     /* int32[hist_n] */
  long long hist2_offset;     /* int32[hist_n] */
  long long hist_n;
  long long ties_offset;      /* int32[1], valid after phase 3 */
} ssdk_loss_ws_layout;
int ssdk_ssd_loss_ws_layout(int B, int P, ssdk_loss_ws_layout* out);
int ssdk_ssd_loss_phase(ssdk_ctx* ctx, int phase, const float* y_true_dev, const float* y_pred_dev, int B, int P,
                        int n_classes_total, int neg_pos_ratio, int n_neg_min, float alpha, void* ws_dev, int global_B,
                        const int* ties_all_dev /* [world], phase 4 */, int rank, const float* upstream_dev,
                        float* out_loss_dev, int* out_stats_dev, float* out_grad_dev, void* stream);

/* Read-only views of the loss kernel, for tests and diagnostics.
 *   ssdk_ssd_loss_plan  the launch a call with these arguments would make (want_grad: bwd / fwd_bwd / phase 4 with a gradient;
 *                       cooperative: the fused entry points, 0 = ssdk_ssd_loss_phase), or the error that call would return.
 *                       stages: shared-memory tile buffers (1 or 2); bulk_ok: tiles are loaded with cp.async.bulk (P*(C+12)
 *                       a multiple of 4 and both inputs 16-byte aligned), else by plain loads.  Launches nothing and changes
 *                       no state of the context (workspace, histogram parity).  Like a call of the same size, it may raise
 *                       the kernels' process-wide cudaFuncAttributeMaxDynamicSharedMemorySize, which the occupancy query
 *                       behind `grid` needs; that attribute only ever grows and changes no result.
 *   ssdk_ssd_loss_read_box_losses  the per-box losses the last call's first phase stored, [B*P] float32 each: cls (the
 *                       log-loss of the box, :93-95) and negl = cls * y_true[..., 0] (:151), the values the hard-negative
 *                       selection ranks.  ws_dev NULL reads the context's own workspace (an error unless its last fused call
 *                       had this (B, P)); otherwise a phase workspace (ssdk_ssd_loss_phase) after its phase 0.  Either output
 *                       may be NULL. */
typedef struct {
  int stages;
  int bulk_ok;
  int grid;
  long long smem_bytes;       /* dynamic shared memory per CTA */
} ssdk_loss_plan;
int ssdk_ssd_loss_plan(ssdk_ctx* ctx, const float* y_true_dev, const float* y_pred_dev, int B, int P, int n_classes_total,
                       int want_grad, int cooperative, ssdk_loss_plan* out);
int ssdk_ssd_loss_read_box_losses(ssdk_ctx* ctx, const void* ws_dev, int B, int P, float* cls_dev, float* negl_dev, void* stream);

/* ------------------------------------------------------------------------------------------
 * Model graph.  Replaces ssd_300 (models/keras_ssd300.py:31-457), ssd_512 (models/keras_ssd512.py:31-477)
 * and build_model (models/keras_ssd7.py:30-430) + L2Normalization
 * (keras_layers/keras_layer_L2Normalization.py:61-63): a static plan of wgmma implicit-GEMM
 * convolutions, pooling, normalisation and the head epilogue producing (B,P,C+12).
 * The graph is described layer by layer by the host (Python mirrors the reference builders).
 * ------------------------------------------------------------------------------------------ */
typedef enum {
  SSDK_OP_INPUT = 0,      /* preprocessing: (x - mean)/std, channel swap; source = user images (B,H,W,3) f32 */
  SSDK_OP_CONV = 1,       /* conv + bias + activation */
  SSDK_OP_MAXPOOL = 2,
  SSDK_OP_L2NORM = 3,     /* x * rsqrt(max(sum_c x^2, 1e-12)) * gamma_c */
  SSDK_OP_HEAD = 4,       /* fused conf+loc 3x3 predictor conv for one source layer -> rows of y_pred */
  SSDK_OP_TENSOR = 5      /* source = a user tensor (B,H,W,C) f32 with any channel count, taken as it is (ssdk_conv2d_fwd / ssdk_maxpool) */
} ssdk_op;

typedef enum { SSDK_ACT_NONE = 0, SSDK_ACT_RELU = 1, SSDK_ACT_ELU = 2 } ssdk_act;

typedef struct {
  int op;                   /* ssdk_op */
  int input;                /* index of the producing layer (-1 for SSDK_OP_INPUT) */
  int cout;                 /* conv/head: output channels (head: n_boxes*(C+4) is derived; give n_boxes) */
  int kh, kw, stride, dilation;
  int pad_t, pad_l, pad_b, pad_r;   /* zero padding (conv) / -inf padding (pool) */
  int act;                  /* ssdk_act */
  int n_boxes;              /* head only */
  /* Parameters, host pointers, copied at build time.  conv: kernel HWIO float32 [kh*kw*cin*cout], bias [cout];
   * optional folded batch-norm scale/shift per output channel (applied after bias, before act);
   * l2norm: gamma [c]; head: conf kernel/bias and loc kernel/bias; input: mean[3]/std[3]/swap[3]. */
  const float* kernel; const float* bias;
  const float* bn_scale; const float* bn_shift;
  const float* kernel2; const float* bias2;      /* head: loc kernel/bias (kernel/bias = conf) */
  const float* mean; const float* stddev; const int* swap;
  /* conv followed by BatchNormalization (models/keras_ssd7.py:277-309), raw parameters [cout] each.  Training plans
   * (ssdk_model_desc.training = 1) run the layer in Keras' training phase: batch statistics over (B,H,W), moving averages
   * updated with `bn_momentum`; inference plans use the folded bn_scale / bn_shift above. */
  const float* bn_gamma; const float* bn_beta; const float* bn_mean; const float* bn_var;
  float bn_eps; float bn_momentum;
} ssdk_layer_desc;

typedef struct {
  int batch;                /* plan is built for this batch size */
  int img_height, img_width, img_channels;
  int n_classes_total;
  int n_layers;
  const ssdk_layer_desc* layers;
  int precision;            /* 0 = bf16x3 split (fp32-faithful, default), 1 = single-pass bf16 */
  const float* anchors_f32; /* host [P*4] */
  float variances[4];
  int training;             /* 1: size the activation borders for the backward pass too (needed by ssdk_trainer_create) */
} ssdk_model_desc;

/* Stand-alone L2Normalization.call (keras_layers/keras_layer_L2Normalization.py:61-63) on a float32 tensor viewed as
 * [rows, C] (rows = B*H*W, channels last): out = x * rsqrt(max(sum_c x^2, 1e-12)) * gamma_c. */
int ssdk_l2_normalize(ssdk_ctx* ctx, const float* x_dev, long long rows, int C, const float* gamma_dev, float* out_dev, void* stream);

/* Stand-alone Conv2D forward (what every `Conv2D(...)` of models/keras_ssd300.py:274-335 computes; SURVEY 8b `ssdk_conv2d_fwd`):
 * y = act(conv(x, kernel) + bias) on float32 NHWC device tensors, kernel HWIO / bias on the HOST (copied and packed by the call).
 * x (B,H,W,Cin) -> y (B,Ho,Wo,Cout), Ho = (H + pad_t + pad_b - dilation*(kh-1) - 1)/stride + 1.  Runs the same wgmma plan the
 * model graphs use (precision 0 = bf16x3, 1 = bf16) as a one-layer graph built and destroyed inside the call: it synchronises
 * the stream and allocates -- a utility for tests and interop; steady-state users describe their layers to ssdk_model_create. */
int ssdk_conv2d_fwd(ssdk_ctx* ctx, const float* x_dev, int B, int H, int W, int Cin, const float* kernel_hwio_host,
                    const float* bias_host /* or NULL */, int Cout, int kh, int kw, int stride, int dilation,
                    int pad_t, int pad_l, int pad_b, int pad_r, int act /* ssdk_act */, int precision, float* y_dev, void* stream);
/* Stand-alone MaxPooling2D forward (models/keras_ssd300.py:276-309; -inf padding, i.e. TensorFlow 'same' when the caller passes
 * the 'same' pads): x (B,H,W,C) -> y (B,Ho,Wo,C), Ho = (H + pad_t + pad_b - kh)/stride + 1.  Same caveats as ssdk_conv2d_fwd. */
int ssdk_maxpool(ssdk_ctx* ctx, const float* x_dev, int B, int H, int W, int C, int kh, int kw, int stride,
                 int pad_t, int pad_l, int pad_b, int pad_r, float* y_dev, void* stream);

/* The two-stream schedule ssdk_model_create gives an inference plan (DESIGN.md 3.5), as a host-only function on plain arrays (no
 * device needed): kind[i] 0 = not a tensor-core GEMM launch (pool, L2Norm, input), 1 = trunk convolution, 2 = predictor head;
 * grid[i] = CTAs of that launch; input[i] = producing layer or -1; R <= 0 selects the default (sm_count / 3 + 1).
 * out_on_side[i] = 1: issued on the second stream; *out_from = first such layer (-1: single stream); *out_grid_cap = grid limit of
 * the GEMM launches that stay on the caller's stream meanwhile.  The reference has no counterpart (Keras/TF schedule their graph). */
int ssdk_schedule_preview(int n_layers, const int* kind, const int* grid, const int* input, int R, int sm_count,
                          unsigned char* out_on_side, int* out_from, int* out_grid_cap);

int ssdk_model_create(ssdk_ctx* ctx, const ssdk_model_desc* desc, ssdk_model** out);
int ssdk_model_destroy(ssdk_model* m);
int ssdk_model_num_priors(const ssdk_model* m, int* out_P);
/* Spatial size / channels of a layer's output (reference: model.get_layer(name).output_shape[1:3]). */
int ssdk_model_layer_shape(const ssdk_model* m, int layer, int* out_h, int* out_w, int* out_c);
/* images_dev (B,H,W,3) float32 NHWC -> y_pred_dev (B,P,C+12) float32. */
int ssdk_model_forward(ssdk_model* m, const float* images_dev, float* y_pred_dev, void* stream);
/* Copy a layer's activation (B,h,w,c) as float32 NHWC to out_dev (tests: per-layer parity). */
int ssdk_model_read_layer(ssdk_model* m, int layer, float* out_dev, void* stream);
/* The raw bf16 activation planes of a layer (what the next launches read, value = hi + lo), borders and padding channels
 * included: geometry (padded rows Hp, row pitch Wp, stored channels Cs, border pad; a plane holds B*Hp*Wp*Cs values), and a
 * copy of hi and lo (lo_dev may be NULL; single-pass bf16 plans have no lo plane).  Heads have no planes. */
int ssdk_model_layer_planes_shape(const ssdk_model* m, int layer, int* out_hp, int* out_wp, int* out_cs, int* out_pad);
int ssdk_model_read_layer_planes(ssdk_model* m, int layer, uint16_t* hi_dev, uint16_t* lo_dev, void* stream);
/* FLOPs of one forward pass (2*MACs of every conv, SURVEY 8d) and MMA flops actually issued. */
int ssdk_model_flops(const ssdk_model* m, double* out_algorithmic, double* out_issued);
/* Time of the conv kernels of the last forward in ms (CUDA events on `stream`), when enabled. */
int ssdk_model_set_timing(ssdk_model* m, int enable);
int ssdk_model_last_conv_ms(ssdk_model* m, float* out_ms);
/* Time in ms of one layer's convolution launch in the last timed forward (0 for layers without a conv_wgmma_kernel launch). */
int ssdk_model_layer_ms(const ssdk_model* m, int layer, float* out_ms);

/* Read-only view of the launch plan ssdk_model_create chose for one convolution or head (host only, no device work), so that a
 * test can pin the kernel variant it exercises.  Non-convolution layers report kernel = SSDK_PLAN_NONE and zeros. */
enum ssdk_plan_kernel {
  SSDK_PLAN_NONE = 0,
  SSDK_PLAN_GEMM = 1,          /* conv_wgmma_kernel on the zero-bordered activation (implicit GEMM) */
  SSDK_PLAN_IM2COL_GEMM = 2,   /* im2col_kernel / im2col8_kernel, then conv_wgmma_kernel on the column matrix */
  SSDK_PLAN_FIRST_TC = 3,      /* conv_first_kernel: image-facing layer, gathered A tile, tensor cores */
  SSDK_PLAN_DIRECT = 4         /* conv_direct_kernel: fp32 FMAs on the float32 master kernel */
};
enum ssdk_plan_epilogue { SSDK_PLAN_EPI_SPLIT = 0, SSDK_PLAN_EPI_F32 = 1, SSDK_PLAN_EPI_ATOMIC = 2, SSDK_PLAN_EPI_HEAD = 3 };
typedef struct ssdk_layer_plan {
  int kernel;                  /* ssdk_plan_kernel */
  int bn;                      /* wgmma N of the tile (GEMM / FIRST_TC) */
  int split;                   /* 1: bf16x3 (hi*hi + hi*lo + lo*hi), 0: one bf16 product */
  int stages;                  /* TMA ring depth (GEMM) */
  int kblocks;                 /* 64-wide K blocks per tap (GEMM: of the input channels or of the im2col row; FIRST_TC: of taps*4) */
  int n_tiles_m, n_tiles_n;    /* scheduled 128-row m-tiles and BN-wide n-tiles */
  int grid;                    /* CTAs of the (persistent) launch */
  int k_split;                 /* work units per tile along K */
  int epilogue;                /* ssdk_plan_epilogue, of GEMM launches */
  int head_fused;              /* 1: softmax / anchors / variances in the GEMM epilogue, straight into y_pred */
  int im2col_vec8;             /* IM2COL_GEMM: 1 = im2col8_kernel (8 channels per thread), 0 = im2col_kernel */
} ssdk_layer_plan;
int ssdk_model_layer_plan(const ssdk_model* m, int layer, ssdk_layer_plan* out);

/* ------------------------------------------------------------------------------------------
 * Training step (BASELINE config 3).  Replaces what Keras/TensorFlow do for the reference in model.fit_generator:
 * autodiff of the graph (models/keras_ssd300.py:263-419) and of SSDLoss (keras_ssd_loss.py:98-211), the kernel_regularizer
 * l2(l2_reg) (models/keras_ssd300.py:274), SGD(lr, momentum) (ssd300_training.ipynb:169) and Adam (ssd7_training.ipynb:153).
 *   ssdk_train_backward  after ssdk_model_forward on the same images: loss + gradients of every kernel / bias / gamma into one
 *                        flat float32 buffer (so that a single NCCL all-reduce covers it).
 *   ssdk_train_apply     g = grad*grad_scale + 2*l2*w (kernels only); v = momentum*v - lr*g; w += v; re-pack the bf16 planes.
 * Parameter order in the flat buffer: layers in graph order, for each conv [kernel as (cout, kh, kw, cin) | bias | BatchNorm
 * gamma | BatchNorm beta], for each head [fused kernel (n_boxes*(C+4), 3, 3, cin) | fused bias], for L2Normalization [gamma].
 * ReLU / linear graphs (SSD300 / SSD512) and conv + BatchNormalization + ELU graphs (SSD7).
 * ------------------------------------------------------------------------------------------ */
typedef struct ssdk_trainer ssdk_trainer;
int ssdk_trainer_create(ssdk_model* m, float* flat_grad_dev /* optional, else allocated */, ssdk_trainer** out);
int ssdk_trainer_destroy(ssdk_trainer* t);
int ssdk_trainer_num_params(const ssdk_trainer* t, long long* out_n);
/* offset (in floats) and element count of a layer's kernel (which=0), bias (1), L2Normalization gamma (2), BatchNormalization
 * gamma (3) or beta (4) inside the flat buffers */
int ssdk_trainer_param_span(const ssdk_trainer* t, int layer, int which, long long* out_offset, long long* out_count);
float* ssdk_trainer_grad_buffer(ssdk_trainer* t);
/* Read-only views of a layer's output gradient (the planes the backward pass writes and the next launches read).
 *   ssdk_trainer_grad_shape        stored geometry of the planes: padded rows Hp, padded row pitch Wp, stored channels Cs
 *                                  (multiple of 8), zero border pad; a plane holds B*Hp*Wp*Cs bf16 values.
 *   ssdk_trainer_read_grad         hi + lo as float32 NHWC (B,H,W,C) into out_dev.
 *   ssdk_trainer_read_grad_planes  the raw bf16 planes, borders and padding channels included; lo_dev may be NULL and is left
 *                                  untouched by a single-pass bf16 trainer, which has no lo plane. */
int ssdk_trainer_grad_shape(const ssdk_trainer* t, int layer, int* out_hp, int* out_wp, int* out_cs, int* out_pad);
int ssdk_trainer_read_grad(ssdk_trainer* t, int layer, float* out_dev, void* stream);
int ssdk_trainer_read_grad_planes(ssdk_trainer* t, int layer, uint16_t* hi_dev, uint16_t* lo_dev, void* stream);
int ssdk_train_backward(ssdk_trainer* t, const float* y_true_dev, const float* y_pred_dev, int neg_pos_ratio, int n_neg_min,
                        float alpha, float* out_loss_dev /* [B] */, void* stream);
/* The step in pieces, for overlapping the gradient exchange with the backward pass:
 *   ssdk_train_backward_begin   loss + d loss / d y_pred (kept inside the trainer), gradient buffer cleared;
 *   ssdk_train_backward_layers  layers hi .. lo (graph indices, top down, consecutive calls cover n_layers-1 .. 0).  In stream
 *                               order after the call the parameter gradients of exactly these layers are final, so their
 *                               span of the flat buffer (ssdk_trainer_param_span) can be all-reduced on another stream while the
 *                               lower layers are still being differentiated.  dypred_dev NULL = the trainer's own. */
int ssdk_train_backward_begin(ssdk_trainer* t, const float* y_true_dev, const float* y_pred_dev, int neg_pos_ratio, int n_neg_min,
                              float alpha, float* out_loss_dev, void* stream);
int ssdk_train_backward_layers(ssdk_trainer* t, const float* dypred_dev, int hi, int lo, void* stream);
/* The same backward pass from a gradient the caller computed: dypred_dev = d loss / d y_pred, (B,P,C+12) float32 (used with the
 * multi-GPU global-batch-exact loss, whose phases run between NCCL collectives, see ssdk_ssd_loss_phase). */
int ssdk_train_backward_dy(ssdk_trainer* t, const float* dypred_dev, void* stream);
int ssdk_train_apply(ssdk_trainer* t, float lr, float momentum, float l2_reg, float grad_scale, void* stream);
/* Adam as Keras applies it (ssd7_training.ipynb:153: Adam(lr=0.001, beta_1=0.9, beta_2=0.999, epsilon=1e-08, decay=0.0)):
 * g = grad*grad_scale + 2*l2*w (kernels); lr_t = lr*sqrt(1-beta2^t)/(1-beta1^t); m = b1*m + (1-b1)*g; v = b2*v + (1-b2)*g^2;
 * w -= lr_t*m/(sqrt(v)+eps).  `step` = t, counted from 1 by the caller. */
int ssdk_train_apply_adam(ssdk_trainer* t, float lr, float beta1, float beta2, float eps, float l2_reg, float grad_scale, int step,
                          void* stream);
/* Moving mean / variance of a BatchNormalization layer as the training passes left them (float32 [cout] each). */
int ssdk_trainer_read_bn_stats(ssdk_trainer* t, int layer, float* mean_dev, float* var_dev, void* stream);
/* The raw convolution output z (B,h,w,c) a BatchNormalization layer normalised in the last forward pass, hi + lo as float32
 * NHWC (read-only; what the BatchNormalization backward reads). */
int ssdk_trainer_read_bn_input(ssdk_trainer* t, int layer, float* out_dev, void* stream);
/* Copy the current float32 master parameters (same order / layout as the gradients) to out_dev. */
int ssdk_trainer_read_params(ssdk_trainer* t, float* out_dev, void* stream);
/* Copy one slot of the optimiser state (same order / layout as the gradients, kernels OHWI) to out_dev (read-only):
 * slot 0 = the SGD velocity or the Adam first moment m, slot 1 = the Adam second moment v (an error before the first Adam
 * update, and for any other slot). */
int ssdk_trainer_read_opt_state(ssdk_trainer* t, int slot, float* out_dev, void* stream);

/* Read-only view of the backward launches ssdk_trainer_create planned for one convolution or head (host only). */
enum ssdk_dgrad_path { SSDK_DGRAD_NONE = 0, SSDK_DGRAD_GEMM = 1 /* implicit GEMM into the producer's gradient planes */,
                       SSDK_DGRAD_STRIDED = 2 /* GEMM to an fp32 column matrix, then col2im */ };
enum ssdk_wgrad_path { SSDK_WGRAD_NONE = 0, SSDK_WGRAD_NATIVE = 1 /* wgrad_wgmma_kernel on dZ / X in place */,
                       SSDK_WGRAD_TRANSPOSED = 2 /* one GEMM per tap on transposed copies of dZ / X */,
                       SSDK_WGRAD_IM2COL = 3 /* one GEMM on transposed copies of dZ and the im2col matrix */,
                       SSDK_WGRAD_DIRECT = 4 /* fp32 image-facing weight-gradient kernel */ };
typedef struct ssdk_backward_plan {
  int dgrad;                   /* ssdk_dgrad_path */
  int dgrad_bn;                /* wgmma N of the data-gradient GEMM */
  int dgrad_mask;              /* 1: ReLU'(producer output) applied in the epilogue */
  int dgrad_accumulate;        /* 1: added to a gradient another consumer of the producer already wrote */
  int dgrad_n_tiles_m, dgrad_n_tiles_n, dgrad_grid;
  int wgrad;                   /* ssdk_wgrad_path */
  int wgrad_bn;                /* NATIVE: input channels per tile (BNc); TRANSPOSED / IM2COL: GEMM tile width */
  int a_boxes;                 /* NATIVE: 64-row output-channel boxes per tile */
  int bw, bh;                  /* NATIVE: pixel patch of one K block (bw * bh = 64) */
  int co_tiles, ci_tiles;      /* NATIVE: output- / input-channel tiles */
  int k_split;                 /* work units per tile along the pixel axis */
  int n_gemms;                 /* TRANSPOSED / IM2COL: GEMM launches */
  int stages, grid;
  int kv;                      /* TRANSPOSED / IM2COL: pixels on the GEMM's K axis (the padded grid); NATIVE: 64-pixel patches */
  int direct_fast;             /* DIRECT: 1 = wgrad_direct3x3_kernel (3x3x3 fast path), 0 = wgrad_direct_kernel */
} ssdk_backward_plan;
int ssdk_trainer_layer_plan(const ssdk_trainer* t, int layer, ssdk_backward_plan* out);

#ifdef __cplusplus
}
#endif
#endif /* SSDK_H_ */
