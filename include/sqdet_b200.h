/*
 * sqdet_b200.h — C ABI of libsqdet_b200.so: the H100 (sm_90a) SqueezeDet
 * inference hot path (conv backbone -> ConvDet -> interpret_output ->
 * filter_prediction / NMS).
 *
 * The reference (BichenWuUCB/squeezeDet) has no FFI of its own: its boundary is
 * the Python object contract of `ModelSkeleton` driven through `sess.run`.  Each
 * entry point below therefore cites the reference *Python* interface it stands
 * in for (paths relative to the reference tree); the binding a maintainer would
 * add on the reference side is a ctypes stub, shown in INTEGRATION.md.
 *
 * Conventions
 *   - every function returns an int status: 0 = SQDET_OK, negative = error;
 *     sqdet_last_error() gives the message of the calling thread's last failure.
 *     Nothing throws across this boundary.
 *   - plain pointers and sizes only; `stream` is a cudaStream_t passed as void*
 *     (NULL = the legacy default stream).
 *   - "_dev" pointers are device memory on the engine's device, everything else
 *     is host memory.  The caller owns every pointer it passes; the engine owns
 *     its weights, activations and result buffers.
 *   - an engine is bound to one device and is NOT thread-safe (one engine per
 *     host thread / stream).  All launches go to the caller's stream; no hidden
 *     host synchronisation except in the functions documented as synchronous.
 *   - layouts are the reference's: activations NHWC fp32, kernels HWIO fp32,
 *     boxes (cx, cy, w, h) fp32, class ids int64.
 */
#ifndef SQDET_B200_H_
#define SQDET_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SQDET_OK                 0
#define SQDET_ERR_INVALID_ARG   (-1)
#define SQDET_ERR_CUDA          (-2)
#define SQDET_ERR_UNSUPPORTED   (-3)
#define SQDET_ERR_STATE         (-4)   /* call order (e.g. forward before finalize) */
#define SQDET_ERR_NOT_FOUND     (-5)
#define SQDET_ERR_OVERFLOW      (-6)   /* threshold branch produced more boxes than capacity */

#define SQDET_PAD_SAME   0
#define SQDET_PAD_VALID  1

/* math_mode of the convolution kernels */
#define SQDET_MATH_FP32_SIMT   0   /* fp32 FFMA direct/implicit-GEMM kernels            */
#define SQDET_MATH_TF32X3_TC   1   /* wgmma tensor cores, 3xTF32 split (fp32-grade)      */

typedef struct sqdet_engine sqdet_engine;   /* opaque */

/* One filtered detection (28 bytes) — the element type of the N-GPU all-gather. */
typedef struct sqdet_det {
  int32_t anchor;   /* index into the image's [A] anchors ("kept-box index")           */
  int32_t cls;      /* class id                                                         */
  float   prob;     /* det_probs[anchor]                                                */
  float   cx, cy, w, h;
} sqdet_det;

/* The inference-relevant keys of the reference's `mc` EasyDict
 * (src/config/config.py:10-142, src/config/kitti_squeezeDet_config.py:9-43). */
typedef struct sqdet_config {
  int32_t batch_size;        /* mc.BATCH_SIZE   (static batch dim, nn_skeleton.py:81-84) */
  int32_t image_height;      /* mc.IMAGE_HEIGHT */
  int32_t image_width;       /* mc.IMAGE_WIDTH  */
  int32_t classes;           /* mc.CLASSES      */
  int32_t anchors_per_grid;  /* mc.ANCHOR_PER_GRID */
  int32_t top_n_detection;   /* mc.TOP_N_DETECTION */
  float   prob_thresh;       /* mc.PROB_THRESH  */
  float   nms_thresh;        /* mc.NMS_THRESH   */
  float   exp_thresh;        /* mc.EXP_THRESH   */
  float   batch_norm_epsilon;/* mc.BATCH_NORM_EPSILON */
  int32_t math_mode;         /* SQDET_MATH_*    */
  int32_t max_dets;          /* per-image record capacity; 0 = derive (top_n, else 1024) */
} sqdet_config;

/* ---- library ---------------------------------------------------------------------- */
const char* sqdet_last_error(void);
const char* sqdet_version(void);
/* Number of CUDA devices visible (0 without a GPU/driver); never fails. */
int sqdet_device_count(void);

/* ---- engine life cycle: replaces `Net(mc, gpu_id)` ---------------------------------
 * ModelSkeleton.__init__ (src/nn_skeleton.py:74-135) + the nets' constructors
 * (src/nets/squeezeDet.py:19-28).  `device` is the reference's `gpu_id`. */
int sqdet_create(const sqdet_config* cfg, int device, sqdet_engine** out);
int sqdet_destroy(sqdet_engine* e);

/* ---- graph construction: one call per reference layer constructor ------------------
 * Tensor ids: 0 is `image_input` [B,H,W,3]; every add_* returns a new id in *out.   */
/* ModelSkeleton._conv_layer (src/nn_skeleton.py:471-563): relu?(conv2d + bias).      */
int sqdet_add_conv(sqdet_engine* e, const char* layer_name, int src, int filters,
                   int size, int stride, int padding, int relu, int* out);
/* ModelSkeleton._conv_bn_layer (src/nn_skeleton.py:374-468): SAME conv [+bias] + frozen BN. */
int sqdet_add_conv_bn(sqdet_engine* e, const char* scope_name, int src, int filters,
                      int size, int stride, int relu, int conv_with_bias, int* out);
/* ModelSkeleton._pooling_layer (src/nn_skeleton.py:565-586): tf.nn.max_pool.          */
int sqdet_add_pool(sqdet_engine* e, const char* layer_name, int src, int size,
                   int stride, int padding, int* out);
/* SqueezeDet._fire_layer (src/nets/squeezeDet.py:81-106).                             */
int sqdet_add_fire(sqdet_engine* e, const char* layer_name, int src, int s1x1,
                   int e1x1, int e3x3, int* out);
/* tf.nn.relu(a + b) of the ResNet shortcuts (src/nets/resnet50_convDet.py:55).        */
int sqdet_add_add_relu(sqdet_engine* e, const char* name, int a, int b, int* out);
/* ModelSkeleton._add_interpretation_graph (src/nn_skeleton.py:142-283): declares
 * `preds` and mc.ANCHOR_BOX ([A,4] float64, as the reference stores it).              */
int sqdet_set_preds(sqdet_engine* e, int preds, const double* anchor_box, int64_t num_anchors);
/* Allocate activations / results, upload + pre-process parameters.  After this the
 * graph is frozen.  Parameters not yet set are zero.                                  */
int sqdet_finalize(sqdet_engine* e);

/* ---- parameters: replaces tf.train.Saver(model.model_params).restore ---------------
 * (src/demo.py:181-184, src/eval.py:205).  Names are the reference's TF variable
 * names: "<layer>/kernels" [kh,kw,Cin,Cout], "<layer>/biases" [Cout], BN
 * "<scope>/gamma|beta|mean|var" [Cout].  Callable before or after finalize.  A change
 * takes effect at the next forward, which first waits for the engine's forwards already
 * in flight.                                                                          */
int sqdet_num_params(sqdet_engine* e);
int sqdet_param_info(sqdet_engine* e, int index, char* name_buf, int name_cap,
                     int64_t shape[4], int* ndim);
int sqdet_set_param(sqdet_engine* e, const char* name, const float* data,
                    const int64_t* shape, int ndim);

/* ---- introspection (model_size_counter / flop_counter / activation_counter,
 * src/nn_skeleton.py:549-561) -------------------------------------------------------- */
int sqdet_num_tensors(sqdet_engine* e);
int sqdet_tensor_info(sqdet_engine* e, int id, char* name_buf, int name_cap,
                      int64_t shape[4]);
int sqdet_read_tensor(sqdet_engine* e, int id, float* host_out);   /* synchronous */
int sqdet_num_ops(sqdet_engine* e);
int sqdet_op_info(sqdet_engine* e, int index, char* name_buf, int name_cap,
                  int64_t* flops, int64_t* params, int64_t* min_bytes);
/* The K split S the plan chose for op `index` (a ConvDet head whose K is summed by a cluster of S
 * CTAs, see sqdet_conv2d_k_split), 1 for every other op; negative on error.  Fixed at
 * sqdet_finalize for BATCH_SIZE images, so every sqdet_forward_n runs the same partition.     */
int sqdet_op_k_split(sqdet_engine* e, int index);

/* ---- execution: replaces sess.run([det_boxes, det_probs, det_class], feed_dict) ----
 * (src/demo.py:193-195, src/eval.py:75-77) and model.filter_prediction on every image
 * (src/demo.py:198-199, src/eval.py:86-87).                                           */
/* Asynchronous on `stream`: backbone + ConvDet + interpret_output + filter for the
 * whole batch.  images_dev [B,H,W,3] fp32 (BGR, mean-subtracted).                     */
int sqdet_forward(sqdet_engine* e, const float* images_dev, void* stream);
/* Partial batch: an engine built for B images runs any n with 1 <= n <= B and processes images
 * [0, n) only.  images_dev then needs to hold just those n images [n,H,W,3]; nothing at or past
 * image n is read.
 *   - Same kernels as the full batch: the plan sqdet_finalize made for B (kernel per layer,
 *     output-channel tile, one-kernel fire or not) runs unchanged; only the grids shrink.  So
 *     image i of an n-image forward is bitwise identical to image i of a full forward whose
 *     first n images are the same.
 *   - No activation row, det_boxes / det_probs / det_class row or record row at or past n is
 *     written: sqdet_read_tensor and sqdet_results_dev still return B rows, and rows [n, B)
 *     hold what the last forward that covered them left there.  counts[n, B) are set to 0 on the
 *     device (inside the forward's CUDA graph), so the all-gather blob stays fully defined.
 *   - sqdet_read_tensor, sqdet_op_info and sqdet_launches_per_forward keep their B-sized meaning.
 *   - SQDET_ERR_INVALID_ARG when n < 1 or n > B.
 * sqdet_forward is sqdet_forward_n with n = B.                                              */
int sqdet_forward_n(sqdet_engine* e, const float* images_dev, int n, void* stream);
/* images_dev: n uint8 BGR images [n,H,W,3] as cv2.imread / cv2.resize leave them (any byte
 * alignment); the engine subtracts mc.BGR_MEANS (src/demo.py:190).  Otherwise sqdet_forward_n:
 * asynchronous on `stream`, graph-captured, the same partial-batch rules, box-scale table and
 * in-forward all-gather, and the same results as sqdet_forward_n on
 * float32(float64(images) - BGR_MEANS), bit for bit.  The plan picks one of two paths:
 *   - when a fused conv+pool first layer is the only reader of the image tensor, that kernel reads
 *     the bytes itself and tensor 0 is not written (sqdet_read_tensor(0) keeps what it held);
 *   - otherwise (a first conv without a pool, VGG16's tensor-core conv1_1, an image read by two
 *     ops) one extra launch converts the n images into tensor 0, which sqdet_read_tensor(0) then
 *     returns, and the forward issues one launch more than sqdet_launches_per_forward counts.
 * A sqdet_set_bgr_means call takes effect at the next sqdet_forward_u8.
 * SQDET_ERR_INVALID_ARG / SQDET_ERR_STATE before any device work as for sqdet_forward_n.     */
int sqdet_forward_u8(sqdet_engine* e, const uint8_t* images_dev, int n, void* stream);
/* sqdet_forward, but records a CUDA event around every op (not graph-captured) and returns
 * per-op milliseconds (synchronous).  op_ms has sqdet_num_ops() entries.              */
int sqdet_forward_profiled(sqdet_engine* e, const float* images_dev, void* stream,
                           float* op_ms);
/* Device result buffers of the last forward (valid until the next one):
 * det_boxes [B,A,4] f32, det_probs [B,A] f32, det_class [B,A] i64,
 * dets [B,max_dets] records, counts [B] i32.                                          */
int sqdet_results_dev(sqdet_engine* e, float** det_boxes, float** det_probs,
                      int64_t** det_class, sqdet_det** dets, int32_t** counts,
                      int32_t* max_dets);
/* Synchronous host-buffer call (the end-to-end path): H2D of images, forward, D2H of
 * whichever outputs are non-NULL.  Host buffers should be pinned for full speed.      */
int sqdet_detect(sqdet_engine* e, const float* images, float* det_boxes,
                 float* det_probs, int64_t* det_class, sqdet_det* dets,
                 int32_t* counts, void* stream);
/* Pipelined host-buffer path (depth 2): sqdet_submit enqueues H2D (own copy stream) ->
 * forward -> D2H of the filtered records and returns at once; sqdet_wait blocks until the
 * OLDEST outstanding submit has delivered into its dets/counts buffers.  With two submits in
 * flight the copy of batch i+1 overlaps the compute of batch i.  img_type SQDET_IMG_F32:
 * [B,H,W,3] fp32 BGR, mean-subtracted (feed_dict semantics, src/demo.py:190-195), uploaded into
 * a buffer of the submission's own, not tensor 0; SQDET_IMG_U8: [B,H,W,3] uint8 BGR exactly as
 * cv2.imread / cv2.resize leave it (src/demo.py:187-189), uploaded as bytes and run by the
 * forward of sqdet_forward_u8, under its rules: the engine applies `im - mc.BGR_MEANS`
 * (src/demo.py:190, src/dataset/imdb.py:88) in the fused first layer, leaving tensor 0 as it
 * was, or in one launch that converts the batch into tensor 0.  Host buffers must stay valid
 * (and should be pinned) until the matching sqdet_wait.  SQDET_ERR_STATE if two submits are
 * already pending.                                                                           */
#define SQDET_IMG_F32 0
#define SQDET_IMG_U8  1
int sqdet_set_bgr_means(sqdet_engine* e, const double bgr_means[3]);   /* mc.BGR_MEANS */
int sqdet_submit(sqdet_engine* e, const void* images, int img_type, sqdet_det* dets,
                 int32_t* counts);
int sqdet_wait(sqdet_engine* e);
/* Variable-size frames in front of the path (SURVEY 8 f-1): B uint8 BGR frames exactly as
 * cv2.imread returns them, frame i = [heights[i], widths[i], 3].  The engine does
 * astype(float32) + cv2.resize(..., (mc.IMAGE_WIDTH, mc.IMAGE_HEIGHT)) (float32 INTER_LINEAR) +
 * `- mc.BGR_MEANS` in the reference order `order` (SQDET_PRE_RESIZE_THEN_SUB: src/demo.py:187-190;
 * SQDET_PRE_SUB_THEN_RESIZE: src/dataset/imdb.py:85-97) on the GPU, then the forward; same
 * depth-2 pipelining and sqdet_wait contract as sqdet_submit.  rescale != 0 additionally divides
 * every det box by (x_scale, y_scale) = (IMAGE_WIDTH / widths[i], IMAGE_HEIGHT / heights[i])
 * BEFORE filter_prediction, i.e. the order of src/eval.py:80-87.  `rescale` applies to this one
 * submission only; the table of sqdet_set_box_scale is never applied here.                  */
int sqdet_submit_frames(sqdet_engine* e, const uint8_t* const* frames,
                        const int32_t* heights, const int32_t* widths, int order,
                        int rescale, sqdet_det* dets, int32_t* counts);
/* sqdet_submit_frames over n frames, 1 <= n <= B, with the partial-batch semantics of
 * sqdet_forward_n: frames/heights/widths have n entries, and n rows of records (dets
 * [n,max_dets]) and n counts are copied back.  Same sqdet_wait contract; submits with different
 * n may be in flight together.  SQDET_ERR_INVALID_ARG when n < 1 or n > B.
 * sqdet_submit_frames is sqdet_submit_frames_n with n = B.                                   */
int sqdet_submit_frames_n(sqdet_engine* e, int n, const uint8_t* const* frames,
                          const int32_t* heights, const int32_t* widths, int order,
                          int rescale, sqdet_det* dets, int32_t* counts);
/* n uint8 BGR frames already in device memory on the engine's device (a hardware decoder's
 * output, torch CUDA tensors, crops of larger frames): frame i is heights[i] rows of widths[i]*3
 * bytes, row r at frames_dev[i] + r*row_pitches[i] (NULL row_pitches = 3*widths[i]; any byte
 * alignment).  Host arrays of n entries, 1 <= n <= B.  Resize + `- mc.BGR_MEANS` in `order` as
 * sqdet_submit_frames_n, bit for bit, into tensor 0, then the forward of sqdet_forward_n on
 * `stream`; rescale != 0 divides det boxes by each frame's scales before the filter (this call
 * only; the sqdet_set_box_scale table is not applied).  Asynchronous; no host synchronisation.
 *   - Afterwards rows [0, n) of tensor 0 (sqdet_read_tensor(0)) hold the resized fp32 images.
 *   - Launches: sqdet_launches_per_forward (without a box-scale table), plus one resize launch
 *     per 64 frames (so one for every n <= B <= 64), plus the rescale launch when rescale != 0.
 *   - Refused before any device work, leaving graphs, pipeline and tensor 0 untouched:
 *     SQDET_ERR_INVALID_ARG for a null engine or array, n outside [1, B], an unknown order, a
 *     null frame, heights[i] or widths[i] <= 0, row_pitches[i] < 3*widths[i], or a frame whose
 *     bytes [p, p + (h-1)*pitch + 3*w) are not device memory of the engine's device inside one
 *     allocation (a host pointer, a frame longer than its buffer); SQDET_ERR_STATE before
 *     sqdet_finalize.
 * Like sqdet_forward_u8, one engine per stream: results are read through sqdet_results_dev.   */
int sqdet_forward_frames_u8(sqdet_engine* e, int n, const uint8_t* const* frames_dev,
                            const int32_t* heights, const int32_t* widths,
                            const int64_t* row_pitches, int order, int rescale, void* stream);
/* n NV12 frames already in device memory on the engine's device, as a hardware video decoder
 * (NVDEC) writes them: frame i is heights[i] x widths[i] (both even), a luma plane of heights[i]
 * rows of widths[i] bytes at luma_dev[i] + r*luma_pitches[i] and a chroma plane of heights[i]/2
 * rows of widths[i] interleaved U,V bytes at chroma_dev[i] + r*chroma_pitches[i] (NULL pitches =
 * widths[i]; either plane may start at any byte).  crops: NULL (whole frames) or n x (x, y, w, h),
 * a non-empty rectangle inside the frame at any origin.  Each crop is exactly
 * cv2.cvtColor(nv12, cv2.COLOR_YUV2BGR_NV12)[y:y+h, x:x+w] (OpenCV's BT.601 limited-range
 * fixed-point conversion; FFmpeg's swscale, inside cv2.VideoCapture, rounds differently), and the
 * call is bit for bit sqdet_forward_frames_u8 on those BGR crops: resize + `- mc.BGR_MEANS` in
 * `order` into tensor 0, rescale by the crop's size, then the forward on `stream`.  No BGR frame
 * is written.  Asynchronous; no host synchronisation.
 *   - Launches: sqdet_launches_per_forward (without a box-scale table), plus one conversion launch
 *     per 56 frames, plus the rescale launch when rescale != 0.
 *   - Refused before any device work, leaving graphs, pipeline and tensor 0 untouched:
 *     SQDET_ERR_INVALID_ARG for a null engine or array, n outside [1, B], an unknown order, a
 *     null plane, a height or width <= 0 or odd, a pitch below the width, an empty crop or one
 *     outside the frame, or a plane whose bytes (luma (H-1)*pitch + W, chroma (H/2-1)*pitch + W)
 *     are not device memory of the engine's device inside one allocation; SQDET_ERR_STATE before
 *     sqdet_finalize.
 * Like sqdet_forward_u8, one engine per stream: results are read through sqdet_results_dev.   */
int sqdet_forward_frames_nv12(sqdet_engine* e, int n, const uint8_t* const* luma_dev,
                              const int64_t* luma_pitches, const uint8_t* const* chroma_dev,
                              const int64_t* chroma_pitches, const int32_t* heights,
                              const int32_t* widths, const int32_t* crops, int order, int rescale,
                              void* stream);
/* Pixel formats of sqdet_forward_frames and the cv2.cvtColor code each frame is converted by.   */
#define SQDET_FMT_BGR        0  /* plane 0: packed B,G,R  (== sqdet_forward_frames_u8)        */
#define SQDET_FMT_RGB        1  /* plane 0: packed R,G,B                  cv2 COLOR_RGB2BGR    */
#define SQDET_FMT_BGRA       2  /* plane 0: packed B,G,R,A, A never read  cv2 COLOR_BGRA2BGR   */
#define SQDET_FMT_RGBA       3  /* plane 0: packed R,G,B,A, A never read  cv2 COLOR_RGBA2BGR   */
#define SQDET_FMT_RGB_PLANAR 4  /* planes 0,1,2: R, G, B, h rows of w bytes (torch [3,h,w])   */
#define SQDET_FMT_NV12       5  /* luma + interleaved U,V (== sqdet_forward_frames_nv12)       */
#define SQDET_FMT_I420       6  /* luma, U, V; U and V h/2 rows of w/2     cv2 COLOR_YUV2BGR_I420 */
/* n frames of pixel format `format` already in device memory on the engine's device: decoder
 * output (torchvision.io.decode_jpeg(device='cuda') gives SQDET_FMT_RGB_PLANAR, NVDEC NV12),
 * render targets and capture surfaces (BGRA, RGBA).  Frame i is heights[i] x widths[i]; its planes
 * are planes[3i + p] (p below the format's plane count; unused entries are not read and may be
 * NULL), plane p's row r at planes[3i + p] + r*pitches[3i + p], any start byte.  Each plane has
 *   - packed BGR, RGB: h rows of 3w bytes; BGRA, RGBA: h rows of 4w bytes;
 *   - RGB_PLANAR: three planes of h rows of w bytes;
 *   - NV12: h rows of w bytes, then h/2 rows of w interleaved U,V bytes (h, w even);
 *   - I420: h rows of w bytes, then U and V of h/2 rows of w/2 bytes (h, w even).
 * NULL pitches = tight rows.  crops: NULL (whole frames) or n x (x, y, w, h), a non-empty
 * rectangle inside the frame at any origin (a 4:2:0 crop at an odd origin reads the frame's own
 * chroma samples).  Each crop is exactly cv2.cvtColor(frame, code)[y:y+h, x:x+w] with the code
 * listed beside the format (the YUV formats by OpenCV's BT.601 limited-range fixed-point
 * conversion), and the call is bit for bit sqdet_forward_frames_u8 on those BGR crops: resize +
 * `- mc.BGR_MEANS` in `order` into tensor 0, rescale by the crop's size, then the forward on
 * `stream`.  No BGR frame is written.  Asynchronous; no host synchronisation.
 *   - sqdet_forward_frames_u8 is this call with SQDET_FMT_BGR and no crops, and
 *     sqdet_forward_frames_nv12 with SQDET_FMT_NV12: same launches, same results.
 *   - Launches: sqdet_launches_per_forward (without a box-scale table), plus one conversion launch
 *     per 64 frames (BGR, RGB, BGRA, RGBA), 56 (NV12) or 45 (RGB_PLANAR, I420), plus the rescale
 *     launch when rescale != 0.
 *   - Refused before any device work, leaving graphs, pipeline and tensor 0 untouched:
 *     SQDET_ERR_INVALID_ARG for a null engine or array, n outside [1, B], an unknown order or
 *     format, a null plane the format needs, a height or width <= 0 (or odd for NV12 and I420), a
 *     pitch below the plane's row bytes, an empty crop or one outside the frame, or a plane whose
 *     bytes ((rows-1)*pitch + row bytes) are not device memory of the engine's device inside one
 *     allocation; SQDET_ERR_STATE before sqdet_finalize.
 * Like sqdet_forward_u8, one engine per stream: results are read through sqdet_results_dev.   */
int sqdet_forward_frames(sqdet_engine* e, int n, int format, const uint8_t* const* planes,
                         const int64_t* pitches, const int32_t* heights, const int32_t* widths,
                         const int32_t* crops, int order, int rescale, void* stream);
/* Detection over whole frames larger than the network input, as overlapping tiles at native
 * scale (an extra "overview" tile of a whole frame, resized, mixes in freely).  n frames in one
 * SQDET_FMT_* format, laid out exactly as sqdet_forward_frames takes them (planes[3f + p],
 * pitches[3f + p], heights[f], widths[f]), and t tiles, tiles[5k .. 5k+4] = (frame, x, y, w, h): a
 * non-empty rectangle inside its frame.  1 <= n <= t <= B, and every frame has a tile.
 *   1. Rows [0, t) of det_boxes / det_probs / det_class and of the per-tile records and counts
 *      (sqdet_results_dev) are bitwise sqdet_forward_frames over the tiles as crops of their
 *      frames, with rescale = 1 (boxes in tile pixels).
 *   2. Frame f's union U_f is its tiles' rows concatenated in call order, union index
 *      j = p * A + anchor for the frame's p-th tile; each box is (cx + float(x), cy + float(y), w,
 *      h), a float32 add (det_boxes itself is not modified).
 *   3. filter_prediction of U_f exactly as sqdet_topk_nms filters one image: the top-N branch
 *      when 0 < TOP_N_DETECTION < |U_f|, else the PROB_THRESH branch in union order (more
 *      candidates than min(1024, max_dets): count -1); same rank order, NMS rule and
 *      class-grouped output.
 *   4. The merged records [B, max_dets] and counts [B] go to a buffer of their own
 *      (sqdet_tile_results_dev): record.anchor is the union index j, so the record came from the
 *      frame's (j / A)-th tile, anchor j % A.  Counts of rows [n, B) are 0; padding as
 *      sqdet_topk_nms writes it.
 * With one tile per frame at (0, 0) the merged records are bitwise the per-tile records.
 * Asynchronous on `stream`, no host synchronisation; a weight reload or sqdet_set_box_scale
 * waits for the merge too.  At most 128 tiles per call (SQDET_ERR_UNSUPPORTED above).
 *   - Launches: those of sqdet_forward_frames over the t tiles with rescale, plus the merge: one
 *     launch, and one per-tile top-N launch before it when some frame's union is longer than
 *     TOP_N_DETECTION > 0.
 *   - Refused before any device work, leaving graphs, tensor 0 and both result buffers
 *     untouched: SQDET_ERR_INVALID_ARG for a null engine or array, t outside [1, B], n outside
 *     [1, t], a tile's frame index outside [0, n), a frame with no tile, an empty tile or one
 *     outside its frame, and every refusal of sqdet_forward_frames (naming "tile k (frame f)");
 *     SQDET_ERR_STATE before sqdet_finalize.                                                  */
int sqdet_forward_tiles(sqdet_engine* e, int n, int format, const uint8_t* const* planes,
                        const int64_t* pitches, const int32_t* heights, const int32_t* widths,
                        int t, const int32_t* tiles, int order, void* stream);
/* sqdet_forward_tiles' merged records [B, max_dets] and counts [B]; valid until the next
 * sqdet_forward_tiles (counts 0 before the first).                                           */
int sqdet_tile_results_dev(sqdet_engine* e, sqdet_det** dets, int32_t** counts,
                           int32_t* max_dets);
/* src/eval.py:83-84 for callers that resize on the host: xy_scales = B pairs (x_scale,
 * y_scale), host memory; every later forward of the paths fed already-resized images
 * (sqdet_forward(_n), sqdet_forward_profiled, sqdet_detect, sqdet_submit) divides
 * det_boxes[b,:,0::2] by x_scale and [b,:,1::2] by y_scale (float32, as numpy does) between
 * interpret_output and filter_prediction, so det_boxes, the records and the NMS all live on the
 * original image.  sqdet_submit_frames(_n) does not use this table: its `rescale` argument
 * decides per submission.  NULL switches it off.  Synchronous (waits for in-flight forwards).
 * sqdet_launches_per_forward counts the rescale launch while a table is set.               */
int sqdet_set_box_scale(sqdet_engine* e, const float* xy_scales);
/* Kernel launches issued by one sqdet_forward (for accounting).                        */
int sqdet_launches_per_forward(sqdet_engine* e);
/* The engine's own compute stream (cudaStream_t as void*): sqdet_detect / sqdet_submit run on
 * it; callers that order foreign work behind those calls record events on it.              */
void* sqdet_engine_stream(sqdet_engine* e);

/* ---- multi-GPU: the ONE collective of the path ---------------------------------------
 * The reference is single-device (`tf.device('/gpu:{}')`, src/nets/squeezeDet.py:21); the
 * path shards over the batch with no data-path exchange, and the only collective is an
 * ncclAllGather of each rank's result blob
 *     [batch * max_dets sqdet_det records][batch int32 counts]
 * NCCL is bound at run time (dlopen of libnccl.so.2, or $SQDET_NCCL_LIB).
 * sqdet_comm_unique_id: rank 0 creates the 128-byte ncclUniqueId; the launcher distributes it
 * (any host channel).  sqdet_comm_init: ncclCommInitRank on the engine's device (collective
 * over all ranks) + the [nranks][blob] receive buffer.  sqdet_comm_attach: use a communicator
 * the caller owns instead (ncclComm_t as void*).  sqdet_set_gather_in_forward(1): every
 * sqdet_forward / sqdet_submit then ends with the all-gather on the SAME stream, captured in
 * the forward's CUDA graph (no host code between filter and collective).  sqdet_allgather:
 * the collective alone on `stream` (comm NULL = the attached one).  sqdet_gathered_dev: the
 * receive buffer, rank-major.                                                              */
int sqdet_comm_unique_id(void* id128);
int sqdet_comm_init(sqdet_engine* e, int nranks, int rank, const void* id128);
int sqdet_comm_attach(sqdet_engine* e, void* nccl_comm, int nranks, int rank);
int sqdet_comm_destroy(sqdet_engine* e);
int sqdet_set_gather_in_forward(sqdet_engine* e, int on);
int sqdet_allgather(sqdet_engine* e, void* nccl_comm, void* stream);
int sqdet_gathered_dev(sqdet_engine* e, void** gathered_dev, int64_t* bytes_per_rank,
                       int32_t* nranks);

/* ---- stage-isolated kernels (device pointers, asynchronous on `stream`) -------------
 * `device` must be current-capable; buffers must live on it.                           */
/* tf.nn.conv2d + bias_add + relu (src/nn_skeleton.py:539-547); scale/shift optional
 * per-channel affine applied before relu (frozen BN, :447-449); y has `y_cstride`
 * channels per pixel and this conv writes channels [y_coff, y_coff+Cout).            */
int sqdet_conv2d(const float* x_dev, const float* w_hwio_dev, const float* bias_dev,
                 const float* scale_dev, const float* shift_dev, float* y_dev,
                 int B, int H, int W, int Cin, int Cout, int size, int stride,
                 int padding, int relu, int y_cstride, int y_coff, int math_mode,
                 void* stream);
/* sqdet_conv2d with the K split of the tensor-core path chosen by the caller.  A stride-1 SAME
 * 3x3 conv of Cin % 32 == 0 and 65..72 output channels (the ConvDet head's 72-wide tile) may sum
 * its Cin / 32 channel chunks over a cluster of S CTAs, each taking a contiguous range of them,
 * and add the S partial sums in rank order.  k_split 0 chooses S as the engine does (from B and
 * the device's resident clusters; sqdet_conv2d), 1 runs unsplit, 2..4 force S (at most Cin / 32,
 * SQDET_MATH_TF32X3_TC and such a shape only).                                               */
int sqdet_conv2d_k_split(const float* x_dev, const float* w_hwio_dev, const float* bias_dev,
                         const float* scale_dev, const float* shift_dev, float* y_dev,
                         int B, int H, int W, int Cin, int Cout, int size, int stride,
                         int padding, int relu, int y_cstride, int y_coff, int math_mode,
                         int k_split, void* stream);
/* SqueezeDet._fire_layer (src/nets/squeezeDet.py:81-106; same in squeezeDetPlus.py) as ONE
 * call: y[..., :E1] = relu(1x1_e1(q)+b), y[..., E1:] = relu(3x3_e3(q)+b), q = relu(1x1_s(x)+b).
 * x [B,H,W,Cin], kernels HWIO, y [B,H,W,E1+E3].  With SQDET_MATH_TF32X3_TC and a shape the
 * one-kernel fire takes (Cin % 16 == 0, S == 16, E1 and E3 together at most 16 chunks of 64
 * channels) this is ONE kernel launch and the squeeze tensor never leaves the SM; other shapes
 * run the squeeze, the 1x1 expand and the 3x3 expand as three sqdet_conv2d launches.
 * Synchronises the stream (test / debug entry, not the hot path).                          */
int sqdet_fire(const float* x_dev, const float* w_sq_dev, const float* b_sq_dev,
               const float* w_e1_dev, const float* b_e1_dev, const float* w_e3_dev,
               const float* b_e3_dev, float* y_dev, int B, int H, int W, int Cin, int S,
               int E1, int E3, int math_mode, void* stream);
/* tf.nn.max_pool NHWC (src/nn_skeleton.py:580-583).                                   */
int sqdet_maxpool_nhwc(const float* x_dev, float* y_dev, int B, int H, int W, int C,
                       int size, int stride, int padding, void* stream);
/* Image pre-processing in front of the path (SURVEY 8 f-1): uint8 BGR [src_h, src_w, 3] ->
 * fp32 [dst_h, dst_w, 3], cv2.resize's float32 INTER_LINEAR plus the mean subtraction.
 * order SQDET_PRE_RESIZE_THEN_SUB: src/demo.py:187-190 (astype(float32), resize, - BGR_MEANS);
 * order SQDET_PRE_SUB_THEN_RESIZE: src/dataset/imdb.py:87-91 (astype(float32), -= BGR_MEANS,
 * resize).  bgr_means: 3 doubles on the host.  dst may point into an engine input batch.  */
#define SQDET_PRE_RESIZE_THEN_SUB 0
#define SQDET_PRE_SUB_THEN_RESIZE 1
int sqdet_preprocess_u8(const uint8_t* src_dev, int src_h, int src_w, float* dst_dev,
                        int dst_h, int dst_w, const double* bgr_means, int order,
                        void* stream);
/* interpret_output (src/nn_skeleton.py:146-238,271-283; util.py:167-196,219-231).     */
int sqdet_interpret(const float* preds_dev, const float* anchors_f32_dev,
                    float* det_boxes_dev, float* det_probs_dev, int64_t* det_class_dev,
                    int B, int grid_h, int grid_w, int anchors_per_grid, int classes,
                    int image_width, int image_height, float exp_thresh, void* stream);
/* ModelSkeleton.filter_prediction + util.nms (src/nn_skeleton.py:696-734,
 * src/utils/util.py:32-76) for B images at once: boxes [B,A,4], probs [B,A],
 * cls [B,A] -> dets [B,max_dets], counts [B] (count<0: SQDET_ERR_OVERFLOW case).
 * Rank order for the top-N cut and NMS: probability descending, -0.0 == +0.0, NaN last,
 * ties by ascending anchor.                                                            */
int sqdet_topk_nms(const float* boxes_dev, const float* probs_dev,
                   const int64_t* cls_dev, int B, int A, int classes, int top_n,
                   float prob_thresh, float nms_thresh, sqdet_det* dets_dev,
                   int32_t* counts_dev, int max_dets, void* stream);
/* The merge of sqdet_forward_tiles (steps 2-4) on its own: boxes [t,A,4], probs [t,A], cls [t,A]
 * are t tile rows, tile k of frame tile_frames[k] at offset (tile_xy[2k], tile_xy[2k+1]) (host
 * arrays) -> dets [n,max_dets], counts [n] for n frames, 1 <= n <= t <= 128.  The per-tile
 * top-N scratch comes from the stream-ordered allocator on `stream`.  Asynchronous.            */
int sqdet_merge_tiles(const float* boxes_dev, const float* probs_dev, const int64_t* cls_dev,
                      int A, int t, const int32_t* tile_frames, const int32_t* tile_xy, int n,
                      int classes, int top_n, float prob_thresh, float nms_thresh,
                      sqdet_det* dets_dev, int32_t* counts_dev, int max_dets, void* stream);
/* Detections drawn onto frames in device memory, as the reference's demo draws them
 * (src/demo.py draw_detections + src/train.py _draw_box: cv2.rectangle + cv2.putText), bit for bit.
 * n <= 128 frames in one SQDET_FMT_* format, laid out exactly as sqdet_forward_frames takes them
 * (planes[3i + p], pitches[3i + p] or NULL for tight rows, heights[i], widths[i], the same
 * refusals).  Frame i's canvas is the frame, or with crops its crop (x, y, w, h): drawing on a crop
 * is cv2 drawing on the numpy view frame[y:y+h, x:x+w], coordinates crop-relative and clipped at
 * the crop's edges (the records of sqdet_forward_frames(..., rescale=1) over the same crops; tile
 * records, sqdet_tile_results_dev, are in frame pixels and draw with no crops).
 * Frame i's records are dets_dev[i * max_dets + k], k < min(counts_dev[i], max_dets) (device
 * memory); count < 0 (the filter's overflow marker) draws nothing.  Each record, in record order,
 * on a uint8 BGR canvas:
 *   - kept only if prob > plot_prob_thresh (float32, as numpy 2 compares np.float32 > float) and
 *     0 <= cls < classes;
 *   - (xmin, ymin, xmax, ymax) = int() of bbox_transform([cx, cy, w, h]): float32 cx - w / 2 etc.
 *     (no contraction), truncated toward zero; skipped if a corner is not finite or |corner| >= 2^31;
 *   - cv2.rectangle(canvas, (xmin, ymin), (xmax, ymax), colour, 1);
 *   - cv2.putText(canvas, name + ": (%.2f)" % prob, (xmin, ymax), FONT_HERSHEY_SIMPLEX,
 *     font_scale, colour, 1) with LINE_8; '%.2f' is correctly rounded (half to even) on the exact
 *     float32 value, e.g. 0.125 -> "0.12", -0.0 -> "-0.00".  A prob outside [0, 1] draws the
 *     rectangle and no label (the engine's probs are always inside);
 *   - later records overwrite earlier ones where they overlap.
 * Formats: BGR is exactly those bytes.  RGB, BGRA, RGBA, RGB_PLANAR: the B, G, R bytes are those of
 * drawing on cv2.cvtColor(frame, -> BGR), written back in the frame's channel order; alpha is never
 * written.  NV12, I420 (no cv2 equivalent): with (Y, U, V) of the colour =
 * cv2.cvtColor(solid 2x2 BGR patch, COLOR_BGR2YUV_I420), a record sets Y on every pixel of its cv2
 * mask and (U, V) on every chroma sample whose 2x2 luma block, in frame coordinates, holds a mask
 * pixel; later records overwrite earlier ones (oracle/draw.py restates the rule).
 * Runs on the device frame 0's first plane lives on, whichever device is current (`stream`
 * belongs to it).  Asynchronous on `stream`, no host synchronisation.  Refused before any device
 * work, leaving every frame untouched: SQDET_ERR_INVALID_ARG for a null array, n outside [1, 128],
 * an unknown format, every frame refusal of sqdet_forward_frames (planes that are not device
 * memory of that device inside one allocation included), max_dets < 1, classes outside [1, 64], a
 * null class name or one that is not printable ASCII of at most 31 characters, a font_scale that
 * is not finite, positive and at most 1024, and dets_dev (n * max_dets records) or counts_dev
 * (n int32) not inside one allocation of device memory on that device.                        */
typedef struct sqdet_draw_style {
  int32_t            classes;          /* 1..64                                              */
  const char* const* class_names;      /* printable ASCII, at most 31 chars each              */
  const uint8_t*     class_bgr;        /* [classes][3]                                        */
  float              plot_prob_thresh; /* mc.PLOT_PROB_THRESH                                 */
  float              font_scale;       /* draw_box's 0.3; thickness is always 1               */
} sqdet_draw_style;
int sqdet_draw_dets(int n, int format, uint8_t* const* planes, const int64_t* pitches,
                    const int32_t* heights, const int32_t* widths, const int32_t* crops,
                    const sqdet_det* dets_dev, const int32_t* counts_dev, int max_dets,
                    const sqdet_draw_style* style, void* stream);

/* ---- JPEG encoding of frames in device memory (no engine needed) -------------------
 * sqdet_encode_jpeg: frame i's crop (x, y, w, h) becomes exactly the bytes of
 *   cv2.imencode('.jpg', cv2.cvtColor(frame, code)[y:y+h, x:x+w], [IMWRITE_JPEG_QUALITY, quality])
 * with `code` the frame format's code of sqdet_forward_frames (BGR: no conversion): cv2's default
 * encoder, libjpeg-turbo's integer pipeline — baseline sequential, 4:2:0, Annex K Huffman tables
 * (not optimized), no restart markers (sqdet_encode_jpeg_params below takes cv2's other settings), JFIF APP0 1.01 with 1:1 density, quantization tables of
 * jpeg_quality_scaling(quality) clamped to 1..255.  Frames are laid out as sqdet_forward_frames
 * takes them.  Frame i's file goes to out_dev + i * cap and its length to lengths_dev[i]; a file
 * longer than cap gives lengths_dev[i] = -1 and unspecified bytes in that frame's slot, and the
 * other frames are unaffected.  cap = sqdet_jpeg_max_bytes(h, w) fits every crop of h x w or less.
 * scratch_dev is 256-byte aligned (as cudaMalloc returns) and holds at least
 * sqdet_jpeg_scratch_bytes(n, heights, widths, crops) bytes; lengths_dev is 8-byte aligned; out_dev
 * may start at any byte.
 * Runs on the device frame 0's first plane lives on (`stream` belongs to it); asynchronous on
 * `stream`, no host synchronisation, no allocation.  Refused before any device work with
 * SQDET_ERR_INVALID_ARG: a null array, n outside [1, 128], an unknown format, every frame refusal of
 * sqdet_forward_frames (planes that are not device memory of that device inside one allocation
 * included), a crop wider or taller than 65500 (libjpeg's JPEG_MAX_DIMENSION: cv2.imencode fails
 * there too), quality outside [1, 100], cap < 1, a misaligned
 * scratch_dev or lengths_dev, scratch_bytes below sqdet_jpeg_scratch_bytes, and out_dev (n * cap bytes), lengths_dev (n int64) or scratch_dev
 * (scratch_bytes) not inside one allocation of device memory on that device.
 * sqdet_jpeg_max_bytes: the largest file of an h x w image, 0xFF stuffing of every byte included
 * (-1 for h or w outside [1, 65500]).  sqdet_jpeg_scratch_bytes: the scratch of that call (-1 when
 * its sizes are refused as sqdet_encode_jpeg refuses them).  Both are worst cases, so that no
 * launch size waits for the device: for 1920 x 1080, about 20 MB of output (a quality-95 file of a
 * natural picture is under 1 MB) and about 17 MB of scratch per frame; frames run in groups of
 * 16 that reuse one scratch, so the scratch is that of the largest group.                     */
int64_t sqdet_jpeg_max_bytes(int h, int w);
int64_t sqdet_jpeg_scratch_bytes(int n, const int32_t* heights, const int32_t* widths,
                                 const int32_t* crops);
int sqdet_encode_jpeg(int n, int format, const uint8_t* const* planes, const int64_t* pitches,
                      const int32_t* heights, const int32_t* widths, const int32_t* crops,
                      int quality, uint8_t* out_dev, int64_t cap, int64_t* lengths_dev,
                      void* scratch_dev, int64_t scratch_bytes, void* stream);

/* ---- JPEG encoding with cv2's other IMWRITE_JPEG_* parameters ----------------------
 * sqdet_encode_jpeg_params: sqdet_encode_jpeg with the file cv2.imencode('.jpg', crop, list)
 * writes for the cv2 parameter list `params` stands for:
 *   quality           IMWRITE_JPEG_QUALITY, 1..100
 *   luma_quality      IMWRITE_JPEG_LUMA_QUALITY, 1..100 or -1 (unset): replaces quality
 *   chroma_quality    IMWRITE_JPEG_CHROMA_QUALITY, 1..100 or -1: counts only with luma_quality
 *                     (unset: the luma quality); when the two differ cv2 writes 4:4:4 whatever
 *                     `sampling` says, and so does this
 *   sampling          IMWRITE_JPEG_SAMPLING_FACTOR: 0x411111, 0x221111 (4:2:0, cv2's default),
 *                     0x211111, 0x121111 or 0x111111 (luma h, v; Cb and Cr are 1x1)
 *   optimize          IMWRITE_JPEG_OPTIMIZE, 0 or 1: each frame's own optimal Huffman tables
 *   restart_interval  IMWRITE_JPEG_RST_INTERVAL, 0..65535 MCUs (0: no restart markers)
 * cv2 clamps out-of-range values and falls back to 4:2:0 for another sampling; these functions
 * refuse them with SQDET_ERR_INVALID_ARG instead (as they refuse a null params), and otherwise
 * refuse what sqdet_encode_jpeg refuses.  Progressive files (IMWRITE_JPEG_PROGRESSIVE) are
 * sqdet_encode_jpeg_progressive's, below.
 * sqdet_jpeg_max_bytes_params and sqdet_jpeg_scratch_bytes_params are the output capacity and
 * scratch of those parameters (-1 when the parameters or sizes are refused).  Sampling, optimize
 * and restart markers raise both: 4:4:4 codes three blocks per 8x8 pixels against 4:2:0's 1.5,
 * optimized DC codes reach 16 + 11 bits, and each restart interval adds a padding byte and RSTn.
 * sqdet_encode_jpeg, sqdet_jpeg_max_bytes and sqdet_jpeg_scratch_bytes are these with
 * {quality, -1, -1, 0x221111, 0, 0} (quality 95 for the sizes).
 * Optimized tables add two launches per group of 16 frames (symbol counts, then the tables) and
 * restart markers two (each interval's first bit, then a scan); neither waits for the device. */
typedef struct {
  int32_t quality;
  int32_t luma_quality;
  int32_t chroma_quality;
  int32_t sampling;
  int32_t optimize;
  int32_t restart_interval;
} sqdet_jpeg_params;
int64_t sqdet_jpeg_max_bytes_params(int h, int w, const sqdet_jpeg_params* params);
int64_t sqdet_jpeg_scratch_bytes_params(int n, const int32_t* heights, const int32_t* widths,
                                        const int32_t* crops, const sqdet_jpeg_params* params);
int sqdet_encode_jpeg_params(int n, int format, const uint8_t* const* planes, const int64_t* pitches,
                             const int32_t* heights, const int32_t* widths, const int32_t* crops,
                             const sqdet_jpeg_params* params, uint8_t* out_dev, int64_t cap,
                             int64_t* lengths_dev, void* scratch_dev, int64_t scratch_bytes,
                             void* stream);

/* ---- progressive JPEG encoding ------------------------------------------------------
 * sqdet_encode_jpeg_progressive: sqdet_encode_jpeg_params with the file cv2.imencode('.jpg', crop,
 * list + [IMWRITE_JPEG_PROGRESSIVE, 1]) writes: SOF2 and jpeg_simple_progression's ten scans (DC
 * first of Y, Cb, Cr; Y 1-5; Cr, Cb 1-63; Y 6-63; Y 1-63 refinement; DC refinement; Cr, Cb, Y
 * 1-63 refinement), each with its own optimal Huffman tables, over the baseline file's quantized
 * coefficients.  `optimize` is checked and has no effect, as in cv2: progressive tables are always
 * optimal.  A restart interval counts MCUs in the two DC scans and blocks in the others, whose
 * scans cover only the component's own blocks; one DRI sits before the first scan.  The refusals are
 * sqdet_encode_jpeg_params'.
 * sqdet_jpeg_max_bytes_progressive is the output capacity: 3055 bytes of headers (SOI .. SOF2 and
 * ten DHT segments of at most 256 symbols, two three-component and eight one-component SOS), 6
 * for the DRI with an interval, twice the bytes of the scans' longest data, 2 per RSTn (each
 * scan's intervals but its first) and 2 for EOI.  A scan's longest data is ceil(units * bits / 8)
 * plus a padding byte per interval, with units its blocks (the DC scans: every block of the MCUs;
 * the others: the component's ceil(w_c / 8) x ceil(h_c / 8)) and bits per unit 27 for the DC first
 * scan (16-bit code, 11 bits), 1 for the DC refinement, 26 n + 30 for a first AC scan of n
 * coefficients (16 + 10 bits per coefficient, the EOBRUN code of 16 + 14 bits after the block) and
 * 17 n + 30 for an AC refinement (16 + 1 bits per newly nonzero coefficient, a correction bit per
 * other, the EOBRUN code; ZRLs cost at most a bit per zero).  Every byte may be stuffed.
 * sqdet_jpeg_scratch_bytes_progressive is the scratch: the coefficients, four 32-bit words per
 * unit of all ten scans, the bit buffers of those longest data, and per frame 11 x 256 64-bit
 * symbol counts and its tables.  -1 when the parameters or sizes are refused.
 * A group of 16 frames takes one memset and fourteen launches for all ten scans; none waits for the
 * device. */
int64_t sqdet_jpeg_max_bytes_progressive(int h, int w, const sqdet_jpeg_params* params);
int64_t sqdet_jpeg_scratch_bytes_progressive(int n, const int32_t* heights, const int32_t* widths,
                                             const int32_t* crops, const sqdet_jpeg_params* params);
int sqdet_encode_jpeg_progressive(int n, int format, const uint8_t* const* planes, const int64_t* pitches,
                                  const int32_t* heights, const int32_t* widths, const int32_t* crops,
                                  const sqdet_jpeg_params* params, uint8_t* out_dev, int64_t cap,
                                  int64_t* lengths_dev, void* scratch_dev, int64_t scratch_bytes,
                                  void* stream);

/* ---- PNG encoding of frames in device memory (no engine needed) ---------------------
 * sqdet_encode_png: frame i's crop (x, y, w, h) becomes exactly the bytes of
 *   cv2.imencode('.png', cv2.cvtColor(frame, code)[y:y+h, x:x+w])
 * with `code` the frame format's code of sqdet_forward_frames (BGR: no conversion): cv2's default
 * PNG writer, libpng 1.6 over zlib 1.2.11 — 8-bit RGB (colour type 2), no interlace, the SUB filter
 * on every row (NONE for a 1-pixel-wide image), zlib level 1 with strategy Z_RLE, 8192-byte IDAT
 * chunks, no ancillary chunk.  Arguments, layout, output slots, lengths (-1 for a file longer than
 * cap, the other frames unaffected), alignment, device and stream rules and refusals are those of
 * sqdet_encode_jpeg without quality, except that a crop may be up to 1000000 pixels wide and high
 * (libpng's user limits: cv2.imencode fails beyond them too).  cap = sqdet_png_max_bytes(h, w) fits
 * every crop of h x w or less.
 * sqdet_png_max_bytes: the largest file of an h x w image, about 9/8 of its 3 h w + h bytes of
 * filtered data (-1 for h or w outside [1, 1000000]).  sqdet_png_scratch_bytes: the scratch of that
 * call (-1 when its sizes are refused as sqdet_encode_png refuses them).  Both are worst cases, so
 * that no launch size waits for the device: for 1920 x 1080, about 7 MB of output and about 26 MB of
 * scratch per frame; frames run in groups of 16 that reuse one scratch, so the scratch is that of
 * the largest group.                                                                      */
int64_t sqdet_png_max_bytes(int h, int w);
int64_t sqdet_png_scratch_bytes(int n, const int32_t* heights, const int32_t* widths,
                                const int32_t* crops);
int sqdet_encode_png(int n, int format, const uint8_t* const* planes, const int64_t* pitches,
                     const int32_t* heights, const int32_t* widths, const int32_t* crops,
                     uint8_t* out_dev, int64_t cap, int64_t* lengths_dev, void* scratch_dev,
                     int64_t scratch_bytes, void* stream);

/* ---- JPEG decoding into frames in device memory (no engine needed) -----------------
 * sqdet_decode_jpeg: file i becomes exactly the pixels of cv2.imdecode(file, cv2.IMREAD_COLOR)
 * (cv2's bundled libjpeg-turbo at its defaults: its SIMD islow IDCT, fancy upsampling, EXIF
 * orientation applied), a BGR uint8 [height, width, 3] frame at out_planes[i] with rows out_pitches[i] bytes
 * apart (pitch >= 3 * width; any start byte).
 *
 * Decoded: SOF0/SOF1 Huffman-coded sequential files with 8-bit samples and one scan of 1 or 3
 * components; luma sampling 1x1, 2x1, 1x2, 2x2 or 4x1 with 1x1 chroma; any DQT and DHT; DRI.
 * APPn and COM segments are skipped; the first APP1 'Exif' segment's Orientation is applied.
 * Everything else is refused before any device work with SQDET_ERR_UNSUPPORTED and a message
 * naming the file; route those files to cv2.imdecode.  Except SQDET_JPEG_TOO_LARGE: a coded side
 * above 65500 (libjpeg's JPEG_MAX_DIMENSION) or more than 2^30 coded pixels (cv2's default
 * CV_IO_MAX_IMAGE_PIXELS) is refused because cv2.imdecode decodes none of these files either (it
 * returns None or raises), and a few header bytes must not size gigabytes of device memory.
 *
 * sqdet_jpeg_parse (host only): the headers of one file.  Returns SQDET_OK for a file
 * sqdet_decode_jpeg decodes, SQDET_ERR_UNSUPPORTED with out->reason set for one it refuses, and
 * SQDET_ERR_INVALID_ARG for a null pointer or len < 0.
 *
 * sqdet_jpeg_decode_staging_bytes / sqdet_jpeg_decode_scratch_bytes: the pinned host staging and
 * the device scratch sqdet_decode_jpeg needs for these files (-1 when a file is refused).  Both
 * come from the headers alone, so nothing on the host waits for the device: the staging holds
 * every file's entropy-coded bytes plus about 9 KiB of tables, and the scratch about 5 bytes per
 * decoded pixel for 4:2:0 and 10 for 4:4:4 (coefficients and sample planes; a quality-95 1080p
 * 4:2:0 file of 0.54 MB takes 0.55 MB of staging and 10.6 MB of scratch).
 *
 * sqdet_decode_jpeg parses every header on the host, builds each file's Huffman lookup tables and
 * quantization tables, packs them and the entropy-coded bytes into staging_pinned, issues one
 * cudaMemcpyAsync of it into scratch_dev and then the kernels, all on `stream`, with no host
 * synchronisation.  Staging reuse: the call returns before the copy has read staging_pinned, so
 * the caller must not write to it again (in another call or otherwise) until that copy is done;
 * record an event on `stream` after the call and wait on it before reusing the staging.
 * status_dev[i] is 0 when file i decoded, negative when its entropy-coded data is corrupt (an
 * invalid code, a DC category above 15, a run past coefficient 63, an RSTn out of sequence or
 * missing, too few blocks in an interval, or data that runs out): its pixels are then unspecified
 * and the other files are unaffected.  As in libjpeg, data after an interval's last block and
 * RSTn markers after the last interval's are skipped.  Files libjpeg refuses when it builds its
 * tables (a Huffman table with more codes than its lengths allow, a DC symbol above 15) are
 * refused as malformed; 3-component files libjpeg takes as RGB (an Adobe transform 0, or ids
 * 'R','G','B', without a JFIF APP0) as SQDET_JPEG_COLOR_TRANSFORM.  n is in [1, 128]; scratch_dev is 256-byte aligned device memory on the device of
 * the outputs, status_dev 4-byte aligned; staging_pinned is page-locked host memory.  Refused
 * with SQDET_ERR_INVALID_ARG before any device work: null arrays, n outside [1, 128], lengths
 * outside [4, 2^28], a pitch below 3 * width, outputs, status or scratch not inside one device
 * allocation of the outputs' device, a misaligned scratch or status, staging that is not pinned
 * host memory, and staging or scratch bytes below the sizes above.                             */
#define SQDET_JPEG_OK               0
#define SQDET_JPEG_MALFORMED        1   /* truncated or malformed header */
#define SQDET_JPEG_PROGRESSIVE      2   /* progressive or hierarchical */
#define SQDET_JPEG_ARITHMETIC       3
#define SQDET_JPEG_LOSSLESS         4
#define SQDET_JPEG_PRECISION        5   /* not 8-bit samples */
#define SQDET_JPEG_COMPONENTS       6   /* not 1 or 3 components (CMYK, YCCK, ...) */
#define SQDET_JPEG_COLOR_TRANSFORM  7   /* RGB-coded: Adobe transform 0 or ids 'R','G','B' */
#define SQDET_JPEG_SAMPLING         8   /* other sampling layouts, multi-scan sequential files */
#define SQDET_JPEG_SIZE             9   /* zero height or width */
#define SQDET_JPEG_TOO_LARGE        10  /* a side above 65500 or more than 2^30 pixels, as coded */
/* progressive entry points only (see below); each names what cv2.imdecode does with the file */
#define SQDET_JPEG_BAD_PROGRESSION  11  /* scan script libjpeg rejects: cv2 returns None */
#define SQDET_JPEG_BOGUS_PROGRESSION 12 /* scan script libjpeg warns on or overwrites: cv2 decodes it */
#define SQDET_JPEG_SMOOTHED         13  /* libjpeg block-smooths it: cv2 decodes it */
#define SQDET_JPEG_TOO_MANY_SCANS   14  /* more than 256 scans: cv2 decodes it */
typedef struct {
  int32_t height, width;              /* of the decoded frame (reduced, see _params), after orientation */
  int32_t coded_height, coded_width;  /* as SOF gives them */
  int32_t components;                 /* 1 or 3 (4 too with any_layout) */
  int32_t h_samp, v_samp;             /* luma sampling factors (chroma is 1x1) */
  int32_t orientation;                /* EXIF Orientation 1..8 (1 without one) */
  int32_t restart_interval;           /* MCUs per restart interval, 0 for none */
  int32_t supported;                  /* 1 when sqdet_decode_jpeg decodes the file */
  int32_t reason;                     /* SQDET_JPEG_* */
  int32_t reserved;
  int64_t scan_offset;                /* the entropy-coded segment's first byte */
} sqdet_jpeg_info;
int sqdet_jpeg_parse(const uint8_t* file, int64_t len, sqdet_jpeg_info* out);
int64_t sqdet_jpeg_decode_staging_bytes(int n, const uint8_t* const* files_host, const int64_t* lengths);
int64_t sqdet_jpeg_decode_scratch_bytes(int n, const uint8_t* const* files_host, const int64_t* lengths);
int sqdet_decode_jpeg(int n, const uint8_t* const* files_host, const int64_t* lengths,
                      uint8_t* const* out_planes, const int64_t* out_pitches, void* staging_pinned,
                      int64_t staging_bytes, void* scratch_dev, int64_t scratch_bytes,
                      int32_t* status_dev, void* stream);
/* Test hook: the bits per subsequence of the parallel Huffman decode (a multiple of 32 in
 * [32, 8192]; 0 restores the default 1024).  Process-wide; sizes from the functions above hold
 * for the value set when they were called.                                                    */
int sqdet_jpeg_decode_set_subsequence_bits(int bits);

/* ---- progressive JPEG decoding (no engine needed) ------------------------------------
 * sqdet_decode_jpeg_progressive decodes SOF2 (progressive Huffman) files as well as every file
 * sqdet_decode_jpeg decodes, in one batch, again exactly to cv2.imdecode's pixels; the sequential
 * files of a batch decode to what sqdet_decode_jpeg gives them.  The four functions take the
 * arguments of their plain counterparts, make the same argument checks and keep the same limits
 * (1 to 128 files, 65500 per side, 2^30 pixels); sqdet_jpeg_decode_set_subsequence_bits applies
 * to the sequential files.  The plain functions keep refusing SOF2 files.
 *
 * A progressive file holds its coefficients in several scans, each a band [Ss, Se] of one or
 * more components at bit Al (Ah: the bit of the scan before, for a refinement).  cv2's
 * libjpeg-turbo reads them all into a whole-image buffer and decodes that as a sequential file
 * of those coefficients, so the sample path (IDCT, upsampling, colour, EXIF orientation) is the
 * sequential one.  Refused besides the sequential refusals, each with what cv2 does:
 *   SQDET_JPEG_BAD_PROGRESSION   libjpeg's JERR_BAD_PROGRESSION (a DC scan with Se != 0, an AC
 *                                scan with Ss > Se, Se > 63 or several components, Ah != 0 with
 *                                Al != Ah - 1, Al > 13): cv2 returns None
 *   SQDET_JPEG_BOGUS_PROGRESSION libjpeg's JWRN_BOGUS_PROGRESSION (an AC scan before the
 *                                component's DC, an Ah that is not the coefficient's last Al),
 *                                and a second first scan (Ah = 0) of a coefficient: cv2 decodes
 *   SQDET_JPEG_SMOOTHED          files libjpeg block-smooths, decided from the scan headers as
 *                                jdcoefct.c's smoothing_ok decides: every component has DC bits
 *                                and nonzero quantizers 0..9 of its latched table, and some
 *                                coefficient 1..9 of some component is never coded or not coded
 *                                down to bit 0.  Complete files are not smoothed
 *   SQDET_JPEG_TOO_MANY_SCANS    more than 256 scans (libjpeg has no cap; a few header bytes
 *                                must not size unbounded staging).  The scans past the cap are
 *                                still checked, so a file libjpeg rejects or warns on is reported
 *                                as such whatever its number of scans
 * Still refused with their plain reasons: SOF6/SOF14 (hierarchical), SOF10 (arithmetic),
 * multi-scan sequential files, and (SQDET_JPEG_SAMPLING, as the plain decoder refuses them) scans
 * whose components are not in the frame's order or repeat one: libjpeg decodes some of these
 * (Cr before Cb) and rejects others (Y, Cr, Cb); route them to cv2.imdecode.  A component's quantization table is the one in force at its
 * first scan, as libjpeg latches it; DHT and DRI may change between scans, and an AC scan's
 * restart interval counts blocks.
 *
 * status_dev[i] is negative, and only file i's pixels unspecified, for the corruptions of
 * sqdet_decode_jpeg and, in a progressive scan, a run past Se, a refinement symbol of a size
 * other than 1, or an EOBRUN past its restart interval.
 *
 * The host reads every scan's bytes to find the next header, removes their stuffing and splits
 * them at their RSTn markers into the staging.  A scan's restart intervals are placed only as far
 * as its markers reach (a scan with fewer markers than its DRI asks for is corrupt), so the
 * staging follows the file's bytes, not its headers: at most 7 bytes per byte of the file (its
 * clean data, and 4 + 8 bytes per restart interval, each of which takes at least the 2 bytes of
 * its RSTn) plus about 5 KiB per scan for its tables and descriptor.  On the stream, with no host synchronisation: one launch decodes
 * every first scan (Ah = 0) of every file, one warp per (scan, restart interval); one launch
 * ORs in every DC refinement, one thread per block; one launch per depth of the longest chain of
 * AC refinements of one component decodes those, one warp per (scan, restart interval); then
 * the sequential IDCT and colour kernels.  A scan without restart markers is one lane's work. */
int sqdet_jpeg_parse_progressive(const uint8_t* file, int64_t len, sqdet_jpeg_info* out);
int64_t sqdet_jpeg_decode_staging_bytes_progressive(int n, const uint8_t* const* files_host,
                                                    const int64_t* lengths);
int64_t sqdet_jpeg_decode_scratch_bytes_progressive(int n, const uint8_t* const* files_host,
                                                    const int64_t* lengths);
int sqdet_decode_jpeg_progressive(int n, const uint8_t* const* files_host, const int64_t* lengths,
                                  uint8_t* const* out_planes, const int64_t* out_pitches,
                                  void* staging_pinned, int64_t staging_bytes, void* scratch_dev,
                                  int64_t scratch_bytes, int32_t* status_dev, void* stream);

/* ---- JPEG decoding with cv2's other colour reads: IMREAD_REDUCED_COLOR_2/4/8 ---------
 * The _params functions take the arguments of their plain counterparts and a
 * sqdet_jpeg_decode_params:
 *   progressive  0: the files sqdet_decode_jpeg decodes; 1: those of sqdet_decode_jpeg_progressive
 *   scale_denom  1, 2, 4 or 8: file i becomes exactly cv2.imdecode(file, IMREAD_REDUCED_COLOR_s)
 *                with s = scale_denom (IMREAD_COLOR for 1); anything else is SQDET_ERR_INVALID_ARG
 *   reserved     0
 * The plain and _progressive functions are these with {0, 1} and {1, 1}.
 *
 * libjpeg-turbo decodes straight to the reduced size with scaled IDCTs; so does sqdet_decode_jpeg_params.
 * The frame is ceil(coded_height / s) x ceil(coded_width / s) before the EXIF orientation, and
 * sqdet_jpeg_info's height and width report it after the orientation.  Luma takes an m x m IDCT
 * per 8 x 8 block, m = 8 / s (jpeg_idct_4x4 and jpeg_idct_2x2 as libjpeg-turbo's SSE2 code
 * computes them, and jpeg_idct_1x1); a chroma component's IDCT doubles from m while it stays
 * below 8 and libjpeg's divisibility rule holds, which 4:2:0 chroma meets (chroma at 2m, not
 * upsampled) and the other samplings do not (chroma at m, upsampled).  Upsampling is fancy
 * (h2v1 and h1v2 triangle filters) at 1/2 and 1/4 and replication at 1/8.  The coefficients are
 * those of the full-size decode; the sample planes in the scratch shrink to the scaled size.
 *
 * Size limits: a coded side above 65500 is SQDET_JPEG_TOO_LARGE at any scale, as in libjpeg.
 * cv2 applies CV_IO_MAX_IMAGE_PIXELS (2^30) to the reduced size: above it the reason is
 * SQDET_JPEG_TOO_LARGE (cv2 refuses the file too).  A file of more than 2^30 coded pixels whose
 * reduced size fits is SQDET_JPEG_CODED_TOO_LARGE, refused before any sizing: cv2 decodes it at
 * that scale, but a few header bytes must not size gigabytes of coefficients (2 bytes per coded
 * sample); route it to cv2.imdecode.                                                          */
#define SQDET_JPEG_CODED_TOO_LARGE  15  /* more than 2^30 coded pixels, fewer reduced: cv2 decodes it */
typedef struct {
  int32_t progressive;
  int32_t scale_denom;
  int32_t reserved[2];
} sqdet_jpeg_decode_params;
int sqdet_jpeg_parse_params(const uint8_t* file, int64_t len, const sqdet_jpeg_decode_params* params,
                            sqdet_jpeg_info* out);
int64_t sqdet_jpeg_decode_staging_bytes_params(int n, const uint8_t* const* files_host,
                                               const int64_t* lengths,
                                               const sqdet_jpeg_decode_params* params);
int64_t sqdet_jpeg_decode_scratch_bytes_params(int n, const uint8_t* const* files_host,
                                               const int64_t* lengths,
                                               const sqdet_jpeg_decode_params* params);
int sqdet_decode_jpeg_params(int n, const uint8_t* const* files_host, const int64_t* lengths,
                             const sqdet_jpeg_decode_params* params, uint8_t* const* out_planes,
                             const int64_t* out_pitches, void* staging_pinned, int64_t staging_bytes,
                             void* scratch_dev, int64_t scratch_bytes, int32_t* status_dev,
                             void* stream);

/* ---- JPEG decoding of every colour space and sampling cv2.imdecode reads -------------
 * The _options functions take the arguments of the _params ones with a
 * sqdet_jpeg_decode_options in place of the params:
 *   progressive, scale_denom  as in sqdet_jpeg_decode_params
 *   any_layout   0: the files the _params functions decode (they are these functions with
 *                any_layout = 0); 1: those and the layouts below; anything else is
 *                SQDET_ERR_INVALID_ARG
 *   reserved     0
 * With any_layout = 1, file i is still exactly cv2.imdecode(file, IMREAD_COLOR or
 * IMREAD_REDUCED_COLOR_s) and these Huffman-coded 8-bit files decode too:
 *   colour space  as libjpeg's default_decompress_parms decides it.  3 components: YCbCr after a
 *                 JFIF APP0, else RGB for an Adobe APP14 transform 0 (any other transform:
 *                 YCbCr), else RGB for component ids 'R','G','B', else YCbCr.  RGB planes come out
 *                 as they are (B, G, R = planes 2, 1, 0).  4 components: YCCK for an Adobe
 *                 transform other than 0, else CMYK.  cv2 reads 4 components as libjpeg's CMYK
 *                 (YCCK through ycck_cmyk_convert: C, M, Y = 255 - the clamped YCbCr->RGB of Y,
 *                 Cb, Cr; K as coded) and converts each pixel with icvCvt_CMYK2BGR:
 *                 B = K - ((255 - Y) * K >> 8), G from M, R from C; no Adobe inversion.
 *   sampling      factors 1..4 with max_h / h and max_v / v integral for every component (the
 *                 largest factors need not be component 0's) and at most 10 blocks in an
 *                 interleaved MCU: a sequential file's scan, and each interleaved progressive
 *                 scan.  Each component is upsampled as jinit_upsampler chooses from its scaled
 *                 IDCT size: not at all when it has the frame's size; h2v1 and h2v2 by the
 *                 triangle filters when fancy upsampling is on and its downsampled width is above
 *                 2, by replication otherwise; h1v2 by the triangle filter when fancy upsampling
 *                 is on; any other integral ratio by replication (int_upsample).  Fancy
 *                 upsampling is on at scales 1, 1/2 and 1/4 and off at 1/8.  Upsampling comes
 *                 before the colour conversion, whatever the colour space.
 * Refused with any_layout = 1, each with what cv2 does:
 *   SQDET_JPEG_BAD_SAMPLING   a ratio that is not integral, or more than 10 blocks in an
 *                             interleaved MCU: libjpeg rejects the file and cv2 returns None
 *   SQDET_JPEG_COMPONENTS     2 components, or more than 4: libjpeg has no conversion of them to
 *                             BGR and cv2 returns None
 * Arithmetic, lossless, 12-bit and multi-scan sequential files keep their refusals.  The plain,
 * _progressive and _params functions keep refusing every file they refused before, with the
 * same reasons.                                                                               */
#define SQDET_JPEG_BAD_SAMPLING     16  /* any_layout: sampling libjpeg rejects: cv2 returns None */
typedef struct {
  int32_t progressive;
  int32_t scale_denom;
  int32_t any_layout;
  int32_t reserved[5];
} sqdet_jpeg_decode_options;
int sqdet_jpeg_parse_options(const uint8_t* file, int64_t len, const sqdet_jpeg_decode_options* options,
                             sqdet_jpeg_info* out);
int64_t sqdet_jpeg_decode_staging_bytes_options(int n, const uint8_t* const* files_host,
                                                const int64_t* lengths,
                                                const sqdet_jpeg_decode_options* options);
int64_t sqdet_jpeg_decode_scratch_bytes_options(int n, const uint8_t* const* files_host,
                                                const int64_t* lengths,
                                                const sqdet_jpeg_decode_options* options);
int sqdet_decode_jpeg_options(int n, const uint8_t* const* files_host, const int64_t* lengths,
                              const sqdet_jpeg_decode_options* options, uint8_t* const* out_planes,
                              const int64_t* out_pitches, void* staging_pinned, int64_t staging_bytes,
                              void* scratch_dev, int64_t scratch_bytes, int32_t* status_dev,
                              void* stream);

/* ---- KITTI 2-D object scoring of filtered records (no engine needed) ---------------
 * sqdet_kitti_eval scores n images of records exactly as the KITTI devkit's evaluate_object does
 * the detection files eval.py writes from them (see oracle/kitti_eval.py for the rules): for each
 * class (car, pedestrian, cyclist) and difficulty (easy, moderate, hard), index 3 * class +
 * difficulty, it gives the threshold count and, per threshold, TP, FP, FN and the similarity sum
 * in image order.  The host forms precision = tp / (double)(tp + fp), aos = similarity /
 * (double)(tp + fp), their suffix maxima and the AP from these (squeezedet_b200.kitti).
 *
 * dets [n, max_dets] and counts [n]: records as the engine writes them, in device memory.
 * class_map [classes] (host): per class id, SQDET_KITTI_CAR / _PEDESTRIAN / _CYCLIST, or -1 for a
 * class the devkit never evaluates; at most one id per KITTI class.  objs [n_objects] and
 * offsets [n + 1] (device): image i's label lines are objs[offsets[i] .. offsets[i + 1]) in file
 * order, with aos_term = (1 + cos(alpha)) / 2 computed by the caller.  scratch: 256-byte aligned,
 * sqdet_kitti_eval_scratch_bytes(n, max_dets, n_objects) bytes (-1 for sizes refused as below).
 * out: one sqdet_kitti_result in device memory.  Everything runs on `stream`, with no host wait.
 *
 * Refused with SQDET_ERR_INVALID_ARG before any launch: n < 1, max_dets outside [1, 1024], null
 * pointers, a bad class map, buffers not on one device.  A record that cannot be scored sets
 * out->status to 8 * image + reason (the first image; -1 when every record is usable): a count
 * outside [0, max_dets] (the filter's -1 overflow marker included), a class id outside the map,
 * a non-finite box or prob, a prob outside [0, 1], offsets that are not increasing in
 * [0, n_objects].  The other outputs are then meaningless, but nothing outside the arguments is
 * read: an image whose offsets are refused is scored as having no objects.                  */
#define SQDET_KITTI_CAR             0
#define SQDET_KITTI_PEDESTRIAN      1
#define SQDET_KITTI_CYCLIST         2
#define SQDET_KITTI_VAN             3
#define SQDET_KITTI_PERSON_SITTING  4
#define SQDET_KITTI_DONTCARE        5
#define SQDET_KITTI_OTHER           6
#define SQDET_KITTI_MAX_THRESHOLDS 41
#define SQDET_KITTI_MAX_CLASSES    64
/* out->status reasons */
#define SQDET_KITTI_BAD_COUNT       1
#define SQDET_KITTI_BAD_CLASS       2
#define SQDET_KITTI_NOT_FINITE      3
#define SQDET_KITTI_BAD_SCORE       4
#define SQDET_KITTI_BAD_OFFSETS     5
#define SQDET_KITTI_TOO_MANY_THRESHOLDS 6   /* never: at most 41 thresholds exist */

typedef struct sqdet_kitti_obj {   /* one label line (56 bytes) */
  double  x1, y1, x2, y2;          /* box, as strtod reads it */
  double  truncation;
  double  aos_term;                /* (1 + cos(alpha)) / 2 */
  int32_t type;                    /* SQDET_KITTI_* type code, case-insensitive */
  int32_t occlusion;
} sqdet_kitti_obj;

typedef struct sqdet_kitti_result {
  double  similarity[9][SQDET_KITTI_MAX_THRESHOLDS];
  int32_t tp[9][SQDET_KITTI_MAX_THRESHOLDS];
  int32_t fp[9][SQDET_KITTI_MAX_THRESHOLDS];
  int32_t fn[9][SQDET_KITTI_MAX_THRESHOLDS];
  int32_t n_thresholds[9];
  int32_t n_gt[9];
  int32_t evaluated[3];            /* a usable record of the class exists */
  int32_t status;
  int32_t reserved;                /* pads the struct to a multiple of 8 bytes (7472) */
} sqdet_kitti_result;

int64_t sqdet_kitti_eval_scratch_bytes(int n, int max_dets, int64_t n_objects);
int sqdet_kitti_eval(int n, int max_dets, const sqdet_det* dets, const int32_t* counts,
                     int classes, const int32_t* class_map, const sqdet_kitti_obj* objs,
                     const int64_t* offsets, int64_t n_objects, void* scratch,
                     int64_t scratch_bytes, sqdet_kitti_result* out, void* stream);

/* ---- KITTI detection error analysis of filtered records (no engine needed) ----------
 * sqdet_kitti_analyze classifies the records of n images exactly as the reference's
 * analyze_detections (src/dataset/kitti.py:182-296, restated in oracle/kitti_analysis.py) does
 * the detection files eval.py writes from them.  Per image, the ground truth is every label line
 * of an analyzed class, in file order; the detections are the records as read back from the file
 * (corners rint(v * 100) / 100, scores k / 1000), ranked by score, then class id, then record
 * index, and only the first G count, G the image's ground-truth count.  Each counted detection is
 * matched to the first object of largest IoU: correct (the first such detection of that object),
 * repeated, localization, classification or background error.
 *
 * The arguments are those of sqdet_kitti_eval, except that every class id must name a distinct
 * analyzed class (class_map entries 0, 1 or 2, so classes <= 3), plus `lines`, a device buffer of
 * line_capacity error lines: in image order, each image's loc / cls / bg detections in ranked
 * order and then its missed objects in label order.  2 x (objects of the analyzed classes) lines
 * always fit; lines past line_capacity are counted in out->n_lines but not written.  scratch:
 * 256-byte aligned, sqdet_kitti_analyze_scratch_bytes(n, max_dets, n_objects) bytes.
 * Everything runs on `stream`, with no host wait.
 *
 * Refused with SQDET_ERR_INVALID_ARG before any launch as sqdet_kitti_eval refuses, and for a
 * class map with a -1 entry.  out->status is 16 * image + reason for the first image refused
 * (-1 when none is): the scorer's reasons, a record with w < 0 or h < 0 (the engine writes none;
 * its IoU union can be 0), or a label box of an analyzed class that is not finite or fails the
 * reference's assertions x1 >= 0, x1 <= x2, y1 >= 0, y1 <= y2.                               */
#define SQDET_KITTI_NEGATIVE_SIZE   7
#define SQDET_KITTI_BAD_LABEL       8
/* error line types */
#define SQDET_KITTI_ERR_LOC         0
#define SQDET_KITTI_ERR_CLS         1
#define SQDET_KITTI_ERR_BG          2
#define SQDET_KITTI_ERR_MISSED      3

typedef struct sqdet_kitti_error_line {   /* one line of det_error_file.txt (56 bytes) */
  int32_t image;
  int32_t type;                    /* SQDET_KITTI_ERR_* */
  int32_t cls;                     /* class id */
  int32_t reserved;
  double  x1, y1, x2, y2;          /* cx - w / 2., cy - h / 2., cx + w / 2., cy + h / 2. */
  double  score;                   /* the read-back score, -1.0 for a missed object */
} sqdet_kitti_error_line;

typedef struct sqdet_kitti_analysis {
  int64_t num_dets, num_objs;      /* counted detections; objects of the analyzed classes */
  int64_t correct, loc, cls, bg, repeated;
  int64_t detected;                /* objects a correct detection claimed */
  int64_t n_lines;                 /* error lines, written or not */
  int32_t status;
  int32_t reserved;
} sqdet_kitti_analysis;

int64_t sqdet_kitti_analyze_scratch_bytes(int n, int max_dets, int64_t n_objects);
int sqdet_kitti_analyze(int n, int max_dets, const sqdet_det* dets, const int32_t* counts,
                        int classes, const int32_t* class_map, const sqdet_kitti_obj* objs,
                        const int64_t* offsets, int64_t n_objects, void* scratch,
                        int64_t scratch_bytes, sqdet_kitti_analysis* out,
                        sqdet_kitti_error_line* lines, int64_t line_capacity, void* stream);

/* ---- tiny device-memory helpers so a ctypes caller needs nothing else -------------- */
int sqdet_malloc(int device, int64_t bytes, void** out_dev);
int sqdet_free(int device, void* dev);
int sqdet_malloc_host(int64_t bytes, void** out_pinned);
int sqdet_free_host(void* pinned);
int sqdet_memcpy_h2d(void* dst_dev, const void* src, int64_t bytes, void* stream);
int sqdet_memcpy_d2h(void* dst, const void* src_dev, int64_t bytes, void* stream);
int sqdet_stream_sync(int device, void* stream);

#ifdef __cplusplus
}
#endif
#endif  /* SQDET_B200_H_ */
