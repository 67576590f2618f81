/* poseengine.h - C ABI of libposeengine.so, the H100-native drop-in for the hot path of
 * examples/rtpose (CMU-Perceptual-Computing-Lab/caffe_rtpose).
 *
 * Every entry point below replaces a call that examples/rtpose/rtpose.cpp makes into Caffe / its own
 * host code for the per-frame path (SURVEY.md section 8b); the reference site is cited on each.
 * Plain C: opaque handle, plain pointers and sizes, int return codes (0 = PE_OK), no exceptions,
 * no torch / CUDA types.  One handle per GPU worker thread (as the reference keeps one caffe::Net per
 * thread, rtpose.cpp:183); calls on one handle must not be concurrent.
 *
 * There is NO CPU fallback: every call needs the CUDA device named at pe_create.
 */
#ifndef POSEENGINE_H
#define POSEENGINE_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define PE_OK 0
#define PE_ERR_INVALID 1   /* bad argument / unsupported configuration */
#define PE_ERR_CUDA 2      /* CUDA runtime / driver failure (message in pe_last_error) */
#define PE_ERR_STATE 3     /* call out of order (e.g. forward before weights) */
#define PE_ERR_IO 4        /* file could not be read / parsed */
#define PE_ERR_RANGE 5     /* fp16 modes: a layer's values left the range of the fp16 planes (see pe_calibrate) */

#define PE_MODEL_MPI_15 0  /* ModelDescriptorFactory::Type::MPI_15  (modelDescriptorFactory.h:16-19) */
#define PE_MODEL_COCO_18 1 /* ModelDescriptorFactory::Type::COCO_18 */

/* arithmetic of the convolution stack */
#define PE_PREC_FP32_SIMT 0 /* fp32 FFMA implicit GEMM (CUDA cores) - the exact-fp32 debugging reference */
#define PE_PREC_BF16X1 1    /* wgmma bf16 x bf16 -> fp32 (fast, NOT parity grade) */
#define PE_PREC_F16X2 2     /* wgmma PARITY mode: activations/weights split in 2 fp16 planes (11+11 bits), 3 MMAs
                             * hi*hi + hi*lo + lo*hi, fp32 accumulation cut into chunks that are summed in registers with
                             * round-to-nearest (the tensor core's own fp32 accumulate truncates): ~1e-5 of the map range
                             * over the whole net, i.e. the level at which two fp32 implementations differ */
#define PE_PREC_BF16X2 PE_PREC_F16X2 /* historical name of the parity mode (its planes were bf16 at first) */
#define PE_PREC_BF16X3 3    /* wgmma, 3 bf16 planes, 6 MMAs: hi*hi chunked as in mode 2, the 5 cross products in a second
                             * accumulator (bf16 planes carry fewer bits: LESS accurate than mode 2) */
#define PE_PREC_F16X1 4     /* wgmma FAST mode: the parity mode's hi plane alone - one fp16 plane (11 bits) of activations and
                             * weights, 1 MMA per MAC, the same per-layer power-of-two weight / range scales (pe_calibrate) and the
                             * same chunked round-to-nearest fp32 accumulation.  Each layer's output is rounded to fp16 (unit
                             * roundoff 2^-11): 1.5e-3 - 2.4e-3 of the map range over the whole net against 1.7e-2 for
                             * PE_PREC_BF16X1 at the same cost, 1.9x the parity mode's frames/s (H100 80GB HBM3, 700 W; DESIGN.md
                             * sections 5, 6).  pe_compare_results measures what that does to the poses. */

#define PE_MAX_PEOPLE 96   /* RENDER_MAX_PEOPLE, renderFunctions.h:6 / rtpose.cpp:88 */

typedef struct pe_engine pe_engine;

typedef struct pe_config {
    int device;          /* CUDA ordinal; Caffe::SetDevice(device_id)                 rtpose.cpp:178 */
    int model;           /* PE_MODEL_*; the reference infers it from nms num_parts    rtpose.cpp:212-229 */
    int net_w, net_h;    /* --net_resolution (multiples of 8)                          rtpose.cpp:64,1693 */
    int disp_w, disp_h;  /* --resolution: joints are reported in display pixels        rtpose.cpp:63,1058-1062 */
    int num_scales;      /* --num_scales == blob dim 0 of one forward                  rtpose.cpp:71,188 */
    double start_scale;  /* --start_scale                                              rtpose.cpp:69 */
    double scale_gap;    /* --scale_gap                                                rtpose.cpp:70 */
    int max_batch;       /* frames per forward on this GPU (1 = the reference's behaviour) */
    int precision;       /* PE_PREC_* */
} pe_config;

/* new caffe::Net(proto, TEST) + Reshape + warmup()                          rtpose.cpp:173-237 */
int pe_create(const pe_config* cfg, pe_engine** out);
/* same, the graph read from a deploy prototxt (--caffeproto, rtpose.cpp:60,183; Net::Init net.cpp:30-280): Convolution /
 * in-place ReLU / 2x2 MAX Pooling / Concat / ImResize / Nms, any number of CPM stages (model/mpi/pose_deploy_linevec_{1,2,4}
 * .prototxt); legacy V1 `layers` blocks are upgraded (upgrade_proto.cpp:957).  cfg->model may be -1: the model follows
 * nms_param.num_parts as in rtpose.cpp:212-229.  nms_param.max_peaks sizes the peak blob (NmsLayer::GetMaxPeaks).
 * Layer types outside the pose path are PE_ERR_INVALID with the layer named in pe_last_error(NULL). */
int pe_create_from_prototxt(const pe_config* cfg, const char* prototxt_path, pe_engine** out);
/* host-only (no GPU): text description of the execution plan of a prototxt (or of the built-in graph of `model` when
 * prototxt_path is NULL); returns the text length (call with buf NULL to size it) or -PE_ERR_* */
int pe_plan_describe(int model, const char* prototxt_path, char* buf, int cap);
void pe_destroy(pe_engine* e);
/* last error text of this handle (or of the failed pe_create / pe_pixels_to_bgr when e == NULL) */
const char* pe_last_error(const pe_engine* e);

/* ---- weights: Net::CopyTrainedLayersFrom                                   rtpose.cpp:184, net.cpp:750-803
 * Layers are matched by name; w is (Cout, Cin, kh, kw) row-major fp32, b is (Cout)  (base_conv_layer.cpp:135-142). */
int pe_num_conv_layers(const pe_engine* e);
int pe_conv_layer_info(const pe_engine* e, int idx, char* name64, int* cout, int* cin, int* ksize);
int pe_set_conv_weights(pe_engine* e, const char* layer_name, const float* w, size_t nw, const float* b, size_t nb);
/* flat file: "RTPW" u32 version=1 u32 nlayers { char name[64]; u32 cout,cin,k; f32 w[]; f32 b[] } */
int pe_load_weights_file(pe_engine* e, const char* path);
/* .caffemodel (binary NetParameter, caffe.proto:92-95 `layer`=100 / legacy `layers`=2): the file rtpose.bin
 * passes to CopyTrainedLayersFrom (rtpose.cpp:59,184).  Matching by layer name, unknown layers ignored,
 * blob-count / shape mismatch is an error (net.cpp:750-786). */
int pe_load_caffemodel(pe_engine* e, const char* path);
/* host-only iteration over a .caffemodel (no GPU needed) */
typedef struct pe_caffemodel pe_caffemodel;
int pe_caffemodel_open(const char* path, pe_caffemodel** out);
void pe_caffemodel_close(pe_caffemodel* m);
int pe_caffemodel_num_layers(const pe_caffemodel* m);
int pe_caffemodel_layer(const pe_caffemodel* m, int idx, char* name64, char* type32, int* num_blobs);
int pe_caffemodel_blob(const pe_caffemodel* m, int layer, int blob, const float** data, size_t* count, int* ndim,
                       long long* dims8);
const char* pe_caffemodel_last_error(void);
/* pack + upload; must be called once after the weights are set and before any forward */
int pe_commit_weights(pe_engine* e);
/* Range management of the fp16 modes (PE_PREC_F16X2, PE_PREC_F16X1; a no-op in the others).  Their activation planes are fp16 x
 * power-of-two scale per layer; the default
 * scale 1 suits the trained pose models.  pe_calibrate runs one forward on the given HOST frames layer by layer, measures every
 * layer's largest |output| in fp32 and sets the scales so that the stored maxima sit in [32, 64) - after that a net of any
 * magnitude (e.g. the prototxt's gaussian(0.01) filler, whose maps are ~3e-11) keeps fp32-level parity.  Exact: scales are powers
 * of two folded into the epilogue's bias / factor.  Call it on the handle that owns the weights, before pe_broadcast_weights /
 * pe_share_weights (the scales travel inside the packed buffer).  Results of the calibration forward are fetchable as usual.
 * pe_range_status: since the previous call, largest |stored value| / 65504 over all layers; PE_ERR_RANGE (and pe_last_error names
 * the layer) if a layer reached the fp16 limit or shrank below 2^-10.  With the environment variable PE_CHECK_RANGE=1 every
 * pe_fetch(idx 0) performs this check, so range problems are errors instead of silent inf / zeros. */
int pe_calibrate(pe_engine* e, const uint8_t* const* frames, int n);
int pe_range_status(pe_engine* e, float* worst_ratio, char* layer64);
/* Net::ShareTrainedLayersWith (net.cpp:682-706): `to` - another handle on the SAME GPU running the same net - uses `from`'s
 * committed weights (the packed device buffer is shared, not copied, and lives until its last user is destroyed). */
int pe_share_weights(pe_engine* from, pe_engine* to);

/* ---- caffe::NmsLayer<float> accessors                                      nms_layer.hpp:24-27, rtpose.cpp:195,207,1145 */
int pe_nms_get_max_peaks(const pe_engine* e);
int pe_nms_get_num_parts(const pe_engine* e);
float pe_nms_get_threshold(const pe_engine* e);
int pe_nms_set_threshold(pe_engine* e, float threshold);
/* ---- caffe::ImResizeLayer<float> accessors                                 imresize_layer.hpp:24-29, rtpose.cpp:201-202 */
int pe_resize_set_start_scale(pe_engine* e, float start_scale);
int pe_resize_set_scale_gap(pe_engine* e, float scale_gap);
float pe_resize_get_start_scale(const pe_engine* e);
float pe_resize_get_scale_gap(const pe_engine* e);
/* ---- global.connect_* thresholds                                           rtpose.cpp:106-111, 212-226 */
int pe_set_connect_params(pe_engine* e, int min_subset_cnt, float min_subset_score, float inter_threshold,
                          int inter_min_above_threshold);

/* ---- per-frame hot loop (processFrame, rtpose.cpp:1099-1203).  All forwards are asynchronous on the
 * engine's stream; pe_fetch* synchronises.  n <= max_batch frames per call.
 *
 * pe_forward_frames: HOST display images, uint8 BGR HWC disp_h x disp_w (what getFrameFromCam holds after
 * warpAffine, rtpose.cpp:484).  Does H2D + the scale loop / INTER_AREA / pad / normalise of rtpose.cpp:508-518
 * on the GPU + net + resize + NMS + connectLimbs*. */
int pe_forward_frames(pe_engine* e, const uint8_t* const* frames, int n);
/* HOST camera/video frames of ANY size (orig_h x orig_w uint8 BGR): first the display image of rtpose.cpp:474-487 -
 * uniform scale s = min(disp_w/cols, disp_h/rows), top-left anchored, cv::warpAffine INTER_CUBIC, black border - is
 * produced on the GPU (OpenCV's fixed-point arithmetic, bit-exact), then as pe_forward_frames.  *scale receives
 * frame.scale (the JSON writer multiplies joints by 1/scale, rtpose.cpp:1384,1399-1400).  = pe_forward_pixels with PE_PIX_BGR. */
int pe_forward_camera_frames(pe_engine* e, const uint8_t* const* frames, int n, int orig_w, int orig_h, double* scale);
/* n JPEG frames of one size as coefficient images (pe_jpeg_read_coefs): copied to the GPU (asynchronously when they were allocated
 * with pe_host_alloc), reconstructed there byte-identically to pe_decode_jpeg, then as pe_forward_frames when the frames are
 * disp_w x disp_h (*scale = 1) and as pe_forward_camera_frames otherwise (GPU warpAffine, *scale = frame.scale).  pe_render
 * with display_bgr == NULL draws on the reconstructed display frame. */
int pe_forward_jpeg_coefs(pe_engine* e, const void* const* coefs, int n, double* scale);
/* the same from scan images (pe_jpeg_read_scan): the Huffman data is decoded on the GPU into coefficient images, then as
 * pe_forward_jpeg_coefs.  A frame whose data the host entropy stage rejects (a DC category above 15) does not stop the batch:
 * pe_fetch of that frame returns PE_ERR_IO (pe_last_error names the frame and the MCU), the other frames' results are unaffected. */
int pe_forward_jpeg_scans(pe_engine* e, const void* const* scans, int n, double* scale);
/* test hook: decode n scan images into coefficient images on the GPU with subsequences of subseq_bits bits (0 = the default) and
 * copy them to coefs_out[i] (coef.total_bytes each).  Synchronous.  status_out[i] (optional): 0, or 1 + the MCU of the first data
 * error of frame i.  The statuses of an earlier pe_forward_jpeg_scans are dropped: pe_fetch no longer reports them. */
int pe_jpeg_decode_scans(pe_engine* e, const void* const* scans, int n, int subseq_bits, void* const* coefs_out, int* status_out);
/* same, frames already resident in device memory (n consecutive disp_h*disp_w*3 images) */
int pe_forward_frames_device(pe_engine* e, const void* d_frames, int n);

/* ---- frames as video decoders hand them out (NVDEC, FFmpeg / PyAV, V4L2, PIL / torchvision), converted to BGR on the GPU with
 * the arithmetic of cv::cvtColor (ITU-R BT.601 studio range, OpenCV's 20-bit fixed point; 4:2:0 chroma nearest-neighbour). */
#define PE_PIX_BGR  0   /* packed uint8 B,G,R (what pe_forward_camera_frames takes)                       */
#define PE_PIX_RGB  1   /* packed uint8 R,G,B            = cv::cvtColor(COLOR_RGB2BGR)                     */
#define PE_PIX_YUYV 2   /* packed 4:2:2 Y0 U Y1 V        = COLOR_YUV2BGR_YUYV; even width                 */
#define PE_PIX_NV12 3   /* Y plane, then interleaved U,V at half size = COLOR_YUV2BGR_NV12; even w, h     */
#define PE_PIX_I420 4   /* Y, then U, then V planes at half size     = COLOR_YUV2BGR_I420; even w, h      */
typedef struct pe_pixel_format {
    int format;              /* PE_PIX_* */
    int width, height;       /* frame size in pixels, 1 .. 16384 */
    long long pitch;         /* bytes between rows of the first plane; 0 = tight (3w, 2w or w); I420: even */
    long long chroma_offset; /* NV12 / I420: bytes from the frame start to the first chroma plane; 0 = pitch * height (an NVDEC
                                surface: pitch * the aligned height).  NV12 chroma rows are `pitch` apart; I420 chroma rows are
                                pitch/2 apart, and V follows U at chroma_offset + (pitch/2) * (height/2).  Ignored otherwise. */
} pe_pixel_format;
/* n <= max_batch frames of one format and size, one pointer per frame.  Each pointer is classified as pe_forward_frames does:
 * device memory on the engine's device (or managed memory) is read in place, asynchronously on the engine's stream; page-locked
 * host memory (pe_host_alloc) is DMA'd; pageable host memory is staged, which drains the stream.  Device memory on another GPU is
 * PE_ERR_INVALID.  Device and page-locked frames must stay unchanged until pe_fetch or pe_sync of this forward returns; work that
 * writes them on another stream is ordered before the forward with pe_stream_wait.  A frame of the display size is converted into
 * the display frame (*scale = 1); any other size is converted at its own size and then warped as pe_forward_camera_frames warps
 * (*scale = frame.scale).  pe_render with display_bgr == NULL draws on the converted display frame.  A format pe_pixels_to_bgr
 * rejects is PE_ERR_INVALID, with the reason in pe_last_error, before anything is queued. */
int pe_forward_pixels(pe_engine* e, const pe_pixel_format* fmt, const void* const* frames, int n, double* scale);
/* later work on e waits for the work queued on cuda_stream (a cudaStream_t of the engine's device; NULL = the legacy default
 * stream) so far: cudaEventRecord there, cudaStreamWaitEvent on the engine's stream.  Nothing blocks the host. */
int pe_stream_wait(pe_engine* e, void* cuda_stream);
/* host reference of pe_forward_pixels's conversion (no GPU): one host frame -> width x height x 3 uint8 BGR when cap suffices.
 * PE_ERR_INVALID for a null pointer, a small cap or a format that fails the checks above; the reason in pe_last_error(NULL). */
int pe_pixels_to_bgr(const pe_pixel_format* fmt, const void* frame, uint8_t* bgr, long long cap);
/* HOST net input as the reference uploads it: n x num_scales x 3 x net_h x net_w fp32 planar
 * (frame.data, rtpose.cpp:1131-1133) */
int pe_forward_net_input(pe_engine* e, const float* net_input, int n);
/* test hook at the concat_stage7 boundary: HOST stride-8 maps n x num_scales x C x net_h/8 x net_w/8;
 * runs resize + NMS + connectLimbs* only (SURVEY.md section 8d "map injection") */
int pe_forward_maps(pe_engine* e, const float* maps8, int n);

/* results of frame `idx` of the last forward.  joints: PE_MAX_PEOPLE x num_parts x 3 (x,y in display pixels,
 * score) as connectLimbs* fills it (rtpose.cpp:1051-1073); peaks (optional): the NMS top blob
 * num_parts x (max_peaks+1) x 3 (nms_layer.cpp:17-29), count in [part][0][0]. */
int pe_fetch(pe_engine* e, int idx, float* joints, int* num_people, float* peaks);
/* stride-8 net output of the last forward, n x num_scales x C x net_h/8 x net_w/8 (blob "concat_stage7") */
int pe_fetch_maps(pe_engine* e, float* maps8, int n);
/* debugging / layer-wise parity: NCHW fp32 copy of an intermediate blob by its prototxt top name, in true values (the range
 * scale of pe_calibrate is divided out).  The stage outputs of the concat buffers that a later stage reuses (for the 6-stage
 * nets: conv5_5_CPM_L1/_L2, Mconv7_stage2_* and Mconv7_stage3_*) are overwritten by every forward: PE_ERR_STATE, and
 * pe_last_error names the layer that reuses the buffer. */
int pe_fetch_blob(pe_engine* e, const char* blob_name, float* out, size_t cap, int* c, int* h, int* w);
/* block until the engine's stream is idle */
int pe_sync(pe_engine* e);

/* page-locked host buffers for frames (the reference `new`s pageable frame buffers, rtpose.cpp:347-354, and pays a
 * staged copy per frame); frames allocated here are DMA'd directly and asynchronously by pe_forward_frames. */
void* pe_host_alloc(size_t bytes);
void pe_host_free(void* p);

/* JSON writer of displayFrame (rtpose.cpp:1383-1416).  Returns the text length (writes if < cap). */
int pe_write_json(const float* joints, int num_people, int num_parts, double frame_scale, char* buf, int cap);

/* Result comparison of two fetched results of one frame (host only, no GPU), e.g. the fast mode against the parity mode.
 * joints_*: people_* x num_parts x 3 as pe_fetch returns them; peaks_*: num_parts x (max_peaks+1) x 3 (count in [part][0][0]).
 * Distances are Euclidean in the units of the inputs (display pixels for pe_fetch).  The results are identical when
 *   - every part has the same peak count in a and b, and peak k of a part lies within tol_px of peak k of b;
 *   - the person counts are equal;
 *   - person i of a has the same present parts (score > 0) as person i of b, each joint within tol_px.
 * Returns PE_OK, or PE_ERR_INVALID for bad arguments. */
typedef struct pe_result_diff {
    int identical;          /* 1 when all three conditions hold */
    int parts_count_differ; /* parts whose peak count differs */
    int peaks_moved;        /* peaks (of parts with equal counts) farther than tol_px from their counterpart */
    int persons_matched;    /* persons i < min(people_a, people_b) with the same present parts */
    float max_joint_dist;   /* largest joint distance over the matched persons */
} pe_result_diff;
int pe_compare_results(const float* joints_a, int people_a, const float* peaks_a, const float* joints_b, int people_b,
                       const float* peaks_b, int num_parts, int max_peaks, float tol_px, pe_result_diff* out);

/* ---- renderers: render() (rtpose.cpp:271-300) + render_mpi_parts / render_coco_parts / render_coco_aff
 * (src/rtpose/renderFunctions.cu:331-389, 978-1080) on the display frame `idx` of the last forward, followed by the
 * float -> uint8 conversion of postProcessFrame (rtpose.cpp:1286-1296).  part_to_show as --part_to_show / the UI keys:
 * 0 = skeletons; MPI: k>0 = heat map of channel k-1; COCO: 1..18 = part heat map, 19 = all parts, 20 = all PAFs,
 * 21..39 = one PAF.  display_bgr: HOST uint8 BGR disp_h x disp_w, or NULL = the frame given to the last
 * pe_forward_frames / _frames_device / _camera_frames (still on the device).  Outputs (either may be NULL): canvas =
 * 3 x disp_h x disp_w float planar BGR (Frame::data_for_mat after render), bgr = disp_h x disp_w x 3 uint8
 * (Frame::data_for_wrap).  After pe_forward_frames_device the caller's device buffer must still be valid.  The cv::putText overlays of displayFrame (rtpose.cpp:1317-1353) are not drawn (= --no_text).
 * Synchronous. */
int pe_render(pe_engine* e, int idx, int part_to_show, int googly_eyes, const uint8_t* display_bgr, float* canvas,
              uint8_t* bgr);

/* render_mpi_parts / render_coco_parts / render_coco_aff with the reference's own DEVICE pointers (include/rtpose/renderFunctions.h:
 * 8-17, call sites rtpose.cpp:277-296): canvas = planar float BGR 3 x h_canvas x w_canvas, heatmaps = full-resolution resized_map
 * (C x h_net x w_net), poses = joints (people x parts x 3), num_people = host array of n_frames counts (frame 0 is rendered, as in
 * the reference).  kind: 0 mpi_parts, 1 coco_parts, 2 coco_aff; extra: googly_eyes (kind 1) / num_parts_accum (kind 2).
 * Runs on the default stream of the current device and synchronises it, like the reference.  C++ callers use the header shim
 * include/rtpose/renderFunctions.h, which has the reference's signatures. */
int pe_render_device(int kind, float* canvas, int w_canvas, int h_canvas, int w_net, int h_net, const float* heatmaps,
                     const float* poses, const int* num_people, int n_frames, int part, int extra);

/* cv::imwrite(fname, frame, {CV_IMWRITE_JPEG_QUALITY, 98}) of displayFrame (rtpose.cpp:1363-1380): baseline JFIF encoder
 * (YCbCr 4:2:0, Annex K tables, libjpeg quality scaling) for the uint8 BGR image pe_render returns.  Host code.  Returns the
 * byte count (the stream is written when it fits in cap), -1 on bad arguments. */
long long pe_encode_jpeg(const uint8_t* bgr, int w, int h, int quality, uint8_t* buf, long long cap);

/* cv::imread of getFrameFromDir (rtpose.cpp:302-391) for .jpg files: Huffman 8-bit JPEG decoder (baseline and progressive) that follows
 * libjpeg's default arithmetic (islow IDCT, fancy chroma upsampling, fixed-point YCbCr->RGB), so the pixels equal what
 * cv::imread returns.  Returns 0 and the image size in *w, *h; pixels (uint8 BGR HWC) are written when bgr != NULL and
 * cap >= w*h*3.  -1: not a JPEG / truncated; -2: arithmetic-coded, lossless, 12-bit, CMYK or unusual chroma sampling. */
int pe_decode_jpeg(const uint8_t* data, long long size, int* w, int* h, uint8_t* bgr, long long cap);

/* ---- JPEG decoding split between host and GPU: the host does only the entropy (Huffman) stage and hands the coefficient image
 * to pe_forward_jpeg_coefs, whose kernels do dequantisation + islow IDCT, fancy chroma upsampling and YCbCr->BGR with
 * pe_decode_jpeg's arithmetic (the pixels are byte-identical).
 * Coefficient image = this 512-byte header followed by the components' int16 coefficients, one after the other (component k
 * at comp[k].offset, comp[0].offset == sizeof(pe_jpeg_coef_header)), each [bh][bw][64] in natural (row-major) order over the
 * MCU-padded block grid: exactly the values libjpeg's IDCT receives. */
#define PE_JPEG_COEF_MAGIC 0x4345504Au /* "JPEC" */
typedef struct pe_jpeg_coef_comp {
    int32_t h, v;        /* sampling factors (1, 1 for a grey image) */
    int32_t bw, bh;      /* blocks per row / column of the MCU-padded plane */
    int32_t dw, dh;      /* real samples of the (downsampled) plane: ceil(width * h / hmax) x ceil(height * v / vmax) */
    int64_t offset;      /* bytes from the start of the buffer to the coefficients */
    uint16_t quant[64];  /* dequantisation table, natural order */
} pe_jpeg_coef_comp;
typedef struct pe_jpeg_coef_header {
    uint32_t magic;      /* PE_JPEG_COEF_MAGIC */
    int32_t width, height;
    int32_t num_comps;   /* 1 (grey) or 3 (YCbCr) */
    int32_t hmax, vmax;  /* largest sampling factors: the MCU is 8*hmax x 8*vmax pixels */
    int64_t total_bytes; /* header + coefficients */
    pe_jpeg_coef_comp comp[3];
} pe_jpeg_coef_header;
/* Entropy stage of pe_decode_jpeg: the coefficient image of a JPEG (host only, thread-safe).  Accepts exactly the files
 * pe_decode_jpeg accepts.  buf == NULL: returns the size needed (parses up to the frame header only).  Otherwise returns the
 * size written; -1 = not a JPEG / truncated / corrupt, or cap too small; -2 = a variant pe_decode_jpeg does not handle. */
long long pe_jpeg_read_coefs(const uint8_t* data, long long size, void* buf, long long cap);
/* host reconstruction of a coefficient image (the same IDCT / upsampling / colour code as pe_decode_jpeg): the reference the GPU
 * kernels are tested against.  Returns 0 and writes width x height x 3 uint8 BGR when cap suffices; -1 = malformed buffer / cap. */
int pe_jpeg_coefs_to_bgr(const void* coefs, uint8_t* bgr, long long cap);

/* ---- JPEG entropy decoding on the GPU: the host parses the headers and finds the restart markers, the GPU decodes the Huffman data
 * into the coefficient image pe_jpeg_read_coefs would write, bit for bit.
 * Scan image = this header, then the segment table at seg_table_offset (num_segments x {int64 offset, int64 length}, offsets from
 * data_offset), then the entropy-coded bytes of the scan at data_offset, still byte-stuffed, RST markers included.  One segment per
 * restart interval (restart_interval == 0: one segment); a segment's bytes end at the first FF xx with xx != 00. */
#define PE_JPEG_SCAN_MAGIC 0x4E43534Au /* "JSCN" */
typedef struct pe_jpeg_scan_header {
    pe_jpeg_coef_header coef; /* the header pe_jpeg_read_coefs writes for this file (geometry, quantisation tables) */
    uint32_t magic;           /* PE_JPEG_SCAN_MAGIC */
    int32_t num_scan_comps;   /* == coef.num_comps */
    int32_t scan_comp[3];     /* SOF index of the scan's k-th component, in SOS order (the order of the blocks in an MCU) */
    int32_t dc_table[3];      /* Huffman table slots of the scan's k-th component */
    int32_t ac_table[3];
    int32_t restart_interval; /* MCUs per segment, 0 = none */
    int32_t mcux, mcuy;       /* MCU grid */
    int32_t num_segments;
    int32_t reserved;
    int64_t seg_table_offset; /* bytes from the start of the buffer */
    int64_t data_offset, data_bytes;
    int64_t total_bytes;      /* header + segment table + data */
    uint8_t dc_bits[4][16], ac_bits[4][16];   /* BITS (codes of length 1..16) of the four DC and four AC slots */
    uint8_t dc_vals[4][256], ac_vals[4][256]; /* HUFFVAL; slots still undefined at the SOS hold the Annex K tables (slots 0, 1) or nothing */
} pe_jpeg_scan_header;
/* The scan image of a JPEG (host only, thread-safe), with pe_jpeg_read_coefs's size-query and cap protocol: buf == NULL returns the
 * size (this parses the whole file).  It covers the streams of pe_jpeg_read_coefs's fast route: SOF0 / SOF1, one scan that names
 * every component once.  -3: valid so far but another kind (progressive, multi-scan): needs the host entropy stage.  Otherwise
 * pe_jpeg_read_coefs's codes; a data error the parser cannot see (a DC category above 15) is reported by the decoder.  Such a
 * stream is one where the codes may differ: pe_jpeg_read_coefs stops at the scan with -1, this call goes on parsing and may
 * return a later header's error instead (e.g. -2 for an SOF3 segment after the scan) or succeed; either way nothing is decoded. */
long long pe_jpeg_read_scan(const uint8_t* data, long long size, void* buf, long long cap);
/* Test hook: the GPU entropy decoder's algorithm run on the host (thread loops in place of threads), subsequences of subseq_bits
 * bits (>= 8).  Writes the coefficient image; returns its size, -1 for a malformed scan image / cap, -4 for data the host entropy
 * stage rejects (a DC category above 15: pe_jpeg_read_coefs returns -1) - the coefficient image is written all the same. */
long long pe_jpeg_scan_to_coefs_host(const void* scan, void* coefs, long long cap, int subseq_bits);

/* same for .png (the third format the reference lists, rtpose.cpp:1743): inflate + PNG filters / Adam7 / all colour types and
 * bit depths, converted as cv::imread(IMREAD_COLOR) does (8-bit BGR, alpha dropped, 16-bit -> high byte). */
int pe_decode_png(const uint8_t* data, long long size, int* w, int* h, uint8_t* bgr, long long cap);

/* cv::VideoCapture of getFrameFromCam for --video (rtpose.cpp:394-411 open / CV_CAP_PROP_FPS / CV_CAP_PROP_POS_FRAMES, :433-446,
 * :525-545 CV_CAP_PROP_FRAME_COUNT, :1677-1682 frame size): RIFF AVI / OpenDML files whose video stream is Motion-JPEG (frames go
 * through pe_decode_jpeg) or uncompressed 24/32-bit DIB.  Other containers / inter-frame codecs: PE_ERR_INVALID, the FourCC in
 * pe_video_last_error() (thread-local).  Frames are addressed by index, pe_video_read is thread-safe on one handle; pixels are
 * uint8 BGR HWC of the video's own size (pe_forward_camera_frames scales them to the display size like the reference's warpAffine). */
typedef struct pe_video pe_video;
int pe_video_open(const char* path, pe_video** out);
void pe_video_close(pe_video* v);
int pe_video_info(const pe_video* v, int* w, int* h, double* fps, int* frame_count, char fourcc[5]);
int pe_video_read(const pe_video* v, int index, uint8_t* bgr, long long cap);
/* Motion-JPEG videos: frame `index` as a coefficient image (pe_jpeg_read_coefs) for pe_forward_jpeg_coefs.  Returns its size; it is
 * written when buf != NULL and cap >= size (call again with a larger buffer otherwise).  -PE_ERR_INVALID: not a Motion-JPEG video,
 * bad index, a JPEG variant the decoder does not handle; -PE_ERR_IO: unreadable / corrupt frame (text in pe_video_last_error()). */
long long pe_video_read_coefs(const pe_video* v, int index, void* buf, long long cap);
/* the same as a scan image (pe_jpeg_read_scan) for pe_forward_jpeg_scans.  A frame that needs the host entropy stage (progressive,
 * multi-scan) gives -3, as pe_jpeg_read_scan; this call never returns -PE_ERR_STATE, so -3 always has that meaning here. */
long long pe_video_read_scan(const pe_video* v, int index, void* buf, long long cap);
const char* pe_video_last_error(void);

/* cv::VideoCapture on a camera index (rtpose.cpp:401-405 cap.open(FLAGS_camera) + CV_CAP_PROP_FRAME_WIDTH/HEIGHT from
 * --camera_resolution, :431 cap >> image): Video4Linux2 streaming capture from /dev/video<index>, Motion-JPEG (pe_decode_jpeg) or YUYV
 * frames.  pe_camera_grab blocks for the next frame (timeout_ms <= 0: 5 s) and returns it as uint8 BGR HWC of the size
 * pe_camera_info reports (the driver may grant another size than asked for).  Errors: PE_ERR_IO / PE_ERR_INVALID, text in
 * pe_camera_last_error() (thread-local; "Couldn't open camera N ..." as the reference's CHECK).
 * pe_yuyv_to_bgr: cv::cvtColor(COLOR_YUV2BGR_YUYV), the conversion OpenCV's V4L2 back end applies to YUYV frames. */
typedef struct pe_camera pe_camera;
int pe_camera_open(int index, int want_w, int want_h, pe_camera** out);
void pe_camera_close(pe_camera* c);
int pe_camera_info(const pe_camera* c, int* w, int* h, char fourcc[5]);
int pe_camera_grab(pe_camera* c, uint8_t* bgr, long long cap, int timeout_ms);
const char* pe_camera_last_error(void);
int pe_yuyv_to_bgr(const uint8_t* yuyv, int w, int h, long long stride, uint8_t* bgr);

/* ---- model descriptor tables (modelDescriptorFactory.cpp:6-28,30-55) */
int pe_model_num_parts(int model);
int pe_model_num_limbs(int model);
const int* pe_model_limb_sequence(int model);
const int* pe_model_map_idx(int model);
const char* pe_model_part_name(int model, int idx);

/* ---- measurement support (bench.py) */
/* device time, CUDA events on the engine stream: slot in [0,16) */
int pe_event_record(pe_engine* e, int slot);
int pe_event_elapsed_ms(pe_engine* e, int slot_a, int slot_b, float* ms);
/* one instrumented forward of the last-submitted batch: per conv-layer device ms (events between launches).
 * names: 64 bytes per layer.  Returns the number of ops written (<= cap). */
int pe_profile_layers(pe_engine* e, int n, float* ms, char* names, double* flops, int cap);
/* kernels launched by this handle since creation (for the bench's gpu_launches claim) */
long long pe_launch_count(const pe_engine* e);
/* algorithmic conv FLOPs of one frame-scale at the configured net size (SURVEY.md section 8d) */
double pe_conv_flops_per_scale(const pe_engine* e);
/* one-time weight replica broadcast for --num_gpu N frame sharding (rank 0's packed weights -> all):
 * exports / imports the packed device buffer so that the host layer (NCCL via torch.distributed or
 * ncclBroadcast in rtpose.bin) can move it.  Returns size in bytes. */
size_t pe_packed_weights_bytes(const pe_engine* e);
/* single-process --num_gpu N: engines[0]'s committed weights -> engines[1..n-1] (one handle per GPU) with one grouped
 * ncclBroadcast over NVLink instead of N file reads (rtpose.cpp:183-184).  The path's only collective. */
int pe_broadcast_weights(pe_engine* const* engines, int n);
void* pe_packed_weights_device_ptr(pe_engine* e);

#ifdef __cplusplus
}
#endif
#endif
