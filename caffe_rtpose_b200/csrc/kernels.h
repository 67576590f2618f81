// Device-side structs and host launchers of the engine's kernels (internal).
#pragma once
#include <cuda_fp8.h>

#include "common.h"
#include "pixels.cuh"    // pe_pix::Colour: the matrix and range of a decoder-format frame
#include "precision.h"   // PlaneFmt: the storage format of the conv stack's activations and packed weights

namespace pe {

#ifdef __CUDACC__
__device__ __forceinline__ float e4m3_to_float(uint8_t b) {
    return __half2float(__half(__nv_cvt_fp8_to_halfraw((__nv_fp8_storage_t)b, __NV_E4M3)));
}
template <bool F16> __device__ __forceinline__ float plane_to_float(uint16_t h) {
    return F16 ? __half2float(__ushort_as_half(h)) : __uint_as_float((uint32_t)h << 16);
}
template <bool F16> __device__ __forceinline__ uint16_t float_to_plane(float x) {
    return F16 ? __half_as_ushort(__float2half_rn(x)) : __bfloat16_as_ushort(__float2bfloat16_rn(x));
}
// two floats -> packed pair of plane values (low half = a) and the residuals a - hi(a), b - hi(b)
template <bool F16> __device__ __forceinline__ uint32_t split_pair(float& a, float& b) {
    if (F16) {
        const __half2 h = __floats2half2_rn(a, b);
        a = __fsub_rn(a, __low2float(h));
        b = __fsub_rn(b, __high2float(h));
        return *reinterpret_cast<const uint32_t*>(&h);
    } else {
        const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
        const uint32_t hu = *reinterpret_cast<const uint32_t*>(&h);
        a = __fsub_rn(a, __uint_as_float(hu << 16));
        b = __fsub_rn(b, __uint_as_float(hu & 0xffff0000u));
        return hu;
    }
}
#endif


struct AxisTap { int i0, i1, i2, i3; float d; };
struct Cand { float conn; int p; };
struct Conn { int a, b; float score; };
struct ModelDev { int limb_seq[40]; int map_idx[40]; };
struct FlipTap { int ch; float sign; };   // the flip test: channel c of the average reads channel ch of a mirrored copy, times sign

struct PostDev {
    PostParams p;
    ModelDev md;
    const float* maps;        // [frames][copies][C][h8][w8]
    int copies;               // stride-8 copies per frame: the S scales, then with the flip test the S mirrored ones
    const FlipTap* flip;      // [C] (model_flip_table)
    const AxisTap* xtab;      // [S][net_w]
    const AxisTap* ytab;      // [S][net_h]
    unsigned* flags;          // [frames][parts][net_h][ceil(net_w/32)]
    float* peaks;             // [frames][parts][max_peaks+1][3]
    Cand* cands;              // [frames][limbs][max_peaks^2]
    int* cand_count;          // [frames][limbs]
    int sort_stride;          // next_pow2(max_peaks^2): sort keys per limb (dynamic shared memory of limb_greedy_kernel)
    Conn* conns;              // [frames][limbs][max_peaks]
    int* conn_count;          // [frames][limbs]
    double* subset;           // [frames][p.max_subset_rows][parts+3]
    int* subset_rows;         // [frames]
    float* joints;            // [frames][PE_MAX_PEOPLE][parts][3]
    int* num_people;          // [frames]
};

void launch_axis_tables(AxisTap* xtab, AxisTap* ytab, const PostParams& p, cudaStream_t st);
int launch_post(const PostDev& pd, int nframes, cudaStream_t st);
cudaError_t post_set_smem_limits();   // on the current device, before the first launch_post

// ---- renderers (render.cu)
int launch_canvas_fill(const uint8_t* bgr, float* canvas, int w, int h, cudaStream_t st);
int launch_canvas_to_u8(const float* canvas, uint8_t* bgr, int w, int h, cudaStream_t st);
int launch_fullres_fill(const PostDev& pd, int frame, int ch0, int nch, float* out, cudaStream_t st);
int launch_skeleton(int model, float* canvas, int w, int h, const float* poses, const int* num_people, int googly, cudaStream_t st,
                    int num_people_host = 0);   // num_people == nullptr: the count is num_people_host
// mode 0: MPI part map, 1: COCO part map, 2: COCO all parts, 3: COCO PAF (render.cu)
int launch_heat_view(float* canvas, int w, int h, float* heat, int w_net, int h_net, int mode, int part, int nch, cudaStream_t st);

// ---- preprocessing (pre.cu)
struct AreaTab {           // OpenCV INTER_AREA decimation tables for one scale, device pointers
    const int* x_ofs; const int* x_si; const float* x_alpha;   // per dst x: [x_ofs[dx], x_ofs[dx+1]) entries
    const int* y_ofs; const int* y_si; const float* y_alpha;
    const int* lin_x; const int* lin_y;                       // linear "area mode" (an axis enlarges): [d][3] = src index, a0, a1
    int tw, th, padw, padh, fast, iscale_x, iscale_y, linear;
};
struct PreArgs {
    const uint8_t* frames;    // [nframes][disp_h][disp_w][3] BGR
    uint8_t* resized;         // [nframes][S][net_h][net_w][3] scratch (only th x tw used)
    AreaTab tab[PE_MAX_SCALES];
    int nframes, S, disp_w, disp_h, net_w, net_h;
    int flip;                 // the flip test: frame f's scale s goes to image 2Sf + s, its mirror in x to image 2Sf + S + s
    // im2col'ed network input, flat padded level-0 geometry
    void* out; int kp; long long out_plane; PlaneFmt fmt;
    int Wp, Hs;
};
int launch_preprocess(const PreArgs& a, cudaStream_t st);
struct WarpArgs {
    const uint8_t* src; uint8_t* dst; int sw, sh, dw, dh;
    const int* adelta; const int* bdelta; const int* x0; const int* y0;   // OpenCV's fixed-point coordinate tables
    const short* tab;                                                      // [32*32][16] bicubic weights
};
int launch_warp_affine(const WarpArgs& a, int nframes, cudaStream_t st);
// planar fp32 net input [N][3][H][W] -> im2col'ed input
int launch_input_from_planar(const float* planar, const PreArgs& a, int nimages, cudaStream_t st);

// ---- JPEG reconstruction (jpeg_gpu.cu): coefficient images of pe_jpeg_read_coefs -> BGR frames
struct JpegArgs {
    const uint8_t* coefs; long long coef_stride;    // [n] coefficient images (pe_jpeg_coef_header + int16), 256-byte aligned
    uint8_t* planes; long long plane_stride;        // [n] component planes: byte 64 * b + k = sample k of block b (coefficient order)
    uint8_t* dst;                                   // [n][H][W][3] uint8 BGR
    int W, H, n;
    long long max_blocks;                           // largest block count of a frame in the batch
};
int launch_jpeg_reconstruct(const JpegArgs& a, cudaStream_t st);   // dequantise + IDCT, then upsample + colour: 2 launches

// ---- JPEG entropy decoding (jpeg_entropy.cu): scan images of pe_jpeg_read_scan -> coefficient images
struct JpegScanArgs {
    const uint8_t* scans; long long scan_stride;    // [n] scan images (checked on the host), 256-byte aligned
    uint8_t* coefs; long long coef_stride;          // [n] coefficient images, zeroed before the launch
    void* tabs;                                     // [n][8] decoder tables (jpeg_huff_tables_bytes() per frame)
    int* seg_sub; long long seg_stride;             // [n][num_segments + 1] first subsequence of every segment
    unsigned long long* pub; int* flags; int ctas_max;   // [n][ctas_max] hand-over between the CTAs of a frame: state, block; flag
    int* tickets;                                   // [n] CTA order
    int* status;                                    // [n] first MCU with a DC category above 15, INT_MAX = none
    int n, S;                                       // frames, subsequence bits
};
size_t jpeg_huff_tables_bytes();
int launch_jpeg_entropy(const JpegScanArgs& a, cudaStream_t st);   // 3 launches

// ---- decoder-format frames (pixels.cu): pe_pixel_format frames -> tight uint8 BGR
constexpr int PIX_MAX_FRAMES = 64;                  // = the largest max_batch: the pointer table travels in the kernel parameters
struct PixArgs {
    const uint8_t* src[PIX_MAX_FRAMES];             // [n] frame starts (device pointers; the host reference reads src[0])
    uint8_t* dst;                                   // [n][h][w][3]
    long long pitch, chroma;                        // a checked pe_pix::Layout's
    int format, w, h;                               // format: PE_PIX_* without the colour flags
    pe_pix::Colour col;                             // the matrix and range the flags chose
};
int launch_pixels_to_bgr(const PixArgs& a, int n, cudaStream_t st);   // every format but PE_PIX_BGR
void pixels_to_bgr_host(const PixArgs& a);                         // every format, frame src[0]

// ---- convolution / pooling (conv_simt.cu, conv_tc.cu, pool.cu)
int launch_conv_simt(const ConvArgs& a, cudaStream_t st);
struct PoolArgs {
    const void* in; void* out; int C; long long in_plane, out_plane; PlaneFmt fmt;
    int Wi, Hi, Wpi, Hsi, Wo, Ho, Wpo, Hso, N;
};
int launch_pool(const PoolArgs& a, cudaStream_t st);
struct CopyArgs { const void* src; void* dst; int pitch, channels, elem_bytes; long long M, plane; PlaneFmt fmt; };
int launch_copy_channels(const CopyArgs& a, cudaStream_t st);
// activation (flat padded, fp32 or 16-bit planes) -> NCHW fp32 (debug / pe_fetch_blob); scale: the inverse of the power-of-two
// range scale the stored values carry (engine.cu, fill_epilogue_fields), so that out holds true values
int launch_act_to_nchw(const void* act, int pitch, int coff, int c, long long plane, PlaneFmt fmt, const Geo& g, float scale,
                       float* out, cudaStream_t st);

}  // namespace pe
