// rtpose.bin - host pipeline over libposeengine.so with the reference's command line
// (examples/rtpose/rtpose.cpp:50-72 flags; :1459-1549 thread topology: one producer, --num_gpu workers each
// owning one engine handle, one re-orderer, one writer).  Host code is plain C++17 (the reference's gflags / glog /
// boost / OpenCV are not available here and are not needed for this path); all math is behind the C ABI.
//
// Supported sources: --image_dir with .jpg / .png / .bmp / .ppm files (own decoders behind the C ABI, pixels identical to
// cv::imread), --video with Motion-JPEG / uncompressed .avi files (csrc/video.cpp), the camera (--camera N: Video4Linux2 capture,
// csrc/camera.cpp), or --synthetic N procedural frames.  Other video codecs need a codec library and are rejected
// with an explicit message; there is no window, so the keyboard UI of handleKey (rtpose.cpp:1551-1671) is served from stdin
// with --keys_from_stdin (same key characters, same step sizes).  --write_frames renders on the GPU (pe_render) and writes
// quality-98 .jpg files like the reference (pe_encode_jpeg; --frame_format bmp for lossless) with displayFrame's text overlays
// (own bitmap font, --no_text turns them off).
// Frames older than 0.1 s are dropped unless --no_frame_drops, as in processFrame (rtpose.cpp:1107-1124).
#include <climits>
#include <dirent.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/stat.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <fstream>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <queue>
#include <string>
#include <thread>
#include <vector>

#include "caffe/cpm/layers/imresize_layer.hpp"
#include "caffe/cpm/layers/nms_layer.hpp"
#include "poseengine.h"
#include "rtpose/modelDescriptorFactory.h"

// ---------------------------------------------------------------------------------------------- flags
struct Flag { std::string value, help; bool is_bool; };
static std::map<std::string, Flag> g_flags;
static void define(const char* name, const char* dflt, const char* help, bool is_bool = false) { g_flags[name] = {dflt, help, is_bool}; }
static std::string F(const char* n) { return g_flags.at(n).value; }
static int Fi(const char* n) { return atoi(F(n).c_str()); }
static double Fd(const char* n) { return atof(F(n).c_str()); }
static bool Fb(const char* n) { const std::string v = F(n); return v == "true" || v == "1"; }

static void define_flags() {
    // names, defaults and help strings of rtpose.cpp:50-72
    define("fullscreen", "false", "Run in fullscreen mode (press f during runtime to toggle)", true);
    define("part_to_show", "0", "Part to show from the start.");
    define("write_frames", "", "Write frames with format prefix%06d.jpg");
    define("probe_image", "", "[extension] decode this image file, print WxH and an FNV-1a hash of the BGR pixels, exit (no GPU)");
    define("num_producers", "0", "[extension] decoder threads for --image_dir / --synthetic: 1 = the reference's single producer, 0 = automatic "
           "(with automatic --batch: 10 per GPU, at most 48 and the host's cores minus the worker threads - one H100 consumes 200-300 frames/s, a thread decodes ~100)");
    define("decode_bench", "false", "[extension] run only the producer stage (decode + queue), print frames/s, exit (no GPU)", true);
    define("gpu_decode", "false", "[extension] JPEG sources (--image_dir .jpg files, Motion-JPEG --video): the producer threads run only the "
           "entropy (Huffman) stage; dequantisation, IDCT, chroma upsampling and colour conversion run on the GPU (pixels identical to the host "
           "decoder). Other files and JPEGs it does not take are decoded on the host as without it", true);
    define("gpu_entropy", "false", "[extension] as --gpu_decode, and for sequential JPEGs (one interleaved scan: cameras, Motion-JPEG, "
           "cv::imwrite) the producer threads only parse the file; the Huffman decoding runs on the GPU too. Progressive / multi-scan "
           "JPEGs take the --gpu_decode route, other files the host decoder", true);
    define("frame_format", "jpg", "[extension] jpg (quality 98, as the reference) or bmp (lossless) for --write_frames");
    define("no_frame_drops", "false", "Dont drop frames.", true);
    define("write_json", "", "Write joint data with json format as prefix%06d.json");
    define("camera", "0", "The camera index for VideoCapture.");
    define("video", "", "Use a video file instead of the camera.");
    define("video_realtime", "true", "[extension] --video: true = the reference's pacing (frames are committed at the file's frame rate, "
           "rtpose.cpp:446-462) and its single producer; false = decode as fast as the GPUs consume (offline processing, combine with "
           "--no_frame_drops)", true);
    define("image_dir", "", "Process a directory of images.");
    define("start_frame", "0", "Skip to frame # of video");
    define("caffemodel", "model/coco/pose_iter_440000.caffemodel", "Caffe model.");
    define("caffeproto", "model/coco/pose_deploy_linevec.prototxt", "Caffe deploy prototxt.");
    define("resolution", "1280x720", "The image resolution (display).");
    define("net_resolution", "656x368", "Multiples of 16.");
    define("camera_resolution", "1280x720", "Size of the camera frames to ask for.");
    define("start_device", "0", "GPU device start number.");
    define("num_gpu", "1", "The number of GPU devices to use.");
    define("start_scale", "1", "Initial scale. Must cv::Match net_resolution");
    define("scale_gap", "0.3", "Scale gap between scales. No effect unless num_scales>1");
    define("num_scales", "1", "Number of scales to average");
    define("no_display", "false", "Do not open a display window.", true);
    define("no_text", "false", "Do not write text on output images.", true);
    define("logtostderr", "false", "glog compatibility: log to stderr", true);
    // extensions of this implementation (not in the reference)
    define("synthetic", "0", "[extension] process N procedurally generated frames instead of a camera/video/image_dir");
    define("random_init", "", "[extension] 'he' or 'caffe': random weights instead of --caffemodel (no checkpoint offline)");
    define("model", "", "[extension] COCO or MPI when --caffeproto is not readable");
    define("precision", "2", "[extension] conv arithmetic: 0 fp32 SIMT, 1 bf16 (A/B only), 2 parity mode (two fp16 planes, 3 MMAs per MAC), "
           "3 three bf16 planes (A/B only), 4 fast mode (one fp16 plane, 1 MMA per MAC; see --audit_every)");
    define("batch", "0", "[extension] frames per forward per GPU: 1 = the reference's behaviour, 0 = automatic (file / synthetic sources "
           "fill two waves of 128-row tiles on the GPU, e.g. 9 frames at 656x368; results do not depend on it)");
    define("engines_per_gpu", "0", "[extension] worker handles per GPU: 1 = the reference's topology (one Net per GPU), 0 = automatic (2 when "
           "--batch is automatic: the copies and the kernel tails of one batch overlap the other; weights are shared, not duplicated)");
    define("calibrate_range", "true", "[extension] fp16 modes (--precision 2 and 4): derive per-layer power-of-two activation scales from one synthetic frame at start-up "
           "(pe_calibrate), so that a model of any magnitude keeps fp32-level results", true);
    define("audit_every", "0", "[extension] N > 0: every worker also holds a parity-mode (--precision 2) handle and forwards every N-th batch "
           "through it too; each frame's peaks, person count and joints are compared with the fast handle's (within 1e-3 net px). The status "
           "line reports how many frames agree, and a summary is printed at exit. Output stays the --precision handle's. 0 = off");
    define("num_writers", "0", "[extension] threads that format / encode and write the --write_json and --write_frames files (a quality-98 720p JPEG takes ~20 ms to encode): "
           "1 = on the display thread like the reference, 0 = automatic (a quarter of the host's cores, at most 16)");
    define("keys_from_stdin", "false", "[extension] read the reference's runtime keys (- = _ + [ ] { } ; ' , . 0-9 q-p a s, ESC or Q to quit) from stdin", true);
}

static int parse_flags(int argc, char** argv) {
    for (int i = 1; i < argc; i++) {
        std::string a = argv[i];
        if (a == "--help" || a == "-help") {
            for (auto& kv : g_flags) printf("  --%s (%s) default: \"%s\"\n", kv.first.c_str(), kv.second.help.c_str(), kv.second.value.c_str());
            exit(0);
        }
        if (a.rfind("--", 0) != 0 && a.rfind("-", 0) == 0) a = "-" + a;   // gflags accepts -flag too
        if (a.rfind("--", 0) != 0) { fprintf(stderr, "ERROR: unexpected argument '%s'\n", argv[i]); return 1; }
        a = a.substr(2);
        std::string name = a, value;
        bool has_value = false;
        const size_t eq = a.find('=');
        if (eq != std::string::npos) { name = a.substr(0, eq); value = a.substr(eq + 1); has_value = true; }
        if (!g_flags.count(name) && name.rfind("no", 0) == 0 && g_flags.count(name.substr(2)) && g_flags[name.substr(2)].is_bool) {
            g_flags[name.substr(2)].value = "false";   // gflags --noflag
            continue;
        }
        if (!g_flags.count(name)) { fprintf(stderr, "ERROR: unknown command line flag '%s'\n", name.c_str()); return 1; }
        Flag& f = g_flags[name];
        if (f.is_bool && !has_value) { f.value = "true"; continue; }
        if (!has_value) {
            if (i + 1 >= argc) { fprintf(stderr, "ERROR: flag '--%s' is missing its argument\n", name.c_str()); return 1; }
            value = argv[++i];
        }
        f.value = value;
    }
    return 0;
}

// one write per line: producers, workers, the key reader and the display thread all log, and a line must not be cut by another one
static void log_line(char level, const char* fmt, ...) __attribute__((format(printf, 2, 3)));
static void log_line(char level, const char* fmt, ...) {
    char buf[2048];
    int n = snprintf(buf, sizeof buf, "%c rtpose] ", level);
    va_list ap;
    va_start(ap, fmt);
    const int m = vsnprintf(buf + n, sizeof buf - (size_t)n - 1, fmt, ap);
    va_end(ap);
    n += m < 0 ? 0 : std::min(m, (int)sizeof buf - n - 2);
    buf[n++] = '\n';
    fwrite(buf, 1, (size_t)n, stderr);
}
#define LOG_INFO(...) log_line('I', __VA_ARGS__)
#define LOG_ERROR(...) log_line('E', __VA_ARGS__)

// ---------------------------------------------------------------------------------------------- frames
struct Frame {
    int index = 0, video_frame_number = 0, w = 0, h = 0;
    double scale = 1.0;                      // display / original (rtpose.cpp:474-480), filled by the engine
    std::vector<uint8_t> bgr;                // display image, HWC BGR (decode buffer)
    std::shared_ptr<uint8_t> pinned;         // same image in page-locked memory (pe_host_alloc) for direct async DMA
    enum Kind { PIXELS, COEFS, SCAN };
    Kind kind = PIXELS;                      // COEFS (--gpu_decode): `pinned` holds the JPEG's coefficient image (pe_jpeg_read_coefs);
                                             // SCAN (--gpu_entropy): its scan image (pe_jpeg_read_scan)
    std::string stem;                        // for <stem>.json with --image_dir
    int num_people = 0;
    std::vector<float> joints;
    std::vector<uint8_t> rendered;           // --write_frames: display image with overlays (pe_render), HWC BGR
    // stage clocks of the reference's latency line (rtpose.cpp:1421-1441)
    double t_commit = 0, t_preprocessed = 0, t_fetched = 0, t_done = 0, t_out_popped = 0, t_buffered = 0;   // t_commit: capture / decode start
};

static double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

static bool read_ppm(const std::string& path, int& w, int& h, std::vector<uint8_t>& bgr) {
    FILE* f = fopen(path.c_str(), "rb");
    if (!f) return false;
    char magic[3] = {0};
    int maxv = 0;
    if (fscanf(f, "%2s", magic) != 1 || strcmp(magic, "P6")) { fclose(f); return false; }
    int vals[3], got = 0;
    while (got < 3) {
        int c = fgetc(f);
        if (c == '#') { while (c != '\n' && c != EOF) c = fgetc(f); continue; }
        if (c == EOF) { fclose(f); return false; }
        if (c >= '0' && c <= '9') { ungetc(c, f); if (fscanf(f, "%d", &vals[got]) != 1) { fclose(f); return false; } got++; }
    }
    w = vals[0]; h = vals[1]; maxv = vals[2];
    fgetc(f);
    if (maxv != 255 || w <= 0 || h <= 0 || (long long)w * h > (1LL << 28)) { fclose(f); return false; }
    std::vector<uint8_t> rgb((size_t)w * h * 3);
    const bool ok = fread(rgb.data(), 1, rgb.size(), f) == rgb.size();
    fclose(f);
    if (!ok) return false;
    bgr.resize(rgb.size());
    for (size_t i = 0; i < rgb.size(); i += 3) { bgr[i] = rgb[i + 2]; bgr[i + 1] = rgb[i + 1]; bgr[i + 2] = rgb[i]; }
    return true;
}

static bool read_bmp(const std::string& path, int& w, int& h, std::vector<uint8_t>& bgr) {
    FILE* f = fopen(path.c_str(), "rb");
    if (!f) return false;
    uint8_t hd[54];
    if (fread(hd, 1, 54, f) != 54 || hd[0] != 'B' || hd[1] != 'M') { fclose(f); return false; }
    const uint32_t off = hd[10] | (hd[11] << 8) | (hd[12] << 16) | ((uint32_t)hd[13] << 24);
    const int32_t bw = (int32_t)(hd[18] | (hd[19] << 8) | (hd[20] << 16) | ((uint32_t)hd[21] << 24));
    const int32_t bh = (int32_t)(hd[22] | (hd[23] << 8) | (hd[24] << 16) | ((uint32_t)hd[25] << 24));
    const int bpp = hd[28] | (hd[29] << 8), comp = hd[30];
    if (bpp != 24 || comp != 0 || bw <= 0 || bh == 0 || bh == INT32_MIN || (long long)bw * (bh < 0 ? -(long long)bh : bh) > (1LL << 28)) { fclose(f); return false; }
    w = bw; h = bh < 0 ? -bh : bh;
    const size_t stride = ((size_t)w * 3 + 3) & ~(size_t)3;
    std::vector<uint8_t> row(stride);
    bgr.resize((size_t)w * h * 3);
    fseek(f, off, SEEK_SET);
    for (int y = 0; y < h; y++) {
        if (fread(row.data(), 1, stride, f) != stride) { fclose(f); return false; }
        const int dy = bh < 0 ? y : h - 1 - y;   // bottom-up unless the height is negative
        memcpy(&bgr[(size_t)dy * w * 3], row.data(), (size_t)w * 3);
    }
    fclose(f);
    return true;
}

static std::string lower_ext(const std::string& p) {
    const size_t dot = p.find_last_of('.');
    std::string e = dot == std::string::npos ? "" : p.substr(dot);
    for (auto& c : e) c = (char)tolower((unsigned char)c);
    return e;
}

// cv::imread (rtpose.cpp:302-391): the decoder is chosen by the file's signature, not its name
// dst_alloc (optional): where the pixels of a .jpg / .png should go (a page-locked buffer of the given size, or nullptr); when it
// delivers one, the decoder writes there directly, *dst is set and bgr stays empty - no staging copy of 2.7 MB per 720p frame
static bool read_image(const std::string& path, int& w, int& h, std::vector<uint8_t>& bgr, const std::function<uint8_t*(size_t)>* dst_alloc = nullptr,
                       uint8_t** dst = nullptr) {
    FILE* f = fopen(path.c_str(), "rb");
    if (!f) return false;
    uint8_t magic[8] = {0};
    const size_t got = fread(magic, 1, 8, f);
    const bool jpg = got >= 2 && magic[0] == 0xFF && magic[1] == 0xD8;
    const bool png = got >= 8 && magic[0] == 0x89 && magic[1] == 'P' && magic[2] == 'N' && magic[3] == 'G';
    if (!jpg && !png) {
        fclose(f);
        return got >= 2 && magic[0] == 'P' && magic[1] == '6' ? read_ppm(path, w, h, bgr) : read_bmp(path, w, h, bgr);
    }
    fseek(f, 0, SEEK_END);
    const long n = ftell(f);
    fseek(f, 0, SEEK_SET);
    std::vector<uint8_t> data((size_t)std::max(n, 0L));
    const bool rd = n > 0 && fread(data.data(), 1, (size_t)n, f) == (size_t)n;
    fclose(f);
    if (!rd) return false;
    auto dec = jpg ? pe_decode_jpeg : pe_decode_png;
    int rc = dec(data.data(), n, &w, &h, nullptr, 0);
    if (rc == 0 && (long long)w * h > (1LL << 28)) { LOG_ERROR("%s: %dx%d is larger than this build accepts", path.c_str(), w, h); return false; }
    if (rc == 0) {
        const size_t bytes = (size_t)w * h * 3;
        uint8_t* out = dst_alloc ? (*dst_alloc)(bytes) : nullptr;
        if (out) *dst = out;
        else { bgr.resize(bytes); out = bgr.data(); }
        rc = dec(data.data(), n, &w, &h, out, (long long)bytes);
    }
    if (rc == -2) LOG_ERROR("%s: JPEG variant not handled (arithmetic-coded / lossless / 12-bit / CMYK / unusual chroma sampling)", path.c_str());
    return rc == 0;
}

static bool write_bmp(const std::string& path, int w, int h, const uint8_t* bgr) {   // 24-bit, bottom-up
    FILE* f = fopen(path.c_str(), "wb");
    if (!f) return false;
    const uint32_t stride = ((uint32_t)w * 3 + 3) & ~3u, size = 54 + stride * (uint32_t)h;
    uint8_t hd[54] = {'B', 'M'};
    auto put32 = [&](int o, uint32_t v) { hd[o] = v & 255; hd[o + 1] = (v >> 8) & 255; hd[o + 2] = (v >> 16) & 255; hd[o + 3] = (v >> 24) & 255; };
    put32(2, size); put32(10, 54); put32(14, 40); put32(18, (uint32_t)w); put32(22, (uint32_t)h);
    hd[26] = 1; hd[28] = 24; put32(34, stride * (uint32_t)h); put32(38, 2835); put32(42, 2835);
    fwrite(hd, 1, 54, f);
    std::vector<uint8_t> row(stride, 0);
    for (int y = h - 1; y >= 0; y--) {
        memcpy(row.data(), bgr + (size_t)y * w * 3, (size_t)w * 3);
        fwrite(row.data(), 1, stride, f);
    }
    fclose(f);
    return true;
}

static void synthetic_frame(int idx, int w, int h, std::vector<uint8_t>& bgr) {
    bgr.resize((size_t)w * h * 3);
    // low-frequency pattern 128 + 100 sin((x + 31 c) / 41) cos((y + 17 idx) / 57) plus LCG noise; the two factors are tabulated per
    // column and per row (the products are the same doubles as when both are evaluated per pixel: 17 -> ~200 frames/s per thread at 720p)
    std::vector<double> sx((size_t)w * 3), cy((size_t)h);
    for (int x = 0; x < w; x++)
        for (int c = 0; c < 3; c++) sx[(size_t)x * 3 + c] = 100.0 * sin((x + 31 * c) / 41.0);
    for (int y = 0; y < h; y++) cy[y] = cos((y + 17 * idx) / 57.0);
    uint32_t s = 0x9E3779B9u * (uint32_t)(idx + 1);
    for (int y = 0; y < h; y++) {
        uint8_t* row = &bgr[(size_t)y * w * 3];
        const double cyy = cy[y];
        for (int i = 0; i < w * 3; i++) {
            s = s * 1664525u + 1013904223u;
            const int low = 128 + (int)(sx[i] * cyy);
            row[i] = (uint8_t)std::min(255, std::max(0, (low + (int)(s >> 24)) / 2));
        }
    }
}

// ---------------------------------------------------------------------------------------------- text overlays
// displayFrame's cv::putText lines (rtpose.cpp:1317-1353): "%4.1f fps" (or "%4.2f s/gpu" with --write_frames) at (25, 35), the
// people count at the top right with a black shadow, the name of the shown part at (W - 175, 55); switched off by --no_text.
// cv::putText draws OpenCV's Hershey strokes (third-party font data); this is a 5x7 bitmap font of our own, scaled to the same
// cap height, so the overlays carry the same information at the same places but are not pixel-identical to OpenCV's.
static const unsigned char kFont5x7[][5] = {   // columns, LSB = top row; ASCII 32..122 subset, missing glyphs are blank
    {0x00,0x00,0x00,0x00,0x00},{0x00,0x00,0x5F,0x00,0x00},{0x00,0x07,0x00,0x07,0x00},{0x14,0x7F,0x14,0x7F,0x14},{0x24,0x2A,0x7F,0x2A,0x12},
    {0x23,0x13,0x08,0x64,0x62},{0x36,0x49,0x55,0x22,0x50},{0x00,0x05,0x03,0x00,0x00},{0x00,0x1C,0x22,0x41,0x00},{0x00,0x41,0x22,0x1C,0x00},
    {0x14,0x08,0x3E,0x08,0x14},{0x08,0x08,0x3E,0x08,0x08},{0x00,0x50,0x30,0x00,0x00},{0x08,0x08,0x08,0x08,0x08},{0x00,0x60,0x60,0x00,0x00},
    {0x20,0x10,0x08,0x04,0x02},{0x3E,0x51,0x49,0x45,0x3E},{0x00,0x42,0x7F,0x40,0x00},{0x42,0x61,0x51,0x49,0x46},{0x21,0x41,0x45,0x4B,0x31},
    {0x18,0x14,0x12,0x7F,0x10},{0x27,0x45,0x45,0x45,0x39},{0x3C,0x4A,0x49,0x49,0x30},{0x01,0x71,0x09,0x05,0x03},{0x36,0x49,0x49,0x49,0x36},
    {0x06,0x49,0x49,0x29,0x1E},{0x00,0x36,0x36,0x00,0x00},{0x00,0x56,0x36,0x00,0x00},{0x08,0x14,0x22,0x41,0x00},{0x14,0x14,0x14,0x14,0x14},
    {0x00,0x41,0x22,0x14,0x08},{0x02,0x01,0x51,0x09,0x06},{0x32,0x49,0x79,0x41,0x3E},{0x7E,0x11,0x11,0x11,0x7E},{0x7F,0x49,0x49,0x49,0x36},
    {0x3E,0x41,0x41,0x41,0x22},{0x7F,0x41,0x41,0x22,0x1C},{0x7F,0x49,0x49,0x49,0x41},{0x7F,0x09,0x09,0x09,0x01},{0x3E,0x41,0x49,0x49,0x7A},
    {0x7F,0x08,0x08,0x08,0x7F},{0x00,0x41,0x7F,0x41,0x00},{0x20,0x40,0x41,0x3F,0x01},{0x7F,0x08,0x14,0x22,0x41},{0x7F,0x40,0x40,0x40,0x40},
    {0x7F,0x02,0x0C,0x02,0x7F},{0x7F,0x04,0x08,0x10,0x7F},{0x3E,0x41,0x41,0x41,0x3E},{0x7F,0x09,0x09,0x09,0x06},{0x3E,0x41,0x51,0x21,0x5E},
    {0x7F,0x09,0x19,0x29,0x46},{0x46,0x49,0x49,0x49,0x31},{0x01,0x01,0x7F,0x01,0x01},{0x3F,0x40,0x40,0x40,0x3F},{0x1F,0x20,0x40,0x20,0x1F},
    {0x3F,0x40,0x38,0x40,0x3F},{0x63,0x14,0x08,0x14,0x63},{0x07,0x08,0x70,0x08,0x07},{0x61,0x51,0x49,0x45,0x43},{0x00,0x7F,0x41,0x41,0x00},
    {0x02,0x04,0x08,0x10,0x20},{0x00,0x41,0x41,0x7F,0x00},{0x04,0x02,0x01,0x02,0x04},{0x40,0x40,0x40,0x40,0x40},{0x00,0x01,0x02,0x04,0x00},
    {0x20,0x54,0x54,0x54,0x78},{0x7F,0x48,0x44,0x44,0x38},{0x38,0x44,0x44,0x44,0x20},{0x38,0x44,0x44,0x48,0x7F},{0x38,0x54,0x54,0x54,0x18},
    {0x08,0x7E,0x09,0x01,0x02},{0x0C,0x52,0x52,0x52,0x3E},{0x7F,0x08,0x04,0x04,0x78},{0x00,0x44,0x7D,0x40,0x00},{0x20,0x40,0x44,0x3D,0x00},
    {0x7F,0x10,0x28,0x44,0x00},{0x00,0x41,0x7F,0x40,0x00},{0x7C,0x04,0x18,0x04,0x78},{0x7C,0x08,0x04,0x04,0x78},{0x38,0x44,0x44,0x44,0x38},
    {0x7C,0x14,0x14,0x14,0x08},{0x08,0x14,0x14,0x18,0x7C},{0x7C,0x08,0x04,0x04,0x08},{0x48,0x54,0x54,0x54,0x20},{0x04,0x3F,0x44,0x40,0x20},
    {0x3C,0x40,0x40,0x20,0x7C},{0x1C,0x20,0x40,0x20,0x1C},{0x3C,0x40,0x30,0x40,0x3C},{0x44,0x28,0x10,0x28,0x44},{0x0C,0x50,0x50,0x50,0x3C},
    {0x44,0x64,0x54,0x4C,0x44}};
// (x, y) = left end of the baseline, like cv::putText; font_scale as OpenCV's (0.75 -> 16-pixel caps); colour BGR
static void put_text(uint8_t* bgr, int W, int H, const char* text, int x, int y, double font_scale, const int color[3], int thickness) {
    const int cell = std::max(1, (int)lrint(font_scale * 22.0 / 7.0));   // Hershey simplex caps are 22 units high at scale 1
    for (const char* p = text; *p; p++, x += 6 * cell) {
        const int ch = (unsigned char)*p;
        if (ch < 32 || ch > 122) continue;
        const unsigned char* g = kFont5x7[ch - 32];
        for (int cx = 0; cx < 5; cx++)
            for (int cy = 0; cy < 7; cy++) {
                if (!((g[cx] >> cy) & 1)) continue;
                const int px0 = x + cx * cell, py0 = y - (7 - cy) * cell, ext = cell + thickness - 1;
                for (int yy = py0; yy < py0 + ext; yy++)
                    for (int xx = px0; xx < px0 + ext; xx++)
                        if (xx >= 0 && xx < W && yy >= 0 && yy < H) { uint8_t* d = bgr + ((size_t)yy * W + xx) * 3; d[0] = (uint8_t)color[0]; d[1] = (uint8_t)color[1]; d[2] = (uint8_t)color[2]; }
            }
    }
}

// ---------------------------------------------------------------------------------------------- queue
template <typename T>
class BlockingQueue {   // the subset of caffe::BlockingQueue the demo uses (push / try_pop / pop / size), std-only
public:
    void push(T v) { { std::lock_guard<std::mutex> l(m_); q_.push(std::move(v)); } cv_.notify_one(); }
    bool try_pop(T* out) { std::lock_guard<std::mutex> l(m_); if (q_.empty()) return false; *out = std::move(q_.front()); q_.pop(); return true; }
    bool pop(T* out, const std::atomic<bool>& quit) {
        std::unique_lock<std::mutex> l(m_);
        cv_.wait(l, [&] { return !q_.empty() || quit.load(); });
        if (q_.empty()) return false;
        *out = std::move(q_.front()); q_.pop(); return true;
    }
    size_t size() { std::lock_guard<std::mutex> l(m_); return q_.size(); }
    void wake() { cv_.notify_all(); }
private:
    std::mutex m_; std::condition_variable cv_; std::queue<T> q_;
};

// Page-locked frame buffers are recycled: cudaMallocHost / cudaFreeHost take the driver lock and cudaFreeHost synchronises the
// device, which would serialise against the workers' asynchronous streams at hundreds of frames per second.
class PinnedPool {
public:
    uint8_t* get(size_t bytes) {
        {
            std::lock_guard<std::mutex> l(m_);
            auto& v = free_[bytes];
            if (!v.empty()) { uint8_t* p = v.back(); v.pop_back(); return p; }
        }
        return (uint8_t*)pe_host_alloc(bytes);
    }
    void put(uint8_t* p, size_t bytes) { std::lock_guard<std::mutex> l(m_); free_[bytes].push_back(p); }
    void clear() { std::lock_guard<std::mutex> l(m_); for (auto& kv : free_) for (uint8_t* p : kv.second) pe_host_free(p); free_.clear(); }
private:
    std::mutex m_;
    std::map<size_t, std::vector<uint8_t*>> free_;
} g_pinned;
static void pin_frame(struct Frame& fr);

struct Global {
    BlockingQueue<Frame> input_queue, output_queue;
    std::priority_queue<int, std::vector<int>, std::greater<int>> dropped_index;
    std::mutex mutex;
    std::atomic<bool> producer_done{false}, quit{false}, failed{false};   // quit: stop all threads (ESC or an error); failed: it was an error
    std::atomic<int> produced{0}, finished{0};
    int disp_w = 0, disp_h = 0, net_w = 0, net_h = 0, model = PE_MODEL_COCO_18, num_parts = 18;
    std::vector<std::string> image_list;
    pe_video* video = nullptr;     // --video (cv::VideoCapture of getFrameFromCam)
    int video_frames = 0, video_w = 0, video_h = 0;
    double video_fps = 0;
    pe_camera* camera = nullptr;   // cap.open(FLAGS_camera) when no --video / --image_dir / --synthetic is given
    int camera_w = 0, camera_h = 0;
    bool proto_readable = false;   // --caffeproto parsed: engines are created from it
    // global.nms_threshold etc. of the reference (rtpose.cpp:106-111), changed at run time by handle_key
    std::atomic<float> nms_threshold{0.05f}, connect_min_subset_score{0.4f}, connect_inter_threshold{0.05f};
    std::atomic<int> connect_min_subset_cnt{3}, connect_inter_min_above_threshold{9}, part_to_show{0}, params_version{0};
    std::atomic<int> dropped{0};
    std::atomic<int> end_index{INT_MAX};   // --gpu_entropy: the run ends before this frame (a video frame the GPU could not decode)
    // global.uistate (rtpose.cpp:96-104): googly eyes, video pause / seek, driven by handle_key
    std::atomic<bool> googly_eyes{false}, video_paused{false};
    std::atomic<int> seek_delta{0};
    int queue_limit = 64, batch = 1, engines_per_gpu = 1;
    // --audit_every: frames compared with the parity mode, how many were identical, the largest joint distance (display px)
    std::mutex audit_mutex;
    long long audit_frames = 0, audit_identical = 0;
    float audit_max_joint = 0.f;
} global;

// --image_dir frame: .jpg / .png decode straight into a page-locked buffer of the pool; other formats (and an exhausted pool) go
// through fr.bgr and pin_frame
static bool read_frame_image(const std::string& path, int& w, int& h, Frame& fr) {
    size_t got_bytes = 0;
    const std::function<uint8_t*(size_t)> alloc = [&](size_t bytes) { got_bytes = bytes; return g_pinned.get(bytes); };
    uint8_t* ph = nullptr;
    const bool ok = read_image(path, w, h, fr.bgr, &alloc, &ph);
    if (ph) {
        const size_t bytes = got_bytes;
        fr.pinned = std::shared_ptr<uint8_t>(ph, [bytes](uint8_t* q) { g_pinned.put(q, bytes); });   // returned to the pool also when decoding failed
    }
    return ok;
}

static int num_producers();
// --gpu_entropy: a frame whose entropy-coded data the GPU rejected (pe_fetch: PE_ERR_IO) is handled as the host route handles a file
// it cannot decode, with the same message: it becomes a dropped index, and with the single --video reader the run ends there.
static void undecodable_frame(const Frame& fr) {
    std::lock_guard<std::mutex> l(global.mutex);
    if (global.video) {
        LOG_ERROR("%s: frame %d is not a decodable JPEG", F("video").c_str(), fr.video_frame_number);
        int cur = global.end_index.load();
        while (num_producers() == 1 && fr.index < cur && !global.end_index.compare_exchange_weak(cur, fr.index)) {}
    } else {
        LOG_ERROR("cannot decode %s (supported: .jpg, .png, 24-bit .bmp, P6 .ppm)", global.image_list[fr.video_frame_number].c_str());
    }
    global.dropped_index.push(fr.index);
}

static void pin_frame(Frame& fr) {
    if (fr.pinned) return;   // decoded in place
    const size_t bytes = fr.bgr.size();
    if (uint8_t* ph = g_pinned.get(bytes)) {   // falls back to the staged copy inside pe_forward_frames if it fails
        memcpy(ph, fr.bgr.data(), bytes);
        fr.pinned = std::shared_ptr<uint8_t>(ph, [bytes](uint8_t* q) { g_pinned.put(q, bytes); });
        std::vector<uint8_t>().swap(fr.bgr);
    }
}

// ---------------------------------------------------------------------------------------------- weights
// The net is built from --caffeproto like `new Net<float>(proto, TEST)` (rtpose.cpp:183); the model follows the Nms layer's
// num_parts (:212-229).  -1: file unreadable, -2: not a pose-path graph (message logged).
static int model_from_prototxt(const std::string& path) {
    std::ifstream f(path);
    if (!f) return -1;
    char buf[64];
    const int n = pe_plan_describe(-1, path.c_str(), nullptr, 0);
    if (n < 0) { LOG_ERROR("%s", pe_last_error(nullptr)); return -2; }
    std::vector<char> text((size_t)n + 1);
    pe_plan_describe(-1, path.c_str(), text.data(), n + 1);
    int model = -2;
    if (sscanf(text.data(), "%63s %d", buf, &model) != 2) return -2;
    global.proto_readable = true;
    return model;
}

static void random_weights(pe_engine* e, const std::string& kind) {
    uint64_t s = 1234;
    auto uni = [&]() { s = s * 6364136223846793005ull + 1442695040888963407ull; return ((s >> 11) + 0.5) / 9007199254740992.0; };
    char name[64];
    int co, ci, k;
    for (int i = 0; i < pe_num_conv_layers(e); i++) {
        pe_conv_layer_info(e, i, name, &co, &ci, &k);
        const double stdv = kind == "caffe" ? 0.01 : sqrt(2.0 / (ci * k * k));
        std::vector<float> w((size_t)co * ci * k * k), b(co, 0.f);
        for (size_t j = 0; j + 1 < w.size(); j += 2) {   // Box-Muller
            const double r = sqrt(-2.0 * log(uni())), t = 6.283185307179586 * uni();
            w[j] = (float)(stdv * r * cos(t)); w[j + 1] = (float)(stdv * r * sin(t));
        }
        pe_set_conv_weights(e, name, w.data(), w.size(), b.data(), b.size());
    }
}

// ---------------------------------------------------------------------------------------------- threads
static int source_frame_count() {
    if (Fi("synthetic") > 0) return Fi("synthetic");
    if (global.video) return global.video_frames;
    if (global.camera) return 0x7fffffff;   // until ESC / a capture error
    return (int)global.image_list.size();
}
// --gpu_decode: frame i of --image_dir / a Motion-JPEG --video as a coefficient image in a page-locked buffer of the pool (the
// reconstruction runs on the GPU, pe_forward_jpeg_coefs); --gpu_entropy: as a scan image (pe_forward_jpeg_scans decodes the Huffman
// data too), or as a coefficient image when the JPEG is not one sequential scan (-3).  false: not a JPEG, or one the coefficient
// stage refuses: the caller decodes the frame on the host instead, which also reports what is wrong with it.
static bool fetch_coefs(int i, Frame& fr) {
    std::vector<uint8_t> data;
    if (!global.video) {
        FILE* f = fopen(global.image_list[i].c_str(), "rb");
        if (!f) return false;
        fseek(f, 0, SEEK_END);
        const long n = ftell(f);
        fseek(f, 0, SEEK_SET);
        data.resize((size_t)std::max(n, 0L));
        const bool rd = n > 4 && fread(data.data(), 1, (size_t)n, f) == (size_t)n;
        fclose(f);
        if (!rd || data[0] != 0xFF || data[1] != 0xD8) return false;
    }
    bool scan = Fb("gpu_entropy");
    auto read = [&](void* buf, long long cap) {
        if (scan) return global.video ? pe_video_read_scan(global.video, i, buf, cap) : pe_jpeg_read_scan(data.data(), (long long)data.size(), buf, cap);
        return global.video ? pe_video_read_coefs(global.video, i, buf, cap) : pe_jpeg_read_coefs(data.data(), (long long)data.size(), buf, cap);
    };
    long long n = read(nullptr, 0);
    if (scan && n == -3) { scan = false; n = read(nullptr, 0); }   // progressive / multi-scan: the host entropy stage
    if (n <= (long long)sizeof(pe_jpeg_coef_header) || n > (3LL << 28)) return false;
    uint8_t* ph = g_pinned.get((size_t)n);   // without page-locked memory the engine stages the copy (as for pixel frames)
    if (ph) fr.pinned = std::shared_ptr<uint8_t>(ph, [n](uint8_t* q) { g_pinned.put(q, (size_t)n); });
    else { fr.bgr.resize((size_t)n); ph = fr.bgr.data(); }
    pe_jpeg_coef_header hd;
    if (read(ph, n) != n) { fr.pinned.reset(); std::vector<uint8_t>().swap(fr.bgr); return false; }
    memcpy(&hd, ph, sizeof hd);
    fr.w = hd.width; fr.h = hd.height;   // (a scan image starts with the same header)
    fr.kind = scan ? Frame::SCAN : Frame::COEFS;
    return true;
}

// frame i of the source (synthetic / --video / --image_dir) into fr; false: could not be decoded (message logged)
static bool fetch_source_frame(int i, Frame& fr) {
    int w = global.disp_w, h = global.disp_h;
    if ((Fb("gpu_decode") || Fb("gpu_entropy")) && (global.video || !global.image_list.empty()) && !global.camera && Fi("synthetic") <= 0 && fetch_coefs(i, fr)) {
        if (!global.video) {
            const std::string& p = global.image_list[i];
            const size_t slash = p.find_last_of('/'), dot = p.find_last_of('.');
            fr.stem = p.substr(slash == std::string::npos ? 0 : slash + 1, dot - (slash == std::string::npos ? 0 : slash + 1));
        }
        return true;
    }
    if (Fi("synthetic") > 0) {
        synthetic_frame(i, w, h, fr.bgr);
    } else if (global.camera) {   // cap >> image_uchar_orig from the capture device
        w = global.camera_w; h = global.camera_h;
        const size_t bytes = (size_t)w * h * 3;
        uint8_t* ph = g_pinned.get(bytes);
        uint8_t* dst = ph;
        if (ph) fr.pinned = std::shared_ptr<uint8_t>(ph, [bytes](uint8_t* q) { g_pinned.put(q, bytes); });
        else { fr.bgr.resize(bytes); dst = fr.bgr.data(); }
        if (pe_camera_grab(global.camera, dst, (long long)bytes, 0)) { LOG_ERROR("%s", pe_camera_last_error()); return false; }
    } else if (global.video) {   // cap >> image_uchar_orig (rtpose.cpp:431): decoded straight into a page-locked buffer
        w = global.video_w; h = global.video_h;
        const size_t bytes = (size_t)w * h * 3;
        uint8_t* ph = g_pinned.get(bytes);
        uint8_t* dst = ph;
        if (ph) fr.pinned = std::shared_ptr<uint8_t>(ph, [bytes](uint8_t* q) { g_pinned.put(q, bytes); });
        else { fr.bgr.resize(bytes); dst = fr.bgr.data(); }
        if (pe_video_read(global.video, i, dst, (long long)bytes)) { LOG_ERROR("%s", pe_video_last_error()); return false; }
    } else {
        const std::string& p = global.image_list[i];
        if (!read_frame_image(p, w, h, fr)) { LOG_ERROR("cannot decode %s (supported: .jpg, .png, 24-bit .bmp, P6 .ppm)", p.c_str()); return false; }
        const size_t slash = p.find_last_of('/'), dot = p.find_last_of('.');
        fr.stem = p.substr(slash == std::string::npos ? 0 : slash + 1, dot - (slash == std::string::npos ? 0 : slash + 1));
    }
    pin_frame(fr);
    fr.w = w; fr.h = h;
    return true;
}

static void producer() {
    const int total = source_frame_count();
    // --video: frames are committed at the file's frame rate (rtpose.cpp:446-462) and the file loops at its end unless results are
    // being written (:525-545; the reference exits only with --write_frames, here also with --write_json: a looping writer would
    // overwrite its own files)
    const bool paced = global.video && Fb("video_realtime");
    const bool loop = global.video && F("write_frames").empty() && F("write_json").empty() && !Fb("decode_bench");
    const double frame_time = global.video_fps > 0 ? 1.0 / global.video_fps : 0;
    double last_frame_time = -1;
    for (int i = Fi("start_frame"); !global.quit; i++) {
        if (global.video) {   // uistate.seek_to_frame / is_video_paused (rtpose.cpp:434-446): a paused video keeps delivering its current frame
            const int d = global.seek_delta.exchange(0);
            if (d) { i = std::max(0, std::min(total - 1, i + d)); LOG_INFO("Seek to frame %d", i); }
            else if (global.video_paused && i > Fi("start_frame")) i--;
        }
        if (i >= total) {
            if (!loop || total <= 0) break;
            LOG_INFO("Looping video after %d frames", total);
            i = 0;
        }
        Frame fr;
        fr.t_commit = now_s();    // frame.commit_time: taken when the frame is grabbed (rtpose.cpp:449)
        fr.index = global.produced; fr.video_frame_number = i;
        if (fr.index >= global.end_index) break;   // --gpu_entropy: a video frame the GPU could not decode ends the run
        if (!fetch_source_frame(i, fr)) {
            if (global.video || global.camera) break;   // a broken frame ends a video / the capture (cap >> returns an empty Mat)
            continue;
        }
        if (global.camera) fr.t_commit = now_s();    // the frame was taken while the call blocked
        if (paced) {
            const double interval = now_s() - last_frame_time;
            if (last_frame_time >= 0 && interval < frame_time) std::this_thread::sleep_for(std::chrono::duration<double>(frame_time - interval));
            last_frame_time = now_s();
            fr.t_commit = last_frame_time;
        }
        fr.t_preprocessed = now_s();
        // the reference's producers wait while more than 10 frames are queued (rtpose.cpp:310-313, 424-429); the bound scales with the batch
        while ((int)global.input_queue.size() > global.queue_limit && !global.quit) std::this_thread::sleep_for(std::chrono::milliseconds(1));
        global.input_queue.push(std::move(fr));
        global.produced++;
    }
    global.producer_done = true;
    global.input_queue.wake();
}

// [extension] --num_producers N > 1.  The reference decodes on ONE thread (getFrameFromDir, rtpose.cpp:302-391); a 720p JPEG
// takes ~12 ms here, i.e. ~80 frames/s per thread against ~740 frames/s that one GPU consumes, so the producer stage is
// what scales with threads.  N threads take frame indices from a shared counter; order is restored downstream by the
// re-orderer through Frame::index, and a frame that fails to decode becomes a dropped index (as dropped frames do).
static void producer_mt(int nthreads) {
    const int total = source_frame_count(), start = Fi("start_frame");
    std::atomic<int> next{start};
    auto body = [&]() {
        while (!global.quit) {
            const int i = next++;
            if (i >= total || i - start >= global.end_index) break;
            Frame fr;
            fr.t_commit = now_s();
            fr.index = i - start; fr.video_frame_number = i;
            if (!fetch_source_frame(i, fr)) {
                std::lock_guard<std::mutex> l(global.mutex);
                global.dropped_index.push(fr.index);
                continue;
            }
            fr.t_preprocessed = now_s();
            while ((int)global.input_queue.size() > global.queue_limit && !global.quit) std::this_thread::sleep_for(std::chrono::milliseconds(1));
            global.input_queue.push(std::move(fr));
            global.produced++;
        }
    };
    std::vector<std::thread> th;
    for (int t = 0; t < nthreads; t++) th.emplace_back(body);
    for (auto& t : th) t.join();
    global.producer_done = true;
    global.input_queue.wake();
}
static int num_producers() {
    if (Fi("num_producers") > 0) return Fi("num_producers");
    if (Fi("batch") > 0) return 1;   // an explicit batch (1 = the reference's behaviour) keeps the reference's single producer
    if (global.camera) return 1;
    if (global.video && (Fb("video_realtime") || (F("write_frames").empty() && F("write_json").empty()))) return 1;   // pacing / looping: one reader, like cap >>
    const int cores = (int)std::thread::hardware_concurrency();
    const int gpus = std::max(1, Fi("num_gpu"));
    return std::max(1, std::min(std::min(48, 10 * gpus), cores - 2 * gpus - 2));
}
static void run_producers() {
    const int n = num_producers();
    if (n > 1) producer_mt(n); else producer();
}

// [extension] --decode_bench: the producer stage alone (decode + queue, no GPU): frames/s of --image_dir with --num_producers
static int decode_bench() {
    std::atomic<long long> bytes{0};
    std::atomic<int> frames{0};
    std::vector<int> order;
    if (uint8_t* warm = g_pinned.get(1 << 20)) g_pinned.put(warm, 1 << 20);   // the first page-locked allocation initialises the CUDA runtime: not part of the decode rate
    const double t0 = now_s();
    std::thread prod(run_producers);
    while (true) {
        Frame fr;
        if (global.input_queue.try_pop(&fr)) { frames++; bytes += (long long)fr.w * fr.h * 3; order.push_back(fr.index); continue; }
        if (global.producer_done && global.input_queue.size() == 0) break;
        std::this_thread::sleep_for(std::chrono::microseconds(100));
    }
    prod.join();
    const double dt = now_s() - t0;
    std::sort(order.begin(), order.end());
    bool contiguous = true;   // every index once, gaps only where a file was dropped
    for (size_t i = 1; i < order.size(); i++) contiguous = contiguous && order[i] != order[i - 1];
    printf("decoded %d frames (%.1f MB) with %d producer(s) in %.3f s: %.1f frames/s, dropped %d, indices_unique %d\n", (int)frames,
           bytes / 1e6, num_producers(), dt, frames / std::max(dt, 1e-9), (int)global.dropped_index.size(), contiguous ? 1 : 0);
    return 0;
}

static int load_weights(pe_engine* e, int device) {   // CopyTrainedLayersFrom (rtpose.cpp:184)
    LOG_INFO("GPU %d: copying to person net", device);
    int rc = 0;
    if (!F("random_init").empty()) random_weights(e, F("random_init"));
    else rc = pe_load_caffemodel(e, F("caffemodel").c_str());
    if (rc || pe_commit_weights(e)) {
        LOG_ERROR("GPU %d: cannot load %s: %s %s", device, F("caffemodel").c_str(), pe_caffemodel_last_error(), pe_last_error(e));
        return 1;
    }
    return 0;
}

// warmup() of every GPU (rtpose.cpp:173-237).  The reference parses the .caffemodel once per GPU; here GPU 0 loads and
// packs it and the replicas receive the packed buffer by one ncclBroadcast (the path's only collective).
// engines[g * per_gpu + k] = handle k of GPU g.  Handle 0 of GPU 0 loads the model; handle 0 of the other GPUs receives the packed
// weights by broadcast; handles k > 0 share their GPU's buffer (Net::ShareTrainedLayersWith).
static bool create_engines(int num_gpu, int per_gpu, int precision, std::vector<pe_engine*>& engines) {
    const int batch = global.batch;
    for (int tid = 0; tid < num_gpu * per_gpu; tid++) {
        pe_config c;
        memset(&c, 0, sizeof c);
        c.device = Fi("start_device") + tid / per_gpu; c.model = global.model; c.net_w = global.net_w; c.net_h = global.net_h;
        c.disp_w = global.disp_w; c.disp_h = global.disp_h; c.num_scales = Fi("num_scales");
        c.start_scale = Fd("start_scale"); c.scale_gap = Fd("scale_gap"); c.max_batch = batch; c.precision = precision;
        pe_engine* e = nullptr;
        const int rc = global.proto_readable ? pe_create_from_prototxt(&c, F("caffeproto").c_str(), &e) : pe_create(&c, &e);
        if (rc) { LOG_ERROR("GPU %d: %s", c.device, pe_last_error(nullptr)); return false; }
        engines.push_back(e);
    }
    if (load_weights(engines[0], Fi("start_device"))) return false;
    if (Fb("calibrate_range") && (precision == PE_PREC_F16X2 || precision == PE_PREC_F16X1)) {   // before the weights are replicated: the scales travel inside the packed buffer
        std::vector<uint8_t> probe;
        synthetic_frame(0, global.disp_w, global.disp_h, probe);
        const uint8_t* ptr = probe.data();
        if (pe_calibrate(engines[0], &ptr, 1)) { LOG_ERROR("GPU %d: range calibration failed: %s", Fi("start_device"), pe_last_error(engines[0])); return false; }
    }
    if (num_gpu > 1) {
        std::vector<pe_engine*> firsts;
        for (int g = 0; g < num_gpu; g++) firsts.push_back(engines[g * per_gpu]);
        if (pe_broadcast_weights(firsts.data(), num_gpu) == PE_OK) {
            LOG_INFO("weights broadcast from GPU %d to %d replicas (%.1f MB, NCCL)", Fi("start_device"), num_gpu - 1,
                     pe_packed_weights_bytes(engines[0]) / 1e6);
        } else {
            LOG_ERROR("weight broadcast unavailable (%s); every GPU loads the model itself", pe_last_error(engines[0]));
            for (int g = 1; g < num_gpu; g++)
                if (load_weights(engines[g * per_gpu], Fi("start_device") + g)) return false;
        }
    }
    for (int g = 0; g < num_gpu; g++)
        for (int k = 1; k < per_gpu; k++)
            if (pe_share_weights(engines[g * per_gpu], engines[g * per_gpu + k])) { LOG_ERROR("GPU %d: %s", Fi("start_device") + g, pe_last_error(engines[g * per_gpu])); return false; }
    return true;
}

// --audit_every: frame i of the last forward of `e` against the parity handle `ref` (same frames)
static bool audit_frame(pe_engine* e, pe_engine* ref, int i, const std::vector<float>& joints, int cnt, const std::vector<float>& peaks) {
    const int P = pe_nms_get_num_parts(e), MP = pe_nms_get_max_peaks(e);
    std::vector<float> rj((size_t)PE_MAX_PEOPLE * P * 3), rp((size_t)P * (MP + 1) * 3);
    int rcnt = 0;
    if (pe_fetch(ref, i, rj.data(), &rcnt, rp.data())) return false;
    // the north-star bar (DESIGN.md section 6): 1e-3 net px, in display px for the joints
    const float tol = 1e-3f * (float)std::max((double)global.disp_w / global.net_w, (double)global.disp_h / global.net_h);
    pe_result_diff d;
    if (pe_compare_results(joints.data(), cnt, peaks.data(), rj.data(), rcnt, rp.data(), P, MP, tol, &d)) return false;
    std::lock_guard<std::mutex> l(global.audit_mutex);
    global.audit_frames++;
    global.audit_identical += d.identical;
    global.audit_max_joint = std::max(global.audit_max_joint, d.max_joint_dist);
    return true;
}

static void worker(int tid, pe_engine* e, pe_engine* ref) {
    const int device = Fi("start_device") + tid / global.engines_per_gpu, batch = global.batch;
    struct Done { ~Done() { global.finished++; global.output_queue.wake(); } } done_guard;   // every exit path counts
    caffe::NmsLayer<float> nms_layer(e);
    caffe::ImResizeLayer<float> resize_layer(e);
    resize_layer.SetStartScale((float)Fd("start_scale"));
    resize_layer.SetScaleGap((float)Fd("scale_gap"));
    LOG_INFO("GPU %d is ready (model %s, max_peaks %d, %d frame(s) per forward)", device, nms_layer.GetNumParts() == 15 ? "MPI" : "COCO",
             nms_layer.GetMaxPeaks(), batch);
    const int P = nms_layer.GetNumParts();
    std::vector<float> joints((size_t)PE_MAX_PEOPLE * P * 3), peaks((size_t)P * (nms_layer.GetMaxPeaks() + 1) * 3);
    const int audit_every = ref ? Fi("audit_every") : 0;
    long long batches = 0;
    Frame pending;
    bool pending_valid = false;
    int seen_version = -1;
    const bool drops = !Fb("no_frame_drops");
    while (!global.quit) {
        std::vector<Frame> frames;
        Frame fr;
        while ((int)frames.size() < batch) {
            if (pending_valid) { fr = std::move(pending); pending_valid = false; }
            else if (!global.input_queue.try_pop(&fr)) break;
            fr.t_fetched = now_s();
            // processFrame drops a frame that waited more than 0.1 s for a GPU unless --no_frame_drops (rtpose.cpp:1107-1124)
            if (drops && fr.t_fetched - fr.t_commit > 0.1) {
                std::lock_guard<std::mutex> l(global.mutex);
                global.dropped_index.push(fr.index);
                global.dropped++;
                continue;
            }
            if (!frames.empty() && (fr.w != frames[0].w || fr.h != frames[0].h || fr.kind != frames[0].kind)) {   // one forward = one frame size and kind
                pending = std::move(fr); pending_valid = true;
                break;
            }
            frames.push_back(std::move(fr));
        }
        if (frames.empty()) {
            if (global.producer_done && global.input_queue.size() == 0 && !pending_valid) break;
            std::this_thread::sleep_for(std::chrono::microseconds(200));
            continue;
        }
        if (seen_version != global.params_version) {   // nms_layer->SetThreshold(global.nms_threshold) + connect_* every frame (rtpose.cpp:1145, 1617-1651)
            seen_version = global.params_version;
            nms_layer.SetThreshold(global.nms_threshold);
            pe_set_connect_params(e, global.connect_min_subset_cnt, global.connect_min_subset_score, global.connect_inter_threshold,
                                  global.connect_inter_min_above_threshold);
        }
        std::vector<const uint8_t*> ptrs;
        for (auto& f : frames) ptrs.push_back(f.pinned ? f.pinned.get() : f.bgr.data());
        double scale = 1.0;
        auto forward = [&](pe_engine* h) {
            if (frames[0].kind == Frame::COEFS) return pe_forward_jpeg_coefs(h, (const void* const*)ptrs.data(), (int)ptrs.size(), &scale);   // GPU JPEG reconstruction
            if (frames[0].kind == Frame::SCAN) return pe_forward_jpeg_scans(h, (const void* const*)ptrs.data(), (int)ptrs.size(), &scale);   // + Huffman decoding
            if (frames[0].w == global.disp_w && frames[0].h == global.disp_h) return pe_forward_frames(h, ptrs.data(), (int)ptrs.size());
            return pe_forward_camera_frames(h, ptrs.data(), (int)ptrs.size(), frames[0].w, frames[0].h, &scale);   // warpAffine on the GPU
        };
        int frc = forward(e);
        for (auto& f : frames) f.scale = scale;
        if (frc) { LOG_ERROR("GPU %d: %s", device, pe_last_error(e)); global.failed = global.quit = true; break; }
        const bool audit = audit_every > 0 && batches++ % audit_every == 0;
        if (audit) {   // the same frames through the parity handle; its results are only compared, never written
            frc = forward(ref);
            if (frc) { LOG_ERROR("GPU %d (audit): %s", device, pe_last_error(ref)); global.failed = global.quit = true; break; }
        }
        for (size_t i = 0; i < frames.size(); i++) {
            int cnt = 0;
            const int frc_i = pe_fetch(e, (int)i, joints.data(), &cnt, audit ? peaks.data() : nullptr);
            if (frc_i == PE_ERR_IO && frames[i].kind == Frame::SCAN) {   // corrupt entropy-coded data: as the host route treats the file
                undecodable_frame(frames[i]);
                frames[i].pinned.reset();
                continue;
            }
            if (frc_i) { LOG_ERROR("GPU %d: %s", device, pe_last_error(e)); global.failed = global.quit = true; break; }
            if (audit && !audit_frame(e, ref, (int)i, joints, cnt, peaks)) {
                LOG_ERROR("GPU %d (audit): %s", device, pe_last_error(ref)); global.failed = global.quit = true; break;
            }
            frames[i].num_people = cnt;
            frames[i].joints.assign(joints.begin(), joints.begin() + (size_t)cnt * P * 3);
            if (!F("write_frames").empty()) {   // render() + postProcessFrame (rtpose.cpp:271-300, 1286-1296) on the GPU
                frames[i].rendered.resize((size_t)global.disp_w * global.disp_h * 3);
                if (pe_render(e, (int)i, global.part_to_show, global.googly_eyes ? 1 : 0, nullptr, nullptr, frames[i].rendered.data())) {
                    LOG_ERROR("GPU %d: %s", device, pe_last_error(e)); global.failed = global.quit = true; break;
                }
            }
            frames[i].pinned.reset();   // back to the pool: the forward has consumed the frame
            frames[i].t_done = now_s();
            global.output_queue.push(std::move(frames[i]));
        }
    }
}

// handleKey (rtpose.cpp:1551-1671) without a window: the same key characters, read from stdin with --keys_from_stdin
static void handle_key(int c) {
    // `global.nms_threshold -= 0.005;` on a float member: the sum is formed in double and rounded to float once (rtpose.cpp:1617-1635)
    auto bump = [](std::atomic<float>& v, double d, const char* name) { v = (float)((double)v.load() + d); LOG_INFO("%s: %g", name, (double)v.load()); };
    auto bumpi = [](std::atomic<int>& v, int d, const char* name) { v = v + d; LOG_INFO("%s: %d", name, v.load()); };
    const int max_show = global.model == PE_MODEL_MPI_15 ? 43 : 39;
    if (c == 27 || c == 'Q') { global.quit = true; return; }   // ESC as in the reference; 'Q' for terminals that cannot send it
    if (c == 'g') { global.googly_eyes = !global.googly_eyes; LOG_INFO("googly eyes: %d", (int)global.googly_eyes.load()); return; }   // rtpose.cpp:1568-1570
    if (c == 'l' || c == 'k' || c == 'L' || c == 'K' || c == ' ') {   // rudimentary seeking in video (:1572-1593): 30 frames, 2 with shift; space pauses
        if (global.video && c != ' ') {
            const int d = (c == 'L' || c == 'K') ? 2 : 30;
            global.seek_delta += (c == 'l' || c == 'L') ? d : -d;
        }
        if (c == ' ') { global.video_paused = !global.video_paused; LOG_INFO("paused: %d", (int)global.video_paused.load()); }
        return;
    }
    if (c == '-' || c == '=') bump(global.nms_threshold, c == '-' ? -0.005 : 0.005, "nms_threshold");
    else if (c == '_' || c == '+') bump(global.connect_min_subset_score, c == '_' ? -0.005 : 0.005, "connect_min_subset_score");
    else if (c == '[' || c == ']') bump(global.connect_inter_threshold, c == '[' ? -0.005 : 0.005, "connect_inter_threshold");
    else if (c == '{' || c == '}') bumpi(global.connect_inter_min_above_threshold, c == '{' ? -1 : 1, "connect_inter_min_above_threshold");
    else if (c == ';' || c == '\'') bumpi(global.connect_min_subset_cnt, c == ';' ? -1 : 1, "connect_min_subset_cnt");
    else if (c == ',' || c == '.') {
        int p = global.part_to_show + (c == '.' ? 1 : -1);
        if (p < 0) p = max_show;
        if (p > max_show) p = 0;
        global.part_to_show = p;
        LOG_INFO("p2s: %d", p);
        return;
    } else {
        static const std::string key2part = "0123456789qwertyuiopas";   // rtpose.cpp:1552, 1607-1615: digit/letter keys pick the view
        const size_t ind = key2part.find((char)c);
        if (ind != std::string::npos && (int)ind <= max_show) { global.part_to_show = (int)ind; LOG_INFO("p2s: %d", (int)ind); }
        return;
    }
    global.params_version++;
}
static void key_reader() {
    int c;
    while (!global.quit && (c = getchar()) != EOF)
        if (c != '\n' && c != '\r') handle_key(c);
}

// [extension] --write_frames images and --write_json files leave the display thread: the reference encodes them there (cv::imwrite inside displayFrame,
// rtpose.cpp:1363-1380), which bounds the whole pipeline by one thread's JPEG encoder (~50 frames/s at 720p, quality 98) while one GPU
// renders hundreds.  The files are independent (the frame number is in the name), so N threads encode and write them; the queue is
// bounded, the display thread waits when the writers fall behind.
struct WriteJob {
    std::string fname;
    std::vector<uint8_t> bgr; int w = 0, h = 0; bool bmp = false;        // an image of --write_frames, or
    std::vector<float> joints; int num_people = -1, num_parts = 0; double scale = 1.0;   // (num_people >= 0) the JSON block of --write_json
};
static void write_image(const WriteJob& j) {
    bool ok;
    if (j.num_people >= 0) {   // displayFrame :1383-1416; one formatting pass into a buffer that holds any frame of this size
        std::vector<char> buf(64 + (size_t)j.num_people * ((size_t)j.num_parts * 48 + 32));
        int need = pe_write_json(j.joints.data(), j.num_people, j.num_parts, j.scale, buf.data(), (int)buf.size());
        if (need >= (int)buf.size()) { buf.resize((size_t)need + 1); need = pe_write_json(j.joints.data(), j.num_people, j.num_parts, j.scale, buf.data(), need + 1); }
        FILE* f = fopen(j.fname.c_str(), "wb");
        ok = f != nullptr;
        if (f) { ok = fwrite(buf.data(), 1, (size_t)need, f) == (size_t)need; fclose(f); }
    } else if (j.bmp) {
        ok = write_bmp(j.fname, j.w, j.h, j.bgr.data());
    } else {
        // one encoding pass: a baseline JPEG never exceeds the raw size by more than its tables and headers
        std::vector<uint8_t> jb((size_t)j.w * j.h * 3 + (1u << 16));
        const long long need = pe_encode_jpeg(j.bgr.data(), j.w, j.h, 98, jb.data(), (long long)jb.size());
        ok = need > 0 && need <= (long long)jb.size();
        FILE* f = ok ? fopen(j.fname.c_str(), "wb") : nullptr;
        ok = f != nullptr;
        if (f) { ok = fwrite(jb.data(), 1, (size_t)need, f) == (size_t)need; fclose(f); }
    }
    if (!ok) LOG_ERROR("cannot write %s", j.fname.c_str());
}
class WriterPool {
public:
    void start(int n) {
        limit_ = (size_t)std::max(2, 4 * n);
        for (int i = 0; i < n; i++) threads_.emplace_back([this] { loop(); });
    }
    void submit(WriteJob&& j) {
        if (threads_.empty()) { write_image(j); return; }   // --num_writers 1: on the caller's thread, as the reference
        std::unique_lock<std::mutex> l(m_);
        space_.wait(l, [&] { return q_.size() < limit_; });
        q_.push(std::move(j));
        l.unlock();
        work_.notify_one();
    }
    void finish() {
        { std::lock_guard<std::mutex> l(m_); done_ = true; }
        work_.notify_all();
        for (auto& t : threads_) t.join();
        threads_.clear();
    }
private:
    void loop() {
        for (;;) {
            WriteJob j;
            {
                std::unique_lock<std::mutex> l(m_);
                work_.wait(l, [&] { return done_ || !q_.empty(); });
                if (q_.empty()) return;
                j = std::move(q_.front());
                q_.pop();
            }
            space_.notify_one();
            write_image(j);
        }
    }
    std::mutex m_;
    std::condition_variable work_, space_;
    std::queue<WriteJob> q_;
    std::vector<std::thread> threads_;
    size_t limit_ = 8;
    bool done_ = false;
};

// re-order by frame index (buffer_and_order, rtpose.cpp:1214-1273) and write JSON (displayFrame, :1383-1416)
static void orderer_and_writer(int num_workers) {
    auto cmp = [](const Frame& a, const Frame& b) { return a.index > b.index; };
    std::priority_queue<Frame, std::vector<Frame>, decltype(cmp)> heap(cmp);
    int next = 0, written = 0;
    const double t0 = now_s();
    double last = t0, fps_now = 0;   // FPS of the last 30 frames, as displayFrame keeps it
    const std::string out = F("write_json");
    WriterPool writers;
    if (!F("write_frames").empty() || !out.empty()) {
        const int nw = Fi("num_writers") > 0 ? Fi("num_writers") : std::max(1, std::min(16, (int)std::thread::hardware_concurrency() / 4));
        if (nw > 1) writers.start(nw);
    }
    auto emit = [&](Frame& fr) {
        if (!out.empty()) {
            char fname[1024];
            if (F("image_dir").empty()) snprintf(fname, sizeof fname, "%s/frame%06d.json", out.c_str(), fr.video_frame_number);
            else snprintf(fname, sizeof fname, "%s/%s.json", out.c_str(), fr.stem.c_str());
            WriteJob job;
            job.fname = fname; job.num_people = fr.num_people; job.num_parts = global.num_parts; job.scale = fr.scale;
            job.joints = fr.joints;   // (the frame keeps its copy: nothing after this reads it, but the status line prints fr.num_people)
            writers.submit(std::move(job));
        }
        if (!F("write_frames").empty() && !fr.rendered.empty() && !Fb("no_text")) {   // displayFrame :1317-1353
            Frame& mfr = fr;
            char tmp[256];
            const int c_fps[3] = {255, 150, 150}, c_black[3] = {0, 0, 0}, c_cnt[3] = {150, 150, 255}, c_white[3] = {255, 255, 255};
            snprintf(tmp, sizeof tmp, "%4.2f s/gpu", fps_now > 0 ? std::max(1, Fi("num_gpu")) * 1.0 / fps_now : 0.0);
            put_text(mfr.rendered.data(), global.disp_w, global.disp_h, tmp, 25, 35, 0.75, c_fps, 1);
            snprintf(tmp, sizeof tmp, "%4d", fr.num_people);
            put_text(mfr.rendered.data(), global.disp_w, global.disp_h, tmp, global.disp_w - 100 + 2, 35 + 2, 0.75, c_black, 2);
            put_text(mfr.rendered.data(), global.disp_w, global.disp_h, tmp, global.disp_w - 100, 35, 0.75, c_cnt, 2);
            const int p2s = global.part_to_show;
            if (p2s != 0) {
                if (p2s - 1 <= global.num_parts) snprintf(tmp, sizeof tmp, "%10s", pe_model_part_name(global.model, p2s - 1));
                else {
                    int aff = ((p2s - 1) - global.num_parts - 1) * 2;
                    if (aff == 0) snprintf(tmp, sizeof tmp, "%10s", "PAFs");
                    else {
                        aff = aff - 2 + 1 + global.num_parts;
                        std::string uv = pe_model_part_name(global.model, aff);
                        snprintf(tmp, sizeof tmp, "%10s", uv.substr(0, uv.find("(")).c_str());
                    }
                }
                put_text(mfr.rendered.data(), global.disp_w, global.disp_h, tmp, global.disp_w - 175 + 1, 55 + 1, 0.5, c_white, 1);
            }
        }
        if (!F("write_frames").empty() && !fr.rendered.empty()) {   // displayFrame :1363-1380 (cv::imwrite, JPEG quality 98)
            WriteJob job;
            job.bmp = F("frame_format") == "bmp";
            char fname[1024];
            if (F("image_dir").empty()) snprintf(fname, sizeof fname, "%s/frame%06d.%s", F("write_frames").c_str(), fr.video_frame_number, job.bmp ? "bmp" : "jpg");
            else snprintf(fname, sizeof fname, "%s/%s.%s", F("write_frames").c_str(), fr.stem.c_str(), job.bmp ? "bmp" : "jpg");
            job.fname = fname; job.w = global.disp_w; job.h = global.disp_h;
            job.bgr = std::move(fr.rendered);
            writers.submit(std::move(job));
        }
        written++;
        if (written % 30 == 0) {   // the reference's line, every 30 frames (rtpose.cpp:1421-1441); stages that run on the GPU here read 0
            const double t = now_s();
            LOG_INFO("# %d, NP %d, Latency %.3f, Preprocess %.3f, QueueA %.3f, GPU %.3f, QueueB %.3f, Postproc %.3f, QueueC %.3f, Buffered %.3f, "
                     "QueueD %.3f, FPS = %.1f", fr.index, fr.num_people, t - fr.t_commit, fr.t_preprocessed - fr.t_commit, fr.t_fetched - fr.t_preprocessed,
                     fr.t_done - fr.t_fetched, fr.t_out_popped - fr.t_done, 0.0, 0.0, fr.t_buffered - fr.t_out_popped, t - fr.t_buffered,
                     30.0 / (t - last));
            fps_now = 30.0 / (t - last);
            last = t;
            if (Fi("audit_every") > 0) {
                std::lock_guard<std::mutex> l(global.audit_mutex);
                LOG_INFO("Audit: %lld/%lld frames identical, max joint \xce\x94 %.3g px", global.audit_identical, global.audit_frames,
                         (double)global.audit_max_joint);
            }
        }
    };
    while (true) {
        Frame fr;
        const bool got = global.output_queue.try_pop(&fr);
        if (got) { fr.t_out_popped = now_s(); heap.push(std::move(fr)); }
        while (true) {
            {
                std::lock_guard<std::mutex> l(global.mutex);
                while (!global.dropped_index.empty() && global.dropped_index.top() == next) { global.dropped_index.pop(); next++; }
            }
            if (!heap.empty() && heap.top().index == next) {
                Frame top = heap.top(); heap.pop(); top.t_buffered = now_s();
                if (top.index < global.end_index) emit(top);
                next++;
            }
            else break;
        }
        if (!got) {
            if (global.finished == num_workers && global.output_queue.size() == 0) {
                while (!heap.empty()) { Frame top = heap.top(); heap.pop(); if (top.index < global.end_index) emit(top); }   // flush (frames lost to an error leave gaps)
                break;
            }
            std::this_thread::sleep_for(std::chrono::microseconds(200));
        }
    }
    writers.finish();   // every image is on disk before the run reports its end
    const double dt = now_s() - t0;
    LOG_INFO("Done, exiting. # frames: %d  (%.1f frames/s overall, %d dropped)", written, written / std::max(dt, 1e-9), global.dropped.load());
    if (Fi("audit_every") > 0)
        LOG_INFO("Audit summary: %lld/%lld audited frames identical to the parity mode, max joint \xce\x94 %.3g px (every %d-th batch)",
                 global.audit_identical, global.audit_frames, (double)global.audit_max_joint, Fi("audit_every"));
}

static bool ensure_dir(const std::string& d) {
    struct stat st;
    if (stat(d.c_str(), &st) == 0) return S_ISDIR(st.st_mode);
    return mkdir(d.c_str(), 0755) == 0;
}

int main(int argc, char** argv) {
    define_flags();
    if (parse_flags(argc, argv)) return 1;
    if (!F("probe_image").empty()) {
        int w = 0, h = 0;
        std::vector<uint8_t> px;
        if (!read_image(F("probe_image"), w, h, px)) { LOG_ERROR("cannot decode %s", F("probe_image").c_str()); return 1; }
        uint64_t hash = 1469598103934665603ull;
        for (uint8_t b : px) { hash ^= b; hash *= 1099511628211ull; }
        printf("%dx%d %016llx\n", w, h, (unsigned long long)hash);
        return 0;
    }
    if (Fb("gpu_decode") && (Fi("synthetic") > 0 || (F("video").empty() && F("image_dir").empty()))) {
        LOG_ERROR("--gpu_decode reconstructs JPEG files on the GPU: it needs --image_dir or a Motion-JPEG --video (not --synthetic or a camera)");
        return 1;
    }
    if (Fb("gpu_entropy") && (Fi("synthetic") > 0 || (F("video").empty() && F("image_dir").empty()))) {
        LOG_ERROR("--gpu_entropy decodes JPEG files on the GPU: it needs --image_dir or a Motion-JPEG --video (not --synthetic or a camera)");
        return 1;
    }
    if (F("video").empty() && F("image_dir").empty() && Fi("synthetic") <= 0) {   // the camera (rtpose.cpp:401-405, 1694-1695)
        int cw = 0, ch = 0;
        if (sscanf(F("camera_resolution").c_str(), "%dx%d", &cw, &ch) != 2) {
            LOG_ERROR("Error, camera resolution format (%s) invalid, should be e.g., 1280x720", F("camera_resolution").c_str());
            return 1;
        }
        if (pe_camera_open(Fi("camera"), cw, ch, &global.camera)) {
            LOG_ERROR("%s; other sources: --video (Motion-JPEG / uncompressed .avi), --image_dir, --synthetic N", pe_camera_last_error());
            return 1;
        }
        char cc[5];
        pe_camera_info(global.camera, &global.camera_w, &global.camera_h, cc);
        LOG_INFO("Camera %d: %dx%d %s", Fi("camera"), global.camera_w, global.camera_h, cc);
    }
    if (F("frame_format") != "jpg" && F("frame_format") != "bmp") { LOG_ERROR("--frame_format must be jpg or bmp"); return 1; }
    if (Fi("audit_every") < 0) { LOG_ERROR("--audit_every must be 0 (off) or a positive number of batches"); return 1; }
    if (Fi("audit_every") > 0 && Fi("precision") == PE_PREC_F16X2) {
        LOG_ERROR("--audit_every compares a faster precision with the parity mode; with --precision 2 there is nothing to compare");
        return 1;
    }
    if (sscanf(F("resolution").c_str(), "%dx%d", &global.disp_w, &global.disp_h) != 2) { LOG_ERROR("Error, resolution format (%s) invalid, should be e.g., 960x540", F("resolution").c_str()); return 1; }
    if (sscanf(F("net_resolution").c_str(), "%dx%d", &global.net_w, &global.net_h) != 2) { LOG_ERROR("Error, net resolution format (%s) invalid, should be e.g., 656x368 (multiples of 16)", F("net_resolution").c_str()); return 1; }
    if (!F("image_dir").empty()) {   // readImageDirIfFlagEnabled (rtpose.cpp:1732-1755): sorted list of image files
        DIR* d = opendir(F("image_dir").c_str());
        if (!d) { LOG_ERROR("Folder %s does not exist.", F("image_dir").c_str()); return -1; }
        while (dirent* ent = readdir(d)) {
            const std::string n = ent->d_name;
            const size_t dot = n.find_last_of('.');
            const std::string ext = dot == std::string::npos ? "" : n.substr(dot);
            const std::string le = lower_ext(n);
            // the reference lists .jpg / .png / .bmp (rtpose.cpp:1743); .jpeg, .ppm and upper-case names are accepted as well
            if (le == ".jpg" || le == ".png" || le == ".bmp" || le == ".jpeg" || le == ".ppm") global.image_list.push_back(F("image_dir") + "/" + n);
        }
        closedir(d);
        std::sort(global.image_list.begin(), global.image_list.end());
        if (global.disp_w == -1 && !global.image_list.empty()) {   // --resolution -1x-1: take it from the first image (:1683-1686)
            std::vector<uint8_t> tmp;
            const std::string& p = global.image_list[0];
            if (!read_image(p, global.disp_w, global.disp_h, tmp)) return 1;
            LOG_INFO("Setting display resolution from first image: %dx%d", global.disp_w, global.disp_h);
        }
    }
    if (!F("video").empty() && F("image_dir").empty() && Fi("synthetic") <= 0) {   // cap.open(FLAGS_video) (rtpose.cpp:406, 1677-1682)
        if (pe_video_open(F("video").c_str(), &global.video)) { LOG_ERROR("Couldn't open video file %s: %s", F("video").c_str(), pe_video_last_error()); return 1; }
        char cc[5];
        pe_video_info(global.video, &global.video_w, &global.video_h, &global.video_fps, &global.video_frames, cc);
        LOG_INFO("Video %s: %dx%d, %d frames, %.3f fps, %s", F("video").c_str(), global.video_w, global.video_h, global.video_frames, global.video_fps, cc);
        if (global.disp_w == -1) { global.disp_w = global.video_w; global.disp_h = global.video_h; }
    }
    if (global.disp_w <= 0 || global.disp_h <= 0) { LOG_ERROR("Invalid resolution without video/images: %dx%d", global.disp_w, global.disp_h); return 1; }
    LOG_INFO("Display resolution: %dx%d", global.disp_w, global.disp_h);
    LOG_INFO("Net resolution: %dx%d", global.net_w, global.net_h);
    if (!F("write_frames").empty() && !ensure_dir(F("write_frames"))) { LOG_ERROR("Could not write to or create directory %s", F("write_frames").c_str()); return 1; }
    if (!F("write_json").empty() && !ensure_dir(F("write_json"))) { LOG_ERROR("Could not write to or create directory %s", F("write_json").c_str()); return 1; }

    int model = model_from_prototxt(F("caffeproto"));
    if (model < 0 && !F("model").empty()) model = F("model") == "MPI" ? PE_MODEL_MPI_15 : PE_MODEL_COCO_18;
    if (model == -1) { LOG_ERROR("cannot read --caffeproto %s (pass --model COCO|MPI to run without it)", F("caffeproto").c_str()); return 1; }
    if (model == -2) { LOG_ERROR("Unknown number of parts! Couldn't set model"); return 1; }
    if (global.proto_readable) LOG_INFO("Net built from %s", F("caffeproto").c_str());
    global.model = model;
    {
        std::unique_ptr<ModelDescriptor> md;
        ModelDescriptorFactory::createModelDescriptor(model == PE_MODEL_MPI_15 ? ModelDescriptorFactory::Type::MPI_15 : ModelDescriptorFactory::Type::COCO_18, md);
        global.num_parts = md->get_number_parts();
        LOG_INFO("Selecting %s model: %d parts, %d limbs.", model == PE_MODEL_MPI_15 ? "MPI" : "COCO", global.num_parts, md->number_limb_sequence());
    }
    // run-time thresholds start from the model defaults of rtpose.cpp:212-226
    if (model == PE_MODEL_MPI_15) { global.nms_threshold = 0.2f; global.connect_inter_threshold = 0.01f; global.connect_inter_min_above_threshold = 8; }
    global.part_to_show = Fi("part_to_show");
    // frames per forward: 1 is the reference's behaviour (lowest latency); file / synthetic sources have no latency to protect, so by
    // default one forward carries as many frames as give two full waves of 128-row tiles on 132 SMs (8 at 656x368); results do not change
    global.batch = Fi("batch");
    if (global.batch <= 0) {   // largest batch whose 128-row tiles still fit two waves of one CTA per SM (one tile more costs a third wave)
        const long long rows = (long long)(global.net_h / 8 + 3) * (global.net_w / 8 + 3) * std::max(1, Fi("num_scales"));
        global.batch = (int)std::min<long long>(16, std::max<long long>(1, (2LL * 132 * 128) / rows));
    }
    global.engines_per_gpu = Fi("engines_per_gpu") > 0 ? std::min(4, Fi("engines_per_gpu")) : (Fi("batch") <= 0 ? 2 : 1);
    global.queue_limit = std::max(10, 4 * global.batch * std::max(1, Fi("num_gpu")) * global.engines_per_gpu);
    if (Fb("keys_from_stdin")) std::thread(key_reader).detach();   // blocks in getchar(): never joined
    if (Fb("decode_bench")) return decode_bench();
    const int num_gpu = std::max(1, Fi("num_gpu"));
    std::vector<pe_engine*> engines, audit;
    const int per_gpu = global.engines_per_gpu, num_workers = num_gpu * per_gpu;
    if (!create_engines(num_gpu, per_gpu, Fi("precision"), engines) ||
        (Fi("audit_every") > 0 && !create_engines(num_gpu, per_gpu, PE_PREC_F16X2, audit))) {
        for (pe_engine* e : engines) pe_destroy(e);
        for (pe_engine* e : audit) pe_destroy(e);
        return 1;
    }
    std::vector<std::thread> workers;
    for (int i = 0; i < num_workers; i++) workers.emplace_back(worker, i, engines[i], audit.empty() ? nullptr : audit[i]);
    std::thread prod(run_producers);
    std::thread ord(orderer_and_writer, num_workers);
    prod.join();
    for (auto& t : workers) t.join();
    ord.join();
    for (pe_engine* e : engines) pe_destroy(e);
    for (pe_engine* e : audit) pe_destroy(e);
    g_pinned.clear();
    pe_video_close(global.video);
    pe_camera_close(global.camera);
    return global.failed ? 1 : 0;   // ESC ends the run with 0 like the reference (rtpose.cpp:1564, 1775-1779)
}
