// cv::VideoCapture for --video (examples/rtpose/rtpose.cpp:394-411, 433-446, 525-545, 1677-1682): open(file), get(FPS /
// FRAME_COUNT / FRAME_WIDTH / FRAME_HEIGHT), set(POS_FRAMES), operator>>.  OpenCV's capture back ends (FFmpeg, GStreamer, V4L2)
// are third-party code that this image does not have for C++; what is written out here is the container and the codecs that
// need nothing beyond this repository's own JPEG decoder:
//   * RIFF AVI 1.0 and OpenDML ('AVIX' extension RIFFs, files > 1 GB), frames located by walking the 'movi' lists (the optional
//     'idx1' / 'indx' indices are not needed and not trusted), 'rec ' lists, first video stream;
//   * Motion-JPEG ('MJPG', 'mjpg', 'AVI1', 'JPEG' ...: every frame a JPEG, decoded by pe_decode_jpeg - libjpeg's arithmetic, i.e.
//     the pixels cv::imdecode / OpenCV's own MJPEG reader return; frames without DHT use the Annex K tables);
//   * uncompressed DIB frames (biCompression BI_RGB, 24 or 32 bits, bottom-up or top-down rows padded to 4 bytes).
// Inter-frame codecs (H.264, MPEG-4 ...) are reported as PE_ERR_INVALID with the FourCC in the message.
// Frames are addressed by index (CV_CAP_PROP_POS_FRAMES), reads are thread-safe (pread), so several decoder threads can work on
// one file.  Host code, no GPU.
#include <fcntl.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <sys/stat.h>
#include <unistd.h>

#include <string>
#include <vector>

#include "../../include/poseengine.h"

namespace {

thread_local std::string g_video_error;

struct FrameRef { uint64_t off; uint32_t size; };

uint32_t rd32(const uint8_t* p) { return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24; }
uint16_t rd16(const uint8_t* p) { return (uint16_t)(p[0] | p[1] << 8); }
bool tag_is(const uint8_t* p, const char* t) { return memcmp(p, t, 4) == 0; }

}  // namespace

struct pe_video {
    int fd = -1;
    uint64_t file_size = 0;
    int w = 0, h = 0, bits = 0, stream = -1;
    bool top_down = false, mjpeg = false;
    double fps = 0;
    char fourcc[5] = {0, 0, 0, 0, 0};
    std::vector<FrameRef> frames;
    std::string path;

    bool read_at(uint64_t off, void* dst, size_t n) const {
        uint8_t* d = (uint8_t*)dst;
        while (n) {
            const ssize_t got = pread(fd, d, n, (off_t)off);
            if (got <= 0) return false;
            d += got; off += (uint64_t)got; n -= (size_t)got;
        }
        return true;
    }
    // Walk the chunks of [off, end): lists are entered, '##dc' / '##db' chunks of the video stream become frames.
    bool walk(uint64_t off, uint64_t end, int depth, bool in_movi, int& n_streams) {
        uint8_t hd[12];
        while (off + 8 <= end) {
            if (!read_at(off, hd, 8)) return false;
            const uint32_t sz = rd32(hd + 4);
            const uint64_t body = off + 8, next = body + sz + (sz & 1u);
            if (body + sz > file_size) {                       // truncated file: keep what is complete (a recording that was cut off)
                if (tag_is(hd, "LIST") || tag_is(hd, "RIFF")) {
                    if (body + 4 <= file_size && read_at(body, hd + 8, 4) && depth < 8)
                        walk(body + 4, file_size, depth + 1, in_movi || tag_is(hd + 8, "movi"), n_streams);
                }
                return true;
            }
            if (tag_is(hd, "RIFF") || tag_is(hd, "LIST")) {
                if (sz >= 4 && depth < 8) {
                    if (!read_at(body, hd + 8, 4)) return false;
                    const bool movi = tag_is(hd + 8, "movi");
                    if (tag_is(hd, "RIFF") && !(tag_is(hd + 8, "AVI ") || tag_is(hd + 8, "AVIX"))) { off = next; continue; }
                    if (!walk(body + 4, body + sz, depth + 1, in_movi || movi, n_streams)) return false;
                }
            } else if (in_movi) {
                // stream chunk: two decimal digits + 'dc' (compressed) / 'db' (uncompressed); 'wb' audio, 'pc' palette changes, 'ix##' indices
                if (hd[0] >= '0' && hd[0] <= '9' && hd[1] >= '0' && hd[1] <= '9' && hd[2] == 'd' && (hd[3] == 'c' || hd[3] == 'b') &&
                    (hd[0] - '0') * 10 + (hd[1] - '0') == stream)
                    frames.push_back({body, sz});
            } else if (tag_is(hd, "avih") && sz >= 40) {
                uint8_t b[40];
                if (!read_at(body, b, 40)) return false;
                const uint32_t us = rd32(b);
                if (us && fps == 0) fps = 1e6 / us;            // the stream header's rate / scale wins when present
            } else if (tag_is(hd, "strh") && sz >= 48) {
                uint8_t b[48];
                if (!read_at(body, b, 48)) return false;
                const int idx = n_streams++;
                if (tag_is(b, "vids") && stream < 0) {
                    stream = idx;
                    memcpy(fourcc, b + 4, 4);
                    const uint32_t scale = rd32(b + 20), rate = rd32(b + 24);
                    if (scale && rate) fps = (double)rate / scale;
                    pending_strf = true;
                }
            } else if (tag_is(hd, "strf") && pending_strf && sz >= 40) {
                uint8_t b[40];
                if (!read_at(body, b, 40)) return false;
                pending_strf = false;
                w = (int)rd32(b + 4);
                const int32_t bh = (int32_t)rd32(b + 8);
                top_down = bh < 0;
                h = bh < 0 ? -bh : bh;
                bits = rd16(b + 14);
                memcpy(compression, b + 16, 4);
            }
            off = next;
        }
        return true;
    }
    bool pending_strf = false;
    uint8_t compression[4] = {0, 0, 0, 0};
};

extern "C" const char* pe_video_last_error(void) { return g_video_error.c_str(); }

extern "C" int pe_video_open(const char* path, pe_video** out) {
    if (!path || !out) { g_video_error = "null argument"; return PE_ERR_INVALID; }
    *out = nullptr;
    pe_video* v = new pe_video;
    v->path = path;
    v->fd = open(path, O_RDONLY);
    struct stat st;
    if (v->fd < 0 || fstat(v->fd, &st) != 0) {
        g_video_error = std::string("Couldn't open video file ") + path;
        if (v->fd >= 0) close(v->fd);
        delete v;
        return PE_ERR_IO;
    }
    v->file_size = (uint64_t)st.st_size;
    uint8_t hd[12];
    auto fail = [&](int code, const std::string& msg) { g_video_error = msg; close(v->fd); delete v; return code; };
    if (v->file_size < 12 || !v->read_at(0, hd, 12) || !tag_is(hd, "RIFF") || !tag_is(hd + 8, "AVI "))
        return fail(PE_ERR_INVALID, std::string(path) + ": not a RIFF AVI file (the containers read here: AVI / OpenDML with Motion-JPEG or "
                                        "uncompressed frames; other containers need a video library this build does not have)");
    int n_streams = 0;
    bool walked = false;
    try { walked = v->walk(0, v->file_size, 0, false, n_streams); } catch (...) { walked = false; }   // no exception crosses the C ABI
    if (!walked) return fail(PE_ERR_IO, std::string(path) + ": read error while indexing");
    if (v->stream < 0 || v->w <= 0 || v->h <= 0 || v->w > 32768 || v->h > 32768) return fail(PE_ERR_INVALID, std::string(path) + ": no video stream");
    char cc[5] = {0, 0, 0, 0, 0};
    memcpy(cc, v->compression, 4);
    for (int i = 0; i < 4; i++) if (cc[i] >= 'a' && cc[i] <= 'z') cc[i] = (char)(cc[i] - 32);
    const uint32_t comp = rd32(v->compression);
    if (!strcmp(cc, "MJPG") || !strcmp(cc, "AVI1") || !strcmp(cc, "AVI2") || !strcmp(cc, "JPEG") || !strcmp(cc, "JPGL") || !strcmp(cc, "IJPG") ||
        !strcmp(cc, "AVRN") || !strcmp(cc, "DMB1")) {
        v->mjpeg = true;
    } else if (comp == 0 /* BI_RGB */ || !strcmp(cc, "DIB ") || !strcmp(cc, "RAW ")) {
        if (v->bits != 24 && v->bits != 32) return fail(PE_ERR_INVALID, std::string(path) + ": uncompressed frames with " + std::to_string(v->bits) + " bits per pixel (24 and 32 are read)");
    } else {
        for (int i = 0; i < 4; i++) if ((uint8_t)cc[i] < 32 || (uint8_t)cc[i] > 126) cc[i] = '?';
        return fail(PE_ERR_INVALID, std::string(path) + ": codec '" + cc + "' needs a video library this build does not have (read here: Motion-JPEG and uncompressed AVI)");
    }
    if (v->mjpeg) memcpy(v->fourcc, "MJPG", 4); else memcpy(v->fourcc, "DIB ", 4);
    if (v->frames.empty()) return fail(PE_ERR_INVALID, std::string(path) + ": no frames in the video stream");
    if (!(v->fps > 0)) v->fps = 30.0;
    *out = v;
    return PE_OK;
}

extern "C" void pe_video_close(pe_video* v) {
    if (!v) return;
    if (v->fd >= 0) close(v->fd);
    delete v;
}

extern "C" int pe_video_info(const pe_video* v, int* w, int* h, double* fps, int* frame_count, char fourcc[5]) {
    if (!v) return PE_ERR_INVALID;
    if (w) *w = v->w;
    if (h) *h = v->h;
    if (fps) *fps = v->fps;
    if (frame_count) *frame_count = (int)v->frames.size();
    if (fourcc) memcpy(fourcc, v->fourcc, 5);
    return PE_OK;
}

extern "C" int pe_video_read(const pe_video* v, int index, uint8_t* bgr, long long cap) {
    if (!v || !bgr) { g_video_error = "null argument"; return PE_ERR_INVALID; }
    if (index < 0 || index >= (int)v->frames.size()) { g_video_error = "frame index outside the video"; return PE_ERR_INVALID; }
    if (cap < (long long)v->w * v->h * 3) { g_video_error = "frame buffer too small"; return PE_ERR_INVALID; }
    // a zero-length chunk repeats the previous frame (dropped frame, as capture tools write them)
    while (index > 0 && v->frames[index].size == 0) index--;
    const FrameRef fr = v->frames[index];
    if (fr.size == 0) { memset(bgr, 0, (size_t)v->w * v->h * 3); return PE_OK; }
    std::vector<uint8_t> buf;
    try { buf.resize(fr.size); } catch (...) { g_video_error = v->path + ": out of memory for a frame"; return PE_ERR_IO; }
    if (!v->read_at(fr.off, buf.data(), fr.size)) { g_video_error = v->path + ": read error"; return PE_ERR_IO; }
    if (v->mjpeg) {
        int jw = 0, jh = 0;
        int rc = pe_decode_jpeg(buf.data(), (long long)buf.size(), &jw, &jh, nullptr, 0);
        if (rc == 0 && (jw != v->w || jh != v->h)) rc = -1;
        if (rc == 0) rc = pe_decode_jpeg(buf.data(), (long long)buf.size(), &jw, &jh, bgr, cap);
        if (rc != 0) { g_video_error = v->path + ": frame " + std::to_string(index) + " is not a decodable JPEG"; return rc == -2 ? PE_ERR_INVALID : PE_ERR_IO; }
        return PE_OK;
    }
    const int bpp = v->bits / 8;
    const size_t stride = ((size_t)v->w * bpp + 3) & ~(size_t)3;
    if ((size_t)fr.size < stride * (size_t)v->h) { g_video_error = v->path + ": short uncompressed frame"; return PE_ERR_IO; }
    for (int y = 0; y < v->h; y++) {
        const uint8_t* src = buf.data() + (size_t)(v->top_down ? y : v->h - 1 - y) * stride;
        uint8_t* dst = bgr + (size_t)y * v->w * 3;
        if (bpp == 3) memcpy(dst, src, (size_t)v->w * 3);
        else for (int x = 0; x < v->w; x++) { dst[3 * x] = src[4 * x]; dst[3 * x + 1] = src[4 * x + 1]; dst[3 * x + 2] = src[4 * x + 2]; }
    }
    return PE_OK;
}

static long long read_jpeg_frame(const pe_video* v, int index, void* buf, long long cap,
                                 long long (*reader)(const uint8_t*, long long, void*, long long));
extern "C" long long pe_video_read_coefs(const pe_video* v, int index, void* buf, long long cap) {
    return read_jpeg_frame(v, index, buf, cap, pe_jpeg_read_coefs);
}
extern "C" long long pe_video_read_scan(const pe_video* v, int index, void* buf, long long cap) {
    return read_jpeg_frame(v, index, buf, cap, pe_jpeg_read_scan);
}
static long long read_jpeg_frame(const pe_video* v, int index, void* buf, long long cap,
                                 long long (*reader)(const uint8_t*, long long, void*, long long)) {
    if (!v) { g_video_error = "null argument"; return -PE_ERR_INVALID; }
    if (!v->mjpeg) { g_video_error = v->path + ": not a Motion-JPEG video"; return -PE_ERR_INVALID; }
    if (index < 0 || index >= (int)v->frames.size()) { g_video_error = "frame index outside the video"; return -PE_ERR_INVALID; }
    while (index > 0 && v->frames[index].size == 0) index--;   // a zero-length chunk repeats the previous frame, as in pe_video_read
    const FrameRef fr = v->frames[index];
    if (fr.size == 0) { g_video_error = v->path + ": the video starts with an empty frame (pe_video_read gives it as black)"; return -PE_ERR_INVALID; }
    std::vector<uint8_t> data;
    try { data.resize(fr.size); } catch (...) { g_video_error = v->path + ": out of memory for a frame"; return -PE_ERR_IO; }
    if (!v->read_at(fr.off, data.data(), fr.size)) { g_video_error = v->path + ": read error"; return -PE_ERR_IO; }
    int jw = 0, jh = 0;
    const int hrc = pe_decode_jpeg(data.data(), (long long)data.size(), &jw, &jh, nullptr, 0);   // frame header only
    long long rc = hrc ? hrc : reader(data.data(), (long long)data.size(), nullptr, 0);
    if (rc == -3) { g_video_error = v->path + ": frame " + std::to_string(index) + " needs the host entropy stage"; return -3; }
    if (rc > 0 && (jw != v->w || jh != v->h)) rc = -1;   // pe_video_read's rule: every frame has the video's size
    if (rc > 0 && buf && cap >= rc && reader(data.data(), (long long)data.size(), buf, cap) != rc) rc = -1;
    if (rc <= 0) { g_video_error = v->path + ": frame " + std::to_string(index) + " is not a decodable JPEG"; return rc == -2 ? -PE_ERR_INVALID : -PE_ERR_IO; }
    return rc;
}
