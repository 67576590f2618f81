// cv::VideoCapture on a camera index, as getFrameFromCam opens it when neither --video nor --image_dir is given
// (examples/rtpose/rtpose.cpp:401-405: cap.open(FLAGS_camera), CV_CAP_PROP_FRAME_WIDTH / HEIGHT from --camera_resolution, then
// cap >> image per frame).  OpenCV's Linux capture back end is Video4Linux2; this is that path written directly against the
// kernel interface (<linux/videodev2.h>, memory-mapped streaming I/O): /dev/video<index>, Motion-JPEG preferred (frames go
// through pe_decode_jpeg, Annex K tables when the camera leaves DHT out), else packed YUYV 4:2:2 converted with the fixed-point
// BT.601 arithmetic of cv::cvtColor(COLOR_YUV2BGR_YUYV) - what OpenCV's V4L2 back end applies (pinned to cv2 in tests/test_abi.py
// through pe_yuyv_to_bgr).  The build container and the GPU boxes have no capture device: the streaming sequence below runs in
// tests/test_camera_device.py against tests/stub/fake_v4l2.c, an LD_PRELOAD stand-in that enforces a driver's state machine; it has
// not met real hardware.  Host code, no GPU.
#include <errno.h>
#include <fcntl.h>
#include <poll.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <sys/ioctl.h>
#include <sys/mman.h>
#include <unistd.h>

#include <linux/videodev2.h>

#include <string>
#include <vector>

#include "../../include/poseengine.h"
#include "pixels.cuh"

namespace {

thread_local std::string g_camera_error;

int xioctl(int fd, unsigned long req, void* arg) {
    int r;
    do r = ioctl(fd, req, arg); while (r == -1 && errno == EINTR);
    return r;
}

}  // namespace

// cv::cvtColor(src, dst, COLOR_YUV2BGR_YUYV) (imgproc color_yuv: ITU-R BT.601, studio range, 20-bit fixed point; pixels.cuh)
extern "C" int pe_yuyv_to_bgr(const uint8_t* yuyv, int w, int h, long long stride, uint8_t* bgr) {
    if (!yuyv || !bgr || w <= 0 || h <= 0 || (w & 1) || stride < 2LL * w) return PE_ERR_INVALID;
    for (int y = 0; y < h; y++) {
        const uint8_t* s = yuyv + (size_t)y * (size_t)stride;
        uint8_t* d = bgr + (size_t)y * w * 3;
        for (int x = 0; x < w; x += 2, s += 4, d += 6) pe_pix::pair422(pe_pix::BT601_STUDIO, s, 0, d);
    }
    return PE_OK;
}

struct pe_camera {
    int fd = -1;
    int w = 0, h = 0;
    uint32_t pixfmt = 0;
    long long stride = 0;
    bool streaming = false;
    struct Buf { void* p = nullptr; size_t len = 0; };
    std::vector<Buf> bufs;
};

extern "C" const char* pe_camera_last_error(void) { return g_camera_error.c_str(); }

extern "C" void pe_camera_close(pe_camera* c) {
    if (!c) return;
    if (c->fd >= 0) {
        if (c->streaming) { int type = V4L2_BUF_TYPE_VIDEO_CAPTURE; xioctl(c->fd, VIDIOC_STREAMOFF, &type); }
        for (auto& b : c->bufs) if (b.p && b.p != MAP_FAILED) munmap(b.p, b.len);
        close(c->fd);
    }
    delete c;
}

extern "C" int pe_camera_open(int index, int want_w, int want_h, pe_camera** out) {
    if (!out || index < 0) { g_camera_error = "bad argument"; return PE_ERR_INVALID; }
    *out = nullptr;
    char dev[64];
    snprintf(dev, sizeof dev, "/dev/video%d", index);
    pe_camera* c = new pe_camera;
    auto fail = [&](int code, const std::string& msg) { g_camera_error = msg; pe_camera_close(c); return code; };
    c->fd = open(dev, O_RDWR | O_NONBLOCK);
    if (c->fd < 0) return fail(PE_ERR_IO, std::string("Couldn't open camera ") + std::to_string(index) + " (" + dev + ": " + strerror(errno) + ")");
    v4l2_capability cap;
    memset(&cap, 0, sizeof cap);
    if (xioctl(c->fd, VIDIOC_QUERYCAP, &cap) < 0 || !(cap.capabilities & V4L2_CAP_VIDEO_CAPTURE) || !(cap.capabilities & V4L2_CAP_STREAMING))
        return fail(PE_ERR_INVALID, std::string(dev) + " is not a streaming video capture device");
    // CV_CAP_PROP_FRAME_WIDTH / HEIGHT (rtpose.cpp:403-404): ask for the size, Motion-JPEG first (full frame rate at 720p over USB), then YUYV
    const uint32_t wanted[2] = {V4L2_PIX_FMT_MJPEG, V4L2_PIX_FMT_YUYV};
    v4l2_format fmt;
    bool ok = false;
    for (int k = 0; k < 2 && !ok; k++) {
        memset(&fmt, 0, sizeof fmt);
        fmt.type = V4L2_BUF_TYPE_VIDEO_CAPTURE;
        fmt.fmt.pix.width = (uint32_t)(want_w > 0 ? want_w : 1280);
        fmt.fmt.pix.height = (uint32_t)(want_h > 0 ? want_h : 720);
        fmt.fmt.pix.pixelformat = wanted[k];
        fmt.fmt.pix.field = V4L2_FIELD_ANY;
        ok = xioctl(c->fd, VIDIOC_S_FMT, &fmt) == 0 && fmt.fmt.pix.pixelformat == wanted[k];
    }
    if (!ok) return fail(PE_ERR_INVALID, std::string(dev) + " offers neither Motion-JPEG nor YUYV frames");
    c->w = (int)fmt.fmt.pix.width; c->h = (int)fmt.fmt.pix.height; c->pixfmt = fmt.fmt.pix.pixelformat;
    c->stride = fmt.fmt.pix.bytesperline ? (long long)fmt.fmt.pix.bytesperline : 2LL * c->w;
    if (c->w <= 0 || c->h <= 0 || c->w > 16384 || c->h > 16384 || (c->pixfmt == V4L2_PIX_FMT_YUYV && (c->w & 1)))
        return fail(PE_ERR_INVALID, std::string(dev) + " reports an unusable frame size");
    v4l2_requestbuffers req;
    memset(&req, 0, sizeof req);
    req.count = 4; req.type = V4L2_BUF_TYPE_VIDEO_CAPTURE; req.memory = V4L2_MEMORY_MMAP;
    if (xioctl(c->fd, VIDIOC_REQBUFS, &req) < 0 || req.count < 2) return fail(PE_ERR_IO, std::string(dev) + ": VIDIOC_REQBUFS failed");
    c->bufs.resize(req.count);
    for (uint32_t i = 0; i < req.count; i++) {
        v4l2_buffer b;
        memset(&b, 0, sizeof b);
        b.type = V4L2_BUF_TYPE_VIDEO_CAPTURE; b.memory = V4L2_MEMORY_MMAP; b.index = i;
        if (xioctl(c->fd, VIDIOC_QUERYBUF, &b) < 0) return fail(PE_ERR_IO, std::string(dev) + ": VIDIOC_QUERYBUF failed");
        c->bufs[i].len = b.length;
        c->bufs[i].p = mmap(nullptr, b.length, PROT_READ | PROT_WRITE, MAP_SHARED, c->fd, b.m.offset);
        if (c->bufs[i].p == MAP_FAILED) { c->bufs[i].p = nullptr; return fail(PE_ERR_IO, std::string(dev) + ": mmap of a capture buffer failed"); }
        if (xioctl(c->fd, VIDIOC_QBUF, &b) < 0) return fail(PE_ERR_IO, std::string(dev) + ": VIDIOC_QBUF failed");
    }
    int type = V4L2_BUF_TYPE_VIDEO_CAPTURE;
    if (xioctl(c->fd, VIDIOC_STREAMON, &type) < 0) return fail(PE_ERR_IO, std::string(dev) + ": VIDIOC_STREAMON failed");
    c->streaming = true;
    *out = c;
    return PE_OK;
}

extern "C" int pe_camera_info(const pe_camera* c, int* w, int* h, char fourcc[5]) {
    if (!c) return PE_ERR_INVALID;
    if (w) *w = c->w;
    if (h) *h = c->h;
    if (fourcc) { memcpy(fourcc, c->pixfmt == V4L2_PIX_FMT_MJPEG ? "MJPG" : "YUYV", 4); fourcc[4] = 0; }
    return PE_OK;
}

// cap >> image: blocks until the driver hands over the next frame (at most timeout_ms), converts it to uint8 BGR HWC
extern "C" int pe_camera_grab(pe_camera* c, uint8_t* bgr, long long cap, int timeout_ms) {
    if (!c || !bgr) { g_camera_error = "null argument"; return PE_ERR_INVALID; }
    if (cap < (long long)c->w * c->h * 3) { g_camera_error = "frame buffer too small"; return PE_ERR_INVALID; }
    for (int attempt = 0; attempt < 8; attempt++) {
        pollfd p;
        p.fd = c->fd; p.events = POLLIN; p.revents = 0;
        const int pr = poll(&p, 1, timeout_ms > 0 ? timeout_ms : 5000);
        if (pr == 0) { g_camera_error = "camera: no frame within the timeout"; return PE_ERR_IO; }
        if (pr < 0) { if (errno == EINTR) continue; g_camera_error = std::string("camera: poll: ") + strerror(errno); return PE_ERR_IO; }
        v4l2_buffer b;
        memset(&b, 0, sizeof b);
        b.type = V4L2_BUF_TYPE_VIDEO_CAPTURE; b.memory = V4L2_MEMORY_MMAP;
        if (xioctl(c->fd, VIDIOC_DQBUF, &b) < 0) {
            if (errno == EAGAIN) continue;
            g_camera_error = std::string("camera: VIDIOC_DQBUF: ") + strerror(errno);
            return PE_ERR_IO;
        }
        int rc = PE_ERR_IO;
        if (b.index < c->bufs.size() && !(b.flags & V4L2_BUF_FLAG_ERROR)) {
            const uint8_t* src = (const uint8_t*)c->bufs[b.index].p;
            const long long used = b.bytesused <= c->bufs[b.index].len ? (long long)b.bytesused : (long long)c->bufs[b.index].len;   // never past the mapping
            if (c->pixfmt == V4L2_PIX_FMT_MJPEG) {
                int jw = 0, jh = 0;
                if (pe_decode_jpeg(src, used, &jw, &jh, nullptr, 0) == 0 && jw == c->w && jh == c->h &&
                    pe_decode_jpeg(src, used, &jw, &jh, bgr, cap) == 0) rc = PE_OK;
            } else if (used >= c->stride * c->h) {
                rc = pe_yuyv_to_bgr(src, c->w, c->h, c->stride, bgr);
            }
        }
        xioctl(c->fd, VIDIOC_QBUF, &b);
        if (rc == PE_OK) return PE_OK;   // a corrupt frame (USB hiccup) is skipped, like cap >> does
    }
    g_camera_error = "camera: eight unusable frames in a row";
    return PE_ERR_IO;
}
