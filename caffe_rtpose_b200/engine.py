"""Host-side mirror of the reference's per-GPU interface over the C ABI (include/poseengine.h).

The reference's worker holds a `caffe::Net`, a `caffe::NmsLayer*`, a `caffe::ImResizeLayer*` and a
`ModelDescriptor` (examples/rtpose/rtpose.cpp:133-142, 173-237) and calls, per frame,
`nms_layer->SetThreshold(...)`, `ForwardFrom(0)`, `connectLimbs*` (rtpose.cpp:1145-1166).  `PoseEngine`
keeps those names and argument meanings (`nms_layer.SetThreshold`, `resize_layer.SetStartScale`,
`model_descriptor.get_limb_sequence()` ...) and routes everything to libposeengine.so, the hand-written
sm_90a implementation.  There is no CPU or PyTorch fallback: if the shared library is missing or no
H100 (sm_90) is visible the constructor raises.
"""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
# PE_LIB: another build of the same library (A/B measurements of two builds in one process tree); never a different implementation
LIB_PATH = os.environ.get("PE_LIB") or os.path.join(HERE, "libposeengine.so")

MPI_15, COCO_18 = 0, 1
PREC_FP32_SIMT, PREC_BF16X1, PREC_BF16X2, PREC_BF16X3 = 0, 1, 2, 3
PREC_F16X2 = PREC_BF16X2   # the parity mode: 2 fp16 planes, chunked round-to-nearest accumulation (poseengine.h)
PREC_F16X1 = 4             # the fast mode: the parity mode's hi plane alone, one MMA per MAC (poseengine.h)
MAX_PEOPLE = 96
# pixel formats of forward_pixels / pixels_to_bgr (PE_PIX_*, poseengine.h)
PIX_BGR, PIX_RGB, PIX_YUYV, PIX_NV12, PIX_I420 = 0, 1, 2, 3, 4

_f32p = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")


class _Config(C.Structure):
    _fields_ = [("device", C.c_int), ("model", C.c_int), ("net_w", C.c_int), ("net_h", C.c_int), ("disp_w", C.c_int),
                ("disp_h", C.c_int), ("num_scales", C.c_int), ("start_scale", C.c_double), ("scale_gap", C.c_double),
                ("max_batch", C.c_int), ("precision", C.c_int)]


class _PixelFormat(C.Structure):
    _fields_ = [("format", C.c_int), ("width", C.c_int), ("height", C.c_int), ("pitch", C.c_longlong), ("chroma_offset", C.c_longlong)]


class PoseEngineError(RuntimeError):
    pass


class _ResultDiff(C.Structure):
    _fields_ = [("identical", C.c_int), ("parts_count_differ", C.c_int), ("peaks_moved", C.c_int), ("persons_matched", C.c_int),
                ("max_joint_dist", C.c_float)]


_lib = None

# every symbol include/poseengine.h declares (checked by tests/test_abi.py)
ABI_SYMBOLS = [
    "pe_create", "pe_destroy", "pe_last_error", "pe_num_conv_layers", "pe_conv_layer_info", "pe_set_conv_weights",
    "pe_load_weights_file", "pe_commit_weights", "pe_share_weights", "pe_calibrate", "pe_range_status", "pe_nms_get_max_peaks", "pe_nms_get_num_parts", "pe_nms_get_threshold",
    "pe_nms_set_threshold", "pe_resize_set_start_scale", "pe_resize_set_scale_gap", "pe_resize_get_start_scale",
    "pe_resize_get_scale_gap", "pe_set_connect_params", "pe_forward_frames", "pe_forward_frames_device",
    "pe_forward_net_input", "pe_forward_maps", "pe_fetch", "pe_fetch_maps", "pe_fetch_blob", "pe_sync", "pe_write_json",
    "pe_model_num_parts", "pe_model_num_limbs", "pe_model_limb_sequence", "pe_model_map_idx", "pe_model_part_name",
    "pe_event_record", "pe_event_elapsed_ms", "pe_profile_layers", "pe_launch_count", "pe_conv_flops_per_scale",
    "pe_packed_weights_bytes", "pe_packed_weights_device_ptr", "pe_load_caffemodel", "pe_caffemodel_open",
    "pe_caffemodel_close", "pe_caffemodel_num_layers", "pe_caffemodel_layer", "pe_caffemodel_blob",
    "pe_caffemodel_last_error", "pe_create_from_prototxt", "pe_plan_describe", "pe_render_device", "pe_host_alloc", "pe_host_free", "pe_forward_camera_frames", "pe_broadcast_weights", "pe_render", "pe_encode_jpeg", "pe_decode_jpeg", "pe_decode_png",
    "pe_video_open", "pe_video_close", "pe_video_info", "pe_video_read", "pe_video_last_error",
    "pe_camera_open", "pe_camera_close", "pe_camera_info", "pe_camera_grab", "pe_camera_last_error", "pe_yuyv_to_bgr",
    "pe_compare_results", "pe_jpeg_read_coefs", "pe_jpeg_coefs_to_bgr", "pe_forward_jpeg_coefs", "pe_video_read_coefs",
    "pe_jpeg_read_scan", "pe_jpeg_scan_to_coefs_host", "pe_forward_jpeg_scans", "pe_jpeg_decode_scans", "pe_video_read_scan",
    "pe_forward_pixels", "pe_stream_wait", "pe_pixels_to_bgr",
]


def lib():
    """Load libposeengine.so.  Fails loudly: the engine has no fallback implementation."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise PoseEngineError("%s is missing - build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                              "(or `make -C caffe_rtpose_b200`); there is no CPU fallback" % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    L.pe_create.argtypes = [C.POINTER(_Config), C.POINTER(C.c_void_p)]
    L.pe_create_from_prototxt.argtypes = [C.POINTER(_Config), C.c_char_p, C.POINTER(C.c_void_p)]
    L.pe_plan_describe.argtypes = [C.c_int, C.c_char_p, C.c_char_p, C.c_int]
    L.pe_destroy.argtypes = [C.c_void_p]
    L.pe_last_error.restype = C.c_char_p
    L.pe_last_error.argtypes = [C.c_void_p]
    L.pe_num_conv_layers.argtypes = [C.c_void_p]
    L.pe_conv_layer_info.argtypes = [C.c_void_p, C.c_int, C.c_char_p] + [C.POINTER(C.c_int)] * 3
    L.pe_set_conv_weights.argtypes = [C.c_void_p, C.c_char_p, _f32p, C.c_size_t, _f32p, C.c_size_t]
    L.pe_load_weights_file.argtypes = [C.c_void_p, C.c_char_p]
    L.pe_commit_weights.argtypes = [C.c_void_p]
    L.pe_share_weights.argtypes = [C.c_void_p, C.c_void_p]
    L.pe_calibrate.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.c_int]
    L.pe_range_status.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.c_char_p]
    L.pe_load_caffemodel.argtypes = [C.c_void_p, C.c_char_p]
    L.pe_caffemodel_open.argtypes = [C.c_char_p, C.POINTER(C.c_void_p)]
    L.pe_caffemodel_close.argtypes = [C.c_void_p]
    L.pe_caffemodel_num_layers.argtypes = [C.c_void_p]
    L.pe_caffemodel_layer.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_char_p, C.POINTER(C.c_int)]
    L.pe_caffemodel_blob.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.POINTER(C.c_float)), C.POINTER(C.c_size_t),
                                     C.POINTER(C.c_int), C.POINTER(C.c_longlong)]
    L.pe_caffemodel_last_error.restype = C.c_char_p
    for f in ("pe_nms_get_max_peaks", "pe_nms_get_num_parts"):
        getattr(L, f).argtypes = [C.c_void_p]
    for f in ("pe_nms_get_threshold", "pe_resize_get_start_scale", "pe_resize_get_scale_gap"):
        getattr(L, f).argtypes = [C.c_void_p]
        getattr(L, f).restype = C.c_float
    for f in ("pe_nms_set_threshold", "pe_resize_set_start_scale", "pe_resize_set_scale_gap"):
        getattr(L, f).argtypes = [C.c_void_p, C.c_float]
    L.pe_set_connect_params.argtypes = [C.c_void_p, C.c_int, C.c_float, C.c_float, C.c_int]
    L.pe_forward_frames.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.c_int]
    L.pe_forward_frames_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    L.pe_forward_camera_frames.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_int, C.POINTER(C.c_double)]
    L.pe_forward_net_input.argtypes = [C.c_void_p, _f32p, C.c_int]
    L.pe_forward_maps.argtypes = [C.c_void_p, _f32p, C.c_int]
    L.pe_fetch.argtypes = [C.c_void_p, C.c_int, _f32p, C.POINTER(C.c_int), C.c_void_p]
    L.pe_fetch_maps.argtypes = [C.c_void_p, _f32p, C.c_int]
    L.pe_fetch_blob.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_size_t] + [C.POINTER(C.c_int)] * 3
    L.pe_sync.argtypes = [C.c_void_p]
    L.pe_host_alloc.argtypes = [C.c_size_t]
    L.pe_host_alloc.restype = C.c_void_p
    L.pe_host_free.argtypes = [C.c_void_p]
    L.pe_write_json.argtypes = [_f32p, C.c_int, C.c_int, C.c_double, C.c_char_p, C.c_int]
    L.pe_compare_results.argtypes = [C.c_void_p, C.c_int, _f32p, C.c_void_p, C.c_int, _f32p, C.c_int, C.c_int, C.c_float,
                                     C.POINTER(_ResultDiff)]
    for f in ("pe_model_num_parts", "pe_model_num_limbs"):
        getattr(L, f).argtypes = [C.c_int]
    for f in ("pe_model_limb_sequence", "pe_model_map_idx"):
        getattr(L, f).argtypes = [C.c_int]
        getattr(L, f).restype = C.POINTER(C.c_int)
    L.pe_model_part_name.argtypes = [C.c_int, C.c_int]
    L.pe_model_part_name.restype = C.c_char_p
    L.pe_event_record.argtypes = [C.c_void_p, C.c_int]
    L.pe_event_elapsed_ms.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_float)]
    L.pe_profile_layers.argtypes = [C.c_void_p, C.c_int, _f32p, C.c_char_p, C.c_void_p, C.c_int]
    L.pe_launch_count.argtypes = [C.c_void_p]
    L.pe_launch_count.restype = C.c_longlong
    L.pe_conv_flops_per_scale.argtypes = [C.c_void_p]
    L.pe_conv_flops_per_scale.restype = C.c_double
    L.pe_packed_weights_bytes.argtypes = [C.c_void_p]
    L.pe_packed_weights_bytes.restype = C.c_size_t
    L.pe_packed_weights_device_ptr.argtypes = [C.c_void_p]
    L.pe_packed_weights_device_ptr.restype = C.c_void_p
    L.pe_broadcast_weights.argtypes = [C.POINTER(C.c_void_p), C.c_int]
    L.pe_render.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    L.pe_render_device.argtypes = [C.c_int, C.c_void_p] + [C.c_int] * 4 + [C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.c_int, C.c_int, C.c_int]
    L.pe_encode_jpeg.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_longlong]
    L.pe_encode_jpeg.restype = C.c_longlong
    L.pe_decode_jpeg.argtypes = [C.c_char_p, C.c_longlong, C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_void_p, C.c_longlong]
    L.pe_decode_png.argtypes = L.pe_decode_jpeg.argtypes
    L.pe_jpeg_read_coefs.argtypes = [C.c_char_p, C.c_longlong, C.c_void_p, C.c_longlong]
    L.pe_jpeg_read_coefs.restype = C.c_longlong
    L.pe_jpeg_coefs_to_bgr.argtypes = [C.c_void_p, C.c_void_p, C.c_longlong]
    L.pe_forward_jpeg_coefs.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.c_int, C.POINTER(C.c_double)]
    L.pe_jpeg_read_scan.argtypes = L.pe_jpeg_read_coefs.argtypes
    L.pe_jpeg_read_scan.restype = C.c_longlong
    L.pe_jpeg_scan_to_coefs_host.argtypes = [C.c_void_p, C.c_void_p, C.c_longlong, C.c_int]
    L.pe_jpeg_scan_to_coefs_host.restype = C.c_longlong
    L.pe_forward_jpeg_scans.argtypes = L.pe_forward_jpeg_coefs.argtypes
    L.pe_jpeg_decode_scans.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.c_int, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_int)]
    L.pe_video_read_scan.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_longlong]
    L.pe_forward_pixels.argtypes = [C.c_void_p, C.POINTER(_PixelFormat), C.POINTER(C.c_void_p), C.c_int, C.POINTER(C.c_double)]
    L.pe_stream_wait.argtypes = [C.c_void_p, C.c_void_p]
    L.pe_pixels_to_bgr.argtypes = [C.POINTER(_PixelFormat), C.c_void_p, C.c_void_p, C.c_longlong]
    L.pe_video_read_scan.restype = C.c_longlong
    if hasattr(L, "pe_video_open") or "PE_LIB" not in os.environ:   # an older A/B build (PE_LIB) may predate the video reader
        L.pe_video_open.argtypes = [C.c_char_p, C.POINTER(C.c_void_p)]
        L.pe_video_close.argtypes = [C.c_void_p]
        L.pe_video_close.restype = None
        L.pe_video_info.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_double), C.POINTER(C.c_int), C.c_char_p]
        L.pe_video_read.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_longlong]
        L.pe_video_last_error.restype = C.c_char_p
    if hasattr(L, "pe_camera_open") or "PE_LIB" not in os.environ:
        L.pe_camera_open.argtypes = [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p)]
        L.pe_camera_close.argtypes = [C.c_void_p]
        L.pe_camera_close.restype = None
        L.pe_camera_last_error.restype = C.c_char_p
        L.pe_yuyv_to_bgr.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_longlong, C.c_void_p]
    _lib = L
    return L


class ModelDescriptor:
    """include/rtpose/modelDescriptor.h API: get_number_parts, number_limb_sequence, get_limb_sequence,
    get_map_idx, get_part_name."""

    def __init__(self, model):
        L = lib()
        self.model = model
        self._np = L.pe_model_num_parts(model)
        self._nl = L.pe_model_num_limbs(model)
        ls, mi = L.pe_model_limb_sequence(model), L.pe_model_map_idx(model)
        self._limb = [ls[i] for i in range(2 * self._nl)]
        self._map = [mi[i] for i in range(2 * self._nl)]

    def get_number_parts(self):
        return self._np

    def number_limb_sequence(self):
        return self._nl

    def get_limb_sequence(self):
        return self._limb

    def get_map_idx(self):
        return self._map

    def get_part_name(self, idx):
        if not 0 <= idx < self._np + 1 + 2 * self._nl:
            raise IndexError(idx)  # std::map::at throws in the reference
        return lib().pe_model_part_name(self.model, idx).decode()


class ModelDescriptorFactory:
    """include/rtpose/modelDescriptorFactory.h: Type::{MPI_15, COCO_18}, createModelDescriptor."""

    class Type:
        MPI_15, COCO_18 = MPI_15, COCO_18

    @staticmethod
    def createModelDescriptor(type_):
        if type_ not in (MPI_15, COCO_18):
            raise RuntimeError("Undefined ModelDescriptor selected.")  # modelDescriptorFactory.cpp:57-60
        return ModelDescriptor(type_)


class NmsLayer:
    """caffe::NmsLayer<float> accessors (nms_layer.hpp:21-27)."""

    def __init__(self, eng):
        self._e = eng

    def type(self):
        return "Nms"

    def GetMaxPeaks(self):
        return lib().pe_nms_get_max_peaks(self._e._h)

    def GetNumParts(self):
        return lib().pe_nms_get_num_parts(self._e._h)

    def GetThreshold(self):
        return lib().pe_nms_get_threshold(self._e._h)

    def SetThreshold(self, t):
        self._e._ck(lib().pe_nms_set_threshold(self._e._h, float(t)))


class ImResizeLayer:
    """caffe::ImResizeLayer<float> accessors (imresize_layer.hpp:20-29)."""

    def __init__(self, eng):
        self._e = eng

    def type(self):
        return "ImResize"

    def SetStartScale(self, s):
        self._e._ck(lib().pe_resize_set_start_scale(self._e._h, float(s)))

    def SetScaleGap(self, g):
        self._e._ck(lib().pe_resize_set_scale_gap(self._e._h, float(g)))

    def GetStartScale(self):
        return lib().pe_resize_get_start_scale(self._e._h)

    def GetScaleGap(self):
        return lib().pe_resize_get_scale_gap(self._e._h)


class PoseEngine:
    """One GPU worker (the reference's NetCopy + warmup(), rtpose.cpp:133-142, 173-237)."""

    def __init__(self, model=COCO_18, net_w=656, net_h=368, disp_w=1280, disp_h=720, num_scales=1, start_scale=1.0,
                 scale_gap=0.3, device=0, max_batch=1, precision=PREC_BF16X2, prototxt=None):
        """prototxt: path of a deploy prototxt (`new caffe::Net(proto, TEST)`, rtpose.cpp:183); model may then be None
        and follows the Nms layer's num_parts (rtpose.cpp:212-229).  Without it the built-in graph of `model` is used."""
        L = lib()
        cfg = _Config(device, -1 if model is None else model, net_w, net_h, disp_w, disp_h, num_scales, start_scale, scale_gap,
                      max_batch, precision)
        h = C.c_void_p()
        if prototxt is not None:
            rc = L.pe_create_from_prototxt(C.byref(cfg), os.fsencode(prototxt), C.byref(h))
        else:
            rc = L.pe_create(C.byref(cfg), C.byref(h))
        if rc != 0:
            raise PoseEngineError("pe_create failed (%d): %s" % (rc, L.pe_last_error(None).decode()))
        self._h = h
        self.cfg = cfg
        if model is None:
            model = {15: MPI_15, 18: COCO_18}[L.pe_nms_get_num_parts(h)]
        self.model = model
        self.num_parts = L.pe_nms_get_num_parts(h)
        self.max_peaks = L.pe_nms_get_max_peaks(h)
        self.num_maps = self.num_parts + 1 + 2 * L.pe_model_num_limbs(model)
        self.nms_layer = NmsLayer(self)
        self.resize_layer = ImResizeLayer(self)
        self.model_descriptor = ModelDescriptorFactory.createModelDescriptor(model)
        self._keep = None
        self._held = []   # frames forward_pixels reads asynchronously: released by the next fetch, sync or close

    def close(self):
        if getattr(self, "_h", None):
            lib().pe_destroy(self._h)
            self._h = None
        self._held = []

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        if rc != 0:
            raise PoseEngineError("poseengine error %d: %s" % (rc, lib().pe_last_error(self._h).decode()))

    # ---- weights (Net::CopyTrainedLayersFrom) -------------------------------------------------
    def conv_layers(self):
        L = lib()
        out = []
        name = C.create_string_buffer(64)
        a, b, k = C.c_int(), C.c_int(), C.c_int()
        for i in range(L.pe_num_conv_layers(self._h)):
            self._ck(L.pe_conv_layer_info(self._h, i, name, C.byref(a), C.byref(b), C.byref(k)))
            out.append((name.value.decode(), a.value, b.value, k.value))
        return out

    def set_weights(self, weights, commit=True):
        for name, (w, b) in weights.items():
            w = np.ascontiguousarray(w, np.float32)
            b = np.ascontiguousarray(b, np.float32)
            self._ck(lib().pe_set_conv_weights(self._h, name.encode(), w, w.size, b, b.size))
        if commit:
            self.commit_weights()

    def load_weights_file(self, path, commit=True):
        self._ck(lib().pe_load_weights_file(self._h, path.encode()))
        if commit:
            self.commit_weights()

    def commit_weights(self):
        self._ck(lib().pe_commit_weights(self._h))

    def load_caffemodel(self, path, commit=True):
        """Net::CopyTrainedLayersFrom(trained_filename) for a binary .caffemodel (rtpose.cpp:184)."""
        rc = lib().pe_load_caffemodel(self._h, path.encode())
        if rc != 0:
            raise PoseEngineError("pe_load_caffemodel failed (%d): %s / %s" % (
                rc, lib().pe_caffemodel_last_error().decode(), lib().pe_last_error(self._h).decode()))
        if commit:
            self.commit_weights()

    def set_connect_params(self, min_subset_cnt, min_subset_score, inter_threshold, inter_min_above):
        self._ck(lib().pe_set_connect_params(self._h, min_subset_cnt, min_subset_score, inter_threshold, inter_min_above))

    # ---- forward ------------------------------------------------------------------------------
    def forward_frames(self, frames):
        """frames: list of uint8 BGR HWC display images (host)."""
        frames = [np.ascontiguousarray(f, np.uint8) for f in frames]
        for f in frames:
            assert f.shape == (self.cfg.disp_h, self.cfg.disp_w, 3), f.shape
        ptrs = (C.c_void_p * len(frames))(*[f.ctypes.data for f in frames])
        self._keep = frames
        self._ck(lib().pe_forward_frames(self._h, ptrs, len(frames)))

    def forward_camera_frames(self, frames):
        """frames: list of uint8 BGR HWC images of one common (arbitrary) size; returns frame.scale (rtpose.cpp:474-487)."""
        frames = [np.ascontiguousarray(f, np.uint8) for f in frames]
        h, w, _ = frames[0].shape
        assert all(f.shape == (h, w, 3) for f in frames)
        ptrs = (C.c_void_p * len(frames))(*[f.ctypes.data for f in frames])
        self._keep = frames
        s = C.c_double()
        self._ck(lib().pe_forward_camera_frames(self._h, ptrs, len(frames), w, h, C.byref(s)))
        return s.value

    def forward_jpeg(self, jpegs, entropy="host"):
        """jpegs: list of JPEG files (bytes) of one common size.  entropy="host": only the entropy stage runs on the host
        (read_jpeg_coefs); the GPU reconstructs the pixels, byte-identical to decode_jpeg, and then runs as forward_frames (display
        size) or forward_camera_frames (any other size).  entropy="gpu": the host only parses the file (read_jpeg_scan) and the GPU
        also decodes the Huffman data; for one interleaved sequential scan per file.  Arrays are taken as coefficient / scan images.
        Returns frame.scale."""
        if entropy not in ("host", "gpu"):
            raise ValueError("entropy must be 'host' or 'gpu'")
        read = read_jpeg_coefs if entropy == "host" else read_jpeg_scan
        bufs = [j if isinstance(j, np.ndarray) else read(j) for j in jpegs]
        ptrs = (C.c_void_p * len(bufs))(*[b.ctypes.data for b in bufs])
        self._keep = bufs
        s = C.c_double()
        fn = lib().pe_forward_jpeg_coefs if entropy == "host" else lib().pe_forward_jpeg_scans
        self._ck(fn(self._h, ptrs, len(bufs), C.byref(s)))
        return s.value

    def forward_pixels(self, frames, fmt, chroma_offset=None):
        """frames: numpy arrays or torch tensors (host or CUDA) of one format and size, in cv2's shapes: (h*3/2, w) for PIX_NV12 /
        PIX_I420, (h, w, 2) for PIX_YUYV, (h, w, 3) for PIX_RGB / PIX_BGR.  The row stride is the pitch, so a column slice of a
        wider allocation is read in place (an I420 array of that shape is copied unless tight: its chroma rows are not pitch/2
        apart).  chroma_offset (NV12 / I420): the frames are the (h, w) luma planes, the row stride is the pitch, and the chroma plane
        starts chroma_offset bytes after each frame's start, e.g. pitch * 1088 in a 1080p NVDEC surface; the caller vouches that
        the allocation reaches that far.  Converted to BGR on the GPU
        as cv2.cvtColor does, then as forward_camera_frames.  CUDA frames are read on the engine's stream after the work queued so
        far on torch's current stream.  Returns frame.scale."""
        views = [_pixel_view(f, fmt, chroma_offset) for f in frames]
        pf = views[0][1]
        if any((v[1].width, v[1].height, v[1].pitch) != (pf.width, pf.height, pf.pitch) for v in views):
            raise ValueError("forward_pixels: the frames of one call share their size and row stride")
        for dev in {v[3] for v in views if v[3] is not None and v[3].index == self.cfg.device}:
            import torch
            self._ck(lib().pe_stream_wait(self._h, C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
        self._held.extend(v[2] for v in views)
        ptrs = (C.c_void_p * len(views))(*[v[0] for v in views])
        s = C.c_double()
        self._ck(lib().pe_forward_pixels(self._h, C.byref(pf), ptrs, len(views), C.byref(s)))
        return s.value

    def decode_jpeg_scans(self, scans, subseq_bits=0):
        """Test hook: scan images (read_jpeg_scan) -> coefficient images decoded on the GPU (subseq_bits 0 = the default
        subsequence length).  Returns (list of coefficient images as uint8 arrays, list of statuses: 0, or 1 + the MCU of the
        first data error)."""
        scans = [np.ascontiguousarray(b, np.uint8) for b in scans]
        outs = [np.zeros(jpeg_coef_header(b[:512])["total_bytes"], np.uint8) for b in scans]
        ptrs = (C.c_void_p * len(scans))(*[b.ctypes.data for b in scans])
        optrs = (C.c_void_p * len(outs))(*[o.ctypes.data for o in outs])
        st = (C.c_int * len(scans))()
        self._ck(lib().pe_jpeg_decode_scans(self._h, ptrs, len(scans), subseq_bits, optrs, st))
        return outs, list(st)

    def render(self, idx=0, part_to_show=0, googly_eyes=False, display_bgr=None, want_canvas=False):
        """render() of rtpose.cpp:271-300 on frame idx of the last forward; returns the uint8 BGR image
        (disp_h, disp_w, 3) and, if want_canvas, also the float planar canvas (3, disp_h, disp_w)."""
        H, W = self.cfg.disp_h, self.cfg.disp_w
        img = np.zeros((H, W, 3), np.uint8)
        canvas = np.zeros((3, H, W), np.float32) if want_canvas else None
        src = None
        if display_bgr is not None:
            src = np.ascontiguousarray(display_bgr, np.uint8)
            assert src.shape == (H, W, 3), src.shape
        self._ck(lib().pe_render(self._h, idx, part_to_show, 1 if googly_eyes else 0, src.ctypes.data if src is not None else None,
                                 canvas.ctypes.data if want_canvas else None, img.ctypes.data))
        return (img, canvas) if want_canvas else img

    def forward_frames_device(self, dev_ptr, n):
        self._ck(lib().pe_forward_frames_device(self._h, C.c_void_p(dev_ptr), n))

    def forward_net_input(self, x):
        x = np.ascontiguousarray(x, np.float32)
        n = x.shape[0] // self.cfg.num_scales
        assert x.shape == (n * self.cfg.num_scales, 3, self.cfg.net_h, self.cfg.net_w), x.shape
        self._ck(lib().pe_forward_net_input(self._h, x, n))

    def forward_maps(self, maps8):
        maps8 = np.ascontiguousarray(maps8, np.float32)
        n = maps8.shape[0] // self.cfg.num_scales
        assert maps8.shape == (n * self.cfg.num_scales, self.num_maps, self.cfg.net_h // 8, self.cfg.net_w // 8), maps8.shape
        self._ck(lib().pe_forward_maps(self._h, maps8, n))

    def calibrate(self, frames):
        """pe_calibrate: per-layer power-of-two activation scales of the parity mode from one forward on `frames`."""
        frames = [np.ascontiguousarray(f, np.uint8) for f in frames]
        arr = (C.c_void_p * len(frames))(*[f.ctypes.data for f in frames])
        self._ck(lib().pe_calibrate(self._h, arr, len(frames)))

    def range_status(self):
        """(rc, worst |stored value| / 65504, layer name); rc != 0 (PE_ERR_RANGE = 5) when a layer left the fp16 range."""
        worst = C.c_float()
        name = C.create_string_buffer(64)
        rc = lib().pe_range_status(self._h, C.byref(worst), name)
        return rc, worst.value, name.value.decode()

    def sync(self):
        self._ck(lib().pe_sync(self._h))
        self._held = []

    def fetch(self, idx=0):
        joints = np.zeros((MAX_PEOPLE, self.num_parts, 3), np.float32)
        peaks = np.zeros((self.num_parts, self.max_peaks + 1, 3), np.float32)
        n = C.c_int()
        self._ck(lib().pe_fetch(self._h, idx, joints, C.byref(n), peaks.ctypes.data_as(C.c_void_p)))
        self._held = []
        return n.value, joints[:n.value].copy(), peaks

    def fetch_maps(self, n=1):
        out = np.zeros((n * self.cfg.num_scales, self.num_maps, self.cfg.net_h // 8, self.cfg.net_w // 8), np.float32)
        self._ck(lib().pe_fetch_maps(self._h, out, n))
        return out

    def fetch_blob(self, name):
        c, h, w = C.c_int(), C.c_int(), C.c_int()
        self._ck(lib().pe_fetch_blob(self._h, name.encode(), None, 0, C.byref(c), C.byref(h), C.byref(w)))
        # number of images of the last forward is not exported; over-allocate for max_batch
        n = self.cfg.max_batch * self.cfg.num_scales
        out = np.zeros((n, c.value, h.value, w.value), np.float32)
        self._ck(lib().pe_fetch_blob(self._h, name.encode(), out.ctypes.data_as(C.c_void_p), out.size, C.byref(c),
                                     C.byref(h), C.byref(w)))
        return out

    def json(self, joints, frame_scale=1.0):
        return write_json(joints, self.num_parts, frame_scale)

    # ---- measurement --------------------------------------------------------------------------
    def event_record(self, slot):
        self._ck(lib().pe_event_record(self._h, slot))

    def event_elapsed_ms(self, a, b):
        ms = C.c_float()
        self._ck(lib().pe_event_elapsed_ms(self._h, a, b, C.byref(ms)))
        return ms.value

    def profile_layers(self, n=1):
        cap = 256
        ms = np.zeros(cap, np.float32)
        names = C.create_string_buffer(64 * cap)
        flops = np.zeros(cap, np.float64)
        k = lib().pe_profile_layers(self._h, n, ms, names, flops.ctypes.data_as(C.c_void_p), cap)
        if k < 0:
            self._ck(-k)
        raw = names.raw
        return [(raw[64 * i:64 * (i + 1)].split(b"\0")[0].decode(), float(ms[i]), float(flops[i])) for i in range(k)]

    def launch_count(self):
        return lib().pe_launch_count(self._h)

    def conv_flops_per_scale(self):
        return lib().pe_conv_flops_per_scale(self._h)

    def packed_weights(self):
        return lib().pe_packed_weights_device_ptr(self._h), lib().pe_packed_weights_bytes(self._h)


def plan_describe(model=None, prototxt=None):
    """Text description of the execution plan (host only, no GPU): built-in graph of `model`, or of a prototxt."""
    L = lib()
    path = os.fsencode(prototxt) if prototxt is not None else None
    n = L.pe_plan_describe(-1 if model is None else model, path, None, 0)
    if n < 0:
        raise PoseEngineError("pe_plan_describe failed (%d): %s" % (-n, L.pe_last_error(None).decode()))
    buf = C.create_string_buffer(n + 1)
    L.pe_plan_describe(-1 if model is None else model, path, buf, n + 1)
    return buf.value.decode()


def write_json(joints, num_parts, frame_scale=1.0):
    """displayFrame's JSON writer (rtpose.cpp:1383-1416)."""
    joints = np.ascontiguousarray(joints, np.float32).reshape(-1, num_parts, 3)
    cap = 64 + joints.shape[0] * (num_parts * 48 + 32)
    buf = C.create_string_buffer(cap)
    src = joints if joints.size else np.zeros(1, np.float32)
    n = lib().pe_write_json(src, joints.shape[0], num_parts, frame_scale, buf, cap)
    assert n < cap
    return buf.value.decode()


def write_weights_file(path, weights, table):
    """Flat RTPW v1 file (see pe_load_weights_file)."""
    import struct
    with open(path, "wb") as f:
        f.write(b"RTPW" + struct.pack("<II", 1, len(table)))
        for name, co, ci, k in table:
            w, b = weights[name]
            f.write(name.encode().ljust(64, b"\0") + struct.pack("<III", co, ci, k))
            f.write(np.ascontiguousarray(w, np.float32).tobytes())
            f.write(np.ascontiguousarray(b, np.float32).tobytes())


def read_caffemodel(path):
    """Host-only: list of (name, type, [(ndarray, shape), ...]) from a binary .caffemodel (no GPU needed)."""
    L = lib()
    h = C.c_void_p()
    rc = L.pe_caffemodel_open(path.encode(), C.byref(h))
    if rc != 0:
        raise PoseEngineError("pe_caffemodel_open failed (%d): %s" % (rc, L.pe_caffemodel_last_error().decode()))
    out = []
    try:
        name, typ = C.create_string_buffer(64), C.create_string_buffer(32)
        nb = C.c_int()
        for i in range(L.pe_caffemodel_num_layers(h)):
            L.pe_caffemodel_layer(h, i, name, typ, C.byref(nb))
            blobs = []
            for j in range(nb.value):
                p = C.POINTER(C.c_float)()
                cnt, nd = C.c_size_t(), C.c_int()
                dims = (C.c_longlong * 8)()
                L.pe_caffemodel_blob(h, i, j, C.byref(p), C.byref(cnt), C.byref(nd), dims)
                arr = np.ctypeslib.as_array(p, shape=(cnt.value,)).copy() if cnt.value else np.zeros(0, np.float32)
                blobs.append((arr, tuple(dims[k] for k in range(nd.value))))
            out.append((name.value.decode(), typ.value.decode(), blobs))
    finally:
        L.pe_caffemodel_close(h)
    return out


def _pb_varint(v):
    out = bytearray()
    while True:
        b = v & 0x7F
        v >>= 7
        if v:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def _pb_len(field, payload):
    return _pb_varint((field << 3) | 2) + _pb_varint(len(payload)) + payload


def write_caffemodel(path, weights, table, legacy_v1=False, legacy_dims=False):
    """Serialise weights as a binary caffe NetParameter (`layer`=100, or V1 `layers`=2), BlobProto.data packed,
    shape as BlobShape or legacy num/channels/height/width - the wire format of pose_iter_*.caffemodel."""
    net = _pb_len(1, b"synthetic_rtpose")
    for name, co, ci, k in table:
        w, b = weights[name]
        blobs = b""
        for arr, shape in ((w, (co, ci, k, k)), (b, (co,))):
            data = _pb_len(5, np.ascontiguousarray(arr, "<f4").tobytes())
            if legacy_dims:
                s4 = (1,) * (4 - len(shape)) + tuple(shape)
                dims = b"".join(_pb_varint((f << 3) | 0) + _pb_varint(v) for f, v in zip((1, 2, 3, 4), s4))
            else:
                dims = _pb_len(7, _pb_len(1, b"".join(_pb_varint(v) for v in shape)))
            blobs += _pb_len(6 if legacy_v1 else 7, dims + data)
        if legacy_v1:
            layer = _pb_len(4, name.encode()) + _pb_varint((5 << 3) | 0) + _pb_varint(4) + blobs   # type CONVOLUTION = 4
            net += _pb_len(2, layer)
        else:
            layer = _pb_len(1, name.encode()) + _pb_len(2, b"Convolution") + blobs
            net += _pb_len(100, layer)
            net += _pb_len(100, _pb_len(1, ("relu_" + name).encode()) + _pb_len(2, b"ReLU"))   # blob-less layer, ignored
    with open(path, "wb") as f:
        f.write(net)


def compare_results(a, b, tol_px):
    """pe_compare_results of two results of one frame, each (num_people, joints, peaks) as PoseEngine.fetch returns it:
    equal peak counts per part with every peak within tol_px, equal person counts, person i of a with the same present parts
    as person i of b and every joint within tol_px.  Joints are in display pixels and peaks in net pixels, both compared
    against tol_px.  Returns a dict with identical, parts_count_differ, peaks_moved, persons_matched, max_joint_dist."""
    (na, ja, pa), (nb, jb, pb) = a, b
    pa = np.ascontiguousarray(pa, np.float32)
    pb = np.ascontiguousarray(pb, np.float32)
    if pa.shape != pb.shape or pa.ndim != 3 or pa.shape[2] != 3:
        raise ValueError("peaks must both be (num_parts, max_peaks + 1, 3), got %s and %s" % (pa.shape, pb.shape))
    num_parts, max_peaks = pa.shape[0], pa.shape[1] - 1
    ja = np.ascontiguousarray(np.asarray(ja, np.float32).reshape(-1, num_parts, 3)[:na])
    jb = np.ascontiguousarray(np.asarray(jb, np.float32).reshape(-1, num_parts, 3)[:nb])
    if ja.shape[0] != na or jb.shape[0] != nb:
        raise ValueError("fewer joint rows than people")
    d = _ResultDiff()
    rc = lib().pe_compare_results(ja.ctypes.data_as(C.c_void_p), int(na), pa, jb.ctypes.data_as(C.c_void_p), int(nb), pb,
                                  num_parts, max_peaks, float(tol_px), C.byref(d))
    if rc != 0:
        raise PoseEngineError("pe_compare_results failed (%d)" % rc)
    return {"identical": bool(d.identical), "parts_count_differ": d.parts_count_differ, "peaks_moved": d.peaks_moved,
            "persons_matched": d.persons_matched, "max_joint_dist": float(d.max_joint_dist)}


def share_weights(src, dst):
    """Net::ShareTrainedLayersWith: `dst` (same GPU, same net) uses `src`'s packed weights without a copy."""
    rc = lib().pe_share_weights(src._h, dst._h)
    if rc != 0:
        raise PoseEngineError("pe_share_weights failed (%d): %s" % (rc, lib().pe_last_error(src._h).decode()))


def broadcast_weights(engines):
    """engines[0]'s committed weights -> the other handles (one per GPU, same process) with one ncclBroadcast."""
    arr = (C.c_void_p * len(engines))(*[e._h for e in engines])
    rc = lib().pe_broadcast_weights(arr, len(engines))
    if rc != 0:
        raise PoseEngineError("pe_broadcast_weights failed (%d): %s" % (rc, lib().pe_last_error(engines[0]._h).decode()))


def encode_jpeg(bgr, quality=98):
    """Baseline JFIF bytes of a uint8 BGR HWC image (what --write_frames stores; cv::imwrite quality 98 in the reference)."""
    bgr = np.ascontiguousarray(bgr, np.uint8)
    h, w, _ = bgr.shape
    n = lib().pe_encode_jpeg(bgr.ctypes.data, w, h, quality, None, 0)
    if n < 0:
        raise PoseEngineError("pe_encode_jpeg: bad arguments")
    buf = np.zeros(n, np.uint8)
    lib().pe_encode_jpeg(bgr.ctypes.data, w, h, quality, buf.ctypes.data, n)
    return buf.tobytes()


def decode_jpeg(data):
    """uint8 BGR HWC pixels of a baseline JPEG, bit-identical to cv::imread / libjpeg defaults (baseline and progressive; what --image_dir feeds)."""
    w, h = C.c_int(), C.c_int()
    rc = lib().pe_decode_jpeg(data, len(data), C.byref(w), C.byref(h), None, 0)
    if rc != 0:
        raise PoseEngineError("pe_decode_jpeg: %s" % ("not a JPEG / truncated" if rc == -1 else "unsupported JPEG variant (arithmetic / lossless / 12-bit / CMYK / unusual sampling)"))
    out = np.zeros((h.value, w.value, 3), np.uint8)
    rc = lib().pe_decode_jpeg(data, len(data), C.byref(w), C.byref(h), out.ctypes.data, out.size)
    if rc != 0:
        raise PoseEngineError("pe_decode_jpeg failed (%d)" % rc)
    return out


def _jpeg_error(fn, rc):
    return PoseEngineError("%s: %s" % (fn, "not a JPEG / truncated" if rc == -1 else "unsupported JPEG variant (arithmetic / lossless / 12-bit / CMYK / unusual sampling)"))


def read_jpeg_coefs(data):
    """Entropy stage of decode_jpeg: the coefficient image (pe_jpeg_coef_header + int16 coefficients, poseengine.h) as a uint8
    array, the input of PoseEngine.forward_jpeg."""
    n = lib().pe_jpeg_read_coefs(data, len(data), None, 0)
    if n < 0:
        raise _jpeg_error("pe_jpeg_read_coefs", n)
    buf = np.zeros(n, np.uint8)
    rc = lib().pe_jpeg_read_coefs(data, len(data), buf.ctypes.data, n)
    if rc != n:
        raise _jpeg_error("pe_jpeg_read_coefs", rc)
    return buf


def read_jpeg_scan(data):
    """Scan image of a JPEG (pe_jpeg_scan_header + segment table + entropy-coded bytes, poseengine.h) as a uint8 array: the input of
    PoseEngine.forward_jpeg(entropy="gpu").  Raises PoseEngineError for files that need the host entropy stage (progressive,
    multi-scan) and for the codes of read_jpeg_coefs."""
    n = lib().pe_jpeg_read_scan(data, len(data), None, 0)
    if n == -3:
        raise PoseEngineError("pe_jpeg_read_scan: not one interleaved sequential scan: needs the host entropy stage")
    if n < 0:
        raise _jpeg_error("pe_jpeg_read_scan", n)
    buf = np.zeros(n, np.uint8)
    rc = lib().pe_jpeg_read_scan(data, len(data), buf.ctypes.data, n)
    if rc != n:
        raise _jpeg_error("pe_jpeg_read_scan", rc)
    return buf


def jpeg_scan_to_coefs_host(scan, subseq_bits=1024):
    """The GPU entropy decoder's algorithm run on the host: scan image -> (coefficient image, ok).  ok is False where
    read_jpeg_coefs rejects the data (a DC category above 15)."""
    scan = np.ascontiguousarray(scan, np.uint8)
    if scan.size < 2784:
        raise PoseEngineError("pe_jpeg_scan_to_coefs_host: truncated scan image")
    n = jpeg_coef_header(scan[:512])["total_bytes"]
    out = np.zeros(max(n, 0), np.uint8)
    rc = lib().pe_jpeg_scan_to_coefs_host(scan.ctypes.data, out.ctypes.data, out.size, subseq_bits)
    if rc == -1:
        raise PoseEngineError("pe_jpeg_scan_to_coefs_host: malformed scan image")
    if rc != n and rc != -4:
        raise PoseEngineError("pe_jpeg_scan_to_coefs_host failed (%d)" % rc)
    return out, rc == n


def jpeg_coef_header(buf):
    """The header fields of a coefficient image: dict with width, height, num_comps, hmax, vmax, total_bytes and comps, a list of
    dicts (h, v, bw, bh, dw, dh, offset, quant) per component."""
    b = np.asarray(buf, np.uint8)
    i32, i64 = b[:32].view(np.int32), b[:32].view(np.int64)
    out = {"magic": int(b[:4].view(np.uint32)[0]), "width": int(i32[1]), "height": int(i32[2]), "num_comps": int(i32[3]),
           "hmax": int(i32[4]), "vmax": int(i32[5]), "total_bytes": int(i64[3]), "comps": []}
    for k in range(out["num_comps"]):
        c = b[32 + 160 * k:32 + 160 * (k + 1)]
        f = c[:24].view(np.int32)
        out["comps"].append({"h": int(f[0]), "v": int(f[1]), "bw": int(f[2]), "bh": int(f[3]), "dw": int(f[4]), "dh": int(f[5]),
                             "offset": int(c[24:32].view(np.int64)[0]), "quant": c[32:].view(np.uint16).reshape(8, 8).copy()})
    return out


def jpeg_coefs_to_bgr(buf):
    """Host reconstruction of a coefficient image with decode_jpeg's own IDCT / upsampling / colour code (the reference of the
    GPU kernels)."""
    buf = np.ascontiguousarray(buf, np.uint8)
    if buf.size < 512 or jpeg_coef_header(buf)["total_bytes"] > buf.size:
        raise PoseEngineError("pe_jpeg_coefs_to_bgr: truncated coefficient image")
    hd = jpeg_coef_header(buf)
    out =np.zeros((max(hd["height"], 0), max(hd["width"], 0), 3), np.uint8)
    if lib().pe_jpeg_coefs_to_bgr(buf.ctypes.data, out.ctypes.data, out.size) != 0:
        raise PoseEngineError("pe_jpeg_coefs_to_bgr: malformed coefficient image")
    return out


class VideoCapture:
    """cv::VideoCapture as getFrameFromCam uses it for --video (rtpose.cpp:394-411, 433-446, 525-545): open / isOpened / get(FPS,
    FRAME_COUNT, FRAME_WIDTH, FRAME_HEIGHT, POS_FRAMES) / set(POS_FRAMES) / read, over pe_video_* (Motion-JPEG and uncompressed AVI)."""
    CAP_PROP_POS_FRAMES, CAP_PROP_FRAME_WIDTH, CAP_PROP_FRAME_HEIGHT, CAP_PROP_FPS, CAP_PROP_FRAME_COUNT = 1, 3, 4, 5, 7

    def __init__(self, path=None):
        self._h = None
        self.error = ""
        if path is not None:
            self.open(path)

    def open(self, path):
        self.release()
        h = C.c_void_p()
        if lib().pe_video_open(os.fsencode(path), C.byref(h)) != 0:
            self.error = lib().pe_video_last_error().decode()
            return False
        self._h = h
        w, hh, n, fps, cc = C.c_int(), C.c_int(), C.c_int(), C.c_double(), C.create_string_buffer(5)
        lib().pe_video_info(h, C.byref(w), C.byref(hh), C.byref(fps), C.byref(n), cc)
        self.width, self.height, self.frame_count, self.fps, self.fourcc, self.pos = w.value, hh.value, n.value, fps.value, cc.value.decode(), 0
        return True

    def isOpened(self):
        return self._h is not None

    def get(self, prop):
        if self._h is None:
            return 0.0
        return float({self.CAP_PROP_POS_FRAMES: self.pos, self.CAP_PROP_FRAME_WIDTH: self.width, self.CAP_PROP_FRAME_HEIGHT: self.height,
                      self.CAP_PROP_FPS: self.fps, self.CAP_PROP_FRAME_COUNT: self.frame_count}.get(prop, 0))

    def set(self, prop, value):
        if self._h is None or prop != self.CAP_PROP_POS_FRAMES:
            return False
        self.pos = max(0, min(int(value), self.frame_count))
        return True

    def read(self):
        """(True, uint8 BGR HWC frame) and the position advances, or (False, None) at the end / on a broken frame."""
        if self._h is None or self.pos >= self.frame_count:
            return False, None
        out = np.empty((self.height, self.width, 3), np.uint8)
        if lib().pe_video_read(self._h, self.pos, out.ctypes.data, out.size) != 0:
            self.error = lib().pe_video_last_error().decode()
            return False, None
        self.pos += 1
        return True, out

    def release(self):
        if self._h is not None:
            lib().pe_video_close(self._h)
            self._h = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


def _pixel_view(frame, fmt, chroma_offset=None):
    """(data pointer, _PixelFormat, the object that owns the pixels, torch device of a CUDA tensor or None) of a uint8 frame in
    forward_pixels's shapes.  Frames whose pixels or channels are not adjacent in memory are copied first."""
    if fmt not in (PIX_BGR, PIX_RGB, PIX_YUYV, PIX_NV12, PIX_I420):
        raise ValueError("pixel format %r is not one of PIX_BGR .. PIX_I420" % (fmt,))
    planar = fmt in (PIX_NV12, PIX_I420)
    ch = 1 if planar else (2 if fmt == PIX_YUYV else 3)
    is_np = isinstance(frame, np.ndarray)
    if not is_np:
        import torch
        if not torch.is_tensor(frame):
            raise TypeError("frames are numpy arrays or torch tensors")
    if (frame.dtype != np.uint8) if is_np else (frame.dtype != torch.uint8):
        raise TypeError("frames are uint8, not %s" % frame.dtype)
    shape = tuple(frame.shape)
    if shape[2:] != (() if planar else (ch,)) or len(shape) < 2:
        raise ValueError("frame shape %s does not fit format %d" % (shape, fmt))

    def strides(f):
        return tuple(f.strides) if is_np else tuple(f.stride())
    h, w = shape[0], shape[1]
    st = strides(frame)
    # In cv2's (h*3/2, w) I420 array one row holds two chroma rows, so only a tight one has the layout's pitch/2 chroma rows
    tight_i420 = fmt == PIX_I420 and chroma_offset is None
    if (w > 1 and st[1] != ch) or (not planar and st[2] != 1) or (h > 1 and st[0] < w * ch) or (tight_i420 and h > 1 and st[0] != w):
        frame = np.ascontiguousarray(frame) if is_np else frame.contiguous()
        st = strides(frame)
    if planar and chroma_offset is None:
        if h % 3:
            raise ValueError("a %s frame has h*3/2 rows, not %d" % ("NV12" if fmt == PIX_NV12 else "I420", h))
        h = h * 2 // 3
    pitch = st[0] if shape[0] > 1 else w * ch
    ptr = frame.ctypes.data if is_np else frame.data_ptr()
    dev = None if is_np or not frame.is_cuda else frame.device
    return ptr, _PixelFormat(fmt, w, h, pitch, chroma_offset or 0), frame, dev


def pixels_to_bgr(frame, fmt):
    """cv2.cvtColor of a host frame in forward_pixels's shapes to uint8 BGR (h, w, 3): the host reference of the GPU conversion."""
    ptr, pf, frame, dev = _pixel_view(frame, fmt)
    if dev is not None:
        raise ValueError("pixels_to_bgr takes host frames")
    out = np.empty((pf.height, pf.width, 3), np.uint8)
    if lib().pe_pixels_to_bgr(C.byref(pf), ptr, out.ctypes.data, out.size) != 0:
        raise PoseEngineError("pe_pixels_to_bgr: %s" % lib().pe_last_error(None).decode())
    return out


def yuyv_to_bgr(yuyv):
    """cv::cvtColor(COLOR_YUV2BGR_YUYV) of an (h, w, 2) uint8 YUYV image - the conversion of camera frames (pe_camera_grab)."""
    yuyv = np.ascontiguousarray(yuyv, np.uint8)
    h, w, _ = yuyv.shape
    out = np.empty((h, w, 3), np.uint8)
    if lib().pe_yuyv_to_bgr(yuyv.ctypes.data, w, h, 2 * w, out.ctypes.data) != 0:
        raise PoseEngineError("pe_yuyv_to_bgr: bad arguments (odd width?)")
    return out


def decode_png(data):
    """uint8 BGR HWC pixels of a PNG as cv::imread(IMREAD_COLOR) returns them."""
    w, h = C.c_int(), C.c_int()
    if lib().pe_decode_png(data, len(data), C.byref(w), C.byref(h), None, 0) != 0:
        raise PoseEngineError("pe_decode_png: not a PNG / corrupt")
    out = np.zeros((h.value, w.value, 3), np.uint8)
    if lib().pe_decode_png(data, len(data), C.byref(w), C.byref(h), out.ctypes.data, out.size) != 0:
        raise PoseEngineError("pe_decode_png: corrupt image data")
    return out
