"""Python mirror of `SIVO::BayesianSegNet` (include/bayesian_segnet/bayesian_segnet.hpp:108-170) over the
C-ABI: same names, argument meaning and error behaviour, so the parity tests read like the reference's
tests/test_bayesian_segnet.cpp."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Optional

import numpy as np

from . import _lib as L


@dataclass
class BayesianSegNetParams:
    """bayesian_segnet.hpp:85-105."""
    model_file: str = ""
    weights_file: str = ""
    use_gpu: bool = True  # kept for signature parity; this backend is GPU only


def sample_ranges(T: int, G: int):
    """Latency mode: the T Monte-Carlo samples of a frame split over G ranks as contiguous (begin, count) blocks whose sizes
    differ by at most one, larger blocks first -- e.g. T=6, G=4 -> [(0, 2), (2, 2), (4, 1), (5, 1)]."""
    if T < 1 or G < 1:
        raise ValueError(f"sample_ranges: T={T} and G={G} must both be >= 1")
    if G > T:
        raise ValueError(f"sample_ranges: {G} ranks for {T} samples would leave a rank without a sample")
    base, extra = divmod(T, G)
    out, b = [], 0
    for g in range(G):
        n = base + (1 if g < extra else 0)
        out.append((b, n))
        b += n
    return out


class BayesianSegNet:
    def __init__(self, params: BayesianSegNetParams, device: int = 0, seed: int = 1234, T: int = 0,
                 precision: str = "fp16", engine: str = "auto", keep_blobs: bool = False, samples=None):
        """`samples` = (begin, count): a latency-mode shard that runs only the samples [begin, begin + count) of a frame of T;
        run it with run_partial() and turn the sum over all shards into maps with finalize()."""
        self._h = C.c_void_p()
        opt = L.SegnetOptions(device=device, T=T, seed=seed,
                              precision={"fp16": L.PRECISION_FP16, "fp32": L.PRECISION_FP32}[precision],
                              engine={"auto": L.ENGINE_AUTO, "simt": L.ENGINE_SIMT, "tcgen05": L.ENGINE_TCGEN05}[engine],
                              keep_blobs=int(keep_blobs), reserved=0)
        if samples is None:
            rc = L.lib().sivo_segnet_create_ex(params.model_file.encode(), params.weights_file.encode(), C.byref(opt),
                                               C.byref(self._h))
        else:
            begin, count = samples
            rc = L.lib().sivo_segnet_create_shard(params.model_file.encode(), params.weights_file.encode(), C.byref(opt), begin, count,
                                                  C.byref(self._h))
        if rc == L.EINVAL:  # the reference throws std::invalid_argument (bayesian_segnet.cpp:66,68,82,86)
            raise ValueError(L.lib().sivo_last_error().decode())
        L.check(rc)
        w, h, t, nc = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        L.check(L.lib().sivo_segnet_geometry(self._h, C.byref(w), C.byref(h), C.byref(t), C.byref(nc)))
        self.width, self.height, self.T, self.n_classes = w.value, h.value, t.value, nc.value
        b, n = C.c_int(), C.c_int()
        L.check(L.lib().sivo_segnet_samples(self._h, C.byref(b), C.byref(n), None))
        self.sample_begin, self.sample_count = b.value, n.value

    def __del__(self):
        if getattr(self, "_h", None) and self._h.value and L is not None and getattr(L, "lib", None):
            try:
                L.lib().sivo_segnet_destroy(self._h)
            except Exception:  # interpreter shutdown: module globals may already be gone
                pass
            self._h = C.c_void_p()

    def getInputGeometry(self):
        return (self.width, self.height)  # cv::Size(width, height)

    def set_frame(self, frame: int):
        L.check(L.lib().sivo_segnet_set_frame(self._h, frame))

    def set_profiling(self, on: bool):
        L.check(L.lib().sivo_segnet_set_profiling(self._h, on))

    def segmentImage(self, image: np.ndarray, out=None):
        """image: HxWx3 u8 BGR.  Returns (classes u8 [H,W], confidence f64 [H,W], entropy f64 [H,W]).
        `out` = (classes, confidence, entropy) reuses caller buffers (like the Eigen matrices the C++ shim resizes
        once); page-locked buffers receive the device copies directly."""
        if image.dtype != np.uint8 or image.ndim != 3 or image.shape[2] != 3:
            raise ValueError("segmentImage expects an HxWx3 uint8 BGR image")
        if image.strides[2] != 1 or image.strides[1] != 3:
            image = np.ascontiguousarray(image)
        if out is not None:
            classes, conf, ent = out
            assert classes.shape == conf.shape == ent.shape == (self.height, self.width)
            assert classes.dtype == np.uint8 and conf.dtype == np.float64 and ent.dtype == np.float64
            assert classes.flags.c_contiguous and conf.flags.c_contiguous and ent.flags.c_contiguous
        else:
            classes = np.empty((self.height, self.width), np.uint8)
            conf = np.empty((self.height, self.width), np.float64)
            ent = np.empty((self.height, self.width), np.float64)
        L.check(L.lib().sivo_segnet_run(self._h, L.ptr(image), image.shape[0], image.shape[1], image.strides[0], L.ptr(classes),
                                        L.ptr(conf), L.ptr(ent)))
        return classes, conf, ent

    def segment_on_device(self, image: np.ndarray):
        """segmentImage without the read-back: the three maps stay on the device for semantic_keys()."""
        if image.dtype != np.uint8 or image.ndim != 3 or image.shape[2] != 3:
            raise ValueError("segmentImage expects an HxWx3 uint8 BGR image")
        if image.strides[2] != 1 or image.strides[1] != 3:
            image = np.ascontiguousarray(image)
        L.check(L.lib().sivo_segnet_run(self._h, L.ptr(image), image.shape[0], image.shape[1], image.strides[0], None, None, None))

    def semantic_keys(self, kps: np.ndarray, max_static_class: int = 8):
        """Frame::SelectSemanticKeys (Frame.cc:177-203) + per-keypoint map reads on the device-resident result of the last
        run.  kps: structured array (orb.KP_DTYPE).  Returns (classes u8 [n], confidence f64 [n], entropy f64 [n], keep int32 [m]):
        keep = indices whose class <= max_static_class (Classes::TERRAIN), in keypoint order."""
        kps = np.ascontiguousarray(kps)
        if kps.dtype.itemsize != 28:
            raise ValueError("keypoints must be the 28-byte sivo_keypoint records")
        n = len(kps)
        cls = np.empty(n, np.uint8)
        conf = np.empty(n, np.float64)
        ent = np.empty(n, np.float64)
        keep = np.empty(max(n, 1), np.int32)
        m = C.c_int(0)
        L.check(L.lib().sivo_segnet_semantic_keys(self._h, L.ptr(kps), n, max_static_class, L.ptr(cls), L.ptr(conf), L.ptr(ent),
                                                  L.ptr(keep), C.byref(m)))
        return cls, conf, ent, keep[:m.value].copy()

    def semantic_keys_device(self, kps_ptr: int, count_ptr: int, cap: int, max_static_class: int = 8, class_ptr: int = 0,
                             conf_ptr: int = 0, ent_ptr: int = 0, keep_ptr: int = 0, n_keep_ptr: int = 0, stream: int = 0):
        """semantic_keys on device buffers (sivo_segnet_semantic_keys_device): kps_ptr holds the keypoint records and count_ptr
        their int64 count (e.g. what ORBextractor.enqueue_device wrote), cap the capacity of the output buffers (u8 classes,
        float64 confidence / entropy, int32 keep indices; 0 = not wanted).  *n_keep_ptr (int64) receives the kept count, or -1
        if the count exceeds cap.  Enqueued on `stream` (0 = the stream of the last run) without a host synchronisation."""
        L.check(L.lib().sivo_segnet_semantic_keys_device(self._h, kps_ptr, count_ptr, cap, max_static_class, class_ptr, conf_ptr,
                                                         ent_ptr, keep_ptr, n_keep_ptr, stream))

    def run_device(self, bgr_ptr: int, classes_ptr: int, conf_ptr: int, ent_ptr: int, stream: int = 0):
        L.check(L.lib().sivo_segnet_run_device(self._h, bgr_ptr, classes_ptr, conf_ptr, ent_ptr, stream))

    def set_record_outputs(self, classes_ptr: int = 0, conf32_ptr: int = 0, ent32_ptr: int = 0):
        """segmentImage additionally leaves classes + f32 maps at these device addresses (a packed multi-GPU record); 0s: off."""
        L.check(L.lib().sivo_segnet_set_record_outputs(self._h, classes_ptr, conf32_ptr, ent32_ptr))

    def run_device_maps(self, bgr_ptr: int, classes_ptr: int, conf_ptr: int, ent_ptr: int, conf32_ptr: int, ent32_ptr: int, stream: int = 0):
        """run_device plus single-precision copies of the two maps (the packed multi-GPU record's layout); any pointer may be 0."""
        L.check(L.lib().sivo_segnet_run_device_maps(self._h, bgr_ptr, classes_ptr, conf_ptr, ent_ptr, conf32_ptr, ent32_ptr, stream))

    def run_partial(self, bgr_ptr: int, sum_ptr: int, stream: int = 0):
        """Latency mode: this handle's samples of the frame at bgr_ptr (device, height x width x 3 u8); sum_ptr (device,
        height*width x 16 float64) receives their sum of per-sample softmax.  Advances the frame counter like run_device."""
        L.check(L.lib().sivo_segnet_run_partial_device(self._h, bgr_ptr, sum_ptr, stream))

    def finalize(self, sum_ptr: int, classes_ptr: int, conf_ptr: int, ent_ptr: int, conf32_ptr: int = 0, ent32_ptr: int = 0,
                 stream: int = 0):
        """Latency mode: the maps of run_device_maps from sum_ptr = the sum over ALL T samples (e.g. reduced over the ranks'
        run_partial sums); any output pointer may be 0."""
        L.check(L.lib().sivo_segnet_finalize_device(self._h, sum_ptr, classes_ptr, conf_ptr, ent_ptr, conf32_ptr, ent32_ptr, stream))

    def computeVariance(self, classes: np.ndarray) -> np.ndarray:
        """bayesian_segnet.cpp:205-260 after segmentImage / segment_on_device: float64 [H, W], per pixel the sample variance
        over the last frame's T samples of the softmax probability of class classes[row, col] (0 where it is >= n_classes)."""
        classes = np.ascontiguousarray(classes)
        if classes.dtype != np.uint8 or classes.shape != (self.height, self.width):
            raise ValueError(f"computeVariance expects a {self.height}x{self.width} uint8 class map")
        var = np.empty((self.height, self.width), np.float64)
        L.check(L.lib().sivo_segnet_variance(self._h, L.ptr(classes), L.ptr(var)))
        return var

    def variance_device(self, classes_ptr: int, var_ptr: int, stream: int = 0):
        """computeVariance on device buffers (height*width u8 in, float64 out), ordered on `stream` after the run it reads."""
        L.check(L.lib().sivo_segnet_variance_device(self._h, classes_ptr, var_ptr, stream))

    def variance_partial(self, classes_ptr: int, moments_ptr: int, stream: int = 0):
        """Latency mode: moments_ptr (device, height*width x 2 float64) receives (sum p, sum p^2) of the given class over this
        shard's samples of its last run_partial."""
        L.check(L.lib().sivo_segnet_variance_partial_device(self._h, classes_ptr, moments_ptr, stream))

    def variance_finalize(self, moments_ptr: int, var_ptr: int, stream: int = 0):
        """Latency mode: the variance map from the moments summed over ALL T samples of the frame."""
        L.check(L.lib().sivo_segnet_variance_finalize_device(self._h, moments_ptr, var_ptr, stream))

    def blob(self, name: str) -> np.ndarray:
        n, c, h, w = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        L.check(L.lib().sivo_segnet_blob(self._h, name.encode(), None, 0, C.byref(n), C.byref(c), C.byref(h), C.byref(w)))
        out = np.empty((n.value, c.value, h.value, w.value), np.float32)
        L.check(L.lib().sivo_segnet_blob(self._h, name.encode(), L.ptr(out), out.size, None, None, None, None))
        return out

    def op_flops_executed(self):
        """Executed conv flops per launch (== algorithmic except for the composed classifier and the split-operand mode)."""
        n = C.c_int()
        L.check(L.lib().sivo_segnet_op_timing(self._h, -1, None, 0, None, None, C.byref(n)))
        out = []
        for i in range(n.value):
            fl = C.c_double()
            L.check(L.lib().sivo_segnet_op_flops_executed(self._h, i, C.byref(fl)))
            out.append(fl.value)
        return out

    def op_timings(self):
        """[(layer names, ms in the last profiled run, algorithmic conv flops)] per launch of the op list."""
        n = C.c_int()
        L.check(L.lib().sivo_segnet_op_timing(self._h, -1, None, 0, None, None, C.byref(n)))
        out = []
        for i in range(n.value):
            buf = C.create_string_buffer(256)
            ms, fl = C.c_float(), C.c_double()
            L.check(L.lib().sivo_segnet_op_timing(self._h, i, buf, 256, C.byref(ms), C.byref(fl), None))
            out.append((buf.value.decode(), ms.value, fl.value))
        return out

    def last_timing(self):
        a, b, c, d, n = C.c_float(), C.c_float(), C.c_float(), C.c_float(), C.c_int()
        L.check(L.lib().sivo_segnet_last_timing(self._h, C.byref(a), C.byref(b), C.byref(c), C.byref(d), C.byref(n)))
        return {"conv_ms": a.value, "other_ms": b.value, "reduce_ms": c.value, "total_ms": d.value, "launches": n.value}

    def flops(self):
        a, b = C.c_double(), C.c_double()
        L.check(L.lib().sivo_segnet_flops(self._h, C.byref(a), C.byref(b)))
        return {"dedup": a.value, "naive": b.value}
