"""The device front end of one stereo frame (Frame.cc:131-145): SegNet's maps, both extractors' keys, the semantic keys and the
stereo matches, resident on the device for the Frame-tail calls, and the stream edges that let several frames be in flight on
rotating DeviceFrames (DESIGN.md, "The Frame tail on the device")."""
import torch

from .orb import KP_DTYPE, stereo_match_device

MAX_STATIC_CLASS = 8  # Classes::TERRAIN: the classes Frame::SelectSemanticKeys keeps
# DeviceFrame's outputs by their C-ABI names: dtype and the sentinel each starts at
OUTPUTS = {"kp_class": (torch.uint8, 77), "kp_conf": (torch.float64, 7.0), "kp_entropy": (torch.float64, 7.0), "keep_idx": (torch.int32, -7),
           "n_keep": (torch.int64, -7), "u_right": (torch.float32, 7.0), "depth": (torch.float32, 7.0)}


class FrameKeys:
    """What ORBextractor.enqueue_device writes for one extractor: capacity() 28-byte keypoint records, their 32-byte descriptors
    and an int64 count."""

    def __init__(self, ext):
        self.cap = ext.capacity()
        self.kps = torch.zeros(self.cap * 28, dtype=torch.uint8, device="cuda")
        self.desc = torch.zeros(self.cap * 32, dtype=torch.uint8, device="cuda")
        self.count = torch.zeros(1, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()  # the extractor's stream does not wait for torch's

    def enqueue(self, ext, gray_dev, rows, cols, pitch):
        ext.enqueue_device(gray_dev.data_ptr(), rows, cols, pitch, self.kps.data_ptr(), self.desc.data_ptr(), self.count.data_ptr())

    def host(self):
        """(keypoints KP_DTYPE [n], descriptors u8 [n, 32]); the caller has waited for the extractor."""
        n = int(self.count.cpu()[0])
        return self.kps[:n * 28].cpu().numpy().view(KP_DTYPE), self.desc[:n * 32].cpu().numpy().reshape(n, 32)


def _ptr(name):
    return property(lambda self: self.out[name].data_ptr(), doc=f"device address of out[{name!r}]")


class DeviceFrame:
    """One stereo frame's device front end for the extractor pair (left, right) on rows x cols images: the three SegNet maps,
    a FrameKeys per side, the five semantic-key outputs (kp_class, kp_conf, kp_entropy, keep_idx, n_keep) and the stereo outputs
    (u_right, depth), each of the left extractor's capacity().  Every buffer starts at a sentinel (classes 77, floats 7.0,
    indices and counts -7), so an entry a call leaves unwritten shows.

    extract() then tail() enqueue the front end on a caller stream S; the properties give the device addresses the Frame-tail
    calls take."""

    def __init__(self, left, right, rows, cols):
        self.el, self.er = left, right
        self.rows, self.cols = rows, cols
        cap, n = left.capacity(), rows * cols
        self.maps = (torch.full((n,), 77, dtype=torch.uint8, device="cuda"), torch.full((n,), 7.0, dtype=torch.float64, device="cuda"),
                     torch.full((n,), 7.0, dtype=torch.float64, device="cuda"))  # classes, confidence, entropy
        self.left, self.right = FrameKeys(left), FrameKeys(right)
        self.out = {k: torch.empty(1 if k == "n_keep" else cap, dtype=dt, device="cuda") for k, (dt, _) in OUTPUTS.items()}
        self.reset()

    def reset(self):
        """Every semantic-key and stereo output back at its sentinel."""
        for k, (_, v) in OUTPUTS.items():
            self.out[k].fill_(v)
        torch.cuda.synchronize()  # the library's streams do not wait for torch's

    kps = property(lambda self: self.left.kps.data_ptr(), doc="device address of the left keypoint records")
    desc = property(lambda self: self.left.desc.data_ptr(), doc="device address of the left descriptors")
    count = property(lambda self: self.left.count.data_ptr(), doc="device address of the left int64 count")
    kp_class, kp_conf, kp_entropy, keep, n_keep, u_right, depth = (
        _ptr(k) for k in ("kp_class", "kp_conf", "kp_entropy", "keep_idx", "n_keep", "u_right", "depth"))

    def extract(self, seg, bgr, gray_left, gray_right, stream):
        """SegNet's maps of `bgr` on `stream`, both extractors on their own streams, then `stream` waits for the left keypoints.
        The extractors first wait for everything already on `stream`: the previous frame's Frame-tail calls read the pyramids
        (and, on the same DeviceFrame, the keys) these enqueues overwrite.  This frame's SegNet is enqueued after that wait, so
        the extractors run beside it.  bgr / gray_left / gray_right: device tensors, complete before the call."""
        self.el.wait_for_stream(stream)
        self.er.wait_for_stream(stream)
        seg.run_device_maps(bgr.data_ptr(), *(m.data_ptr() for m in self.maps), 0, 0, stream)
        self.left.enqueue(self.el, gray_left, self.rows, self.cols, self.cols)
        self.right.enqueue(self.er, gray_right, self.rows, self.cols, self.cols)
        self.el.stream_wait(stream)  # the semantic keys read the left keypoints

    def tail(self, seg, mb, mbf, stream):
        """Frame::SelectSemanticKeys then Frame::ComputeStereoMatches over the kept keys, on `stream` after extract().  The stereo
        call makes `stream` wait for both extractors itself."""
        seg.semantic_keys_device(self.kps, self.count, self.left.cap, MAX_STATIC_CLASS, self.kp_class, self.kp_conf, self.kp_entropy,
                                 self.keep, self.n_keep, stream)
        stereo_match_device(self.el, self.er, self.kps, self.desc, self.keep, self.n_keep, self.right.kps.data_ptr(),
                            self.right.desc.data_ptr(), self.right.count.data_ptr(), mb, mbf, self.u_right, self.depth, stream)

    def host(self):
        """(n_keep, keep_idx [n_keep], u_right [n_keep], depth [n_keep]) as host arrays; the caller has synchronised the stream."""
        n = int(self.out["n_keep"].cpu()[0])
        m = max(n, 0)
        return (n, self.out["keep_idx"][:m].cpu().numpy(), self.out["u_right"][:m].cpu().numpy(), self.out["depth"][:m].cpu().numpy())
