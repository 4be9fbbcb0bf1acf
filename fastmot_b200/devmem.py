"""Device-memory plumbing: torch tensors are used only as containers (allocation, streams, pinned memory).

`Uplink` packs many small host arrays into one pinned block and ships them with a single async H2D copy;
`ptr()` turns tensors into raw addresses for the C-ABI.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib


def ptr(t):
    """Raw device (or pinned-host) address of a torch tensor, or None."""
    if t is None:
        return None
    return C.c_void_p(t.data_ptr())


def stream_ptr(stream=None):
    s = torch.cuda.current_stream() if stream is None else stream
    return C.c_void_p(s.cuda_stream)


class Uplink:
    """Ring of pinned staging blocks -> one device block each; one cudaMemcpyAsync per `flush`."""

    ALIGN = 256

    def __init__(self, nbytes=1 << 20, depth=4, device="cuda"):
        self.nbytes = nbytes
        self.host = [torch.empty(nbytes, dtype=torch.uint8).pin_memory() for _ in range(depth)]
        self.host_np = [h.numpy() for h in self.host]
        self.dev = [torch.empty(nbytes, dtype=torch.uint8, device=device) for _ in range(depth)]
        self.events = [None] * depth
        self.cur = 0
        self.off = 0
        self._begin()

    def _begin(self):
        ev = self.events[self.cur]
        if ev is not None:
            ev.synchronize()
        self.off = 0

    def put(self, arr):
        """Stage a host ndarray; returns the device address (c_void_p) it will have after flush()."""
        arr = np.ascontiguousarray(arr)
        n = arr.nbytes
        off = self.off
        if off + n > self.nbytes:
            raise MemoryError("Uplink block overflow")
        if n:
            self.host_np[self.cur][off:off + n] = arr.view(np.uint8).reshape(-1)
        self.off = (off + n + self.ALIGN - 1) // self.ALIGN * self.ALIGN
        return C.c_void_p(self.dev[self.cur].data_ptr() + off)

    def flush(self):
        if self.off:
            self.dev[self.cur][:self.off].copy_(self.host[self.cur][:self.off], non_blocking=True)
            ev = torch.cuda.Event()
            ev.record()
            self.events[self.cur] = ev
        self.cur = (self.cur + 1) % len(self.host)
        self._begin()


class Downlink:
    """Device scratch block mirrored by a pinned host block; kernels write results at `alloc`ed offsets,
    `fetch()` brings the used prefix back with one D2H copy + stream synchronize."""

    ALIGN = 256

    def __init__(self, nbytes=1 << 20, device="cuda"):
        self.nbytes = nbytes
        self.dev = torch.empty(nbytes, dtype=torch.uint8, device=device)
        self.host = torch.empty(nbytes, dtype=torch.uint8).pin_memory()
        self.host_np = self.host.numpy()
        self.off = 0
        self.items = []

    def reset(self):
        self.off = 0
        self.items = []

    def alloc(self, shape, dtype):
        dtype = np.dtype(dtype)
        n = int(np.prod(shape)) * dtype.itemsize
        off = self.off
        if off + n > self.nbytes:
            raise MemoryError("Downlink block overflow")
        self.off = (off + n + self.ALIGN - 1) // self.ALIGN * self.ALIGN
        self.items.append((off, n, tuple(shape), dtype))
        return C.c_void_p(self.dev.data_ptr() + off), len(self.items) - 1

    def fetch(self):
        """Returns list of ndarrays (views into the pinned block — copy if kept across fetches)."""
        if self.off:
            self.host[:self.off].copy_(self.dev[:self.off], non_blocking=True)
        torch.cuda.current_stream().synchronize()
        out = []
        for off, n, shape, dtype in self.items:
            out.append(self.host_np[off:off + n].view(dtype).reshape(shape))
        return out


PIXEL_FORMATS = ("BGR", "NV12")


def check_pixel_format(pixel_format):
    """'BGR' or 'NV12' (any case) -> the upper-case name; anything else raises ValueError."""
    fmt = str(pixel_format).upper()
    if fmt not in PIXEL_FORMATS:
        raise ValueError(f"pixel_format must be one of {PIXEL_FORMATS}, got {pixel_format!r}")
    return fmt


class Frame:
    """One camera frame as the pre-processing kernels read it: pixel format, size and planes.

    BGR: `y` is an HxWx3 uint8 cuda tensor (tight rows); `uv` is None.
    NV12 (hardware video decoders): `y` is the H x W luma plane and `uv` the H/2 x W plane of interleaved U, V at half
    resolution, each with its own row pitch in bytes (`y_pitch`, `uv_pitch` >= W).  Build NV12 frames with
    `nv12_frame`; the planes are views of the caller's memory, nothing is copied.
    A host frame (`on_device` False) holds its ndarray in `y` (HxWx3 BGR or (3H/2, W) NV12); `device_frame` uploads it.
    """
    __slots__ = ("format", "w", "h", "y", "uv", "y_pitch", "uv_pitch", "_fm")

    def __init__(self, format, w, h, y, uv=None, y_pitch=0, uv_pitch=0):
        self.format, self.w, self.h = format, int(w), int(h)
        self.y, self.uv, self.y_pitch, self.uv_pitch = y, uv, int(y_pitch), int(uv_pitch)
        self._fm = None

    @classmethod
    def bgr(cls, t):
        """A contiguous HxWx3 uint8 cuda tensor as a Frame."""
        if not (torch.is_tensor(t) and t.is_cuda and t.dtype == torch.uint8 and t.dim() == 3 and t.shape[2] == 3
                and t.is_contiguous()):
            raise ValueError("every BGR frame must be a contiguous HxWx3 uint8 cuda tensor")
        return cls("BGR", t.shape[1], t.shape[0], t)

    @property
    def size(self):
        return (self.w, self.h)

    @property
    def on_device(self):
        return torch.is_tensor(self.y)

    def fm(self):
        """The FmFrame of this device frame, which every C entry point that reads camera pixels takes (built on the
        first call).  It holds raw plane addresses: keep this Frame referenced until the kernels that read them ran."""
        if self._fm is None:
            nv12 = self.format == "NV12"
            self._fm = _lib.FmFrame(self.y.data_ptr(), self.uv.data_ptr() if nv12 else None, self.w, self.h,
                                    self.y_pitch, self.uv_pitch, _lib.FM_PIX_NV12 if nv12 else _lib.FM_PIX_BGR)
        return self._fm


def _plane(t, rows, w, what):
    """Checks one NV12 plane: a 2-D uint8 tensor of `rows` x w with unit column stride and any row stride >= w."""
    if not torch.is_tensor(t):
        raise ValueError(f"NV12 {what}: expected a uint8 cuda tensor, got {type(t).__name__}")
    if t.dtype != torch.uint8 or t.dim() != 2:
        raise ValueError(f"NV12 {what}: expected a 2-D uint8 tensor, got {t.dtype} of shape {tuple(t.shape)}")
    if tuple(t.shape) != (rows, w):
        raise ValueError(f"NV12 {what}: expected shape {(rows, w)}, got {tuple(t.shape)}")
    if t.stride(1) != 1 or t.stride(0) < w:
        raise ValueError(f"NV12 {what}: expected stride(1) == 1 and stride(0) >= {w} (the width), got strides "
                         f"{tuple(t.stride())}")


def _even(w, h):
    if w < 2 or h < 2 or w % 2 or h % 2:
        raise ValueError(f"NV12 needs an even width and height, got {w}x{h}")


def nv12_layout(frame):
    """Checks the shape, dtype and strides of an NV12 frame in one of the forms `nv12_frame` takes and returns its
    Frame, without looking at the device its tensors live on."""
    if isinstance(frame, Frame):
        if frame.format != "NV12":
            raise ValueError(f"expected an NV12 frame, got a {frame.format} Frame")
        return frame
    if isinstance(frame, (tuple, list)):
        if len(frame) != 2:
            raise ValueError(f"NV12 planes: expected a pair (Y (H, W), UV (H/2, W)), got {len(frame)} items")
        y, uv = frame
        if not torch.is_tensor(y) or y.dim() != 2:
            raise ValueError("NV12 Y plane: expected a 2-D uint8 cuda tensor (H, W)")
        h, w = y.shape
        _even(w, h)
        _plane(y, h, w, "Y plane")
        _plane(uv, h // 2, w, "UV plane")
        return Frame("NV12", w, h, y, uv, y.stride(0), uv.stride(0))
    if isinstance(frame, np.ndarray):
        if frame.dtype != np.uint8 or frame.ndim != 2 or frame.shape[0] % 3:
            raise ValueError(f"NV12 host frame: expected a (3H/2, W) uint8 ndarray, got {frame.dtype} of shape "
                             f"{frame.shape}")
        h, w = frame.shape[0] * 2 // 3, frame.shape[1]
        _even(w, h)
        return Frame("NV12", w, h, frame)
    if torch.is_tensor(frame):
        if frame.dim() != 2 or frame.shape[0] % 3:
            raise ValueError(f"NV12 frame: expected a (3H/2, W) uint8 cuda tensor, got shape {tuple(frame.shape)}")
        h, w = frame.shape[0] * 2 // 3, frame.shape[1]
        _even(w, h)
        _plane(frame, 3 * h // 2, w, "frame")
        return Frame("NV12", w, h, frame[:h], frame[h:], frame.stride(0), frame.stride(0))
    raise ValueError(f"NV12 frame: expected a (3H/2, W) uint8 ndarray or cuda tensor, or a (Y, UV) pair of cuda "
                     f"tensors, got {type(frame).__name__}")


def nv12_frame(frame):
    """The Frame of an NV12 frame given as
      - a host ndarray (3H/2, W) uint8 (Y rows, then UV rows);
      - a cuda tensor (3H/2, W) uint8 with stride(1) == 1 and any stride(0) >= W (pitched surfaces);
      - a pair (Y, UV) of cuda tensors (H, W) and (H/2, W), each with its own row stride (decoder surfaces whose UV
        plane does not follow row H, e.g. 1080p decoded into 1088-row surfaces).
    A Frame passes through.  Anything else (wrong shape, dtype or device, odd size, row stride below W) raises
    ValueError naming what was expected."""
    f = nv12_layout(frame)
    if f.on_device:
        if not f.y.is_cuda or not f.uv.is_cuda:
            raise ValueError(f"NV12 frame: expected cuda tensors, got tensors on {f.y.device} and {f.uv.device} "
                             "(host frames are (3H/2, W) uint8 ndarrays)")
        if f.y.device != f.uv.device:
            raise ValueError(f"NV12 planes on different devices: {f.y.device} and {f.uv.device}")
    return f


class FrameUploader:
    """Host frame -> device tensor with one async copy: HxWx3 u8 BGR frames, or (pixel_format 'NV12') (3H/2, W) u8
    NV12 frames, which move half the bytes.  Page-locked sources (detected with cudaPointerGetAttributes) are copied
    directly; pageable ones are staged through an internal pinned ring."""

    def __init__(self, size, depth=2, device="cuda", pixel_format="BGR"):
        self._lib = _lib.load()
        self.pixel_format = check_pixel_format(pixel_format)
        self.shape = self.frame_shape(size, self.pixel_format)
        self.nbytes = int(np.prod(self.shape))
        self.bytes_copied = 0              # host-to-device bytes of every copy made so far
        self.dev = [torch.empty(self.shape, dtype=torch.uint8, device=device) for _ in range(depth)]
        self.host = [torch.empty(self.shape, dtype=torch.uint8).pin_memory() for _ in range(depth)]
        self.host_np = [t.numpy() for t in self.host]
        self.events = [None] * depth
        self.cur = 0
        # read-ahead (GPU-resident ingest, role of the reference's VideoIO frame queue, fastmot/videoio.py:125-142):
        # prefetch(frame) starts the H2D copy of a FUTURE frame on a dedicated upload stream while the current step
        # computes; upload() of that same frame then only waits for the copy's event.  Every prefetched frame keeps its
        # copy until it is uploaded or its slot is taken again, so prefetch(frame t + 1) issued before upload(frame t)
        # does not discard frame t's read-ahead.
        self._up_stream = torch.cuda.Stream(device=device)
        self._prefetched = {}              # key -> (slot, event)

    @staticmethod
    def frame_shape(size, pixel_format):
        """Shape of a host frame of size (width, height): (h, w, 3) for BGR, (3h/2, w) for NV12."""
        w, h = size
        return (h, w, 3) if pixel_format == "BGR" else (3 * h // 2, w)

    @staticmethod
    def _key(frame):
        return (frame.ctypes.data, frame.shape)

    def _copy(self, frame, k, stream):
        src = frame.ctypes.data
        if not self._lib.fm_host_is_pinned(C.c_void_p(src)):
            ev = self.events[k]
            if ev is not None:
                ev.synchronize()
            np.copyto(self.host_np[k], frame)
            src = self.host[k].data_ptr()
        self._lib.fm_memcpy_async(C.c_void_p(self.dev[k].data_ptr()), C.c_void_p(src), self.nbytes,
                                  C.c_void_p(stream.cuda_stream))
        self.bytes_copied += self.nbytes
        ev = torch.cuda.Event()
        ev.record(stream)
        self.events[k] = ev
        return ev

    def _next_slot(self):
        """Takes the next ring slot; a read-ahead still parked there is dropped (its frame would be copied again)."""
        k = self.cur
        self.cur = (k + 1) % len(self.dev)
        for key, (slot, _) in list(self._prefetched.items()):
            if slot == k:
                del self._prefetched[key]
        return k

    def prefetch(self, frame):
        """Starts the upload of a frame that a later upload() call will ask for (the same ndarray)."""
        frame = np.ascontiguousarray(frame)
        if frame.shape != self.shape or frame.dtype != np.uint8:
            raise ValueError(f"frame must be uint8 {self.shape}, got {frame.dtype} {frame.shape}")
        key = self._key(frame)
        self._prefetched.pop(key, None)          # the array may hold a new frame: copy it again
        k = self._next_slot()
        # the slot's previous contents may still be read by kernels of the main stream
        self._up_stream.wait_stream(torch.cuda.current_stream())
        self._prefetched[key] = (k, self._copy(frame, k, self._up_stream))

    def upload(self, frame):
        frame = np.ascontiguousarray(frame)
        hit = self._prefetched.pop(self._key(frame), None)
        if hit is not None:
            k, ev = hit
            torch.cuda.current_stream().wait_event(ev)
            return self.dev[k]
        if frame.shape != self.shape or frame.dtype != np.uint8:
            raise ValueError(f"frame must be uint8 {self.shape}, got {frame.dtype} {frame.shape}")
        k = self._next_slot()
        self._copy(frame, k, torch.cuda.current_stream())
        return self.dev[k]

    def upload_frame(self, f):
        """A host Frame of this uploader's format and size -> its device Frame."""
        t = self.upload(f.y)
        return nv12_frame(t) if self.pixel_format == "NV12" else Frame.bgr(t)


class UploadSlot:
    """Uploads host Frames of any format and size: keeps the FrameUploader of the last one and builds a new one when the
    format or size changes (a stage used on its own, whose caller may change the frame size between calls)."""

    def __init__(self, uploader=None):
        self.uploader = uploader

    def upload_frame(self, f):
        up = self.uploader
        if up is None or up.pixel_format != f.format or up.shape != FrameUploader.frame_shape(f.size, f.format):
            self.uploader = up = FrameUploader(f.size, pixel_format=f.format)
        return up.upload_frame(f)


def check_capture_size(capture_size, size, pixel_format):
    """The (width, height) a tracker's frames arrive at: `size` (the tracking size) when capture_size is None, else
    capture_size as a tuple of two positive ints (even for NV12).  Anything else raises ValueError."""
    if capture_size is None:
        return tuple(int(v) for v in size)
    if not (isinstance(capture_size, (tuple, list)) and len(capture_size) == 2
            and all(np.isscalar(v) and int(v) == v and v > 0 for v in capture_size)):
        raise ValueError(f"capture_size must be (width, height) with positive integers, got {capture_size!r}")
    w, h = (int(v) for v in capture_size)
    if pixel_format == "NV12" and (w % 2 or h % 2):
        raise ValueError(f"an NV12 capture size must be even, got {w}x{h}")
    return w, h


class FrameResizer:
    """Device Frames of any size and format -> BGR Frames of one size (`size`, the tracking size): cv2.resize with the
    default INTER_LINEAR of the frame (of its cv2.cvtColor decode for NV12), bit for bit, one fm_frame_resize launch on
    the current stream into the next slot of a ring of `depth` device frames.

    Slot reuse: a tracker resizes on the main stream at the start of a step, and every stage reads the resized frame
    either on the main stream or on a stream that waits on an event recorded after the resize (the detector and ReID
    streams wait on `_main_ready`).  Before the next step's resize is enqueued, the host has waited for the detector
    stream's last event and the main stream has joined the ReID stream, so every read of a slot is ordered before the
    next write on the main stream.  One slot would therefore do; with two, a resize never overwrites the frame the
    previous step's stages were handed, whatever a later stage does with it."""

    def __init__(self, size, depth=2, device="cuda"):
        self._lib = _lib.load()
        self.size = w, h = tuple(int(v) for v in size)
        self.dev = [torch.empty((h, w, 3), dtype=torch.uint8, device=device) for _ in range(depth)]
        self.cur = 0

    def resize(self, frame):
        """The device Frame `frame` at this resizer's size, as a BGR Frame (valid until `depth` more resizes)."""
        out = self.dev[self.cur]
        self.cur = (self.cur + 1) % len(self.dev)
        _lib.check(self._lib.fm_frame_resize(C.byref(frame.fm()), ptr(out), self.size[0], self.size[1], stream_ptr()),
                   "fm_frame_resize")
        return Frame.bgr(out)


def as_frame(frame, pixel_format="BGR", size=None):
    """A caller's frame as a Frame, nothing copied.  A Frame passes through; otherwise `frame` is in pixel_format:
    'BGR' -- an HxWx3 uint8 cuda tensor (contiguous) or host ndarray; 'NV12' -- any form nv12_frame accepts.  size:
    the (width, height) the frame must have; another size raises ValueError."""
    if isinstance(frame, Frame):
        f = frame
    elif pixel_format == "NV12":
        f = nv12_frame(frame)
    elif torch.is_tensor(frame):
        f = Frame.bgr(frame)
    else:
        if not (isinstance(frame, np.ndarray) and frame.dtype == np.uint8 and frame.ndim == 3 and frame.shape[2] == 3):
            raise ValueError(f"BGR host frame: expected an HxWx3 uint8 ndarray, got {type(frame).__name__} "
                             f"{getattr(frame, 'dtype', '')} {getattr(frame, 'shape', '')}")
        f = Frame("BGR", frame.shape[1], frame.shape[0], frame)
    if size is not None and f.size != tuple(size):
        raise ValueError(f"{f.format} frame of size {f.size}, expected {tuple(size)}")
    return f


def device_frame(frame, uploader=None, pixel_format="BGR", size=None):
    """The device Frame of a caller's frame (any input as_frame takes, checked against `size` as there).  A host frame
    is uploaded through `uploader`: a FrameUploader of its format and size, or an UploadSlot; without one a host frame
    raises ValueError."""
    f = as_frame(frame, pixel_format, size)
    if f.on_device:
        return f
    if uploader is None:
        raise ValueError("expected a frame in device memory, got a host frame")
    return uploader.upload_frame(f)


def prefetch_frame(frame, uploader, pixel_format="BGR", size=None):
    """Starts the upload (FrameUploader.prefetch) of the host frame a later device_frame call will get; a device frame
    needs none."""
    f = as_frame(frame, pixel_format, size)
    if not f.on_device:
        uploader.prefetch(f.y)
