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


class _PixelFormat:
    """One row of the pixel-format table: the FmFrame format code, the shape of a host frame of size (w, h), whether
    the width and the height must be even, and the parser of the frame forms the format accepts."""
    __slots__ = ("code", "shape", "even_w", "even_h", "layout")

    def __init__(self, code, shape, even_w, even_h, layout):
        self.code, self.shape, self.even_w, self.even_h, self.layout = code, shape, even_w, even_h, layout


def check_pixel_format(pixel_format):
    """One of PIXEL_FORMATS (any case) -> the upper-case name; anything else raises ValueError."""
    fmt = str(pixel_format).upper()
    if fmt not in PIXEL_FORMATS:
        raise ValueError(f"pixel_format must be one of {PIXEL_FORMATS}, got {pixel_format!r}")
    return fmt


def _check_size(fmt, w, h):
    """Raises ValueError unless (w, h) is a frame size `fmt` can have."""
    p = _FORMATS[fmt]
    if w < 1 or h < 1 or (p.even_w and w % 2) or (p.even_h and h % 2):
        need = ("an even width and height" if p.even_h else "an even width") if p.even_w else "a non-empty size"
        raise ValueError(f"{fmt} needs {need}, got {w}x{h}")


class Frame:
    """One camera frame as the pre-processing kernels read it: pixel format, size and planes.

    BGR: `y` is an HxWx3 uint8 cuda tensor (tight rows); `uv` is None.
    NV12 (hardware video decoders): `y` is the H x W luma plane and `uv` the H/2 x W plane of interleaved U, V at half
    resolution, each with its own row pitch in bytes (`y_pitch`, `uv_pitch` >= W).
    I420 (software decoders): `y` is the H x W luma plane, `uv` the H/2 x W/2 U plane and `v` the V plane, U and V
    with one row pitch `uv_pitch` >= W/2.
    YUY2 (USB cameras) and BGRX (nvvidconv): `y` is the H x W x 2 or H x W x 4 packed plane, row pitch `y_pitch`.
    Build them with `pixel_frame` (or `nv12_frame`); the planes are views of the caller's memory, nothing is copied.
    A host frame (`on_device` False) holds its ndarray in `y` (the host shape of its format, FrameUploader.frame_shape);
    `device_frame` uploads it.
    """
    __slots__ = ("format", "w", "h", "y", "uv", "y_pitch", "uv_pitch", "v", "_fm")

    def __init__(self, format, w, h, y, uv=None, y_pitch=0, uv_pitch=0, v=None):
        self.format, self.w, self.h = format, int(w), int(h)
        self.y, self.uv, self.y_pitch, self.uv_pitch, self.v = y, uv, int(y_pitch), int(uv_pitch), v
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
            addr = lambda t: None if t is None else t.data_ptr()
            self._fm = _lib.FmFrame(self.y.data_ptr(), addr(self.uv), self.w, self.h, self.y_pitch, self.uv_pitch,
                                    _FORMATS[self.format].code, addr(self.v))
        return self._fm


def _plane(t, rows, cols, what):
    """Checks one plane: a 2-D uint8 tensor of rows x cols with unit column stride and any row stride >= cols."""
    if not torch.is_tensor(t):
        raise ValueError(f"{what}: expected a uint8 cuda tensor, got {type(t).__name__}")
    if t.dtype != torch.uint8 or t.dim() != 2:
        raise ValueError(f"{what}: expected a 2-D uint8 tensor, got {t.dtype} of shape {tuple(t.shape)}")
    if tuple(t.shape) != (rows, cols):
        raise ValueError(f"{what}: expected shape {(rows, cols)}, got {tuple(t.shape)}")
    if t.stride(1) != 1 or t.stride(0) < cols:
        raise ValueError(f"{what}: expected stride(1) == 1 and stride(0) >= {cols} (the row length), got strides "
                         f"{tuple(t.stride())}")


def _is_u8(a):
    return a.dtype == (torch.uint8 if torch.is_tensor(a) else np.uint8)


def _yuv420_size(fmt, frame):
    """(w, h) of a (3H/2, W) uint8 4:2:0 frame (ndarray or tensor), checked."""
    if not _is_u8(frame) or frame.ndim != 2 or frame.shape[0] % 3:
        kind = "ndarray" if isinstance(frame, np.ndarray) else "cuda tensor"
        raise ValueError(f"{fmt} frame: expected a (3H/2, W) uint8 {kind}, got {frame.dtype} of shape "
                         f"{tuple(frame.shape)}")
    w, h = int(frame.shape[1]), int(frame.shape[0]) * 2 // 3
    _check_size(fmt, w, h)
    return w, h


def _bgr_layout(frame):
    if torch.is_tensor(frame):
        return Frame.bgr(frame)
    if not (isinstance(frame, np.ndarray) and frame.dtype == np.uint8 and frame.ndim == 3 and frame.shape[2] == 3):
        raise ValueError(f"BGR host frame: expected an HxWx3 uint8 ndarray, got {type(frame).__name__} "
                         f"{getattr(frame, 'dtype', '')} {getattr(frame, 'shape', '')}")
    return Frame("BGR", frame.shape[1], frame.shape[0], frame)


def _nv12_layout(frame):
    if isinstance(frame, (tuple, list)):
        if len(frame) != 2:
            raise ValueError(f"NV12 planes: expected a pair (Y (H, W), UV (H/2, W)), got {len(frame)} items")
        y, uv = frame
        if not torch.is_tensor(y) or y.dim() != 2:
            raise ValueError("NV12 Y plane: expected a 2-D uint8 cuda tensor (H, W)")
        h, w = y.shape
        _check_size("NV12", w, h)
        _plane(y, h, w, "NV12 Y plane")
        _plane(uv, h // 2, w, "NV12 UV plane")
        return Frame("NV12", w, h, y, uv, y.stride(0), uv.stride(0))
    if isinstance(frame, np.ndarray):
        w, h = _yuv420_size("NV12", frame)
        return Frame("NV12", w, h, frame)
    if torch.is_tensor(frame):
        w, h = _yuv420_size("NV12", frame)
        _plane(frame, 3 * h // 2, w, "NV12 frame")
        return Frame("NV12", w, h, frame[:h], frame[h:], frame.stride(0), frame.stride(0))
    raise ValueError(f"NV12 frame: expected a (3H/2, W) uint8 ndarray or cuda tensor, or a (Y, UV) pair of cuda "
                     f"tensors, got {type(frame).__name__}")


def _i420_layout(frame):
    if isinstance(frame, (tuple, list)):
        if len(frame) != 3:
            raise ValueError(f"I420 planes: expected a triple (Y (H, W), U (H/2, W/2), V (H/2, W/2)), got "
                             f"{len(frame)} items")
        y, u, v = frame
        if not torch.is_tensor(y) or y.dim() != 2:
            raise ValueError("I420 Y plane: expected a 2-D uint8 cuda tensor (H, W)")
        h, w = y.shape
        _check_size("I420", w, h)
        _plane(y, h, w, "I420 Y plane")
        _plane(u, h // 2, w // 2, "I420 U plane")
        _plane(v, h // 2, w // 2, "I420 V plane")
        if u.stride(0) != v.stride(0):
            raise ValueError(f"I420 U and V planes: expected equal row strides, got {u.stride(0)} and {v.stride(0)}")
        return Frame("I420", w, h, y, u, y.stride(0), u.stride(0), v)
    if isinstance(frame, np.ndarray):
        w, h = _yuv420_size("I420", frame)
        return Frame("I420", w, h, frame)
    if torch.is_tensor(frame):
        w, h = _yuv420_size("I420", frame)
        if not frame.is_contiguous():
            raise ValueError(f"I420 frame: expected a tight (3H/2, W) tensor (strides ({w}, 1)), got strides "
                             f"{tuple(frame.stride())}; give pitched planes as a (Y, U, V) triple")
        q = h * w // 4
        chroma = frame[h:].reshape(-1)
        u, v = chroma[:q].view(h // 2, w // 2), chroma[q:].view(h // 2, w // 2)
        return Frame("I420", w, h, frame[:h], u, w, w // 2, v)
    raise ValueError(f"I420 frame: expected a (3H/2, W) uint8 ndarray or cuda tensor, or a (Y, U, V) triple of cuda "
                     f"tensors, got {type(frame).__name__}")


def _packed_layout(fmt, ch):
    """The parser of a packed format of `ch` bytes per pixel: a host (H, W, ch) uint8 ndarray, or a cuda tensor of that
    shape with strides (>= ch W, ch, 1) (rows may be pitched)."""
    form = f"(H, W, {ch}) uint8"

    def layout(frame):
        if isinstance(frame, np.ndarray) or torch.is_tensor(frame):
            kind = "ndarray" if isinstance(frame, np.ndarray) else "cuda tensor"
            if not _is_u8(frame) or frame.ndim != 3 or frame.shape[2] != ch:
                raise ValueError(f"{fmt} frame: expected an {form} {kind}, got {frame.dtype} of shape "
                                 f"{tuple(frame.shape)}")
            h, w = int(frame.shape[0]), int(frame.shape[1])
            _check_size(fmt, w, h)
            if isinstance(frame, np.ndarray):
                return Frame(fmt, w, h, frame)
            if frame.stride(2) != 1 or frame.stride(1) != ch or frame.stride(0) < ch * w:
                raise ValueError(f"{fmt} frame: expected strides (>= {ch * w}, {ch}, 1), got {tuple(frame.stride())}")
            return Frame(fmt, w, h, frame, y_pitch=frame.stride(0))
        raise ValueError(f"{fmt} frame: expected an {form} ndarray or cuda tensor, got {type(frame).__name__}")
    return layout


# The one table of pixel formats: every other place asks it.
_FORMATS = {
    "BGR": _PixelFormat(_lib.FM_PIX_BGR, lambda w, h: (h, w, 3), False, False, _bgr_layout),
    "NV12": _PixelFormat(_lib.FM_PIX_NV12, lambda w, h: (3 * h // 2, w), True, True, _nv12_layout),
    "I420": _PixelFormat(_lib.FM_PIX_I420, lambda w, h: (3 * h // 2, w), True, True, _i420_layout),
    "YUY2": _PixelFormat(_lib.FM_PIX_YUY2, lambda w, h: (h, w, 2), True, False, _packed_layout("YUY2", 2)),
    "BGRX": _PixelFormat(_lib.FM_PIX_BGRX, lambda w, h: (h, w, 4), False, False, _packed_layout("BGRX", 4)),
}
PIXEL_FORMATS = tuple(_FORMATS)


def frame_layout(frame, pixel_format):
    """Checks the shape, dtype and strides of a frame in one of the forms `pixel_frame` takes for `pixel_format` and
    returns its Frame, without looking at the device its tensors live on.  A Frame of that format passes through."""
    fmt = check_pixel_format(pixel_format)
    if isinstance(frame, Frame):
        if frame.format != fmt:
            raise ValueError(f"expected a {fmt} frame, got a {frame.format} Frame")
        return frame
    return _FORMATS[fmt].layout(frame)


def pixel_frame(frame, pixel_format):
    """The Frame of a frame in `pixel_format`, given as
      - BGR : a host ndarray (H, W, 3) uint8, or a contiguous cuda tensor of that shape;
      - NV12: any form `nv12_frame` takes;
      - I420: a host ndarray (3H/2, W) uint8 (Y rows, then the U and the V plane: cv2's layout), a tight cuda tensor
        (3H/2, W), or a triple (Y, U, V) of cuda tensors (H, W), (H/2, W/2), (H/2, W/2) with unit column stride, any
        Y row stride >= W and one U / V row stride >= W/2;
      - YUY2: a host ndarray (H, W, 2) uint8 (Y0 U Y1 V per pixel pair: cv2's layout), or a cuda tensor of that shape
        with strides (>= 2W, 2, 1); W even;
      - BGRX: a host ndarray (H, W, 4) uint8, or a cuda tensor of that shape with strides (>= 4W, 4, 1).
    NV12 and I420 need an even width and height.  A Frame of that format passes through.  Anything else (wrong shape,
    dtype or device, odd size, row stride too small) raises ValueError naming what was expected."""
    f = frame_layout(frame, pixel_format)
    if f.on_device:
        planes = [t for t in (f.y, f.uv, f.v) if t is not None]
        if not all(t.is_cuda for t in planes):
            raise ValueError(f"{f.format} frame: expected cuda tensors, got tensors on "
                             f"{' and '.join(str(t.device) for t in planes)} (host frames are uint8 ndarrays)")
        if len({t.device for t in planes}) > 1:
            raise ValueError(f"{f.format} planes on different devices: "
                             f"{' and '.join(str(t.device) for t in planes)}")
    return f


def nv12_layout(frame):
    """frame_layout(frame, 'NV12')."""
    return frame_layout(frame, "NV12")


def nv12_frame(frame):
    """The Frame of an NV12 frame given as
      - a host ndarray (3H/2, W) uint8 (Y rows, then UV rows);
      - a cuda tensor (3H/2, W) uint8 with stride(1) == 1 and any stride(0) >= W (pitched surfaces);
      - a pair (Y, UV) of cuda tensors (H, W) and (H/2, W), each with its own row stride (decoder surfaces whose UV
        plane does not follow row H, e.g. 1080p decoded into 1088-row surfaces).
    A Frame passes through.  Anything else (wrong shape, dtype or device, odd size, row stride below W) raises
    ValueError naming what was expected."""
    return pixel_frame(frame, "NV12")


class FrameUploader:
    """Host frame -> device tensor with one async copy, of the host shape of `pixel_format` (frame_shape): HxWx3 u8
    BGR frames, or raw camera frames, which move fewer bytes (NV12, I420: half; YUY2: two thirds) or, for BGRX, a
    third more.  Page-locked sources (detected with cudaPointerGetAttributes) are copied
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
        """Shape of a host frame of size (width, height): (h, w, 3) for BGR, (3h/2, w) for NV12 and I420, (h, w, 2)
        for YUY2, (h, w, 4) for BGRX."""
        w, h = size
        return _FORMATS[pixel_format].shape(w, h)

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
        return pixel_frame(self.upload(f.y), self.pixel_format)


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
    capture_size as a tuple of two positive ints (even where pixel_format needs it: NV12 and I420 an even width and
    height, YUY2 an even width).  Anything else raises ValueError."""
    if capture_size is None:
        return tuple(int(v) for v in size)
    if not (isinstance(capture_size, (tuple, list)) and len(capture_size) == 2
            and all(np.isscalar(v) and int(v) == v and v > 0 for v in capture_size)):
        raise ValueError(f"capture_size must be (width, height) with positive integers, got {capture_size!r}")
    w, h = (int(v) for v in capture_size)
    try:
        _check_size(pixel_format, w, h)
    except ValueError as e:
        raise ValueError(f"capture_size: {e}") from None
    return w, h


class FrameResizer:
    """Device Frames of any size and format -> BGR Frames of one size (`size`, the tracking size): cv2.resize with the
    default INTER_LINEAR of the frame (of its cv2.cvtColor decode for the raw formats), bit for bit, one fm_frame_resize
    launch on the current stream into the next slot of a ring of `depth` device frames.

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
    """A caller's frame as a Frame, nothing copied.  A Frame passes through; otherwise `frame` is in pixel_format, in
    any form pixel_frame accepts ('BGR': an HxWx3 uint8 cuda tensor (contiguous) or host ndarray).  size: the (width,
    height) the frame must have; another size raises ValueError."""
    f = frame if isinstance(frame, Frame) else pixel_frame(frame, pixel_format)
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
