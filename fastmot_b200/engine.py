"""Conv-stack executors that take the place of the reference's TensorRT engines
(fastmot/utils/inference.py:39-125): `YoloEngine` runs a Darknet layer list, `OSNetEngine` the OSNet op list,
both on NHWC fp16 device tensors through the C-ABI layer kernels (csrc/nn.cu, csrc/conv_tc.cu).

The launch sequence of a network is recorded once (static shapes) and replayed per call; with `use_graph=True`
the replay is captured into a CUDA graph so a 170-layer detector costs one launch.
"""
import ctypes as C
import os

import numpy as np
import torch

from . import _lib
from .devmem import ptr, stream_ptr
from .models import darknet, osnet
from .models.yolo import check_heads

_ACT = darknet.ACTS
ACT_AFTER_RESIDUAL = 0x100
IN_C_PAD = 8      # network inputs are NHWC with 3 real + 5 zero channels: one 16-byte chunk per pixel


class _Launch:
    """A recorded C-ABI call: function + fully bound arguments."""
    __slots__ = ("fn", "args", "what")

    def __init__(self, fn, args, what):
        self.fn, self.args, self.what = fn, args, what

    def __call__(self, s):
        rc = self.fn(*self.args, s)
        if rc:
            _lib.check(rc, self.what)


class View:
    """One tensor a recorded launch reads or writes, as the kernel addresses it (metadata for tests and tools).
    Layouts: 'nhwc' fp16 [B][h][w][c_stride] (channels c_off .. c_off + c), 'nhwc4b' the fused stem's bordered NHWC4
    input [B][h + 8][w + 8][4], 'planar8' fp16 chunk-planar [B][c / 8][h][w][8] (fm_osb_streams tails), 'gap_part' fp32
    [B][strips][4][c] per-strip channel sums, 'f32' fp32 vectors [B][c]."""
    __slots__ = ("name", "t", "layout", "c", "h", "w", "c_stride", "c_off", "strips")

    def __init__(self, name, t, layout, c, h=1, w=1, c_stride=None, c_off=0, strips=None):
        self.name, self.t, self.layout, self.c, self.h, self.w = name, t, layout, c, h, w
        self.c_stride = c if c_stride is None else c_stride
        self.c_off, self.strips = c_off, strips

    def array(self, n):
        """The first n rows of the batch, shaped by the layout (a view into the buffer, not a copy)."""
        t, c, h, w = self.t.reshape(-1), self.c, self.h, self.w
        if self.layout == 'nhwc':
            return t[:n * h * w * self.c_stride].view(n, h, w, self.c_stride)[..., self.c_off:self.c_off + c]
        if self.layout == 'nhwc4b':
            return t[:n * (h + 8) * (w + 8) * 4].view(n, h + 8, w + 8, 4)
        if self.layout == 'planar8':
            return t[:n * h * w * c].view(n, c // 8, h, w, 8)
        if self.layout == 'gap_part':
            return t[:n * self.strips * 4 * c].view(n, self.strips, 4, c)
        if self.layout == 'f32':
            return t[:n * c].view(n, c)
        raise ValueError(self.layout)


class TraceEntry:
    """What one recorded launch computes: `kind` ('stem', 'S' = fm_osb_streams, 'G' = fm_osb_merge, 'conv', 'conv+add'
    = conv with the residual add + ReLU in its epilogue, 'gate4_pooled', or the op kind of models/osnet.py; for the
    detector 'conv', 'conv+shortcut', 'maxpool', 'upsample', 'copy', 'shortcut'), the indices of the ops (Darknet
    layers) it implements, the views it reads and writes, and kind-specific details in `info` (the conv path, the
    window a max-pool launches)."""
    __slots__ = ("kind", "ops", "ins", "outs", "info")

    def __init__(self, kind, ops, ins, outs, info=None):
        self.kind, self.ops, self.ins, self.outs = kind, tuple(ops), list(ins), list(outs)
        self.info = dict(info or {})


def _conv_desc(n, hi, wi, cin, cin_stride, cin_off, ho, wo, cout, cout_stride, cout_off, k, stride, pad, act, ws=None):
    d = _lib.FmConvDesc()
    if ws is not None:       # fp32 split-K scratch (a torch uint8 tensor owned by the caller)
        d.ws, d.ws_bytes = ws.data_ptr(), ws.numel()
    d.n, d.hi, d.wi, d.cin, d.cin_stride, d.cin_offset = n, hi, wi, cin, cin_stride, cin_off
    d.ho, d.wo, d.cout, d.cout_stride, d.cout_offset = ho, wo, cout, cout_stride, cout_off
    d.kh = d.kw = k
    d.stride, d.pad, d.act = stride, pad, act
    d.res_stride = d.res_offset = 0
    return d


class _Net:
    """Shared plumbing: recorded launches, optional CUDA-graph replay, conv dispatch (wgmma when supported)."""
    WS_BYTES = 32 << 20

    def __init__(self, use_tc=True, use_graph=False, ws=None):
        self._lib = _lib.require_device()
        self.use_tc = use_tc
        self.use_graph = use_graph
        self.launches = []
        self._graph = None
        self._keep = []
        self.n_tc = self.n_simt = self.n_tma = 0
        self.use_tma = os.environ.get("FM_CONV_TMA", "1") != "0"     # A/B switch: 0 = every conv through conv_tc.cu
        self.layer_bytes = 0        # algorithmic HBM bytes of the conv / depthwise layers (each tensor moved once)
        self.dev = torch.device("cuda")
        # split-K scratch of the wgmma conv: one per engine, so engines on different streams never share partials
        # (`ws` given: an engine that only ever runs on the same stream as its owner, one after the other)
        self.ws = ws if ws is not None else torch.empty(self.WS_BYTES, dtype=torch.uint8, device=self.dev)

    def _conv(self, desc, x, w, b, out, residual=None):
        """Records the conv on the path that supports it; returns that path: 'tma', 'tc' or 'simt'."""
        lib = self._lib
        desc.ws, desc.ws_bytes = self.ws.data_ptr(), self.ws.numel()
        self._keep.append(desc)
        self.layer_bytes += 2 * (desc.n * desc.hi * desc.wi * desc.cin + desc.n * desc.ho * desc.wo * desc.cout
                                 * (2 if residual is not None else 1) + desc.kh * desc.kw * desc.cin * desc.cout)
        if self.use_tc and self.use_tma and lib.fm_conv2d_tma_supported(C.byref(desc)):
            fn, path = lib.fm_conv2d_tma, 'tma'         # TMA-fed, cluster split-K (csrc/conv_tma.cu)
            self.n_tc += 1
            self.n_tma += 1
        elif self.use_tc and lib.fm_conv2d_tc_supported(C.byref(desc)):
            fn, path = lib.fm_conv2d_tc, 'tc'
            self.n_tc += 1
        else:
            fn, path = lib.fm_conv2d_simt, 'simt'
            self.n_simt += 1
        self.launches.append(_Launch(fn, (C.byref(desc), ptr(x), ptr(w), ptr(b), ptr(residual), ptr(out)), "conv"))
        return path

    def kernels_per_replay(self):
        extra = {'fm_channel_gate': 2, 'fm_channel_gate4': 2, 'fm_channel_gate4_pooled': 1, 'fm_osb_merge': 1}
        return sum(1 + extra.get(l.what, 0) for l in self.launches)

    def _add(self, fn_name, *args):
        self.launches.append(_Launch(getattr(self._lib, fn_name), args, fn_name))

    def warm(self, n=3):
        """Replays the recorded network n times (graph capture included) so the first timed call is steady state."""
        for _ in range(n):
            self.replay()
        torch.cuda.synchronize()

    def replay(self):
        _lib.count_graph_kernels(self.kernels_per_replay() if self.use_graph and self._graph is not None else 0)
        if self.use_graph:
            if self._graph is None:
                s = torch.cuda.Stream()
                s.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(s):
                    sp = stream_ptr()
                    for l in self.launches:      # warm-up outside capture
                        l(sp)
                torch.cuda.current_stream().wait_stream(s)
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    sp = stream_ptr()
                    for l in self.launches:
                        l(sp)
                self._graph = g
            self._graph.replay()
        else:
            sp = stream_ptr()
            for l in self.launches:
                l(sp)


class YoloEngine(_Net):
    """Darknet graph executor.  forward(inp NHWC8 fp16) -> list of head tensors [H, W, (5+C)*A] fp16.

    With batch = B > 1 every tensor gains a leading image dimension: the input is [B][H][W][8], the heads are
    [B][H][W][(5+C)*A], and every launch covers the B images (conv descriptors, pools, upsample and route copies get
    n = B; route buffers are [B][h][w][c]).  Each conv keeps the path the kernels' own `supported` checks pick at n = B.

    share = an engine of the same network at a larger batch (see `with_batch`): this engine allocates nothing on the
    device.  It runs on share's weights and split-K workspace, and its input, route and activation buffers are the
    first B images of share's.  The plan below is deterministic, so both engines allocate the same buffers in the same
    order and the i-th buffer of this engine is a prefix of share's i-th."""
    heads_nhwc = True

    def __init__(self, layers, input_hw, weights, use_tc=True, use_graph=False, batch=1, share=None):
        if share is not None and not (1 <= batch < share.batch):
            raise ValueError(f"a shared engine runs fewer images than its owner ({share.batch}), got batch {batch}")
        super().__init__(use_tc, use_graph, ws=None if share is None else share.ws)
        H, W = input_hw
        B = self.batch = batch
        self._src = (layers, tuple(input_hw))
        lead = () if B == 1 else (B,)        # batch 1 keeps the unbatched shapes
        self._bufs = []                      # the device buffers in allocation order (share's, when shared)

        def alloc(shape):
            if share is None:
                t = torch.zeros(lead + shape, dtype=torch.float16, device=self.dev)
                self._bufs.append(t)
                return t
            if len(self._bufs) >= len(share._bufs) or tuple(share._bufs[len(self._bufs)].shape[1:]) != shape:
                raise ValueError("the shared engine's buffer plan differs from its owner's")
            t = share._bufs[len(self._bufs)]
            self._bufs.append(t)
            return t[:B] if B > 1 else t[0]

        self.layers, self.shapes = darknet.infer_shapes(layers, 3, H, W)
        # (c, h, w) of each head per image, in the order forward() returns them
        self.head_shapes = [self.shapes[i] for i, l in enumerate(self.layers) if l['type'] == 'yolo']
        self.inp = alloc((H, W, IN_C_PAD))
        self.flops = darknet.count_flops(layers, 3, H, W) * B
        L = self.layers
        n = len(L)
        # ---- plan: which layers are written straight into a concat buffer ----
        home = {}       # layer -> (route index, channel offset)
        strided_ok = ('convolutional', 'maxpool', 'upsample')
        for i, l in enumerate(L):
            if l['type'] == 'route' and len(l['layers_abs']) > 1 and l.get('groups', 1) == 1:
                off = 0
                for s in l['layers_abs']:
                    if s not in home and L[s]['type'] in strided_ok:
                        home[s] = (i, off)
                    off += self.shapes[s][0]
        bufs = {}       # route index -> tensor

        def route_buf(i):
            if i not in bufs:
                c, h, w = self.shapes[i]
                bufs[i] = alloc((h, w, c))
            return bufs[i]

        self.views = []     # per layer: (tensor, c, c_stride, c_off, h, w)
        self.params = {}
        self.heads = []
        # shortcut layers (yolo2onnx.py:707-731) whose first operand is the convolution right before them and is read
        # by nothing else: the add moves into that conv's epilogue (residual after the activation), one launch less
        refs = {}
        for i, l in enumerate(L):
            if l['type'] == 'route':
                for s_ in l['layers_abs']:
                    refs.setdefault(s_, set()).add(i)
            elif l['type'] == 'shortcut':
                refs.setdefault(l['from_abs'], set()).add(i)
        self.fused_shortcuts = set()
        for i, l in enumerate(L[:-1]):
            nx = L[i + 1]
            if l['type'] == 'convolutional' and nx['type'] == 'shortcut' and i not in home and \
                    nx.get('activation', 'linear') == 'linear' and not refs.get(i) and nx['from_abs'] < i and \
                    self.shapes[nx['from_abs']] == self.shapes[i]:
                self.fused_shortcuts.add(i + 1)
        # self.trace[k] describes self.launches[k] (TraceEntry): the layers it implements, the views it reads and writes
        self.trace = []

        def vw(j, v=None):
            """The View of layer j's output (j = -1: the network input), or of the view tuple v named after j."""
            t_, c_, cs_, co_, h_, w_ = v if v is not None else (self.views[j] if j >= 0 else
                                                                (self.inp, IN_C_PAD, IN_C_PAD, 0, H, W))
            return View('input' if j < 0 else f"L{j}", t_, 'nhwc', c_, h_, w_, cs_, co_)

        spp_prev = {}
        for i, l in enumerate(L):
            t = l['type']
            c, h, w = self.shapes[i]
            if i in home:
                ri, off = home[i]
                out = (route_buf(ri), c, self.shapes[ri][0], off, h, w)
            elif t in ('convolutional', 'maxpool', 'upsample', 'shortcut') and i not in self.fused_shortcuts:
                out = (alloc((h, w, c)), c, c, 0, h, w)
            else:
                out = None
            src = self.views[i - 1] if i else (self.inp, IN_C_PAD, IN_C_PAD, 0, H, W)
            if t == 'convolutional':
                k = l['size']
                cin = src[1]
                if share is not None:
                    wd, bd = share.params[i]
                else:
                    wt, bs = weights[i]
                    if i == 0:   # physical input has IN_C_PAD channels (the extra ones are zero)
                        wt = np.concatenate([wt, np.zeros(wt.shape[:3] + (IN_C_PAD - wt.shape[3],), np.float32)], -1)
                    wd = torch.as_tensor(np.ascontiguousarray(wt)).to(self.dev).half().contiguous()
                    bd = torch.as_tensor(bs).to(self.dev).float().contiguous()
                self.params[i] = (wd, bd)
                pad = k // 2 if l.get('pad', 0) else 0
                d = _conv_desc(B, src[4], src[5], cin, src[2], src[3], h, w, c, out[2], out[3], k, l.get('stride', 1),
                               pad, _ACT[l.get('activation', 'linear')])
                if i + 1 in self.fused_shortcuts:
                    fr = L[i + 1]['from_abs']
                    b = self.views[fr]
                    d.res_stride, d.res_offset = b[2], b[3]
                    path = self._conv(d, src[0], wd, bd, out[0], residual=b[0])
                    self.trace.append(TraceEntry('conv+shortcut', (i, i + 1), [vw(i - 1), vw(fr)], [vw(i, out)],
                                                 {'path': path}))
                else:
                    path = self._conv(d, src[0], wd, bd, out[0])
                    self.trace.append(TraceEntry('conv', (i,), [vw(i - 1)], [vw(i, out)], {'path': path}))
            elif t == 'maxpool':
                ksz, psrc, pj = l['size'], src, i - 1
                key = (src[0].data_ptr(), src[1], src[2], src[3])
                if l['stride'] == 1 and ksz % 2 == 1:
                    # SPP (5 / 9 / 13 on the same tensor): a k x k stride-1 max over a k0 x k0 max is the
                    # (k + k0 - 1) window, so 9 = 5 o 5 and 13 = 5 o 9 -- each pool reads 25 taps instead of 81 / 169
                    prev = spp_prev.get(key)
                    if prev is not None and ksz > prev[0]:
                        ksz, psrc, pj = ksz - prev[0] + 1, prev[1], prev[2]
                    spp_prev[key] = (l['size'], out, i)
                self._add('fm_maxpool', ptr(psrc[0]), ptr(out[0]), B, psrc[4], psrc[5], psrc[1], psrc[2], psrc[3],
                          ksz, l['stride'], out[2], out[3])
                # ins[0] is the declared source; a composed SPP pool also reads the smaller pool's output
                self.trace.append(TraceEntry('maxpool', (i,), [vw(i - 1)] + ([vw(pj)] if pj != i - 1 else []),
                                             [vw(i, out)], {'size': l['size'], 'src': i - 1, 'stride': l['stride'],
                                                            'launch_size': ksz, 'launch_src': pj}))
            elif t == 'upsample':
                self._add('fm_upsample_copy', ptr(src[0]), ptr(out[0]), B, src[4], src[5], src[1], src[2], src[3],
                          l['stride'], out[2], out[3])
                self.trace.append(TraceEntry('upsample', (i,), [vw(i - 1)], [vw(i, out)], {'stride': l['stride']}))
            elif t == 'shortcut' and i in self.fused_shortcuts:
                out = self.views[i - 1]          # already holds conv + residual
            elif t == 'shortcut':
                a, b = self.views[i - 1], self.views[l['from_abs']]
                self._add('fm_add_act_strided', ptr(a[0]), a[2], a[3], ptr(b[0]), b[2], b[3], ptr(out[0]), out[2],
                          out[3], B * h * w, c, _ACT[l.get('activation', 'linear')])
                self.trace.append(TraceEntry('shortcut', (i,), [vw(i - 1), vw(l['from_abs'])], [vw(i, out)]))
            elif t == 'route':
                srcs = l['layers_abs']
                g = l.get('groups', 1)
                if len(srcs) == 1:
                    sv = self.views[srcs[0]]
                    cg = sv[1] // g
                    out = (sv[0], cg, sv[2], sv[3] + l.get('group_id', 0) * cg, sv[4], sv[5])
                else:
                    buf = route_buf(i)
                    off = 0
                    for s in srcs:
                        sv = self.views[s]
                        cs = sv[1] // g
                        if home.get(s, (None,))[0] != i:
                            self._add('fm_upsample_copy', ptr(sv[0]), ptr(buf), B, sv[4], sv[5], cs, sv[2],
                                      sv[3] + l.get('group_id', 0) * cs, 1, c, off)
                            self.trace.append(TraceEntry(
                                'copy', (i,), [vw(s, (sv[0], cs, sv[2], sv[3] + l.get('group_id', 0) * cs) + sv[4:])],
                                [vw(i, (buf, cs, c, off, h, w))], {'src': s}))
                        off += cs
                    out = (buf, c, c, 0, h, w)
            elif t == 'yolo':
                out = self.views[i - 1]
                assert out[2] == out[1] and out[3] == 0
                self.heads.append(out[0])
            self.views.append(out)
        if share is not None and len(self._bufs) != len(share._bufs):
            raise ValueError("the shared engine's buffer plan differs from its owner's")

    def with_batch(self, k, use_graph=None):
        """The engine of this network at batch k < self.batch that shares this engine's device weights, split-K
        workspace and buffers (the first k images of each): one more launch list (and graph), no activation memory.
        Each conv keeps the path its kernel picks at n = k.  It overwrites this engine's buffers, so the two must run
        one after the other on one stream."""
        layers, input_hw = self._src
        return YoloEngine(layers, input_hw, None, use_tc=self.use_tc,
                          use_graph=self.use_graph if use_graph is None else use_graph, batch=k, share=self)

    def forward(self, inp):
        if inp.data_ptr() != self.inp.data_ptr():
            self.inp.copy_(inp)
        self.replay()
        return self.heads


def build_yolo_engine(model, weights=None, use_tc=True, use_graph=True, head_obj_bias=-5.0, batch=1):
    """Engine for a `models.YOLO` descriptor (`batch` images per forward).  Without a Darknet .weights file the
    weights are synthetic (seeded He-normal, detection-prior objectness bias) — there are no trained weights offline."""
    if isinstance(model.CFG, str) and model.CFG in darknet.BUILDERS:
        layers = darknet.BUILDERS[model.CFG](num_classes=model.NUM_CLASSES,
                                             anchors_per_head=len(model.ANCHORS[0]) // 2)
    else:
        _, layers = darknet.parse_cfg(open(model.CFG).read())
    check_heads(model, darknet.head_shapes(layers, *model.INPUT_SHAPE[1:]))
    if weights is None:
        if model.WEIGHTS_PATH:
            weights = darknet.load_weights(model.WEIGHTS_PATH, layers, 3)
        else:
            # FM_SYNTH_OBJ_BIAS: objectness prior of the SYNTHETIC heads (how many random-weight candidates pass
            # conf_thresh); bench.py lowers it for the big-input models so the candidate count stays realistic
            # FM_SYNTH_HEAD_GAIN: scale of the synthetic head weights (logit variance on real frames)
            head_obj_bias = float(os.environ.get("FM_SYNTH_OBJ_BIAS", head_obj_bias))
            weights = darknet.synthetic_weights(layers, 3, head_obj_bias=head_obj_bias,
                                                num_classes=model.NUM_CLASSES,
                                                head_gain=float(os.environ.get("FM_SYNTH_HEAD_GAIN", 1.0)))
    return YoloEngine(layers, model.INPUT_SHAPE[1:], weights, use_tc=use_tc, use_graph=use_graph, batch=batch)


class LaunchGroup:
    """One launch of an OSNet engine: its trace `kind`, the range of `ops` it implements, the (c, h, w) `shape` its
    last op writes, and the kind-specific details its emitter needs in `info`."""
    __slots__ = ("kind", "ops", "shape", "info")

    def __init__(self, kind, ops, shape, info):
        self.kind, self.ops, self.shape, self.info = kind, ops, shape, info


def _reads(op):
    """The buffer names an OSNet op reads."""
    kind = op[0]
    if kind == 'conv':
        return [op[8]]
    if kind == 'dw':
        return [op[4]]
    if kind in ('maxpool3s2', 'avgpool2', 'gap'):
        return [op[1]]
    if kind == 'gate':
        return [op[3], op[4]]
    if kind == 'gate4':
        return list(op[3])
    if kind == 'add_relu':
        return [op[1], op[2]]
    if kind == 'fc':
        return [op[4]]
    return []


def _match_osblock(ops, k):
    """ops[k] = '<blk>.conv1'; returns (tail buffer names of the four streams, index of the gate4 op) when the next
    twenty ops are the Lite-3x3 chains a.0, b.0, b.1, c.0 .. d.3 feeding that gate, else None."""
    if k + 21 >= len(ops):
        return None
    x1 = ops[k][9]
    mid = ops[k][3]
    tails = []
    i = k + 1
    for s_ in range(4):
        prev = x1
        for j in range(s_ + 1):
            pw, dw = ops[i], ops[i + 1]
            if pw[0] != 'conv' or dw[0] != 'dw' or pw[2] != mid or pw[3] != mid or pw[4] != 1 or pw[7] != 'linear' \
                    or pw[8] != prev or dw[4] != pw[9] or dw[2] != mid or dw[3] != 'relu':
                return None
            prev = dw[5]
            i += 2
        tails.append(prev)
    g = ops[i]
    if g[0] != 'gate4' or tuple(g[3]) != tuple(tails):
        return None
    return tails, i


def _match_merge(ops, k):
    """ops[k] = gate4 of an OSBlock; returns (downsample conv or None, conv3, add_relu, index of add_relu) when
    the ops that follow are [downsample 1x1] conv3 1x1 (linear, reads the gate output) and add_relu."""
    acc = ops[k][4]
    i = k + 1
    ds = None
    if i < len(ops) and ops[i][0] == 'conv' and ops[i][8] != acc:      # a conv beside conv3: the downsample branch
        ds = ops[i]
        i += 1
    if i + 1 >= len(ops):
        return None
    c3, add = ops[i], ops[i + 1]
    if c3[0] != 'conv' or c3[4] != 1 or c3[7] != 'linear' or c3[8] != acc or add[0] != 'add_relu':
        return None
    if c3[9] not in (add[1], add[2]):
        return None
    other = add[2] if add[1] == c3[9] else add[1]
    if ds is not None and (ds[4] != 1 or ds[7] != 'linear' or ds[9] != other or ds[2] % 64):
        return None
    return ds, c3, add, i + 1


def plan_osnet(ops, input_hw, fuse_osb, lib):
    """The launches an OSNet op list becomes, in order: LaunchGroups whose op ranges cover every op exactly once.
    Every fusion decision of the engine is taken here, from the ops and their shapes alone (no device):
      'stem'          the 7x7/2 conv + 3x3/2 max-pool of a 256x128 input in one launch (fm_osnet_stem);
      'S'             an OSBlock's conv1 and its four Lite-3x3 streams (fm_osb_streams), which also writes the strip
                      sums of the tails; info: the tail names and the strip count;
      'G'             the gate4 over S's tails, [downsample,] conv3 and the residual add + ReLU (fm_osb_merge); info:
                      the downsample (or None), conv3 and add_relu ops and the output channels per CTA;
      'gate4_pooled'  a gate4 over S's tails that the merge kernel cannot take, reading S's strip sums;
      'conv+add'      a linear conv whose output feeds add_relu next: the add and ReLU run in the conv epilogue;
      and one group per remaining op, of that op's kind.
    `fuse_osb` False keeps one launch per op apart from conv+add.  `lib` answers which geometries the fused OSBlock
    kernels support (fm_osb_streams_strips, fm_osb_merge_ncta: host-only functions)."""
    shapes = osnet.infer_shapes(ops, *input_hw)
    groups, strips_of = [], {}      # strips_of: first tail name of an S group -> its strip count

    def group(kind, k, end, **info):
        groups.append(LaunchGroup(kind, tuple(range(k, end)), shapes[end - 1], info))
        return end

    k = 0
    if fuse_osb and tuple(input_hw) == (256, 128) and len(ops) > 1 and ops[0][0] == 'conv' \
            and ops[0][2:8] == (3, 64, 7, 2, 3, 'relu') and ops[1][0] == 'maxpool3s2' and ops[1][1] == ops[0][9]:
        k = group('stem', 0, 2)
    while k < len(ops):
        op = ops[k]
        nxt = ops[k + 1] if k + 1 < len(ops) else ('end',)
        if op[0] == 'conv':
            # kernel S computes conv1 as a 1x1, stride-1, unpadded conv: at its input's shape
            blk = _match_osblock(ops, k) if fuse_osb and op[4:8] == (1, 1, 0, 'relu') and op[2] % 64 == 0 else None
            strips = lib.fm_osb_streams_strips(shapes[k][1], shapes[k][2], op[3]) if blk else 0
            if strips > 0:
                strips_of[blk[0][0]] = strips
                k = group('S', k, blk[1], tails=blk[0], strips=strips)
            elif nxt[0] == 'add_relu' and nxt[1] == op[9] and nxt[2] != op[9] and op[7] == 'linear':
                k = group('conv+add', k, k + 2)
            else:
                k = group('conv', k, k + 1)
        elif op[0] == 'gate4' and op[3][0] in strips_of:
            m = _match_merge(ops, k)
            ncta = lib.fm_osb_merge_ncta(op[2], m[1][3]) if m else 0
            if ncta > 0:
                k = group('G', k, m[3] + 1, ds=m[0], c3=m[1], add=m[2], ncta=ncta)
            else:
                k = group('gate4_pooled', k, k + 1)
        else:
            k = group(op[0], k, k + 1)
    return groups


class OSNetEngine(_Net):
    """OSNet executor for up to `max_batch` crops per call: forward(x [n,256,128,8] fp16, n) -> [n, 512] f32
    L2-normalised embeddings (feature_extractor.py:62-74)."""

    def __init__(self, width, weights=None, input_hw=(256, 128), feature_dim=512, max_batch=256, use_tc=True,
                 use_graph=False, ops=None):
        """`ops` (+ `weights`): an op list in the vocabulary of models/osnet.py, e.g. from
        models.onnx_import.import_reid_onnx; default: the published OSNet of the given width."""
        super().__init__(use_tc, use_graph)
        # The ReID stack's stand-alone convs are thousands of tiles with 1-8 K slices each: the one-tile-per-CTA TMA
        # kernel pays its per-CTA set-up many times per SM there; it is the batch-1 detector layers it was written for.
        self.use_tma = False
        if ops is not None and weights is None:
            raise ValueError("a custom op list needs its weights")
        self.ops = list(ops) if ops is not None else osnet.build_osnet(width, feature_dim)
        self.weights = weights if weights is not None else osnet.synthetic_weights(self.ops)
        self.max_batch = max_batch
        self.feature_dim = feature_dim
        self.macs_per_crop = osnet.count_macs(self.ops, *input_hw)
        B, (H, W) = max_batch, input_hw
        dev = self.dev
        # FM_OSB_FUSED=0 falls back to one launch per layer (r01 path); default: fused stem (fm_osnet_stem), one
        # fm_osb_streams + fm_osb_merge pair per OSBlock (csrc/osnet_fused.cu, csrc/osnet_stem.cu)
        self.fuse_osb = os.environ.get("FM_OSB_FUSED", "1") != "0" and use_tc
        plan = plan_osnet(self.ops, (H, W), self.fuse_osb, self._lib)
        self.fuse_stem = plan[0].kind == 'stem'
        # network input: NHWC8 (layout 1 of fm_roi_resize_norm) or, for the fused stem, NHWC4 inside a zero border
        self.inp_layout = 2 if self.fuse_stem else 1
        if self.fuse_stem:
            self.inp = torch.zeros(B, H + 8, W + 8, 4, dtype=torch.float16, device=dev)
        else:
            self.inp = torch.zeros(B, H, W, IN_C_PAD, dtype=torch.float16, device=dev)
        self.out = torch.zeros(B, feature_dim, dtype=torch.float32, device=dev)
        self.pooled = torch.zeros(4 * B, 512, dtype=torch.float32, device=dev)
        self.gate_tmp = torch.zeros(4 * B, 512, dtype=torch.float32, device=dev)
        self._params = {}
        self._bufs = []     # every activation buffer must outlive the recorded launches (raw pointers!)
        self._free = {}     # (numel, dtype) -> released activation buffers, reused by the next _alloc of that size
        # name -> (tensor, channels, h, w) of the buffers a later launch still reads
        self._live = {'input': (self.inp, IN_C_PAD, H, W)}
        # name -> the View its last writer recorded; self.trace[i] describes self.launches[i] through these views
        self._views = {'input': View('input', self.inp, 'nhwc4b', 4, H, W) if self.fuse_stem
                       else View('input', self.inp, 'nhwc', IN_C_PAD, H, W)}
        self.trace = []
        self.n_osb = 0
        last = {name: k for k, op in enumerate(self.ops) for name in _reads(op)}
        for g in plan:
            # a group allocates its outputs before its inputs are released, so no launch writes into its own input
            defs = self._EMIT[g.kind](self, g)
            for k in g.ops:
                for name in _reads(self.ops[k]):
                    if last[name] == k and defs.get(name) is not self._live.get(name):   # not the in-place gate
                        self._release(name)
            for name, entry in defs.items():
                if self._live.get(name) is not entry:
                    self._release(name)     # the previous holder of a rebound name
                    self._live[name] = entry

    def _alloc(self, numel, dtype=torch.float16):
        free = self._free.get((numel, dtype))
        if free:
            return free.pop()
        t = torch.zeros(numel, dtype=dtype, device=self.dev)
        self._bufs.append(t)
        return t

    def _release(self, name):
        t = self._live.pop(name, None)
        if t is not None and name != 'input':
            self._free.setdefault((t[0].numel(), t[0].dtype), []).append(t[0])

    def _param(self, name):
        """The device copies of a layer's weights, uploaded once."""
        if name not in self._params:
            self._params[name] = tuple(torch.as_tensor(a).to(self.dev) for a in self.weights[name])
        return self._params[name]

    def _record(self, g, ins, outs):
        """Appends the trace entry of group g: the names of the views it reads, the Views it writes."""
        self.trace.append(TraceEntry(g.kind, g.ops, [self._views[name] for name in ins], outs))
        self._views.update((v.name, v) for v in outs)

    def _bind(self, g, ins, name, entry):
        """Records g as writing entry = (tensor, c, h, w) NHWC under name; returns the group's definitions."""
        self._record(g, ins, [View(name, entry[0], 'nhwc', *entry[1:])])
        return {name: entry}

    def _emit_stem(self, g):
        from .packing import pack_b_sw64
        w7, b7 = self.weights[self.ops[0][1]]                        # [64][7][7][3]
        wk = np.zeros((64, 7, 8, 4), np.float32)
        wk[:, :, 1:8, :3] = w7
        img = torch.as_tensor(pack_b_sw64(wk.reshape(64, 224))).to(self.dev)
        b_d = torch.as_tensor(np.ascontiguousarray(b7, np.float32)).to(self.dev)
        c, h, w = g.shape
        y = self._alloc(self.max_batch * c * h * w)
        self._keep += [img, b_d]
        self._add('fm_osnet_stem', ptr(self.inp), self.max_batch, ptr(img), ptr(b_d), ptr(y))
        self.n_tc += 1
        self.layer_bytes += 2 * (self.inp.numel() + y.numel())
        return self._bind(g, ['input'], self.ops[1][2], (y, c, h, w))

    def _emit_S(self, g):
        from .packing import pack_b_sw128
        k, B, dev = g.ops[0], self.max_batch, self.dev
        op = self.ops[k]
        x, xc, h, w = self._live[op[8]]
        mid, strips, names = op[3], g.info['strips'], g.info['tails']
        w1, b1 = self.weights[op[1]]
        w1_img = torch.as_tensor(pack_b_sw128(w1.reshape(mid, xc))).to(dev)
        b1_d = torch.as_tensor(np.ascontiguousarray(b1, np.float32)).to(dev)
        pw_imgs, dw_blobs = [], []
        for i in range(10):
            pw_op, dw_op = self.ops[k + 1 + 2 * i], self.ops[k + 2 + 2 * i]
            wp, bp = self.weights[pw_op[1]]
            wd, bd = self.weights[dw_op[1]]
            pw_imgs.append(pack_b_sw128(wp.reshape(mid, mid)))
            dw_blobs.append(np.concatenate([np.ascontiguousarray(wd, np.float32).astype(np.float16)
                                            .reshape(-1).view(np.uint8),
                                            np.ascontiguousarray(bp, np.float32).view(np.uint8),
                                            np.ascontiguousarray(bd, np.float32).view(np.uint8)]))
        pw_d = torch.as_tensor(np.concatenate(pw_imgs)).to(dev)
        dw_d = torch.as_tensor(np.concatenate(dw_blobs)).to(dev)
        tails = [self._alloc(B * h * w * mid) for _ in range(4)]
        gap = torch.zeros(B * strips * 4 * mid, dtype=torch.float32, device=dev)
        d = _lib.FmOsbStreams()
        d.x, d.n, d.h, d.w, d.cin, d.mid = x.data_ptr(), B, h, w, xc, mid
        d.w1, d.b1, d.pw, d.dw = w1_img.data_ptr(), b1_d.data_ptr(), pw_d.data_ptr(), dw_d.data_ptr()
        for i in range(4):
            d.tails[i] = tails[i].data_ptr()
        d.gap_part = gap.data_ptr()
        self._keep += [d, w1_img, b1_d, pw_d, dw_d, gap]
        self._add('fm_osb_streams', C.byref(d))
        self.n_tc += 1
        self.n_osb += 1
        self.layer_bytes += 2 * (B * h * w * (xc + 4 * mid))
        # the strip sums: read by the G or gate4_pooled launch that follows, under the first tail's name + '.gap'
        self._record(g, [op[8]], [View(tn, t, 'planar8', mid, h, w) for tn, t in zip(names, tails)]
                     + [View(names[0] + '.gap', gap, 'gap_part', mid, h, w, strips=strips)])
        return {tn: (t, mid, h, w) for tn, t in zip(names, tails)}

    def _emit_G(self, g):
        from .packing import pack_b_sw128
        B, dev = self.max_batch, self.dev
        _, name, c, srcs, acc = self.ops[g.ops[0]]
        ds_op, c3_op, add_op, ncta = g.info['ds'], g.info['c3'], g.info['add'], g.info['ncta']
        cout, h, w = g.shape
        gap = self._views[srcs[0] + '.gap']
        gw1, gb1, gw2, gb2 = self._param(name)
        w3, b3 = self.weights[c3_op[1]]
        wcat = w3.reshape(cout, c)
        bias = np.asarray(b3, np.float32).copy()
        ident_name = add_op[2] if add_op[1] == c3_op[9] else add_op[1]
        d = _lib.FmOsbMerge()
        if ds_op is not None:
            wdn, bdn = self.weights[ds_op[1]]
            cin = ds_op[2]
            wcat = np.concatenate([wdn.reshape(cout, cin), wcat], 1)
            bias += np.asarray(bdn, np.float32)
            d.x, d.res, d.cin = self._live[ds_op[8]][0].data_ptr(), None, cin
        else:
            d.x, d.res, d.cin = None, self._live[ident_name][0].data_ptr(), cout
        img = np.concatenate([pack_b_sw128(wcat[r:r + ncta]) for r in range(0, cout, ncta)])
        img_d = torch.as_tensor(img).to(dev)
        bias_d = torch.as_tensor(bias).to(dev)
        y = self._alloc(B * h * w * cout)
        d.n, d.hw, d.cout, d.mid, d.cr, d.strips = B, h * w, cout, c, gw1.shape[0], gap.strips
        for i in range(4):
            d.tails[i] = self._live[srcs[i]][0].data_ptr()
        d.gap_part = gap.t.data_ptr()
        d.gw1, d.gb1, d.gw2, d.gb2 = (t_.data_ptr() for t_ in (gw1, gb1, gw2, gb2))
        d.wimg, d.bias, d.out = img_d.data_ptr(), bias_d.data_ptr(), y.data_ptr()
        d.gate_scratch = self.gate_tmp.data_ptr()
        self._keep += [d, img_d, bias_d]
        self._add('fm_osb_merge', C.byref(d))
        self.n_tc += 1
        self.layer_bytes += 2 * (B * h * w * (4 * c + 2 * cout))
        return self._bind(g, list(srcs) + [gap.name, ds_op[8] if ds_op else ident_name], add_op[3], (y, cout, h, w))

    def _emit_conv(self, g):
        """'conv', and 'conv+add': relu(conv(x) + residual) with the residual and the activation in the epilogue."""
        _, name, cin, cout, ks, stride, pad, act, src, dst = self.ops[g.ops[0]]
        B = self.max_batch
        x, xc, h, w = self._live[src]
        _, ho, wo = g.shape
        wt, bs = self.weights[name]
        if xc != cin:  # stem: physical 4 channels
            wt = np.concatenate([wt, np.zeros(wt.shape[:3] + (xc - cin,), np.float32)], -1)
        wd = torch.as_tensor(np.ascontiguousarray(wt)).to(self.dev).half().contiguous()
        bd = torch.as_tensor(bs).to(self.dev).float().contiguous()
        self._params[name] = (wd, bd)
        y = self._alloc(B * ho * wo * cout)
        if g.kind == 'conv':
            self._conv(_conv_desc(B, h, w, xc, xc, 0, ho, wo, cout, cout, 0, ks, stride, pad, _ACT[act]), x, wd, bd, y)
            return self._bind(g, [src], dst, (y, cout, ho, wo))
        _, _, res, out = self.ops[g.ops[1]]
        d = _conv_desc(B, h, w, xc, xc, 0, ho, wo, cout, cout, 0, ks, stride, pad, _ACT['relu'] | ACT_AFTER_RESIDUAL)
        d.res_stride, d.res_offset = cout, 0
        self._conv(d, x, wd, bd, y, residual=self._live[res][0])
        return self._bind(g, [src, res], out, (y, cout, ho, wo))

    def _emit_dw(self, g):
        _, name, c, act, src, dst = self.ops[g.ops[0]]
        B = self.max_batch
        x, _, h, w = self._live[src]
        wd, bd = self._param(name)
        wd = wd.half().contiguous()
        self._params[name] = (wd, bd)
        y = self._alloc(B * h * w * c)
        self._add('fm_dwconv3', ptr(x), ptr(wd), ptr(bd), ptr(y), B, h, w, c, _ACT[act])
        self.layer_bytes += 2 * (2 * B * h * w * c + 9 * c)
        return self._bind(g, [src], dst, (y, c, h, w))

    def _emit_pool(self, g):
        """'maxpool3s2' and 'avgpool2'."""
        _, src, dst = self.ops[g.ops[0]]
        B = self.max_batch
        x, xc, h, w = self._live[src]
        _, ho, wo = g.shape
        y = self._alloc(B * ho * wo * xc)
        if g.kind == 'maxpool3s2':
            self._add('fm_maxpool_pad', ptr(x), ptr(y), B, h, w, xc, 3, 2, 1)
        else:
            self._add('fm_avgpool2', ptr(x), ptr(y), B, h, w, xc)
        return self._bind(g, [src], dst, (y, xc, ho, wo))

    def _emit_gate(self, g):
        """acc (+)= src * gate(src), in place into acc once the first gate of a chain has allocated it."""
        _, name, c, src, acc, accumulate = self.ops[g.ops[0]]
        B = self.max_batch
        x, _, h, w = self._live[src]
        w1, b1, w2, b2 = self._param(name)
        entry = self._live[acc] if acc in self._live else (self._alloc(B * h * w * c), c, h, w)
        self._add('fm_channel_gate', ptr(x), ptr(self.pooled), ptr(self.gate_tmp), ptr(w1), ptr(b1), ptr(w2),
                  ptr(b2), ptr(entry[0]), B, h * w, c, w1.shape[0], accumulate)
        return self._bind(g, [src, acc] if accumulate else [src], acc, entry)

    def _emit_gate4(self, g):
        """'gate4', and 'gate4_pooled': the channel sums come from the S launch that wrote the four streams."""
        _, name, c, srcs, acc = self.ops[g.ops[0]]
        B = self.max_batch
        xs = [ptr(self._live[s_][0]) for s_ in srcs]
        _, h, w = g.shape
        w1, b1, w2, b2 = self._param(name)
        a = self._alloc(B * h * w * c)
        if g.kind == 'gate4_pooled':
            gap = self._views[srcs[0] + '.gap']
            self._add('fm_channel_gate4_pooled', *xs, ptr(gap.t), gap.strips, ptr(self.gate_tmp), ptr(w1), ptr(b1),
                      ptr(w2), ptr(b2), ptr(a), B, h * w, c, w1.shape[0])
            return self._bind(g, list(srcs) + [gap.name], acc, (a, c, h, w))
        self._add('fm_channel_gate4', *xs, ptr(self.pooled), ptr(self.gate_tmp), ptr(w1), ptr(b1), ptr(w2), ptr(b2),
                  ptr(a), B, h * w, c, w1.shape[0])
        return self._bind(g, list(srcs), acc, (a, c, h, w))

    def _emit_add_relu(self, g):
        _, a_name, b_name, dst = self.ops[g.ops[0]]
        a, ac, h, w = self._live[a_name]
        n = self.max_batch * h * w * ac
        y = self._alloc(n)
        self._add('fm_add_act', ptr(a), ptr(self._live[b_name][0]), ptr(y), n, _ACT['relu'])
        return self._bind(g, [a_name, b_name], dst, (y, ac, h, w))

    def _emit_gap(self, g):
        _, src, dst = self.ops[g.ops[0]]
        x, xc, h, w = self._live[src]
        y = self._alloc(self.max_batch * xc, torch.float32)
        self._add('fm_global_avgpool', ptr(x), ptr(y), self.max_batch, h * w, xc)
        self._record(g, [src], [View(dst, y, 'f32', xc)])
        return {dst: (y, xc, 1, 1)}

    def _emit_fc(self, g):
        """Writes the embeddings into self.out, which no later launch reads: defines no buffer."""
        _, name, cin, cout, src, dst = self.ops[g.ops[0]]
        wd, bd = self._param(name)
        self._add('fm_fc_norm', ptr(self._live[src][0]), ptr(wd), ptr(bd), ptr(self.out), self.max_batch, cin, cout,
                  1, 1)
        self._record(g, [src], [View(dst, self.out, 'f32', cout)])
        return {}

    # group kind -> emitter: allocates the group's outputs, records its launch, trace entry and counters, and returns
    # {name: (tensor, c, h, w)} of the buffers it defines
    _EMIT = {'stem': _emit_stem, 'S': _emit_S, 'G': _emit_G, 'conv': _emit_conv, 'conv+add': _emit_conv,
             'dw': _emit_dw, 'maxpool3s2': _emit_pool, 'avgpool2': _emit_pool, 'gate': _emit_gate,
             'gate4': _emit_gate4, 'gate4_pooled': _emit_gate4, 'add_relu': _emit_add_relu, 'gap': _emit_gap,
             'fc': _emit_fc}

    def load_nhwc8(self, x):
        """Copies crops given as [n][256][128][>= 3] fp16 (RGB first) into the engine's input buffer, whatever its
        layout (tests and tools; the product path writes the buffer with fm_roi_resize_norm)."""
        n = x.shape[0]
        if self.inp_layout == 2:
            self.inp[:n, 4:-4, 4:-4, :3].copy_(x[..., :3])
        else:
            self.inp[:n].copy_(x)

    def forward(self, n=None):
        """Runs the recorded network on self.inp (all max_batch rows; rows >= n are don't-care)."""
        self.replay()
        return self.out if n is None else self.out[:n]


def build_reid_engine(model, max_batch=256, use_tc=True, use_graph=True):
    """Engine for a `models.ReID` descriptor.  `MODEL_PATH` (an ONNX file, the reference's reid.py:20-23) is lowered
    by models.onnx_import; without it the descriptor's `ARCH` selects the built-in OSNet with synthetic weights."""
    if getattr(model, 'MODEL_PATH', None) is not None:
        from .models.onnx_import import import_reid_onnx
        ops, weights, in_shape, dim = import_reid_onnx(str(model.MODEL_PATH))
        if tuple(in_shape) != tuple(model.INPUT_SHAPE):
            raise ValueError(f"{model.__name__}: ONNX input {in_shape} != INPUT_SHAPE {model.INPUT_SHAPE}")   # reid.py:66
        if dim != model.OUTPUT_LAYOUT:
            raise ValueError(f"{model.__name__}: ONNX feature dim {dim} != OUTPUT_LAYOUT {model.OUTPUT_LAYOUT}")
        return OSNetEngine(None, weights=weights, input_hw=in_shape[1:], feature_dim=dim, max_batch=max_batch,
                           use_tc=use_tc, use_graph=use_graph, ops=ops)
    arch, width = model.ARCH
    assert arch == 'osnet'
    return OSNetEngine(width, input_hw=model.INPUT_SHAPE[1:], feature_dim=model.OUTPUT_LAYOUT, max_batch=max_batch,
                       use_tc=use_tc, use_graph=use_graph)


# ------------------------------------------------------------------------------------------------ stage profiling
class _Profiler:
    """CUDA-event timers around the conv stacks (recorded on the stream each stack is launched on)."""

    def __init__(self):
        self.reset()

    def reset(self):
        self.records = []

    def add(self, kind, e0, e1, flops, path, nbytes=0.0):
        self.records.append((kind, e0, e1, flops, path, nbytes))

    def summary(self):
        torch.cuda.synchronize()
        out = {"yolo_ms": 0.0, "osnet_ms": 0.0, "yolo_flops": 0.0, "osnet_flops": 0.0, "yolo_bytes": 0.0,
               "osnet_bytes": 0.0, "yolo_calls": 0, "osnet_calls": 0, "detector_frames": 0}
        path = set()
        for kind, e0, e1, flops, p, nbytes in self.records:
            out[kind + "_ms"] += e0.elapsed_time(e1)
            out[kind + "_flops"] += flops
            out[kind + "_bytes"] += nbytes
            out[kind + "_calls"] += 1
            out["detector_frames"] += kind == "yolo"
            path.add(p)
        out["conv_path"] = "+".join(sorted(path)) if path else None
        return out


_PROF = None


def enable_profiling():
    global _PROF
    _PROF = _Profiler()
    return _PROF


def _profiled(kind):
    def deco(fn):
        def wrapper(self, *a, **k):
            if _PROF is None:
                return fn(self, *a, **k)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            r = fn(self, *a, **k)
            e1.record()
            if kind == "yolo":
                flops = float(self.flops)
            else:
                n = a[0] if a and a[0] is not None else self.max_batch
                flops = 2.0 * self.macs_per_crop * n
            path = "wgmma" if self.n_tc >= self.n_simt else "simt"
            _PROF.add(kind, e0, e1, flops, f"{kind}:{path}({self.n_tc}tc/{self.n_simt}simt)", float(self.layer_bytes))
            return r
        return wrapper
    return deco


YoloEngine.forward = _profiled("yolo")(YoloEngine.forward)
OSNetEngine.forward = _profiled("osnet")(OSNetEngine.forward)
