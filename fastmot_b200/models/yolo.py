"""YOLO model descriptors: same class-attribute "plugin" API and auto-registry as fastmot/models/yolo.py:11-58
(subclass -> registered by name -> selected by the `model` string of the config).  TensorRT engine paths are
replaced by a Darknet-cfg graph description consumed by fastmot_b200.engine (no TensorRT here).

Descriptor values (NUM_CLASSES, LETTERBOX, NEW_COORDS, INPUT_SHAPE, LAYER_FACTORS, SCALES, ANCHORS) follow
fastmot/models/yolo.py:154-299, with one deviation: YOLOv3 and YOLOv3SPP get a third SCALES entry (see YOLOv3).
"""


class YOLO:
    __registry = {}

    CFG = None            # callable returning Darknet cfg text (fastmot_b200/models/darknet_cfgs.py)
    WEIGHTS_PATH = None   # optional Darknet .weights; None -> seeded synthetic weights
    NUM_CLASSES = None
    LETTERBOX = False
    NEW_COORDS = False
    INPUT_SHAPE = None
    LAYER_FACTORS = None
    SCALES = None
    ANCHORS = None

    def __init_subclass__(cls, **kwargs):
        super().__init_subclass__(**kwargs)
        cls.__registry[cls.__name__] = cls

    @classmethod
    def get_model(cls, name):
        return cls.__registry[name]


MAX_ANCHORS = 6     # FM_MAX_ANCHORS (include/fastmot_b200.h): the anchors one head decode holds


def check_heads(model, head_shapes=None):
    """Raises ValueError naming the model unless its head table describes its heads: LAYER_FACTORS, ANCHORS and SCALES
    have one entry per head (per [yolo] layer of the graph when head_shapes, the graph's [(c, h, w)] of each head in
    graph order, is given), no head has more than MAX_ANCHORS anchors, and each graph head has the grid
    INPUT_SHAPE // factor and (5 + NUM_CLASSES) * anchors channels.  A table that disagrees with the graph would
    otherwise drop heads or decode them with the wrong grid."""
    name = model.__name__
    n = len(model.LAYER_FACTORS) if head_shapes is None else len(head_shapes)
    for what in ('LAYER_FACTORS', 'ANCHORS', 'SCALES'):
        if len(getattr(model, what)) != n:
            raise ValueError(f"{name}: {what} has {len(getattr(model, what))} entries for "
                             f"{n} {'[yolo] layers in the graph' if head_shapes is not None else 'LAYER_FACTORS'}")
    _, in_h, in_w = model.INPUT_SHAPE
    for i, (factor, anchors) in enumerate(zip(model.LAYER_FACTORS, model.ANCHORS)):
        na = len(anchors) // 2
        if len(anchors) % 2 or not 1 <= na <= MAX_ANCHORS:
            raise ValueError(f"{name}: head {i} lists {len(anchors)} anchor values; a head takes 1 to {MAX_ANCHORS} "
                             "(w, h) pairs")
        if head_shapes is None:
            continue
        c, h, w = head_shapes[i]
        if (h, w) != (in_h // factor, in_w // factor):
            raise ValueError(f"{name}: head {i} has a {h}x{w} grid in the graph, but INPUT_SHAPE {model.INPUT_SHAPE} "
                             f"// LAYER_FACTORS[{i}] = {factor} gives {in_h // factor}x{in_w // factor}")
        if c != (5 + model.NUM_CLASSES) * na:
            raise ValueError(f"{name}: head {i} has {c} channels in the graph, but (5 + NUM_CLASSES) * anchors = "
                             f"{(5 + model.NUM_CLASSES) * na}")


class YOLOv4(YOLO):
    CFG = 'yolov4'
    NUM_CLASSES = 2
    INPUT_SHAPE = (3, 512, 512)
    LAYER_FACTORS = [8, 16, 32]
    SCALES = [1.2, 1.1, 1.05]
    ANCHORS = [[11, 22, 24, 60, 37, 116],
               [54, 186, 69, 268, 89, 369],
               [126, 491, 194, 314, 278, 520]]


class YOLOv4CSP(YOLO):
    CFG = 'yolov4-csp'
    NUM_CLASSES = 1
    LETTERBOX = True
    NEW_COORDS = True
    INPUT_SHAPE = (3, 640, 640)
    LAYER_FACTORS = [8, 16, 32]
    SCALES = [2.0, 2.0, 2.0]
    ANCHORS = [[12, 16, 19, 36, 40, 28],
               [36, 75, 76, 55, 72, 146],
               [142, 110, 192, 243, 459, 401]]


class YOLOv4P5(YOLO):
    CFG = 'yolov4-p5'
    NUM_CLASSES = 1
    LETTERBOX = True
    NEW_COORDS = True
    INPUT_SHAPE = (3, 896, 896)
    LAYER_FACTORS = [8, 16, 32]
    SCALES = [2.0, 2.0, 2.0]
    ANCHORS = [[13, 17, 31, 25, 24, 51, 61, 45],
               [48, 102, 119, 96, 97, 189, 217, 184],
               [171, 384, 324, 451, 616, 618, 800, 800]]


class YOLOv4P5_1280(YOLOv4P5):
    """BASELINE.json config 4 quotes 'YOLOv4-p5 1280x'; same graph at a 1280 input (SURVEY.md §8)."""
    INPUT_SHAPE = (3, 1280, 1280)


class YOLOv4Tiny(YOLO):
    CFG = 'yolov4-tiny'
    NUM_CLASSES = 1
    INPUT_SHAPE = (3, 416, 416)
    LAYER_FACTORS = [32, 16]
    SCALES = [1.05, 1.05]
    ANCHORS = [[81, 82, 135, 169, 344, 319],
               [23, 27, 37, 58, 81, 82]]


class YOLOv4xMish(YOLO):
    CFG = 'yolov4x-mish'
    NUM_CLASSES = 1
    LETTERBOX = True
    NEW_COORDS = True
    INPUT_SHAPE = (3, 640, 640)
    LAYER_FACTORS = [8, 16, 32]
    SCALES = [2.0, 2.0, 2.0]
    ANCHORS = [[12, 16, 19, 36, 40, 28],
               [36, 75, 76, 55, 72, 146],
               [142, 110, 192, 243, 459, 401]]


class YOLOv4CSPSwish(YOLO):
    CFG = 'yolov4-csp-swish'
    NUM_CLASSES = 1
    LETTERBOX = True
    NEW_COORDS = True
    INPUT_SHAPE = (3, 640, 640)
    LAYER_FACTORS = [8, 16, 32]
    SCALES = [2.0, 2.0, 2.0]
    ANCHORS = [[12, 16, 19, 36, 40, 28],
               [36, 75, 76, 55, 72, 146],
               [142, 110, 192, 243, 459, 401]]


class YOLOv4CSPxSwish(YOLO):
    CFG = 'yolov4-csp-x-swish'
    NUM_CLASSES = 1
    LETTERBOX = True
    NEW_COORDS = True
    INPUT_SHAPE = (3, 640, 640)
    LAYER_FACTORS = [8, 16, 32]
    SCALES = [2.0, 2.0, 2.0]
    ANCHORS = [[12, 16, 19, 36, 40, 28],
               [36, 75, 76, 55, 72, 146],
               [142, 110, 192, 243, 459, 401]]


class YOLOv4P6(YOLO):
    CFG = 'yolov4-p6'
    NUM_CLASSES = 1
    LETTERBOX = True
    NEW_COORDS = True
    INPUT_SHAPE = (3, 1280, 1280)
    LAYER_FACTORS = [8, 16, 32, 64]
    SCALES = [2.0, 2.0, 2.0, 2.0]
    ANCHORS = [[13, 17, 31, 25, 24, 51, 61, 45],
               [61, 45, 48, 102, 119, 96, 97, 189],
               [97, 189, 217, 184, 171, 384, 324, 451],
               [324, 451, 545, 357, 616, 618, 1024, 1024]]


class YOLOv3(YOLO):
    """The reference lists two SCALES for three heads (yolo.py:273), which its own add_plugin rejects
    (yolo.py:70); the third head takes Darknet's default scale_x_y = 1.0."""
    CFG = 'yolov3'
    NUM_CLASSES = 1
    INPUT_SHAPE = (3, 416, 416)
    LAYER_FACTORS = [32, 16, 8]
    SCALES = [1.0, 1.0, 1.0]
    ANCHORS = [[116, 90, 156, 198, 373, 326],
               [30, 61, 62, 45, 59, 119],
               [10, 13, 16, 30, 33, 23]]


class YOLOv3SPP(YOLO):
    """Third SCALES entry added as for YOLOv3 (the reference lists two, yolo.py:285)."""
    CFG = 'yolov3-spp'
    NUM_CLASSES = 1
    INPUT_SHAPE = (3, 608, 608)
    LAYER_FACTORS = [32, 16, 8]
    SCALES = [1.0, 1.0, 1.0]
    ANCHORS = [[116, 90, 156, 198, 373, 326],
               [30, 61, 62, 45, 59, 119],
               [10, 13, 16, 30, 33, 23]]


class YOLOv3Tiny(YOLO):
    CFG = 'yolov3-tiny'
    NUM_CLASSES = 1
    INPUT_SHAPE = (3, 416, 416)
    LAYER_FACTORS = [32, 16]
    SCALES = [1.0, 1.0]
    ANCHORS = [[81, 82, 135, 169, 344, 319],
               [10, 14, 23, 27, 37, 58]]
