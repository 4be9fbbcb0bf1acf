// YOLO detector post-processing on the device: head decode fused with score threshold + compaction,
// (class, objectness) sort, per-class DIoU-NMS with a bit-mask, final box rounding and area/aspect filters.
//
// Reference: fastmot/plugins/yolo_layer.cu:127-230 (CalDetection, CalDetection_NewCoords),
//            fastmot/detector.py:322-365 (_filter_dets), fastmot/utils/rect.py:198-244 (diou_nms),
//            rect.py:48-57 (to_tlbr), :21-32 (aspect_ratio, area).
// The reference copies all K0 decoded candidates to the host and filters there; here only the D survivors
// (48 B each) leave the device.
//
// Every kernel handles a batch of images: image b owns its own segment of each buffer (heads + b * head_stride,
// dense rows + b * cand_stride, keys + b * key_cap, counter[b], mask + b * key_cap * words, outputs + b * max_out,
// out_count[b], status[b]) and the grid carries b.  The one-image entries launch the same kernels with one image, so
// a batched image's keys, rows and detections are those of the one-image path on the same head slice, and NMS never
// compares boxes of different images.  The batched decode (fm_yolo_decode_filter_geom) reads each image's pixel scale
// and letterbox offset from a device FmFrameGeom table, so the images of one batch may come from frames of any sizes.
#include "common.cuh"
#include "../../include/fastmot_b200.h"

int fm_launch_nms_scan(int batch, const unsigned long long* keys, const float* dense, int cand_stride,
                       const int* counter, int key_cap, const unsigned long long* mask, int words, double max_area,
                       double min_ar, int max_out, double* out_tlbr, long long* out_label, double* out_conf,
                       int* out_count, int* status, cudaStream_t s);

namespace {

__device__ __forceinline__ float sigmoidf_fast(float x) { return 1.0f / (1.0f + __expf(-x)); }

// One thread per (anchor, cell); blockIdx.y = image.  Input NCHW-style head tensor [(5+C)*A, H, W] in fp32 or fp16.
template <typename T>
__global__ void yolo_decode_filter_kernel(const T* __restrict__ in, long long head_stride, int cand_stride,
                                          int yolo_w, int yolo_h, int num_anchors,
                                          FmYoloHead head, int num_classes, int input_w, int input_h, int new_coords,
                                          int nhwc,
                                          int cand_base, const unsigned char* __restrict__ label_mask,
                                          double conf_thresh, float size_w, float size_h, float off_x, float off_y,
                                          const FmFrameGeom* __restrict__ geom, float* __restrict__ dense, unsigned long long* __restrict__ keys,
                                          int* __restrict__ counter, int key_cap) {
    const int total = yolo_w * yolo_h;
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total * num_anchors) return;
    const int img = blockIdx.y;
    in += img * head_stride;
    dense += (size_t)img * cand_stride * 8;
    keys += (size_t)img * key_cap;
    counter += img;
    const int info_len = 5 + num_classes;
    const int anchor = idx / total, cell = idx - anchor * total;
    // planar [(5+C)*A, H, W] (the TensorRT plugin's input) or channels-last [H, W, (5+C)*A] (our conv engine)
    const size_t as = nhwc ? 1 : (size_t)total;
    const T* cur = nhwc ? in + (size_t)cell * info_len * num_anchors + (size_t)anchor * info_len
                        : in + (size_t)anchor * info_len * total + cell;
    int class_id = 0;
    float best = -INFINITY;
    for (int i = 5; i < info_len; ++i) {
        float l = (float)cur[(size_t)i * as];
        if (l > best) { best = l; class_id = i - 5; }
    }
    const float t0 = (float)cur[0], t1 = (float)cur[as], t2 = (float)cur[2 * as], t3 = (float)cur[3 * as],
                t4 = (float)cur[4 * as];
    const int row = cell / yolo_w, col = cell - row * yolo_w;
    const float s = head.scale_x_y;
    float cls_prob, box_prob, bx, by, bw, bh;
    // explicit _rn intrinsics: no FMA contraction, so the fp32 results equal the numpy oracle bit for bit
    const float half_sm1 = __fmul_rn(s - 1.0f, 0.5f);
    float ex, ey;
    if (new_coords) {
        cls_prob = best;
        box_prob = t4;
        ex = t0; ey = t1;
        bw = __fdiv_rn(__fmul_rn(__fmul_rn(__fmul_rn(t2, t2), 4.0f), head.anchors[2 * anchor]), (float)input_w);
        bh = __fdiv_rn(__fmul_rn(__fmul_rn(__fmul_rn(t3, t3), 4.0f), head.anchors[2 * anchor + 1]), (float)input_h);
    } else {
        cls_prob = sigmoidf_fast(best);
        box_prob = sigmoidf_fast(t4);
        ex = sigmoidf_fast(t0); ey = sigmoidf_fast(t1);
        bw = __fdiv_rn(__fmul_rn(__expf(t2), head.anchors[2 * anchor]), (float)input_w);
        bh = __fdiv_rn(__fmul_rn(__expf(t3), head.anchors[2 * anchor + 1]), (float)input_h);
    }
    bx = __fdiv_rn(__fadd_rn((float)col, __fsub_rn(__fmul_rn(s, ex), half_sm1)), (float)yolo_w);
    by = __fdiv_rn(__fadd_rn((float)row, __fsub_rn(__fmul_rn(s, ey), half_sm1)), (float)yolo_h);
    bx = __fsub_rn(bx, __fdiv_rn(bw, 2.0f));
    by = __fsub_rn(by, __fdiv_rn(bh, 2.0f));
    // detector.py:331-336: class mask and score threshold
    if (!label_mask[class_id]) return;
    const float score = __fmul_rn(box_prob, cls_prob);
    if (!((double)score >= conf_thresh)) return;
    // detector.py:339-341: scale to pixels (f32 <- f64 product), subtract letterbox offset.  The f64 product of two
    // floats is exact, so its f32 rounding is __fmul_rn; likewise the f32 rounding of the f64 difference is __fsub_rn.
    // Written as f64 casts the compiler lowered both to plain mul.f32 / sub.f32, which ptxas contracted into one FFMA:
    // the product was never rounded and py differed from the reference by up to half an ulp of by * size_h.
    if (geom != nullptr) {
        const FmFrameGeom& g = geom[img];
        size_w = g.size_w; size_h = g.size_h; off_x = g.off_x; off_y = g.off_y;
    }
    const float px = __fsub_rn(__fmul_rn(bx, size_w), off_x);
    const float py = __fsub_rn(__fmul_rn(by, size_h), off_y);
    const float pw = __fmul_rn(bw, size_w);
    const float ph = __fmul_rn(bh, size_h);
    const int gidx = cand_base + idx;
    float* d = dense + (size_t)gidx * 8;
    d[0] = px; d[1] = py; d[2] = pw; d[3] = ph; d[4] = box_prob; d[5] = (float)class_id; d[6] = cls_prob;
    const int slot = atomicAdd(counter, 1);
    if (slot < key_cap) {
        // ascending u64 order == class asc, objectness desc, candidate index asc
        unsigned int sb = ~__float_as_uint(box_prob);   // objectness is >= 0
        keys[slot] = ((unsigned long long)(unsigned)class_id << 56) | ((unsigned long long)sb << 24) |
                     (unsigned long long)(gidx & 0xffffff);
    }
}

// Bitonic sort of up to 16384 keys in shared memory, one CTA per image.
__global__ void __launch_bounds__(1024) sort_keys_kernel(unsigned long long* __restrict__ keys,
                                                          const int* __restrict__ counter, int key_cap,
                                                          int* __restrict__ status) {
    extern __shared__ unsigned long long sk[];
    keys += (size_t)blockIdx.x * key_cap;
    counter += blockIdx.x;
    status += blockIdx.x;
    int n = *counter;
    if (n > key_cap) {
        if (threadIdx.x == 0) status[0] = 1;   // overflow: host raises
        n = key_cap;
    }
    if (n <= 1) return;
    int np2 = 1;
    while (np2 < n) np2 <<= 1;
    for (int i = threadIdx.x; i < np2; i += blockDim.x) sk[i] = i < n ? keys[i] : ~0ull;
    __syncthreads();
    for (int k = 2; k <= np2; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int t = threadIdx.x; t < (np2 >> 1); t += blockDim.x) {
                int lo = ((t & ~(j - 1)) << 1) | (t & (j - 1));
                int hi = lo | j;
                bool asc = (lo & k) == 0;
                unsigned long long a = sk[lo], b = sk[hi];
                if ((a > b) == asc) { sk[lo] = b; sk[hi] = a; }
            }
            __syncthreads();
        }
    }
    for (int i = threadIdx.x; i < n; i += blockDim.x) keys[i] = sk[i];
}

// rect.py:198-244 in fp64 on fp32-valued inputs (Numba promotes `tl + wh - 1` with an int literal to f64).
__device__ __forceinline__ bool diou_suppresses(const float* a, const float* b, double thresh) {
    const double ax = a[0], ay = a[1], bx = b[0], by = b[1];
    const double abx = (double)(a[0] + a[2]) - 1.0, aby = (double)(a[1] + a[3]) - 1.0;
    const double bbx = (double)(b[0] + b[2]) - 1.0, bby = (double)(b[1] + b[3]) - 1.0;
    const double iw = fmax(0.0, fmin(abx, bbx) - fmax(ax, bx) + 1.0);
    const double ih = fmax(0.0, fmin(aby, bby) - fmax(ay, by) + 1.0);
    const double inter = iw * ih;
    const double area_a = (double)(a[2] * a[3]), area_b = (double)(b[2] * b[3]);
    const double iou = inter / ((double)(float)(area_a + area_b) - inter);
    if (!(iou > thresh)) return false;  // DIoU <= IoU
    const double ew = fmax(abx, bbx) - fmin(ax, bx) + 1.0, eh = fmax(aby, bby) - fmin(ay, by) + 1.0;
    const double c = ew * ew + eh * eh;
    const double dx = (ax + abx) / 2 - (bx + bbx) / 2, dy = (ay + aby) / 2 - (by + bby) / 2;
    const double d = dx * dx + dy * dy;
    return iou - pow(d / c, 0.6) > thresh;
}

// mask[i][w] bit b set  <=>  sorted candidate j = 64 w + b (j > i, same class) is suppressed by i.  blockIdx.y = image.
__global__ void __launch_bounds__(64) nms_mask_kernel(const unsigned long long* __restrict__ keys,
                                                       const float* __restrict__ dense, int cand_stride,
                                                       const int* __restrict__ counter, int key_cap, double thresh,
                                                       unsigned long long* __restrict__ mask, int mask_words) {
    __shared__ float sb[64][4];
    __shared__ int scls[64];
    const int img = blockIdx.y;
    keys += (size_t)img * key_cap;
    dense += (size_t)img * cand_stride * 8;
    counter += img;
    mask += (size_t)img * key_cap * mask_words;
    int n = min(*counter, key_cap);
    const int nb = (n + 63) >> 6;
    const int ntiles = nb * nb;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int rb = tile / nb, cb = tile - rb * nb;
        if (cb < rb) continue;  // only j > i matters
        __syncthreads();
        const int j = cb * 64 + threadIdx.x;
        if (j < n) {
            unsigned long long kj = keys[j];
            const float* d = dense + (size_t)(kj & 0xffffff) * 8;
            sb[threadIdx.x][0] = d[0]; sb[threadIdx.x][1] = d[1]; sb[threadIdx.x][2] = d[2]; sb[threadIdx.x][3] = d[3];
            scls[threadIdx.x] = (int)(kj >> 56);
        }
        __syncthreads();
        const int i = rb * 64 + threadIdx.x;
        if (i < n) {
            unsigned long long ki = keys[i];
            const float* a = dense + (size_t)(ki & 0xffffff) * 8;
            float av[4] = {a[0], a[1], a[2], a[3]};
            const int ci = (int)(ki >> 56);
            unsigned long long bits = 0;
            const int jn = min(64, n - cb * 64);
            for (int b = 0; b < jn; ++b) {
                int jj = cb * 64 + b;
                if (jj > i && scls[b] == ci && diou_suppresses(av, sb[b], thresh)) bits |= 1ull << b;
            }
            mask[(size_t)i * mask_words + cb] = bits;
        }
    }
}

}  // namespace

static int launch_decode(const void* head_out, int batch, long long head_stride, int cand_stride, int is_fp16, int nhwc,
                         int yolo_w, int yolo_h, int num_anchors, const FmYoloHead& head, int num_classes, int input_w,
                         int input_h, int new_coords, int cand_base, const unsigned char* label_mask,
                         double conf_thresh, float size_w, float size_h, float off_x, float off_y,
                         const FmFrameGeom* geom, float* dense, unsigned long long* keys, int* counter, int key_cap,
                         void* stream, const char* what) {
    int total = yolo_w * yolo_h * num_anchors;
    if (total <= 0) return FM_OK;
    dim3 grid(fm_cdiv(total, 128), batch);
    if (is_fp16)
        yolo_decode_filter_kernel<__half><<<grid, 128, 0, (cudaStream_t)stream>>>(
            (const __half*)head_out, head_stride, cand_stride, yolo_w, yolo_h, num_anchors, head, num_classes, input_w,
            input_h, new_coords, nhwc, cand_base, label_mask, conf_thresh, size_w, size_h, off_x, off_y, geom, dense,
            keys, counter, key_cap);
    else
        yolo_decode_filter_kernel<float><<<grid, 128, 0, (cudaStream_t)stream>>>(
            (const float*)head_out, head_stride, cand_stride, yolo_w, yolo_h, num_anchors, head, num_classes, input_w,
            input_h, new_coords, nhwc, cand_base, label_mask, conf_thresh, size_w, size_h, off_x, off_y, geom, dense,
            keys, counter, key_cap);
    FM_CHECK_LAUNCH(what);
    return FM_OK;
}

extern "C" int fm_yolo_decode_filter(const void* head_out, int is_fp16, int nhwc, int yolo_w, int yolo_h, int num_anchors,
                                     const FmYoloHead* head, int num_classes, int input_w, int input_h,
                                     int new_coords, int cand_base, const unsigned char* label_mask,
                                     double conf_thresh, float size_w, float size_h, float off_x, float off_y,
                                     float* dense, unsigned long long* keys, int* counter, int key_cap, void* stream) {
    FM_REQUIRE(head != nullptr, "fm_yolo_decode_filter: head is NULL");
    FM_REQUIRE(num_anchors <= FM_MAX_ANCHORS, "fm_yolo_decode_filter: too many anchors");
    FM_REQUIRE(cand_base + yolo_w * yolo_h * num_anchors <= (1 << 24), "fm_yolo_decode_filter: > 2^24 candidates");
    return launch_decode(head_out, 1, 0, 0, is_fp16, nhwc, yolo_w, yolo_h, num_anchors, *head, num_classes, input_w,
                         input_h, new_coords, cand_base, label_mask, conf_thresh, size_w, size_h, off_x, off_y, nullptr,
                         dense, keys, counter, key_cap, stream, "fm_yolo_decode_filter");
}

extern "C" int fm_yolo_decode_filter_geom(const void* head_out, int batch, long long head_stride, int is_fp16,
                                          int nhwc, int yolo_w, int yolo_h, int num_anchors, const FmYoloHead* head,
                                          int num_classes, int input_w, int input_h, int new_coords, int cand_base,
                                          int cand_stride, const unsigned char* label_mask, double conf_thresh,
                                          const FmFrameGeom* geom, float* dense, unsigned long long* keys,
                                          int* counters, int key_cap, void* stream) {
    FM_REQUIRE(head != nullptr, "fm_yolo_decode_filter_geom: head is NULL");
    FM_REQUIRE(geom != nullptr, "fm_yolo_decode_filter_geom: geometry table is NULL");
    FM_REQUIRE(num_anchors <= FM_MAX_ANCHORS, "fm_yolo_decode_filter_geom: too many anchors");
    FM_REQUIRE(batch > 0 && batch <= 65535, "fm_yolo_decode_filter_geom: batch must be in [1, 65535]");
    FM_REQUIRE(cand_base + yolo_w * yolo_h * num_anchors <= cand_stride && cand_stride <= (1 << 24),
               "fm_yolo_decode_filter_geom: the head's candidates do not fit in cand_stride (<= 2^24) rows per image");
    FM_REQUIRE(head_stride >= (long long)yolo_w * yolo_h * num_anchors * (5 + num_classes),
               "fm_yolo_decode_filter_geom: head_stride is smaller than one image's head");
    return launch_decode(head_out, batch, head_stride, cand_stride, is_fp16, nhwc, yolo_w, yolo_h, num_anchors, *head,
                         num_classes, input_w, input_h, new_coords, cand_base, label_mask, conf_thresh, 0.f, 0.f, 0.f,
                         0.f, geom, dense, keys, counters, key_cap, stream, "fm_yolo_decode_filter_geom");
}

extern "C" long long fm_nms_mask_bytes(int key_cap) {
    long long words = (key_cap + 63) / 64;
    return (long long)key_cap * words * 8;
}

static int launch_nms(int batch, unsigned long long* keys, const float* dense, int cand_stride, const int* counter,
                      int key_cap, double nms_thresh, double max_area, double min_aspect_ratio,
                      unsigned long long* mask, int max_out, double* out_tlbr, long long* out_label, double* out_conf,
                      int* out_count, int* status, void* stream) {
    static bool attr_set = false;
    if (!attr_set) {
        cudaFuncSetAttribute(sort_keys_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 16384 * 8);
        attr_set = true;
    }
    cudaStream_t s = (cudaStream_t)stream;
    int np2 = 1;
    while (np2 < key_cap) np2 <<= 1;
    cudaMemsetAsync(status, 0, sizeof(int) * batch, s);
    sort_keys_kernel<<<batch, 1024, (size_t)np2 * 8, s>>>(keys, counter, key_cap, status);
    FM_CHECK_LAUNCH("sort_keys_kernel");
    const int words = (key_cap + 63) / 64;
    nms_mask_kernel<<<dim3(FM_NUM_SMS * 8, batch), 64, 0, s>>>(keys, dense, cand_stride, counter, key_cap, nms_thresh,
                                                                mask, words);
    FM_CHECK_LAUNCH("nms_mask_kernel");
    fm_launch_nms_scan(batch, keys, dense, cand_stride, counter, key_cap, mask, words, max_area, min_aspect_ratio,
                       max_out, out_tlbr, out_label, out_conf, out_count, status, s);   // blocked scan, detect_nms.cu
    FM_CHECK_LAUNCH("nms_scan_blocked_kernel");
    return FM_OK;
}

extern "C" int fm_diou_nms_filter(unsigned long long* keys, const float* dense, const int* counter, int key_cap,
                                  double nms_thresh, double max_area, double min_aspect_ratio,
                                  unsigned long long* mask, int max_out, double* out_tlbr, long long* out_label,
                                  double* out_conf, int* out_count, int* status, void* stream) {
    FM_REQUIRE(key_cap > 0 && key_cap <= 16384, "fm_diou_nms_filter: key_cap must be in (0, 16384]");
    return launch_nms(1, keys, dense, 0, counter, key_cap, nms_thresh, max_area, min_aspect_ratio, mask, max_out,
                      out_tlbr, out_label, out_conf, out_count, status, stream);
}

extern "C" int fm_diou_nms_filter_batch(int batch, unsigned long long* keys, const float* dense, int cand_stride,
                                        const int* counters, int key_cap, double nms_thresh, double max_area,
                                        double min_aspect_ratio, unsigned long long* mask, int max_out,
                                        double* out_tlbr, long long* out_label, double* out_conf, int* out_count,
                                        int* status, void* stream) {
    FM_REQUIRE(key_cap > 0 && key_cap <= 16384, "fm_diou_nms_filter_batch: key_cap must be in (0, 16384]");
    FM_REQUIRE(batch > 0 && batch <= 65535, "fm_diou_nms_filter_batch: batch must be in [1, 65535]");
    FM_REQUIRE(cand_stride > 0 && cand_stride <= (1 << 24), "fm_diou_nms_filter_batch: cand_stride must be in (0, 2^24]");
    return launch_nms(batch, keys, dense, cand_stride, counters, key_cap, nms_thresh, max_area, min_aspect_ratio, mask,
                      max_out, out_tlbr, out_label, out_conf, out_count, status, stream);
}
