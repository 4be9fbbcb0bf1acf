// Host-side runner for the KLT stage: the whole enqueue sequence of Flow.predict (fastmot/flow.py:135-264) behind ONE
// C-ABI call.  The kernels are the ones the per-call API exposes (klt_image.cu, klt_feat.cu, klt_lk.cu,
// klt_ransac.cu); what this file removes is ~22 Python -> C transitions per frame (the tracking-only frame is host
// bound), not any GPU work.  No allocation, no synchronisation; two private events fork /
// join the camera-motion RANSAC onto the caller's side stream.
#include "common.cuh"
#include "../../include/fastmot_b200.h"
#include <new>

namespace {
struct FlowRunner {
    FmFlowPlan p;
    cudaEvent_t ev_lk = nullptr, ev_h = nullptr;
    // pyramid + Scharr chain of buffer k as a CUDA graph: pyrDown levels on one branch, the Scharr images on a second
    // (each needs only its own level), one launch instead of 2 * levels - 1.  0 = not built, 1 = ready, -1 = unavailable
    cudaGraphExec_t pyr_graph[2] = {nullptr, nullptr};
    int pyr_state[2] = {0, 0};
    int pyr_nodes = 0;
};

// Records pyr_level / scharr of buffer k into a graph by stream capture on two private streams.  Any failure leaves
// the runner on plain launches (state -1); nothing here touches the caller's streams.
void build_pyr_graph(FlowRunner* r, int k) {
    const FmPyramid& py = r->p.pyr[k];
    r->pyr_state[k] = -1;
    cudaStream_t s1 = nullptr, s2 = nullptr;
    cudaEvent_t ev[FM_MAX_PYR_LEVELS + 1] = {};
    cudaGraph_t graph = nullptr;
    bool ok = cudaStreamCreateWithFlags(&s1, cudaStreamNonBlocking) == cudaSuccess &&
              cudaStreamCreateWithFlags(&s2, cudaStreamNonBlocking) == cudaSuccess;
    for (int i = 0; ok && i <= py.n_levels; ++i) ok = cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming) == cudaSuccess;
    if (ok && cudaStreamBeginCapture(s1, cudaStreamCaptureModeThreadLocal) == cudaSuccess) {
        int nodes = 0;
        for (int i = 0; ok && i < py.n_levels; ++i) {
            ok = cudaEventRecord(ev[i], s1) == cudaSuccess && cudaStreamWaitEvent(s2, ev[i], 0) == cudaSuccess &&
                 fm_scharr(py.img[i], py.w[i], py.h[i], (short*)py.deriv[i], s2) == FM_OK;
            ++nodes;
            if (ok && i + 1 < py.n_levels) {
                ok = fm_pyr_level(py.img[i], py.w[i], py.h[i], (unsigned char*)py.img[i + 1], s1) == FM_OK;
                ++nodes;
            }
        }
        ok = ok && cudaEventRecord(ev[py.n_levels], s2) == cudaSuccess &&
             cudaStreamWaitEvent(s1, ev[py.n_levels], 0) == cudaSuccess;
        const cudaError_t e = cudaStreamEndCapture(s1, &graph);       // always end the capture, even after a failure
        ok = ok && e == cudaSuccess && graph != nullptr;
        if (ok && cudaGraphInstantiate(&r->pyr_graph[k], graph, 0) == cudaSuccess) {
            r->pyr_state[k] = 1;
            r->pyr_nodes = nodes;
        }
        fm_count_launches(-nodes);                                    // recording is not launching
    }
    if (graph) cudaGraphDestroy(graph);
    for (int i = 0; i <= FM_MAX_PYR_LEVELS; ++i)
        if (ev[i]) cudaEventDestroy(ev[i]);
    if (s1) cudaStreamDestroy(s1);
    if (s2) cudaStreamDestroy(s2);
    cudaGetLastError();
}
}  // namespace

extern "C" void* fm_flow_plan_create(const FmFlowPlan* plan) {
    if (!plan) { fm_set_last_error("fm_flow_plan_create: null plan"); return nullptr; }
    if (plan->pyr[0].n_levels < 1 || plan->pyr[0].n_levels > FM_MAX_PYR_LEVELS ||
        plan->pyr[1].n_levels != plan->pyr[0].n_levels || plan->rounds_ahead < 0 || (plan->rounds_ahead & 3)) {
        fm_set_last_error("fm_flow_plan_create: bad pyramid depth or rounds_ahead (multiple of 4)");
        return nullptr;
    }
    FlowRunner* r = new (std::nothrow) FlowRunner;
    if (!r) { fm_set_last_error("fm_flow_plan_create: out of host memory"); return nullptr; }
    r->p = *plan;
    if (cudaEventCreateWithFlags(&r->ev_lk, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&r->ev_h, cudaEventDisableTiming) != cudaSuccess) {
        fm_set_last_error("fm_flow_plan_create: cudaEventCreate failed");
        if (r->ev_lk) cudaEventDestroy(r->ev_lk);
        delete r;
        return nullptr;
    }
    return r;
}

extern "C" void fm_flow_plan_destroy(void* h) {
    FlowRunner* r = (FlowRunner*)h;
    if (!r) return;
    cudaEventDestroy(r->ev_lk);
    cudaEventDestroy(r->ev_h);
    for (int k = 0; k < 2; ++k)
        if (r->pyr_graph[k]) cudaGraphExecDestroy(r->pyr_graph[k]);
    delete r;
}

#define FM_TRY(call)            \
    do {                        \
        int rc__ = (call);      \
        if (rc__ != FM_OK) return rc__; \
    } while (0)

#define FM_CUDA_TRY(call, what)                     \
    do {                                            \
        cudaError_t e__ = (call);                   \
        if (e__ != cudaSuccess) {                   \
            char buf__[256];                        \
            snprintf(buf__, sizeof buf__, "%s: %s", what, cudaGetErrorString(e__)); \
            fm_set_last_error(buf__);               \
            return FM_ERR_CUDA;                     \
        }                                           \
    } while (0)

namespace {
// gray + optical-flow image + LK pyramid with Scharr derivatives for buffer k (flow.py:129-131 / :153-154).  An
// optical-flow image of exactly half the frame in both directions is the 2x2 mean (what cv2.resize computes there);
// any other size is the general INTER_LINEAR resize.
int preprocess(FlowRunner* r, const FmFrame* f, int k, void* stream) {
    const FmFlowPlan& p = r->p;
    const FmPyramid& py = p.pyr[k];
    unsigned char* small = (unsigned char*)py.img[0];
    if (2 * py.w[0] == p.frame_w && 2 * py.h[0] == p.frame_h)
        FM_TRY(fm_gray_half(f, p.gray[k], small, stream));
    else
        FM_TRY(fm_gray_resize(f, p.gray[k], small, py.w[0], py.h[0], stream));
    if (r->pyr_state[k] == 0) build_pyr_graph(r, k);
    if (r->pyr_state[k] == 1) {
        FM_CUDA_TRY(cudaGraphLaunch(r->pyr_graph[k], (cudaStream_t)stream), "fm_flow_predict: pyramid graph");
        fm_count_launches(r->pyr_nodes);
        return FM_OK;
    }
    for (int i = 0; i < py.n_levels; ++i) {
        if (i + 1 < py.n_levels)
            FM_TRY(fm_pyr_level(py.img[i], py.w[i], py.h[i], (unsigned char*)py.img[i + 1], stream));
        FM_TRY(fm_scharr(py.img[i], py.w[i], py.h[i], (short*)py.deriv[i], stream));
    }
    return FM_OK;
}

int predict(FlowRunner* r, const FmFrame* f, int prev, int n_trk, double* H_out, int* h_ok, void* s_main,
            void* s_side) {
    const FmFlowPlan& p = r->p;
    const int cur = 1 - prev;
    cudaStream_t sm = (cudaStream_t)s_main, ss = (cudaStream_t)s_side;
    FM_TRY(preprocess(r, f, cur, s_main));
    FM_CUDA_TRY(cudaMemsetAsync(p.klt_ok, 0, (size_t)p.klt_ok_bytes, sm), "fm_flow_predict: klt_ok clear");
    FM_TRY(fm_flow_keypoints_cfg(p.gray[prev], p.frame_w, p.frame_h, p.tlbr_pool, p.slots, n_trk, p.owner, p.kp_pool,
                                 p.kp_count, p.max_kp, p.feat_density, p.feat_dist_factor, p.quality, p.max_corners,
                                 p.block_size, p.gradient_size, p.use_harris, p.harris_k, p.jobs, p.scratch,
                                 p.scratch_cap, p.flags, p.flags + 1, s_main));
    FM_TRY(fm_bg_small(p.gray[prev], p.owner, p.frame_w, p.frame_h, p.bg, p.bg_mask, p.bg_w, p.bg_h, s_main));
    FM_TRY(fm_fast_detect(p.bg, p.bg_mask, p.bg_w, p.bg_h, p.bg_thresh, p.unscale_x, p.unscale_y, p.bg_score, p.bg_pts,
                          p.bg_count, p.max_bg, s_main));
    FM_TRY(fm_gather_points(p.kp_pool, p.kp_count, p.max_kp, p.slots, n_trk, p.bg_pts, p.bg_count, p.all_prev,
                            p.trk_begin, p.meta, p.max_points, s_main));
    FM_TRY(fm_lk_track(&p.pyr[prev], &p.pyr[cur], p.all_prev, p.meta, p.pt_scale_x, p.pt_scale_y, p.win_w, p.win_h,
                       p.lk_max_count, p.lk_epsilon, p.lk_min_eig, p.max_error, p.all_cur, p.status, p.err, s_main));
    // camera-motion RANSAC on the side stream, next to the per-track affine rounds (read-only sharing of LK outputs)
    FM_CUDA_TRY(cudaEventRecord(r->ev_lk, sm), "fm_flow_predict: event record");
    FM_CUDA_TRY(cudaStreamWaitEvent(ss, r->ev_lk, 0), "fm_flow_predict: side stream wait");
    FM_TRY(fm_ransac_homography(p.all_prev, p.all_cur, p.status, p.meta, p.ransac_max_iter, p.ransac_conf,
                                p.ransac_thresh, p.inlier_thresh, p.good_idx, p.inl_idx, H_out, h_ok, p.bg_kp,
                                p.bg_kp_prev, p.bg_kp_count, p.max_bg, s_side));
    FM_CUDA_TRY(cudaEventRecord(r->ev_h, ss), "fm_flow_predict: event record");
    for (int first = 0; first < p.rounds_ahead; first += 4)
        FM_TRY(fm_ransac_affine_partial_batch(p.all_prev, p.all_cur, p.status, p.trk_begin, p.slots, n_trk, 4,
                                              p.flags + 8, nullptr, p.est_boxes, p.sig, (double*)p.tlbr_pool, p.klt_tlbr,
                                              p.klt_ok, p.inlier_ratio, p.kp_pool, p.kp_prev_pool, p.kp_count, p.max_kp,
                                              p.frame_w, p.frame_h, p.ransac_max_iter, p.ransac_conf, p.ransac_thresh,
                                              p.inlier_thresh, p.refine_iters, first, s_main));
    FM_CUDA_TRY(cudaStreamWaitEvent(sm, r->ev_h, 0), "fm_flow_predict: join");   // H / h_ok feed the Kalman step
    return FM_OK;
}
}  // namespace

extern "C" int fm_flow_predict(void* h, const FmFrame* frame, int prev, int n_trk, double* H_out, int* h_ok,
                               void* s_main, void* s_side) {
    FlowRunner* r = (FlowRunner*)h;
    FM_REQUIRE(r && frame && (prev == 0 || prev == 1) && n_trk >= 0 && H_out && h_ok,
               "fm_flow_predict: bad handle / frame / buffer index / track count");
    FM_REQUIRE(frame->w == r->p.frame_w && frame->h == r->p.frame_h,
               "fm_flow_predict: the frame is not the plan's frame_w x frame_h");
    return predict(r, frame, prev, n_trk, H_out, h_ok, s_main, s_side);
}
