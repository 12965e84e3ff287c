// One front-end step over a batch of frame pairs as a single ABI call: what VisualFrontEnd does per
// frame (preprocessImage -> kltTracking, /root/reference/src/visual_front_end.cpp:65-128,1143-1177) plus
// MapManager::extractKeypoints' detect + describe on the current image (src/map_manager.cpp:286-341),
// composed from the operator entry points in batch mode: one round of H2D copies, the kernels, one
// round of D2H copies and ONE synchronisation.
//
// The step is a fixed DAG for a fixed argument block (same buffers every frame batch), so from its
// second call on it is captured into a CUDA graph and replayed with one cudaGraphLaunch: ~40 driver
// calls per step shrink to one, which is what limits throughput when several host threads feed one
// GPU (the CUDA context lock serialises them).
#include "ov2_common.cuh"

#include <condition_variable>
#include <mutex>
#include <string.h>

namespace {
// Several host threads drive several contexts (one per chunk of the batch).  If they all start their
// uploads at once the copy engine round-robins between the streams, every chunk receives its images
// only when (almost) all bytes of the batch have crossed PCIe, and copies never overlap compute.  The
// upload token makes image uploads FIFO per chunk: a chunk holds it from issuing its two H2D copies
// until they have landed (it keeps enqueueing its kernels meanwhile), so chunk k computes while chunk
// k+1 uploads.
// Two tokens: while one chunk's copies drain, the next chunk's are already queued behind them, so the
// copy engine never idles on a host-thread wake-up (measured: one token leaves ~80 us gaps per chunk).
struct UploadTokens {
    std::mutex mu;
    std::condition_variable cv;
    int free_tokens = 2;
    void acquire() { std::unique_lock<std::mutex> lk(mu); cv.wait(lk, [&] { return free_tokens > 0; }); --free_tokens; }
    void release() { { std::lock_guard<std::mutex> lk(mu); ++free_tokens; } cv.notify_one(); }
} g_upload_tokens;

// enqueue everything after the image uploads on ctx->stream (batch mode must be on); returns with the
// D2H copies enqueued
ov2_status enqueue_step(ov2_ctx* ctx, ov2_pyr* prev, ov2_pyr* cur, const ov2_frontend_step_args* a) {
    ov2_status st;
#define STEP(call) do { st = (call); if (st != OV2_OK) return st; } while (0)
    STEP(ov2_pyr_make_levels(ctx, prev, 0, a->count));
    STEP(ov2_pyr_make_levels(ctx, cur, 0, a->count));
    if (a->n_kps > 0)
        STEP(ov2_fb_klt(ctx, prev, cur, &a->klt, a->n_kps, nullptr, 0, a->kps_per_frame, a->nbpyrlvl, a->nbpyrlvl_all, a->kps,
                        a->priors_inout, a->status_out));
    if (a->cellsize > 0)
        STEP(ov2_grid_fast(ctx, cur, 0, a->count, a->cellsize, nullptr, nullptr, a->fast_th_inout, a->max_per_frame, a->new_pts,
                           a->new_counts, nullptr, 1));
    if (a->n_kps > 0 && a->desc_tracked)
        STEP(ov2_describe(ctx, cur, a->n_kps, nullptr, 0, a->kps_per_frame, a->priors_inout, a->desc_tracked, a->valid_tracked));
    if (a->cellsize > 0 && a->desc_new)
        STEP(ov2_describe(ctx, cur, a->count * a->max_per_frame, nullptr, 0, a->max_per_frame, a->new_pts, a->desc_new, a->valid_new));
#undef STEP
    return ov2_batch_flush_outputs(ctx);
}

}  // namespace

extern "C" ov2_status ov2_frontend_step(ov2_ctx* ctx, ov2_pyr* prev, ov2_pyr* cur, const ov2_frontend_step_args* a) {
    if (!ctx || !prev || !cur || !a || a->count <= 0) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_frontend_step: bad arguments");
    if (ctx->batch) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_frontend_step: a batch is already open on this context");
    // graph cache key: the argument block and the two pyramids
    std::vector<unsigned char> key(sizeof(*a) + 2 * sizeof(void*));
    memcpy(key.data(), a, sizeof(*a));
    memcpy(key.data() + sizeof(*a), &prev, sizeof(void*));
    memcpy(key.data() + sizeof(*a) + sizeof(void*), &cur, sizeof(void*));
    ov2_ctx::StepGraph* g = nullptr;
    for (auto& e : ctx->step_graphs)
        if (e.key == key) { g = &e; break; }
    const bool use_graphs = !ctx->profiling;
    const bool host_images = !ov2_is_device_ptr(a->prev_images);

    ov2_status st = ov2_batch_begin(ctx);     // resets the arena, opens batch mode
    if (st != OV2_OK) return st;
    auto abort_batch = [&](ov2_status s) { ctx->batch = false; ctx->pending.clear(); return s; };

    // ---- 1. image uploads, FIFO across contexts
    struct TokenGuard {
        bool held = false;
        void take() { g_upload_tokens.acquire(); held = true; }
        void drop() { if (held) { g_upload_tokens.release(); held = false; } }
        ~TokenGuard() { drop(); }
    } token;
    if (host_images) token.take();
    if ((st = ov2_pyr_load_level0(ctx, prev, a->prev_images, a->row_stride, a->frame_stride, 0, a->count)) != OV2_OK) return abort_batch(st);
    if ((st = ov2_pyr_load_level0(ctx, cur, a->cur_images, a->row_stride, a->frame_stride, 0, a->count)) != OV2_OK) return abort_batch(st);
    if (host_images) {
        if (!ctx->upload_ev && cudaEventCreateWithFlags(&ctx->upload_ev, cudaEventDisableTiming) != cudaSuccess)
            return abort_batch(ov2_fail(ctx, OV2_ERR_CUDA, "cudaEventCreate"));
        if (cudaEventRecord(ctx->upload_ev, ctx->stream) != cudaSuccess) return abort_batch(ov2_fail(ctx, OV2_ERR_CUDA, "cudaEventRecord"));
    }

    // ---- 2. everything else: replay the captured graph, capture it (second call), or enqueue eagerly
    bool done = false;
    if (g && g->state == 1 && use_graphs) {
        ctx->batch = false;
        ctx->pending.clear();
        if (cudaGraphLaunch(g->exec, ctx->stream) != cudaSuccess) return ov2_fail(ctx, OV2_ERR_CUDA, "cudaGraphLaunch", cudaGetLastError());
        ctx->launches += g->launches;
        done = true;
    } else if (g && g->state == 0 && use_graphs) {
        // second call with these arguments: every buffer (arena, pyramid level 0, tables) exists now, so the
        // rest of the step can be captured without allocations.  Any failure -> eager path for this key.
        const uint64_t l0 = ctx->launches;
        cudaGraph_t graph = nullptr;
        cudaGraphExec_t exec = nullptr;
        bool ok = cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeRelaxed) == cudaSuccess;
        if (ok) {
            st = enqueue_step(ctx, prev, cur, a);
            cudaError_t ce = cudaStreamEndCapture(ctx->stream, &graph);
            ok = st == OV2_OK && ce == cudaSuccess && graph != nullptr;
        }
        if (ok) ok = cudaGraphInstantiate(&exec, graph, 0) == cudaSuccess;
        if (graph) cudaGraphDestroy(graph);
        ctx->pending.clear();
        if (ok) {
            ctx->batch = false;
            g->exec = exec;
            g->launches = ctx->launches - l0;
            ctx->launches = l0;
            g->state = 1;
            if (cudaGraphLaunch(g->exec, ctx->stream) != cudaSuccess) return ov2_fail(ctx, OV2_ERR_CUDA, "cudaGraphLaunch", cudaGetLastError());
            ctx->launches += g->launches;   // capture did not execute anything
            done = true;
        } else {
            cudaGetLastError();
            g->state = -1;
            ctx->launches = l0;
            // the arena offsets consumed during the failed capture are simply re-used below
            ctx->chunk_off = 0;
        }
    }
    if (!done) {
        if (!g) {
            // bounded cache: argument blocks that change every call (per-frame buffers) must not grow it without limit
            if (ctx->step_graphs.size() >= 16) {
                auto& old = ctx->step_graphs.front();
                if (old.state == 1 && old.exec) cudaGraphExecDestroy(old.exec);
                ctx->step_graphs.erase(ctx->step_graphs.begin());
            }
            ctx->step_graphs.push_back({key, nullptr, 0, 0});
        }
        st = enqueue_step(ctx, prev, cur, a);
        if (st != OV2_OK) return abort_batch(st);
        ctx->batch = false;
    }
    // ---- 3. release the upload token once this chunk's images are on the device, then wait for the step
    if (host_images) {
        cudaError_t ce = cudaEventSynchronize(ctx->upload_ev);
        token.drop();
        if (ce != cudaSuccess) return ov2_fail(ctx, OV2_ERR_CUDA, "cudaEventSynchronize(upload)", ce);
    }
    return ov2_wait_stream(ctx);
}
