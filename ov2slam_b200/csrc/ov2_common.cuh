// Shared host/device plumbing for libov2b200 (context, scratch arenas, argument staging).
// Product code: nothing here may include or call anything under oracle/.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <functional>
#include <string>
#include <vector>

#include "../../include/ov2b200.h"

#define OV2_MAX_LEVELS 8

struct ov2_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = true;
    std::string err;
    uint64_t launches = 0;
    int sm_count = 132;
    // device scratch: bump allocator, reset at the start of every API call
    struct Chunk { char* p; size_t cap; };
    std::vector<Chunk> chunks;
    size_t chunk_off = 0;
    // pending device->host copies of the current call
    struct Pending { void* host; const void* dev; size_t bytes; };
    std::vector<Pending> pending;
    // batch mode (ov2_batch_begin / ov2_batch_end): calls only enqueue; host outputs are copied back and
    // the stream is synchronised ONCE at batch end; a host pointer written by an earlier call of the
    // batch and read by a later one is served from its device staging buffer (no round trip)
    bool batch = false;
    // CUDA graphs of ov2_frontend_step (one per distinct argument block): the whole step - H2D copies,
    // kernels, D2H copies - is captured on its second call and replayed with one cudaGraphLaunch afterwards
    struct StepGraph { std::vector<unsigned char> key; cudaGraphExec_t exec; uint64_t launches; int state; };  // state 0 seen once, 1 captured, -1 not capturable
    std::vector<StepGraph> step_graphs;
    cudaEvent_t sync_ev = nullptr;   // blocking-sync event: waiting threads sleep instead of spinning
    cudaEvent_t upload_ev = nullptr; // "images of this step are on the device" (ov2_frontend_step's upload token)
    // persistent small device blocks (tables)
    void* ba_ws = nullptr; size_t ba_ws_cap = 0;
    int desc_mode = 0;            // OV2_DESC_* (ov2_describe_config)
    int8_t* desc_table = nullptr; // device copy of the BRIEF-32 test pairs [256][4]
    int* ba_stop = nullptr;       // mapped pinned int: stop request polled by the persistent solve kernel
    // optional per-kernel CUDA-event timing (ov2_profile_enable): serialises launches
    bool profiling = false;
    cudaEvent_t pe0 = nullptr, pe1 = nullptr;
    struct Prof { std::string name; double ms; uint64_t n; };
    std::vector<Prof> prof;
};

struct ov2_pyr {
    ov2_ctx* ctx = nullptr;
    int batch = 0, nlev = 0;
    int w[OV2_MAX_LEVELS] = {0}, h[OV2_MAX_LEVELS] = {0};
    size_t pitch[OV2_MAX_LEVELS] = {0}, fstride[OV2_MAX_LEVELS] = {0};
    uint8_t* own[OV2_MAX_LEVELS] = {nullptr};   // own[0] allocated lazily (host-image path only)
    const uint8_t* l0 = nullptr;                 // level-0 base (own[0] or caller's device images)
    size_t l0_pitch = 0, l0_fstride = 0;
    int l0_mode = 0;                             // 0 unset, 1 own, 2 external
};

// What kernels see of a pyramid.
struct PyrView {
    const uint8_t* lvl[4];
    int w[4], h[4];
    int pitch[4];
    long long fstride[4];
    int nlev;
};

static inline PyrView make_view(const ov2_pyr* p) {
    PyrView v;
    for (int l = 0; l < 4; ++l) {
        int ll = l < p->nlev ? l : p->nlev - 1;
        v.lvl[l] = ll == 0 ? p->l0 : p->own[ll];
        v.w[l] = p->w[ll];
        v.h[l] = p->h[ll];
        v.pitch[l] = (int)(ll == 0 ? p->l0_pitch : p->pitch[ll]);
        v.fstride[l] = (long long)(ll == 0 ? p->l0_fstride : p->fstride[ll]);
    }
    v.nlev = p->nlev < 4 ? p->nlev : 4;
    return v;
}

ov2_status ov2_fail(ov2_ctx* ctx, ov2_status st, const char* what, cudaError_t ce = cudaSuccess);

#define OV2_CUDA(ctx, call)                                                         \
    do {                                                                            \
        cudaError_t _e = (call);                                                    \
        if (_e != cudaSuccess) return ov2_fail((ctx), OV2_ERR_CUDA, #call, _e);     \
    } while (0)

#define OV2_CHECK_LAUNCH(ctx, name)                                                 \
    do {                                                                            \
        (ctx)->launches++;                                                          \
        cudaError_t _e = cudaGetLastError();                                        \
        if (_e != cudaSuccess) return ov2_fail((ctx), OV2_ERR_CUDA, name, _e);      \
    } while (0)

void ov2_prof_begin(ov2_ctx* ctx);
void ov2_prof_end(ov2_ctx* ctx, const char* name);

// Launch wrapper: counts the launch, checks the launch error and, when profiling is on, times
// the kernel with CUDA events on the launching stream.
#define OV2_LAUNCH(ctx, name, ...)                                                  \
    do {                                                                            \
        if ((ctx)->profiling) ov2_prof_begin(ctx);                                  \
        __VA_ARGS__;                                                                \
        (ctx)->launches++;                                                          \
        cudaError_t _e = cudaGetLastError();                                        \
        if (_e != cudaSuccess) return ov2_fail((ctx), OV2_ERR_CUDA, name, _e);      \
        if ((ctx)->profiling) ov2_prof_end(ctx, name);                              \
    } while (0)

// --- call scope: scratch + staging ------------------------------------------------------
ov2_status ov2_begin(ov2_ctx* ctx);                               // reset scratch, bind device
ov2_status ov2_scratch(ov2_ctx* ctx, size_t bytes, void** out);   // 256-byte aligned device scratch
bool       ov2_is_device_ptr(const void* p);
// input: returns a device pointer holding `bytes` of *p (p itself if already on the device)
ov2_status ov2_stage_in(ov2_ctx* ctx, const void* p, size_t bytes, const void** dev);
// output: returns a device pointer to write; host destinations are copied back by ov2_end()
ov2_status ov2_stage_out(ov2_ctx* ctx, void* p, size_t bytes, void** dev, bool copy_in = false);
ov2_status ov2_end(ov2_ctx* ctx);                                 // D2H of pending outputs + sync if any
ov2_status ov2_wait_stream(ov2_ctx* ctx);                         // sleep-wait for the context's stream
ov2_status ov2_batch_flush_outputs(ov2_ctx* ctx);                 // batch mode: enqueue the D2H copies (no wait)

// The same, typed: counts are in elements of T.
template <class T> ov2_status ov2_stage_in(ov2_ctx* ctx, const void* p, size_t count, const T*& dev) {
    const void* d = nullptr;
    const ov2_status st = ov2_stage_in(ctx, p, sizeof(T) * count, &d);
    dev = static_cast<const T*>(d);
    return st;
}
template <class T> ov2_status ov2_stage_out(ov2_ctx* ctx, void* p, size_t count, T*& dev, bool copy_in = false) {
    void* d = nullptr;
    const ov2_status st = ov2_stage_out(ctx, p, sizeof(T) * count, &d, copy_in);
    dev = static_cast<T*>(d);
    return st;
}
template <class T> ov2_status ov2_scratch(ov2_ctx* ctx, size_t count, T*& dev) {
    void* d = nullptr;
    const ov2_status st = ov2_scratch(ctx, sizeof(T) * count, &d);
    dev = static_cast<T*>(d);
    return st;
}

// A call composed of other calls: runs enqueue inside the caller's open batch, or inside a batch of its own, so that the
// calls it makes only enqueue, scratch survives between them, and host outputs come back with one synchronisation at the
// end.  With device outputs only, the call returns without waiting, as every other call with device pointers.
ov2_status ov2_in_batch(ov2_ctx* ctx, const std::function<ov2_status()>& enqueue);

// A host table of count + 1 offsets that start at 0 and never decrease: each frame of a batch owns
// [t[f], t[f + 1]) of arrays sized t[count].
enum ov2_offsets_check { OV2_OFFSETS_OK, OV2_OFFSETS_ON_DEVICE, OV2_OFFSETS_NOT_ASCENDING };
ov2_offsets_check ov2_check_offsets(const int32_t* t, int count);

// Two pyramids one tracker can read together: both built, same depth and level-0 size.
static inline bool ov2_pyr_pair_ok(const ov2_pyr* a, const ov2_pyr* b) {
    return a->nlev == b->nlev && a->w[0] == b->w[0] && a->h[0] == b->h[0] && a->l0 && b->l0;
}

// pyramid build in two halves (frontend_step.cu orders the uploads of concurrent contexts)
ov2_status ov2_pyr_load_level0(ov2_ctx* ctx, ov2_pyr* p, const uint8_t* images, size_t row_stride, size_t frame_stride,
                               int first, int count);
ov2_status ov2_pyr_make_levels(ov2_ctx* ctx, ov2_pyr* p, int first, int count);

// --- device helpers ------------------------------------------------------------------
__device__ __forceinline__ int reflect101(int i, int n) {
    // BORDER_REFLECT_101: ... 2 1 | 0 1 2 ... n-2 n-1 | n-2 n-3 ...   (|overshoot| < n assumed)
    i = i < 0 ? -i : i;
    return i >= n ? 2 * (n - 1) - i : i;
}
__device__ __forceinline__ int clampi(int i, int lo, int hi) { return i < lo ? lo : (i > hi ? hi : i); }

static inline int div_up(int a, int b) { return (a + b - 1) / b; }
