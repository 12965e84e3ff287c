// Context, scratch arena, host<->device argument staging, pyramid storage.
#include "ov2_common.cuh"

#include <string.h>

ov2_status ov2_fail(ov2_ctx* ctx, ov2_status st, const char* what, cudaError_t ce) {
    if (ctx) {
        ctx->err = what ? what : "";
        if (ce != cudaSuccess) {
            ctx->err += ": ";
            ctx->err += cudaGetErrorString(ce);
        }
    }
    return st;
}

extern "C" const char* ov2_version(void) { return "ov2b200 0.1 (sm_90a)"; }

extern "C" ov2_status ov2_create(int device, ov2_ctx** out) {
    if (!out) return OV2_ERR_INVALID;
    *out = nullptr;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0) return OV2_ERR_NO_DEVICE;  // no CPU path exists
    if (device < 0 || device >= ndev) return OV2_ERR_INVALID;
    if (cudaSetDevice(device) != cudaSuccess) return OV2_ERR_CUDA;
    ov2_ctx* c = new ov2_ctx();
    c->device = device;
    if (cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess) {
        delete c;
        return OV2_ERR_CUDA;
    }
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) c->sm_count = prop.multiProcessorCount;
    *out = c;
    return OV2_OK;
}

extern "C" void ov2_destroy(ov2_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    for (auto& ch : ctx->chunks) cudaFree(ch.p);
    if (ctx->ba_stop) cudaFreeHost(ctx->ba_stop);
    if (ctx->ba_ws) cudaFreeHost(ctx->ba_ws);   // pinned staging block of the BA path
    if (ctx->desc_table) cudaFree(ctx->desc_table);
    if (ctx->pe0) { cudaEventDestroy(ctx->pe0); cudaEventDestroy(ctx->pe1); }
    if (ctx->sync_ev) cudaEventDestroy(ctx->sync_ev);
    if (ctx->upload_ev) cudaEventDestroy(ctx->upload_ev);
    for (auto& g : ctx->step_graphs) if (g.state == 1 && g.exec) cudaGraphExecDestroy(g.exec);
    if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
}

extern "C" const char* ov2_last_error(const ov2_ctx* ctx) { return ctx ? ctx->err.c_str() : "no context"; }

extern "C" ov2_status ov2_set_stream(ov2_ctx* ctx, void* s) {
    if (!ctx) return OV2_ERR_INVALID;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
    if (s) {
        ctx->stream = (cudaStream_t)s;
        ctx->own_stream = false;
    } else {
        OV2_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
        ctx->own_stream = true;
    }
    return OV2_OK;
}

extern "C" ov2_status ov2_sync(ov2_ctx* ctx) {
    if (!ctx) return OV2_ERR_INVALID;
    OV2_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return OV2_OK;
}

extern "C" ov2_status ov2_host_alloc(ov2_ctx* ctx, size_t bytes, void** out) {
    if (!ctx || !out) return OV2_ERR_INVALID;
    OV2_CUDA(ctx, cudaSetDevice(ctx->device));
    OV2_CUDA(ctx, cudaHostAlloc(out, bytes, cudaHostAllocDefault));
    return OV2_OK;
}

extern "C" ov2_status ov2_host_free(ov2_ctx* ctx, void* p) {
    if (!ctx) return OV2_ERR_INVALID;
    OV2_CUDA(ctx, cudaFreeHost(p));
    return OV2_OK;
}

void ov2_prof_begin(ov2_ctx* ctx) { cudaEventRecord(ctx->pe0, ctx->stream); }

void ov2_prof_end(ov2_ctx* ctx, const char* name) {
    cudaEventRecord(ctx->pe1, ctx->stream);
    cudaEventSynchronize(ctx->pe1);
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ctx->pe0, ctx->pe1);
    for (auto& p : ctx->prof)
        if (p.name == name) { p.ms += ms; p.n++; return; }
    ctx->prof.push_back({name, (double)ms, 1});
}

extern "C" ov2_status ov2_profile_enable(ov2_ctx* ctx, int on) {
    if (!ctx) return OV2_ERR_INVALID;
    OV2_CUDA(ctx, cudaSetDevice(ctx->device));
    if (on && !ctx->pe0) {
        OV2_CUDA(ctx, cudaEventCreate(&ctx->pe0));
        OV2_CUDA(ctx, cudaEventCreate(&ctx->pe1));
    }
    ctx->profiling = on != 0;
    if (on) ctx->prof.clear();
    return OV2_OK;
}

extern "C" int ov2_profile_query(const ov2_ctx* ctx, int idx, char* name_out, int name_cap, double* total_ms,
                                 uint64_t* launches) {
    if (!ctx || idx < 0 || idx >= (int)ctx->prof.size()) return 0;
    const auto& p = ctx->prof[idx];
    if (name_out && name_cap > 0) {
        snprintf(name_out, name_cap, "%s", p.name.c_str());
    }
    if (total_ms) *total_ms = p.ms;
    if (launches) *launches = p.n;
    return 1;
}

extern "C" uint64_t ov2_launch_count(const ov2_ctx* ctx) { return ctx ? ctx->launches : 0; }

// ------------------------------------------------------------------------ call scope
ov2_status ov2_begin(ov2_ctx* ctx) {
    if (!ctx) return OV2_ERR_INVALID;
    OV2_CUDA(ctx, cudaSetDevice(ctx->device));
    if (ctx->batch) return OV2_OK;     // batch mode: keep the arena and the pending outputs of earlier calls
    ctx->pending.clear();
    if (ctx->chunks.size() > 1) {
        // consolidate: previous call outgrew the arena
        OV2_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        size_t total = 0;
        // captured step graphs hold arena addresses: drop them before the arena moves
        for (auto& g : ctx->step_graphs) { if (g.state == 1 && g.exec) cudaGraphExecDestroy(g.exec); g.exec = nullptr; g.state = 0; }
        for (auto& ch : ctx->chunks) { total += ch.cap; cudaFree(ch.p); }
        ctx->chunks.clear();
        char* p = nullptr;
        OV2_CUDA(ctx, cudaMalloc(&p, total));
        ctx->chunks.push_back({p, total});
    }
    ctx->chunk_off = 0;
    return OV2_OK;
}

ov2_status ov2_scratch(ov2_ctx* ctx, size_t bytes, void** out) {
    bytes = (bytes + 255) & ~(size_t)255;
    if (bytes == 0) bytes = 256;
    if (ctx->chunks.empty() || ctx->chunk_off + bytes > ctx->chunks.back().cap) {
        size_t cap = ctx->chunks.empty() ? (size_t)(4 << 20) : ctx->chunks.back().cap * 2;
        if (cap < bytes) cap = bytes;
        char* p = nullptr;
        OV2_CUDA(ctx, cudaMalloc(&p, cap));
        ctx->chunks.push_back({p, cap});
        ctx->chunk_off = 0;
    }
    *out = ctx->chunks.back().p + ctx->chunk_off;
    ctx->chunk_off += bytes;
    return OV2_OK;
}

bool ov2_is_device_ptr(const void* p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

ov2_status ov2_stage_in(ov2_ctx* ctx, const void* p, size_t bytes, const void** dev) {
    if (!p || bytes == 0) { *dev = nullptr; return OV2_OK; }
    if (ov2_is_device_ptr(p)) { *dev = p; return OV2_OK; }
    if (ctx->batch) {
        // produced by an earlier call of this batch? then its device staging buffer IS the data
        for (auto it = ctx->pending.rbegin(); it != ctx->pending.rend(); ++it)
            if (it->host == p && it->bytes >= bytes) { *dev = it->dev; return OV2_OK; }
    }
    void* d = nullptr;
    ov2_status st = ov2_scratch(ctx, bytes, &d);
    if (st != OV2_OK) return st;
    OV2_CUDA(ctx, cudaMemcpyAsync(d, p, bytes, cudaMemcpyHostToDevice, ctx->stream));
    *dev = d;
    return OV2_OK;
}

ov2_status ov2_stage_out(ov2_ctx* ctx, void* p, size_t bytes, void** dev, bool copy_in) {
    if (!p || bytes == 0) { *dev = nullptr; return OV2_OK; }
    if (ov2_is_device_ptr(p)) { *dev = p; return OV2_OK; }
    if (ctx->batch) {
        // in/out buffer already staged by an earlier call of the batch: keep working on that copy
        for (auto it = ctx->pending.rbegin(); it != ctx->pending.rend(); ++it)
            if (it->host == p && it->bytes >= bytes) { *dev = const_cast<void*>(it->dev); return OV2_OK; }
    }
    void* d = nullptr;
    ov2_status st = ov2_scratch(ctx, bytes, &d);
    if (st != OV2_OK) return st;
    if (copy_in) OV2_CUDA(ctx, cudaMemcpyAsync(d, p, bytes, cudaMemcpyHostToDevice, ctx->stream));
    ctx->pending.push_back({p, d, bytes});
    *dev = d;
    return OV2_OK;
}

ov2_status ov2_wait_stream(ov2_ctx* ctx) {
    // sleep-wait (blocking-sync event) so many host threads can drive many contexts without burning
    // a core each in a spin loop
    if (!ctx->sync_ev) OV2_CUDA(ctx, cudaEventCreateWithFlags(&ctx->sync_ev, cudaEventBlockingSync | cudaEventDisableTiming));
    OV2_CUDA(ctx, cudaEventRecord(ctx->sync_ev, ctx->stream));
    OV2_CUDA(ctx, cudaEventSynchronize(ctx->sync_ev));
    return OV2_OK;
}

ov2_status ov2_end(ov2_ctx* ctx) {
    if (ctx->batch) return OV2_OK;     // deferred to ov2_batch_end
    if (ctx->pending.empty()) return OV2_OK;
    for (auto& pd : ctx->pending)
        OV2_CUDA(ctx, cudaMemcpyAsync(pd.host, pd.dev, pd.bytes, cudaMemcpyDeviceToHost, ctx->stream));
    ctx->pending.clear();
    return ov2_wait_stream(ctx);
}

extern "C" ov2_status ov2_batch_begin(ov2_ctx* ctx) {
    if (!ctx) return OV2_ERR_INVALID;
    if (ctx->batch) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_batch_begin: batch already open");
    ov2_status st = ov2_begin(ctx);    // resets the arena / pending list
    if (st != OV2_OK) return st;
    ctx->batch = true;
    return OV2_OK;
}

// D2H copies of everything the open batch produced into host buffers (no wait)
ov2_status ov2_batch_flush_outputs(ov2_ctx* ctx) {
    for (size_t i = 0; i < ctx->pending.size(); ++i) {
        bool superseded = false;
        for (size_t j = i + 1; j < ctx->pending.size(); ++j)
            if (ctx->pending[j].host == ctx->pending[i].host && ctx->pending[j].bytes >= ctx->pending[i].bytes) superseded = true;
        if (superseded) continue;
        auto& pd = ctx->pending[i];
        OV2_CUDA(ctx, cudaMemcpyAsync(pd.host, pd.dev, pd.bytes, cudaMemcpyDeviceToHost, ctx->stream));
    }
    ctx->pending.clear();
    return OV2_OK;
}

extern "C" ov2_status ov2_batch_end(ov2_ctx* ctx) {
    if (!ctx) return OV2_ERR_INVALID;
    if (!ctx->batch) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_batch_end: no batch open");
    ctx->batch = false;
    ov2_status fst = ov2_batch_flush_outputs(ctx);
    if (fst != OV2_OK) return fst;
    return ov2_wait_stream(ctx);
}

ov2_status ov2_in_batch(ov2_ctx* ctx, const std::function<ov2_status()>& enqueue) {
    const bool own_batch = !ctx->batch;
    ov2_status st = own_batch ? ov2_batch_begin(ctx) : ov2_begin(ctx);
    if (st != OV2_OK) return st;
    st = enqueue();
    if (!own_batch) return st;
    ctx->batch = false;
    if (st != OV2_OK) {
        ctx->pending.clear();
        return st;
    }
    if (ctx->pending.empty()) return OV2_OK;
    if ((st = ov2_batch_flush_outputs(ctx)) != OV2_OK) return st;
    return ov2_wait_stream(ctx);
}

ov2_offsets_check ov2_check_offsets(const int32_t* t, int count) {
    if (ov2_is_device_ptr(t)) return OV2_OFFSETS_ON_DEVICE;
    if (t[0] != 0) return OV2_OFFSETS_NOT_ASCENDING;
    for (int k = 0; k < count; ++k)
        if (t[k + 1] < t[k]) return OV2_OFFSETS_NOT_ASCENDING;
    return OV2_OFFSETS_OK;
}

// ------------------------------------------------------------------------ pyramid storage
extern "C" ov2_status ov2_pyr_create(ov2_ctx* ctx, int batch, int width, int height, int nlevels_extra,
                                     ov2_pyr** out) {
    if (!ctx || !out || batch <= 0 || width < 16 || height < 16 || nlevels_extra < 0 ||
        nlevels_extra + 1 > OV2_MAX_LEVELS)
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_pyr_create: bad arguments");
    OV2_CUDA(ctx, cudaSetDevice(ctx->device));
    ov2_pyr* p = new ov2_pyr();
    p->ctx = ctx;
    p->batch = batch;
    p->nlev = nlevels_extra + 1;
    int w = width, h = height;
    for (int l = 0; l < p->nlev; ++l) {
        p->w[l] = w;
        p->h[l] = h;
        p->pitch[l] = ((size_t)w + 127) & ~(size_t)127;
        p->fstride[l] = p->pitch[l] * (size_t)h;
        if (l > 0) {
            cudaError_t e = cudaMalloc(&p->own[l], p->fstride[l] * (size_t)batch);
            if (e != cudaSuccess) {
                for (int k = 1; k < l; ++k) cudaFree(p->own[k]);
                delete p;
                return ov2_fail(ctx, OV2_ERR_NOMEM, "ov2_pyr_create: cudaMalloc", e);
            }
        }
        w = (w + 1) / 2;
        h = (h + 1) / 2;
    }
    *out = p;
    return OV2_OK;
}

extern "C" void ov2_pyr_destroy(ov2_pyr* p) {
    if (!p) return;
    cudaSetDevice(p->ctx->device);
    cudaStreamSynchronize(p->ctx->stream);
    {
        // captured step graphs of this context hold the pyramid's device pointers: drop the ones keyed on it (the key ends
        // with the two pyramid handles), so a new pyramid at the same address can never replay a graph over freed levels
        auto& gs = p->ctx->step_graphs;
        for (size_t i = 0; i < gs.size();) {
            bool mine = false;
            if (gs[i].key.size() >= 2 * sizeof(void*)) {
                void* h[2];
                memcpy(h, gs[i].key.data() + gs[i].key.size() - 2 * sizeof(void*), sizeof(h));
                mine = h[0] == (void*)p || h[1] == (void*)p;
            }
            if (mine) {
                if (gs[i].state == 1 && gs[i].exec) cudaGraphExecDestroy(gs[i].exec);
                gs.erase(gs.begin() + i);
            } else {
                ++i;
            }
        }
    }
    for (int l = 0; l < p->nlev; ++l)
        if (p->own[l]) cudaFree(p->own[l]);
    delete p;
}

extern "C" ov2_status ov2_pyr_download(ov2_ctx* ctx, const ov2_pyr* p, int frame, int level, uint8_t* out,
                                       int* level_w, int* level_h) {
    if (!ctx || !p || frame < 0 || frame >= p->batch || level < 0 || level >= p->nlev || !out)
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_pyr_download: bad arguments");
    OV2_CUDA(ctx, cudaSetDevice(ctx->device));
    const uint8_t* base = level == 0 ? p->l0 : p->own[level];
    if (!base) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_pyr_download: pyramid not built");
    size_t pitch = level == 0 ? p->l0_pitch : p->pitch[level];
    size_t fs = level == 0 ? p->l0_fstride : p->fstride[level];
    OV2_CUDA(ctx, cudaMemcpy2DAsync(out, p->w[level], base + fs * (size_t)frame, pitch, p->w[level],
                                    p->h[level], cudaMemcpyDeviceToHost, ctx->stream));
    OV2_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (level_w) *level_w = p->w[level];
    if (level_h) *level_h = p->h[level];
    return OV2_OK;
}
