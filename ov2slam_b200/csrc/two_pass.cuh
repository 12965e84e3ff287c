// The two-pass tracking protocol of VisualFrontEnd::kltTracking and MapManager::stereoMatching: a guided pass 1 at depth 1
// from a prior, then pass 2 at full depth over every keypoint pass 1 did not track.  A composed call runs one CTA of
// THREADS threads per frame, each thread striding over the frame's keypoints, and keeps the slot arrays below in scratch.
// A slot with x < 0 is empty: ov2_fb_klt skips it at no cost, writes status 0 and leaves its prior alone.
#pragma once

#include "ov2_common.cuh"

namespace two_pass {

constexpr int THREADS = 256;

struct TwoPass {
    int32_t* frame_idx;                // [n] pyramid slot of each keypoint
    float2* kp1; float2* pri1; uint8_t* st1;   // pass 1: keypoints, priors (forward results after the pass), statuses
    float2* kp2; uint8_t* st2;                 // pass 2: keypoints, statuses; its priors are the caller's output array

    ov2_status stage(ov2_ctx* ctx, size_t n) {
        ov2_status st;
        if ((st = ov2_scratch(ctx, n, frame_idx)) != OV2_OK) return st;
        if ((st = ov2_scratch(ctx, n, kp1)) != OV2_OK) return st;
        if ((st = ov2_scratch(ctx, n, pri1)) != OV2_OK) return st;
        if ((st = ov2_scratch(ctx, n, st1)) != OV2_OK) return st;
        if ((st = ov2_scratch(ctx, n, kp2)) != OV2_OK) return st;
        return ov2_scratch(ctx, n, st2);
    }
    ov2_status pass1(ov2_ctx* ctx, const ov2_pyr* prev, const ov2_pyr* cur, const ov2_klt_params* prm, int n) const {
        return ov2_fb_klt(ctx, prev, cur, prm, n, frame_idx, 0, 0, nullptr, 1, (const float*)kp1, (float*)pri1, st1);
    }
    // out holds each pass-2 slot's prior and receives its tracked position
    ov2_status pass2(ov2_ctx* ctx, const ov2_pyr* prev, const ov2_pyr* cur, const ov2_klt_params* prm, int n, int nklt_pyr_lvl,
                     float2* out) const {
        return ov2_fb_klt(ctx, prev, cur, prm, n, frame_idx, 0, 0, nullptr, nklt_pyr_lvl, (const float*)kp2, (float*)out, st2);
    }

    // Keypoint i's pass-1 slot: px tracked from proj when guided, an empty slot otherwise.
    __device__ __forceinline__ void set_pass1(int i, int frame, float2 px, bool guided, float2 proj) const {
        frame_idx[i] = frame;
        kp1[i] = guided ? px : make_float2(-1.f, -1.f);
        pri1[i] = guided ? proj : px;
    }
    // Keypoint i's pass-2 slot and its output: tracked in pass 1, an empty slot that keeps the pass-1 result (pass 1); a
    // member, px tracked from restart (pass 2); otherwise an empty slot, output px (pass 0).
    __device__ __forceinline__ void set_pass2(int i, float2 px, bool member, float2 restart, float2* out, uint8_t* pass) const {
        if (kp1[i].x >= 0.f && st1[i]) {
            kp2[i] = make_float2(-1.f, -1.f);
            out[i] = pri1[i];
            pass[i] = 1;
        } else if (member) {
            kp2[i] = px;
            out[i] = restart;
            pass[i] = 2;
        } else {
            kp2[i] = make_float2(-1.f, -1.f);
            out[i] = px;
            pass[i] = 0;
        }
    }
};

// The sum of v over the CTA, returned to every thread (integers: order independent).  s: THREADS / 32 ints of shared
// memory for this sum alone.
__device__ __forceinline__ int cta_sum(int v, int* s) {
    v = __reduce_add_sync(0xffffffffu, v);
    if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = v;
    __syncthreads();
    v = 0;
    for (int k = 0; k < THREADS / 32; ++k) v += s[k];
    return v;
}

}  // namespace two_pass
