// ceresPnP ("next" row 2, SURVEY.md 8f): batched motion-only bundle adjustment, one thread block per pose
// problem, the whole Ceres-faithful Levenberg-Marquardt loop ON THE DEVICE (no host round trip per
// iteration: a PnP is ~5 iterations over 100-700 points, pure latency on the host).
//
// Reference behaviour replaced: MultiViewGeometry::ceresPnP
// (/root/reference/src/multi_view_geometry.cpp:492-588; called on every frame from
// src/visual_front_end.cpp:791-801).  The solve itself is pnp_math.cuh (shared with the host test);
// this file only provides the thread-block context (strided point ownership, block all-reduce) and
// the ABI entry.  Every thread runs the LM controller redundantly on the block-reduced sums, so the
// control flow is uniform and no thread waits for a "master".
//
// STATUS: host-validated against oracle/pnp_ref.py through pnp_math.cuh (tests/test_host_logic.py);
#include "ov2_common.cuh"
#include "pnp_math.cuh"

namespace {

constexpr int PNP_THREADS = 128;
constexpr unsigned FULL = 0xffffffffu;

struct BlockPar {
    double* sred;    // shared: [PNP_THREADS / 32][32]
    __device__ int begin() const { return (int)threadIdx.x; }
    __device__ int stride() const { return (int)blockDim.x; }
    __device__ void sync() { __syncthreads(); }
    // all-reduce (sum) of n <= 32 doubles; every thread gets the same bits (one fixed summation order)
    __device__ void reduce(double* v, int n) {
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        for (int k = 0; k < n; ++k) {
            double s = v[k];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(FULL, s, o);
            if (lane == 0) sred[warp * 32 + k] = s;
        }
        __syncthreads();
        for (int k = 0; k < n; ++k) {
            double s = 0.0;
            for (int w = 0; w < PNP_THREADS / 32; ++w) s += sred[w * 32 + k];
            v[k] = s;
        }
        __syncthreads();
    }
};

struct PnpArgs {
    int nprob;
    const int32_t* offsets;   // [nprob + 1]
    const double* unpx;       // [N][2]
    const double* wpts;       // [N][3]
    const int32_t* scales;    // [N] or NULL
    const double* K;          // [nprob][4]
    double* pose;             // [nprob][7] in/out
    int nmaxiter;
    float chi2th;
    int use_robust, apply_l2;
    uint8_t* flags;           // [N] out: 1 = rejected block
    uint8_t* success;         // [nprob]
    int32_t* iterations;      // [nprob] LM iterations of the last solve that ran
    double* chi2;             // [N] scratch
    uint8_t* depth;           // [N] scratch
    uint8_t* work;            // [N] scratch
};

__global__ void __launch_bounds__(PNP_THREADS) pnp_kernel(PnpArgs A) {
    __shared__ double sred[(PNP_THREADS / 32) * 32];
    const int pb = blockIdx.x;
    const int o0 = A.offsets[pb], o1 = A.offsets[pb + 1];
    pnp::Problem P;
    P.n = o1 - o0;
    P.unpx = A.unpx + 2 * (size_t)o0;
    P.wpts = A.wpts + 3 * (size_t)o0;
    P.scales = A.scales ? A.scales + o0 : nullptr;
    for (int i = 0; i < 4; ++i) P.K[i] = A.K[4 * pb + i];
    double pose[7];
    for (int i = 0; i < 7; ++i) pose[i] = A.pose[7 * pb + i];
    BlockPar par{sred};
    pnp::Summary S;
    S.iterations = 0; S.termination = 0; S.initial_cost = 0.0; S.final_cost = 0.0;
    bool ok = false;
    if (P.n > 0)
        ok = pnp::ceres_pnp(par, P, pose, A.nmaxiter, A.chi2th, A.use_robust != 0, A.apply_l2 != 0, A.chi2 + o0, A.depth + o0,
                            A.flags + o0, A.work + o0, S);
    if (threadIdx.x == 0) {
        for (int i = 0; i < 7; ++i) A.pose[7 * pb + i] = pose[i];
        A.success[pb] = ok ? 1 : 0;
        A.iterations[pb] = S.iterations;
    }
}

}  // namespace

extern "C" ov2_status ov2_pnp_solve(ov2_ctx* ctx, int nprob, const int32_t* offsets, const double* unpx, const double* wpts,
                                    const int32_t* scales, const double* K, double* pose_inout, int nmaxiter, float chi2th,
                                    int use_robust, int apply_l2_after_robust, uint8_t* outlier_flags, uint8_t* success_out,
                                    int32_t* iterations_out) {
    if (!ctx || nprob < 0 || (nprob > 0 && (!offsets || !K || !pose_inout || !success_out)))
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_pnp_solve: bad arguments");
    if (nprob == 0) return OV2_OK;
    // every block reads offsets[pb] .. offsets[pb + 1] of buffers sized offsets[nprob]: a descending pair would read past them
    const ov2_offsets_check oc = ov2_check_offsets(offsets, nprob);
    if (oc == OV2_OFFSETS_ON_DEVICE) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_pnp_solve: offsets must be a host pointer");
    if (oc != OV2_OFFSETS_OK) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_pnp_solve: offsets must start at 0 and be ascending");
    const int N = offsets[nprob];
    if (N > 0 && (!unpx || !wpts || !outlier_flags)) return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_pnp_solve: null array");
    ov2_status st = ov2_begin(ctx);
    if (st != OV2_OK) return st;
    PnpArgs A;
    A.nprob = nprob; A.nmaxiter = nmaxiter; A.chi2th = chi2th; A.use_robust = use_robust; A.apply_l2 = apply_l2_after_robust;
    const size_t np = (size_t)nprob, nn = (size_t)N;
    if ((st = ov2_stage_in(ctx, offsets, np + 1, A.offsets)) != OV2_OK) return st;
    if ((st = ov2_stage_in(ctx, K, 4 * np, A.K)) != OV2_OK) return st;
    A.unpx = nullptr; A.wpts = nullptr; A.scales = nullptr; A.flags = nullptr; A.chi2 = nullptr; A.depth = nullptr; A.work = nullptr;
    if (N > 0) {
        if ((st = ov2_stage_in(ctx, unpx, 2 * nn, A.unpx)) != OV2_OK) return st;
        if ((st = ov2_stage_in(ctx, wpts, 3 * nn, A.wpts)) != OV2_OK) return st;
        if (scales && (st = ov2_stage_in(ctx, scales, nn, A.scales)) != OV2_OK) return st;
        if ((st = ov2_stage_out(ctx, outlier_flags, nn, A.flags)) != OV2_OK) return st;
        if ((st = ov2_scratch(ctx, nn, A.chi2)) != OV2_OK) return st;
        if ((st = ov2_scratch(ctx, nn, A.depth)) != OV2_OK) return st;
        if ((st = ov2_scratch(ctx, nn, A.work)) != OV2_OK) return st;
        OV2_CUDA(ctx, cudaMemsetAsync(A.flags, 0, nn, ctx->stream));
    }
    if ((st = ov2_stage_out(ctx, pose_inout, 7 * np, A.pose, true)) != OV2_OK) return st;
    if ((st = ov2_stage_out(ctx, success_out, np, A.success)) != OV2_OK) return st;
    if ((st = iterations_out ? ov2_stage_out(ctx, iterations_out, np, A.iterations) : ov2_scratch(ctx, np, A.iterations)) != OV2_OK)
        return st;
    OV2_LAUNCH(ctx, "pnp_kernel", pnp_kernel<<<nprob, PNP_THREADS, 0, ctx->stream>>>(A));
    return ov2_end(ctx);
}
