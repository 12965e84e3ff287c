// P: image pyramid (cv::pyrDown semantics), one launch per level over the whole frame batch.
//
// Reference behaviour replaced: cv::buildOpticalFlowPyramid(img, pyr, Size(9,9), 3)
// (/root/reference/src/visual_front_end.cpp:1172).  out(y,x) = (sum_{i,j} k_i k_j in(2y+i-2,
// 2x+j-2) + 128) >> 8, k = [1 4 6 4 1], BORDER_REFLECT_101, size ((W+1)/2, (H+1)/2): pure
// integer arithmetic, bit-exact against cv2.pyrDown.  HBM-bound: reads the level once (through
// a shared-memory tile with a 2-px halo), writes a quarter of it.
#include "ov2_common.cuh"
#include "tma_util.cuh"

#include <string.h>

namespace {

constexpr int TX = 32, TY = 4;          // threads: each computes 4 pixels of TWO output rows
constexpr int OUT_W = TX * 4;           // 128 output pixels per tile row
constexpr int OUT_H = 2 * TY;           // 8 output rows
constexpr int IN_ROWS = 2 * OUT_H + 3;  // 19
constexpr int IN_WORDS = 66;            // 264 bytes: input cols [2*x0-4, 2*x0+260)

// 5-tap [1 4 6 4 1] on packed bytes with dp4a: the four outputs of a thread read input bytes
// 2*x0-2 .. 2*x0+8, i.e. bytes 2.. of word W0 up to byte 0 of word W3 (W0 = tile word 2*tx)
__device__ __forceinline__ void hrow4(const uint32_t* w, int& h0, int& h1, int& h2, int& h3) {
    const uint32_t W0 = w[0], W1 = w[1], W2 = w[2], W3 = w[3];
    h0 = (int)__dp4a(W0, 0x04010000u, __dp4a(W1, 0x00010406u, 0u));   // bytes: W0[2]*1 + W0[3]*4 + W1[0]*6 + W1[1]*4 + W1[2]*1
    h1 = (int)__dp4a(W1, 0x04060401u, __dp4a(W2, 0x00000001u, 0u));   // W1[0..3]*(1,4,6,4) + W2[0]*1
    h2 = (int)__dp4a(W1, 0x04010000u, __dp4a(W2, 0x00010406u, 0u));
    h3 = (int)__dp4a(W2, 0x04060401u, __dp4a(W3, 0x00000001u, 0u));
}

__global__ void __launch_bounds__(TX* TY)
pyr_down_kernel(const uint8_t* __restrict__ src, int sw, int sh, int spitch, long long sfstride,
                uint8_t* __restrict__ dst, int dw, int dh, int dpitch, long long dfstride, int first) {
    __shared__ uint32_t tile[IN_ROWS][IN_WORDS];
    const int frame = first + blockIdx.z;
    src += sfstride * frame;
    dst += dfstride * frame;
    const int ox0 = blockIdx.x * OUT_W, oy0 = blockIdx.y * OUT_H;
    const int ix0 = 2 * ox0 - 4;  // input column of tile byte 0 (multiple of 4)
    const int iy0 = 2 * oy0 - 2;

    // Fixed 2-D mapping (no divisions): rows ty, ty+8, ty+16; words tx, tx+32 and the 2 tail words.
    // BORDER_REFLECT_101 in y only changes which row is read, so whole words are still loaded;
    // only words that stick out of [0, sw) in x are assembled byte by byte.
    const bool aligned = ((reinterpret_cast<uintptr_t>(src) | (uintptr_t)spitch) & 3) == 0;
    for (int r = threadIdx.y; r < IN_ROWS; r += TY) {
        int y = reflect101(iy0 + r, sh);
        y = clampi(y, 0, sh - 1);
        const uint8_t* grow = src + (size_t)y * spitch;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const int c = threadIdx.x + 32 * k;
            if (c >= IN_WORDS) break;
            const int x0 = ix0 + 4 * c;
            uint32_t wv;
            if (x0 > sw + 1) {
                wv = 0;   // beyond the last column any existing output reads (2*(dw-1)+2 <= sw+1)
            } else if (aligned && x0 >= 0 && x0 + 4 <= sw) {
                wv = __ldg(reinterpret_cast<const uint32_t*>(grow + x0));
            } else {
                wv = 0;
#pragma unroll
                for (int b = 0; b < 4; ++b) {
                    int x = reflect101(x0 + b, sw);
                    x = clampi(x, 0, sw - 1);   // far outside: only beyond what any in-range output needs
                    wv |= (uint32_t)__ldg(grow + x) << (8 * b);
                }
            }
            tile[r][c] = wv;
        }
    }
    __syncthreads();

    // two output rows per thread (oy, oy+1) share 3 of their 5 input rows: 7 horizontal passes (dp4a)
    // instead of 10, then the vertical [1 4 6 4 1] on the running sums
    const int oy = oy0 + 2 * threadIdx.y;
    const int ox = ox0 + 4 * threadIdx.x;
    if (oy >= dh || ox >= dw) return;
    const int r0 = 4 * threadIdx.y;
    int h[7][4];
#pragma unroll
    for (int r = 0; r < 7; ++r) hrow4(&tile[r0 + r][2 * threadIdx.x], h[r][0], h[r][1], h[r][2], h[r][3]);
#pragma unroll
    for (int o = 0; o < 2; ++o) {
        if (oy + o >= dh) break;
        int v[4];
#pragma unroll
        for (int j = 0; j < 4; ++j)
            v[j] = h[2 * o][j] + 4 * h[2 * o + 1][j] + 6 * h[2 * o + 2][j] + 4 * h[2 * o + 3][j] + h[2 * o + 4][j];
        const uint32_t packed = (uint32_t)((v[0] + 128) >> 8) | ((uint32_t)((v[1] + 128) >> 8) << 8) |
                                ((uint32_t)((v[2] + 128) >> 8) << 16) | ((uint32_t)((v[3] + 128) >> 8) << 24);
        uint8_t* drow = dst + (size_t)(oy + o) * dpitch + ox;
        if (ox + 3 < dw && ((reinterpret_cast<uintptr_t>(drow)) & 3) == 0) {
            *reinterpret_cast<uint32_t*>(drow) = packed;
        } else {
            for (int j = 0; j < 4 && ox + j < dw; ++j) drow[j] = (uint8_t)(packed >> (8 * j));
        }
    }
}


// ------------------------------------------------------------------------------------------------
// Fused pyramid: levels 1, 2 and 3 from level 0 in ONE launch.  A tile owns T3W x T3H pixels of level 3 and the
// matching 2x / 4x regions of levels 2 and 1; the level-0 region it needs (8 T3 + 21 pixels per side) is fetched by TMA
// (one cp.async.bulk.tensor per tile, double buffered: the next tile's image lands while this one is reduced), the
// intermediate levels live in shared memory, so level 0 is read from HBM once and levels 1-2 are never re-read.
// BORDER_REFLECT_101 is applied per level exactly as cv::pyrDown does: TMA zero-fills outside the image and the (at
// most two) out-of-range rows / columns a level needs are patched in shared memory from their mirror positions.
//
// Shared-memory convention: tile column c of every level is stored at byte c + 2 of its row, so the four outputs of a
// "strip" (tile columns 4k-2 .. 4k+1, bytes 4k .. 4k+3: one aligned word) read source bytes 8k-2 .. 8k+8, i.e. bytes
// 2.. of source word 2k-1 up to byte 0 of word 2k+2 - the pattern hrow4() reduces with dp4a.  The vertical
// [1 4 6 4 1] runs on two 16-bit lanes per register (sums stay below 2^16), one PRMT picks the four result bytes.
constexpr int T3W = 28, T3H = 16;
constexpr int W2T = 2 * T3W + 3, H2T = 2 * T3H + 3;        // 59 x 35
constexpr int W1T = 4 * T3W + 9, H1T = 4 * T3H + 9;        // 121 x 73
constexpr int W0T = 8 * T3W + 21, H0T = 8 * T3H + 21;      // 245 x 149 (TMA box: 256 x 149, starting 2 bytes early)
constexpr int P0 = 256, P1 = 128, P2 = 64, P3 = 32;
constexpr int FUSED_THREADS = 256;
constexpr int SLACK = 128;                                  // guard bytes before / after every tile (strip 0 reads word -1)
constexpr int L0_BYTES = P0 * H0T;                          // 38144
constexpr int OFF_L0A = SLACK, OFF_L0B = OFF_L0A + L0_BYTES + SLACK;
constexpr int OFF_L1 = OFF_L0B + L0_BYTES + SLACK;
constexpr int OFF_L2 = OFF_L1 + P1 * H1T + SLACK;
constexpr int OFF_L3 = OFF_L2 + P2 * H2T + SLACK;
constexpr int FUSED_SMEM = OFF_L3 + P3 * T3H + SLACK;

struct FusedArgs {
    uint8_t* l1; uint8_t* l2; uint8_t* l3;
    int w[4], h[4];
    int pitch1, pitch2, pitch3;
    long long fs1, fs2, fs3;
    int first, count, ntx, nty;
};

// horizontal [1 4 6 4 1] for the four outputs of a strip, packed as two 16-bit lanes per register
__device__ __forceinline__ void hrow_packed(const uint32_t* w, uint32_t& a, uint32_t& b) {
    int h0, h1, h2, h3;
    hrow4(w, h0, h1, h2, h3);
    a = (uint32_t)h0 | ((uint32_t)h1 << 16);
    b = (uint32_t)h2 | ((uint32_t)h3 << 16);
}

// One reduction stage inside shared memory: dst(i, j) = pyrDown of src at tile columns 2i .. 2i+4, rows 2j .. 2j+4.
template <int SP, int DP, int DWT, int DHT>
__device__ __forceinline__ void down_stage(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst) {
    constexpr int NS = (DWT + 2 + 3) / 4;                    // strips per row
    constexpr int NSEG = FUSED_THREADS / NS;
    constexpr int RPS = (DHT + NSEG - 1) / NSEG;             // rows per segment
    const int k = threadIdx.x % NS, seg = threadIdx.x / NS;
    if (seg >= NSEG) return;
    const int j0 = seg * RPS;
    int j1 = j0 + RPS;
    if (j1 > DHT) j1 = DHT;
    if (j0 >= j1) return;
    const uint32_t* s = reinterpret_cast<const uint32_t*>(src) + (2 * k - 1);
    constexpr int SW = SP / 4;
    uint32_t a0, b0, a1, b1, a2, b2, a3, b3, a4, b4;
    hrow_packed(s + (size_t)(2 * j0) * SW, a0, b0);
    hrow_packed(s + (size_t)(2 * j0 + 1) * SW, a1, b1);
    hrow_packed(s + (size_t)(2 * j0 + 2) * SW, a2, b2);
    for (int j = j0; j < j1; ++j) {
        hrow_packed(s + (size_t)(2 * j + 3) * SW, a3, b3);
        hrow_packed(s + (size_t)(2 * j + 4) * SW, a4, b4);
        const uint32_t va = a0 + a4 + 4u * (a1 + a3) + 6u * a2 + 0x00800080u;   // both lanes < 2^16: no carry between them
        const uint32_t vb = b0 + b4 + 4u * (b1 + b3) + 6u * b2 + 0x00800080u;
        *reinterpret_cast<uint32_t*>(dst + (size_t)j * DP + 4 * k) = __byte_perm(va, vb, 0x7531);   // (v >> 8) of the 4 lanes
        a0 = a2; b0 = b2; a1 = a3; b1 = b3; a2 = a4; b2 = b4;
    }
}

// BORDER_REFLECT_101 patch of a level tile whose column 0 / row 0 are global (gx0, gy0): positions -2, -1, n, n+1.
template <int PITCH, int WT, int HT>
__device__ __forceinline__ void reflect_cols(uint8_t* t, int gx0, int w) {
    for (int e = threadIdx.x; e < HT * 4; e += FUSED_THREADS) {
        const int j = e >> 2, q = e & 3;
        const int x = q < 2 ? q - 2 : w + (q - 2);
        const int c = x - gx0;
        if (c < 0 || c >= WT) continue;
        const int sx = x < 0 ? -x : 2 * (w - 1) - x;
        const int sc = sx - gx0;
        if (sc < 0 || sc >= WT) continue;
        t[(size_t)j * PITCH + c + 2] = t[(size_t)j * PITCH + sc + 2];
    }
}
template <int PITCH, int WT, int HT>
__device__ __forceinline__ void reflect_rows(uint8_t* t, int gy0, int h) {
    for (int e = threadIdx.x; e < 4 * (PITCH / 4); e += FUSED_THREADS) {
        const int q = e / (PITCH / 4), wd = e - q * (PITCH / 4);
        const int y = q < 2 ? q - 2 : h + (q - 2);
        const int r = y - gy0;
        if (r < 0 || r >= HT) continue;
        const int sy = y < 0 ? -y : 2 * (h - 1) - y;
        const int sr = sy - gy0;
        if (sr < 0 || sr >= HT) continue;
        reinterpret_cast<uint32_t*>(t + (size_t)r * PITCH)[wd] = reinterpret_cast<const uint32_t*>(t + (size_t)sr * PITCH)[wd];
    }
}

// store the owned part of a level tile (tile columns [c0, c0 + ow), rows [r0, r0 + oh)) to the level image at (gx, gy)
template <int PITCH, int VEC>
__device__ __forceinline__ void store_owned(const uint8_t* t, int c0, int r0, int ow, int oh, uint8_t* img, int pitch, int gx, int gy,
                                            int w, int h) {
    const int nv = ow / VEC;
    for (int e = threadIdx.x; e < nv * oh; e += FUSED_THREADS) {
        const int j = e / nv, v = e - j * nv;
        const int y = gy + j, x = gx + v * VEC;
        if (y >= h || x >= w) continue;
        const uint8_t* sp = t + (size_t)(r0 + j) * PITCH + c0 + 2 + v * VEC;
        uint8_t* dp = img + (size_t)y * pitch + x;
        if (x + VEC <= w) {
            if (VEC == 16) {
                const uint2 lo = *reinterpret_cast<const uint2*>(sp), hi = *reinterpret_cast<const uint2*>(sp + 8);
                *reinterpret_cast<uint4*>(dp) = make_uint4(lo.x, lo.y, hi.x, hi.y);
            } else if (VEC == 4) {
                *reinterpret_cast<uint32_t*>(dp) = *reinterpret_cast<const uint32_t*>(sp);
            } else {
                *reinterpret_cast<uint16_t*>(dp) = *reinterpret_cast<const uint16_t*>(sp);
            }
        } else {
            for (int b = 0; b < VEC && x + b < w; ++b) dp[b] = sp[b];
        }
    }
}

__global__ void __launch_bounds__(FUSED_THREADS, 2) pyr_levels_kernel(FusedArgs A, const __grid_constant__ CUtensorMap tmap) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ __align__(8) uint64_t s_bar[2];
    uint8_t* t1 = smem + OFF_L1; uint8_t* t2 = smem + OFF_L2; uint8_t* t3 = smem + OFF_L3;
    const int tiles_per_frame = A.ntx * A.nty, ntiles = tiles_per_frame * A.count;
    if (threadIdx.x == 0) { tma::mbar_init(&s_bar[0], 1); tma::mbar_init(&s_bar[1], 1); }
    __syncthreads();
    auto issue = [&](int tile, int buf) {
        const int fr = tile / tiles_per_frame, rem = tile - fr * tiles_per_frame;
        const int ty = rem / A.ntx, tx = rem - ty * A.ntx;
        tma::mbar_expect_tx(&s_bar[buf], (uint32_t)L0_BYTES);
        tma::load_3d(smem + (buf ? OFF_L0B : OFF_L0A), &tmap, &s_bar[buf], 8 * tx * T3W - 16, 8 * ty * T3H - 14, A.first + fr);
    };
    int it = 0;
    if ((int)blockIdx.x < ntiles && threadIdx.x == 0) issue(blockIdx.x, 0);
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
        const int buf = it & 1;
        const int next = tile + gridDim.x;
        // the other buffer was last touched (generic proxy) two barriers ago at least; order those accesses before the
        // async-proxy write of the next tile
        if (next < ntiles && threadIdx.x == 0) {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            issue(next, buf ^ 1);
        }
        const int fr = tile / tiles_per_frame, rem = tile - fr * tiles_per_frame;
        const int ty = rem / A.ntx, tx = rem - ty * A.ntx;
        const int x3 = tx * T3W, y3 = ty * T3H;
        tma::mbar_wait(&s_bar[buf], (uint32_t)((it >> 1) & 1));
        uint8_t* t0 = smem + (buf ? OFF_L0B : OFF_L0A);      // (no pointer array: keeps the accesses LDS, not generic LD)
        // ---- level 0 -> 1
        reflect_cols<P0, W0T, H0T>(t0, 8 * x3 - 14, A.w[0]);
        __syncthreads();
        reflect_rows<P0, W0T, H0T>(t0, 8 * y3 - 14, A.h[0]);
        __syncthreads();
        down_stage<P0, P1, W1T, H1T>(t0, t1);
        __syncthreads();
        reflect_cols<P1, W1T, H1T>(t1, 4 * x3 - 6, A.w[1]);
        __syncthreads();
        reflect_rows<P1, W1T, H1T>(t1, 4 * y3 - 6, A.h[1]);
        __syncthreads();
        store_owned<P1, 16>(t1, 6, 6, 4 * T3W, 4 * T3H, A.l1 + A.fs1 * (A.first + fr), A.pitch1, 4 * x3, 4 * y3, A.w[1], A.h[1]);
        // ---- level 1 -> 2
        down_stage<P1, P2, W2T, H2T>(t1, t2);
        __syncthreads();
        reflect_cols<P2, W2T, H2T>(t2, 2 * x3 - 2, A.w[2]);
        __syncthreads();
        reflect_rows<P2, W2T, H2T>(t2, 2 * y3 - 2, A.h[2]);
        __syncthreads();
        store_owned<P2, 4>(t2, 2, 2, 2 * T3W, 2 * T3H, A.l2 + A.fs2 * (A.first + fr), A.pitch2, 2 * x3, 2 * y3, A.w[2], A.h[2]);
        // ---- level 2 -> 3
        down_stage<P2, P3, T3W, T3H>(t2, t3);
        __syncthreads();
        store_owned<P3, 2>(t3, 0, 0, T3W, T3H, A.l3 + A.fs3 * (A.first + fr), A.pitch3, x3, y3, A.w[3], A.h[3]);
        __syncthreads();
    }
}

}  // namespace

// level 0: alias device images / upload host images (H2D on the context's stream)
ov2_status ov2_pyr_load_level0(ov2_ctx* ctx, ov2_pyr* p, const uint8_t* images, size_t row_stride, size_t frame_stride,
                               int first, int count) {
    if (!ctx || !p || !images || first < 0 || count <= 0 || first + count > p->batch ||
        row_stride < (size_t)p->w[0])
        return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_pyr_build: bad arguments");
    if (ov2_is_device_ptr(images)) {
        const uint8_t* base = images - (ptrdiff_t)frame_stride * first;
        if (p->l0_mode == 1)
            return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_pyr_build: pyramid already owns level 0 (host images)");
        p->l0 = base;
        p->l0_pitch = row_stride;
        p->l0_fstride = frame_stride;
        p->l0_mode = 2;
    } else {
        if (p->l0_mode == 2)
            return ov2_fail(ctx, OV2_ERR_INVALID, "ov2_pyr_build: pyramid aliases device images; cannot mix host images");
        if (!p->own[0]) {
            OV2_CUDA(ctx, cudaMalloc(&p->own[0], p->fstride[0] * (size_t)p->batch));
            p->l0 = p->own[0];
            p->l0_pitch = p->pitch[0];
            p->l0_fstride = p->fstride[0];
            p->l0_mode = 1;
        }
        if (frame_stride == row_stride * (size_t)p->h[0] && row_stride == p->pitch[0]) {
            // fully contiguous on both sides: ONE linear copy (a pitched copy is issued as W-byte rows and
            // reaches a fraction of the PCIe bandwidth)
            OV2_CUDA(ctx, cudaMemcpyAsync(p->own[0] + p->fstride[0] * (size_t)first, images, frame_stride * (size_t)count,
                                          cudaMemcpyHostToDevice, ctx->stream));
        } else if (frame_stride == row_stride * (size_t)p->h[0]) {
            OV2_CUDA(ctx, cudaMemcpy2DAsync(p->own[0] + p->fstride[0] * (size_t)first, p->pitch[0], images, row_stride,
                                            p->w[0], (size_t)p->h[0] * count, cudaMemcpyHostToDevice, ctx->stream));
        } else {
            for (int k = 0; k < count; ++k)
                OV2_CUDA(ctx, cudaMemcpy2DAsync(p->own[0] + p->fstride[0] * (size_t)(first + k), p->pitch[0],
                                                images + frame_stride * (size_t)k, row_stride, p->w[0], p->h[0],
                                                cudaMemcpyHostToDevice, ctx->stream));
        }
    }
    return OV2_OK;
}

// levels 1.. from level 0 (kernels only)
ov2_status ov2_pyr_make_levels(ov2_ctx* ctx, ov2_pyr* p, int first, int count) {
    // fused path: the reference's pyramid depth (3 extra levels), level 3 at least 8 x 8, level 0 TMA-addressable
    if (p->nlev == 4 && p->w[3] >= 8 && p->h[3] >= 8) {
        CUtensorMap tmap;
        memset(&tmap, 0, sizeof(tmap));
        if (tma::make_u8_3d(&tmap, p->l0, p->w[0], p->h[0], p->batch, p->l0_pitch, p->l0_fstride, P0, H0T)) {
            FusedArgs A;
            A.l1 = p->own[1]; A.l2 = p->own[2]; A.l3 = p->own[3];
            for (int l = 0; l < 4; ++l) { A.w[l] = p->w[l]; A.h[l] = p->h[l]; }
            A.pitch1 = (int)p->pitch[1]; A.pitch2 = (int)p->pitch[2]; A.pitch3 = (int)p->pitch[3];
            A.fs1 = (long long)p->fstride[1]; A.fs2 = (long long)p->fstride[2]; A.fs3 = (long long)p->fstride[3];
            A.first = first; A.count = count;
            A.ntx = div_up(p->w[3], T3W); A.nty = div_up(p->h[3], T3H);
            static bool attr_set = false;
            if (!attr_set) {
                OV2_CUDA(ctx, cudaFuncSetAttribute(pyr_levels_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FUSED_SMEM));
                attr_set = true;
            }
            const int ntiles = A.ntx * A.nty * count;
            int grid = 2 * ctx->sm_count;
            if (grid > ntiles) grid = ntiles;
            OV2_LAUNCH(ctx, "pyr_levels_kernel", pyr_levels_kernel<<<grid, FUSED_THREADS, FUSED_SMEM, ctx->stream>>>(A, tmap));
            return OV2_OK;
        }
    }
    for (int l = 1; l < p->nlev; ++l) {
        const uint8_t* s = l == 1 ? p->l0 : p->own[l - 1];
        int spitch = (int)(l == 1 ? p->l0_pitch : p->pitch[l - 1]);
        long long sfs = (long long)(l == 1 ? p->l0_fstride : p->fstride[l - 1]);
        dim3 grid(div_up(p->w[l], OUT_W), div_up(p->h[l], OUT_H), count);
        OV2_LAUNCH(ctx, "pyr_down_kernel", pyr_down_kernel<<<grid, dim3(TX, TY), 0, ctx->stream>>>(s, p->w[l - 1], p->h[l - 1], spitch, sfs, p->own[l],
                                                               p->w[l], p->h[l], (int)p->pitch[l],
                                                               (long long)p->fstride[l], first));
    }
    return OV2_OK;
}

extern "C" ov2_status ov2_pyr_build(ov2_ctx* ctx, ov2_pyr* p, const uint8_t* images, size_t row_stride,
                                    size_t frame_stride, int first, int count) {
    if (!ctx) return OV2_ERR_INVALID;
    ov2_status st = ov2_begin(ctx);
    if (st != OV2_OK) return st;
    if ((st = ov2_pyr_load_level0(ctx, p, images, row_stride, frame_stride, first, count)) != OV2_OK) return st;
    if ((st = ov2_pyr_make_levels(ctx, p, first, count)) != OV2_OK) return st;
    return ov2_end(ctx);
}
