// eft_ops.cu -- the non-GEMM operators of the Epipolar Feature Transformer (sparsefusion/eft.py, SURVEY.md §8f row 4), NHWC fp32, sm_90a.
//
// The EFT builds the per-view conditioning cache once per scene (sparsefusion/distillation.py:92-127): a ResNet-18 pyramid over the input views
// (eft.py:172-204), bilinear look-ups of that pyramid at the projections of every ray sample (F.grid_sample, eft.py:248-275), and three small
// transformer encoders over (input views) / (depth samples) / (input views) (eft.py:396-440).  Convolutions and every nn.Linear run on the
// wgmma implicit-GEMM engine (conv_wgmma.cu); this file holds what is left: 3x3/2 max-pooling, bilinear resize (align_corners), the
// grid-sample gather, the single-head attention core over short sequences, and the in-place activations.  All latency / L2-gather bound.
#include "common.cuh"
#include "../../include/sparsefusion_b200.h"

namespace sfb {

// y[n][oh][ow][c] = max over the 3x3 window at stride 2, padding 1 (torchvision resnet maxpool; padded positions never win; a NaN in the
// window gives NaN, as F.max_pool2d does)
__global__ void maxpool3x3s2_kernel(const float4* __restrict__ x, float4* __restrict__ y, int H, int W, int Ho, int Wo, int C4, int64_t total) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % C4);
        int64_t r = i / C4;
        const int ow = (int)(r % Wo); r /= Wo;
        const int oh = (int)(r % Ho);
        const int n = (int)(r / Ho);
        float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
#pragma unroll
        for (int dy = 0; dy < 3; ++dy) {
            const int ih = oh * 2 - 1 + dy;
            if (ih < 0 || ih >= H) continue;
#pragma unroll
            for (int dx = 0; dx < 3; ++dx) {
                const int iw = ow * 2 - 1 + dx;
                if (iw < 0 || iw >= W) continue;
                const float4 v = __ldg(x + (((int64_t)n * H + ih) * W + iw) * C4 + c);
                m.x = max_keep_nan(m.x, v.x); m.y = max_keep_nan(m.y, v.y); m.z = max_keep_nan(m.z, v.z); m.w = max_keep_nan(m.w, v.w);
            }
        }
        y[i] = m;
    }
}

// F.interpolate(x, (Ho, Wo), mode='bilinear', align_corners=True) in NHWC, written into a channel slice of a wider tensor (ldo): eft.py:194-202
__global__ void resize_bilinear_ac_kernel(const float* __restrict__ x, int64_t ldx, float* __restrict__ y, int64_t ldo, int H, int W, int Ho, int Wo, int C4,
                                          float sh, float sw, int64_t total) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % C4);
        int64_t r = i / C4;
        const int ow = (int)(r % Wo); r /= Wo;
        const int oh = (int)(r % Ho);
        const int n = (int)(r / Ho);
        const float fy = sh * oh, fx = sw * ow;                      // area_pixel_compute_source_index with align_corners: scale * dst_index
        const int y0 = min((int)fy, H - 1), x0 = min((int)fx, W - 1);
        const int y1 = min(y0 + 1, H - 1), x1 = min(x0 + 1, W - 1);
        const float ly = fy - y0, lx = fx - x0, hy = 1.f - ly, hx = 1.f - lx;
        const float* b = x + (int64_t)n * H * W * ldx + c * 4;
        const float4 v00 = __ldg(reinterpret_cast<const float4*>(b + ((int64_t)y0 * W + x0) * ldx));
        const float4 v01 = __ldg(reinterpret_cast<const float4*>(b + ((int64_t)y0 * W + x1) * ldx));
        const float4 v10 = __ldg(reinterpret_cast<const float4*>(b + ((int64_t)y1 * W + x0) * ldx));
        const float4 v11 = __ldg(reinterpret_cast<const float4*>(b + ((int64_t)y1 * W + x1) * ldx));
        float4 o;
        o.x = hy * (hx * v00.x + lx * v01.x) + ly * (hx * v10.x + lx * v11.x);
        o.y = hy * (hx * v00.y + lx * v01.y) + ly * (hx * v10.y + lx * v11.y);
        o.z = hy * (hx * v00.z + lx * v01.z) + ly * (hx * v10.z + lx * v11.z);
        o.w = hy * (hx * v00.w + lx * v01.w) + ly * (hx * v10.w + lx * v11.w);
        *reinterpret_cast<float4*>(y + (((int64_t)n * Ho + oh) * Wo + ow) * ldo + c * 4) = o;
    }
}

// F.grid_sample(mode='bilinear', padding_mode='border', align_corners=True) at one point (gx, gy) in [-1, 1] of an NHWC image b [H][W]
// (channel stride ldx): the four corner rows and their weights.  Out-of-range corners contribute zero (their weight is zero anyway).
struct BorderBilinear {
    const float *p00, *p01, *p10, *p11;
    float w00, w01, w10, w11;
    __device__ __forceinline__ float operator()(int c) const {
        return __ldg(p00 + c) * w00 + __ldg(p01 + c) * w01 + __ldg(p10 + c) * w10 + __ldg(p11 + c) * w11;
    }
};

__device__ __forceinline__ BorderBilinear border_bilinear(const float* b, int64_t ldx, int H, int W, float gx, float gy) {
    float ix = (gx + 1.f) * 0.5f * (W - 1), iy = (gy + 1.f) * 0.5f * (H - 1);      // grid_sampler_unnormalize, align_corners
    ix = fminf(fmaxf(ix, 0.f), (float)(W - 1));                                     // clip_coordinates (border)
    iy = fminf(fmaxf(iy, 0.f), (float)(H - 1));
    const float fx0 = floorf(ix), fy0 = floorf(iy);
    const int x0 = (int)fx0, y0 = (int)fy0, x1 = x0 + 1, y1 = y0 + 1;
    const float wx1 = ix - fx0, wy1 = iy - fy0, wx0 = 1.f - wx1, wy0 = 1.f - wy1;
    const bool vx1 = x1 <= W - 1, vy1 = y1 <= H - 1;
    BorderBilinear s;
    s.p00 = b + ((int64_t)y0 * W + x0) * ldx;
    s.p01 = b + ((int64_t)y0 * W + (vx1 ? x1 : x0)) * ldx;
    s.p10 = b + ((int64_t)(vy1 ? y1 : y0) * W + x0) * ldx;
    s.p11 = b + ((int64_t)(vy1 ? y1 : y0) * W + (vx1 ? x1 : x0)) * ldx;
    s.w00 = wx0 * wy0; s.w01 = vx1 ? wx1 * wy0 : 0.f; s.w10 = vy1 ? wx0 * wy1 : 0.f; s.w11 = (vx1 && vy1) ? wx1 * wy1 : 0.f;
    return s;
}

// F.grid_sample(x, grid, mode='bilinear', padding_mode='border', align_corners=True) with NHWC input and point-major output:
// out[n][m][c] = bilinear(x[n], grid[n][m] = (gx, gy) in [-1, 1]).  One warp per point, lanes over channels (scalar channels: C need not be a
// multiple of 4 -- the RGB look-up has 3).  eft.py:248-275.
__global__ void grid_sample_kernel(const float* __restrict__ x, int64_t ldx, const float* __restrict__ grid, float* __restrict__ out, int64_t ldo, int H, int W,
                                   int C, int64_t M, int64_t total_pts) {
    const int64_t pt = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
    if (pt >= total_pts) return;
    const int lane = threadIdx.x & 31;
    const int n = (int)(pt / M);
    const BorderBilinear s = border_bilinear(x + (int64_t)n * H * W * ldx, ldx, H, W, __ldg(grid + pt * 2), __ldg(grid + pt * 2 + 1));
    float* o = out + pt * ldo;
    for (int c = lane; c < C; c += 32) o[c] = s(c);
}

// column j of HarmonicEmbedding (utils/common_utils.py:68-140, 6 frequencies f_k = omega0 2^k) over n coordinates v: sin of all (coordinate,
// k) pairs coordinate-major, then cos of all, then the coordinates themselves.  v is indexed by an unrolled select, so it stays in registers.
template <int n>
__device__ __forceinline__ float harmonic(const float (&v)[n], int j, float omega0) {
    constexpr int nf = 6 * n;
    const int q = j >= 2 * nf ? j - 2 * nf : (j % nf) / 6;
    float x = v[0];
#pragma unroll
    for (int i = 1; i < n; ++i) x = q == i ? v[i] : x;
    if (j >= 2 * nf) return x;
    const float a = x * ((float)(1 << (j % nf % 6)) * omega0);
    return j < nf ? sinf(a) : cosf(a);
}

// T1 token rows of the view-batched EFT feature cache: one warp per (camera c, view v, ray n, depth d) row, lanes over the row's columns.
// The point, its projection and the camera centre are computed by every lane (a few dozen flops); each of the row's 91 embedding columns by
// one lane; the latent / image look-ups lanes-over-channels like grid_sample_kernel.  Arithmetic in the order of the eager assembly in
// EpipolarFeatureTransformer.forward (no FMA contraction where the eager ops round twice).
__global__ void __launch_bounds__(256) eft_t1_tokens_kernel(const float* __restrict__ cams, const float* __restrict__ origins,
                                                            const float* __restrict__ directions, const float* __restrict__ lengths,
                                                            const float* __restrict__ latent, int64_t ldl, int h, int w, int C,
                                                            const float* __restrict__ images, int64_t ldi, int H, int W, int Ci, float omega0,
                                                            float* __restrict__ out, int64_t ldo, int V, int NC, int N, int D) {
    const int64_t VND = (int64_t)V * N * D;
    const int64_t row = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= (int64_t)NC * VND) return;
    const int lane = threadIdx.x & 31;
    const int c = (int)(row / VND);
    const int64_t r = row % VND;                       // (v, n, d)
    const int64_t ray = r / D;                         // v * N + n
    const int v = (int)(ray / N);
    const float* cam = cams + ((int64_t)v * NC + c) * 16;
    float R[9], T[3];
#pragma unroll
    for (int i = 0; i < 9; ++i) R[i] = __ldg(cam + i);
#pragma unroll
    for (int i = 0; i < 3; ++i) T[i] = __ldg(cam + 9 + i);
    const float l = __ldg(lengths + r);
    float x[3], oc[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) x[i] = __fadd_rn(__ldg(origins + ray * 3 + i), __fmul_rn(l, __ldg(directions + ray * 3 + i)));
#pragma unroll
    for (int i = 0; i < 3; ++i) oc[i] = -(T[0] * R[i * 3 + 0] + T[1] * R[i * 3 + 1] + T[2] * R[i * 3 + 2]);     // centre = -T R^T
    // reference Pluecker coordinates (u, oc x u), u = normalize(x - oc) (F.normalize, eps 1e-12)
    float u[3] = {__fsub_rn(x[0], oc[0]), __fsub_rn(x[1], oc[1]), __fsub_rn(x[2], oc[2])};
    const float nrm = fmaxf(sqrtf(u[0] * u[0] + u[1] * u[1] + u[2] * u[2]), 1e-12f);
    float pl[6];
#pragma unroll
    for (int i = 0; i < 3; ++i) pl[i] = u[i] / nrm;
    pl[3] = __fsub_rn(__fmul_rn(oc[1], pl[2]), __fmul_rn(oc[2], pl[1]));
    pl[4] = __fsub_rn(__fmul_rn(oc[2], pl[0]), __fmul_rn(oc[0], pl[2]));
    pl[5] = __fsub_rn(__fmul_rn(oc[0], pl[1]), __fmul_rn(oc[1], pl[0]));
    float* o = out + row * ldo;
    const float lv[1] = {l};
    for (int j = lane; j < 91; j += 32) o[j] = j < 78 ? harmonic(pl, j, omega0) : harmonic(lv, j - 78, omega0);
    // NDC projection by camera (v, c): x_view = x R + T, ndc = f x_view.xy / z + p; look-ups at -ndc (eft.py:241-272)
    float xv[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) xv[i] = x[0] * R[0 * 3 + i] + x[1] * R[1 * 3 + i] + x[2] * R[2 * 3 + i] + T[i];
    const float gx = -(__ldg(cam + 12) * xv[0] / xv[2] + __ldg(cam + 14));
    const float gy = -(__ldg(cam + 13) * xv[1] / xv[2] + __ldg(cam + 15));
    const BorderBilinear sl = border_bilinear(latent + (int64_t)c * h * w * ldl, ldl, h, w, gx, gy);
    for (int k = lane; k < C; k += 32) o[91 + k] = sl(k);
    const BorderBilinear si = border_bilinear(images + (int64_t)c * H * W * ldi, ldi, H, W, gx, gy);
    for (int k = lane; k < Ci; k += 32) o[91 + C + k] = si(k);
    for (int64_t k = 91 + C + Ci + lane; k < ldo; k += 32) o[k] = 0.f;
}

// nn.MultiheadAttention core, ONE head, sequence-first layout (nn.TransformerEncoderLayer default): qkv [S][B][3E] (in_proj output: q | k | v),
// out [S][B][E] = softmax(q k^T / sqrt(E)) v over the S positions of batch element b.  One warp per (b, s); S <= 32, E % 128 == 0 handled in
// float4 chunks (E = 256 here).  eft.py:30-33 (n_hidden 256, nhead 1).
constexpr int kSeqMax = 32;
__global__ void __launch_bounds__(256) seq_attention_kernel(const float* __restrict__ qkv, float* __restrict__ out, int S, int B, int E, float scale) {
    const int64_t w = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
    if (w >= (int64_t)S * B) return;
    const int lane = threadIdx.x & 31;
    const int s = (int)(w / B), b = (int)(w % B);
    const int E4 = E >> 2;
    const float4* q = reinterpret_cast<const float4*>(qkv + ((int64_t)s * B + b) * 3 * E);
    float sc[kSeqMax];
    float mx = -INFINITY;
#pragma unroll 1
    for (int t = 0; t < S; ++t) {
        const float4* k = reinterpret_cast<const float4*>(qkv + ((int64_t)t * B + b) * 3 * E + E);
        float d = 0.f;
        for (int e = lane; e < E4; e += 32) {
            const float4 a = __ldg(q + e), c = __ldg(k + e);
            d += a.x * c.x + a.y * c.y + a.z * c.z + a.w * c.w;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
        d *= scale;
        sc[t] = d;
        mx = fmaxf(mx, d);
    }
    float sum = 0.f;
#pragma unroll 1
    for (int t = 0; t < S; ++t) { sc[t] = __expf(sc[t] - mx); sum += sc[t]; }
    const float inv = 1.f / sum;
    float4* o = reinterpret_cast<float4*>(out + ((int64_t)s * B + b) * E);
    for (int e = lane; e < E4; e += 32) {
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
        for (int t = 0; t < S; ++t) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(qkv + ((int64_t)t * B + b) * 3 * E + 2 * E) + e);
            const float p = sc[t];
            acc.x += p * v.x; acc.y += p * v.y; acc.z += p * v.z; acc.w += p * v.w;
        }
        o[e] = make_float4(acc.x * inv, acc.y * inv, acc.z * inv, acc.w * inv);
    }
}

// in place: kind 0 = ReLU (NaN stays NaN, as F.relu), 1 = GELU (erf form, nn.GELU default)
__global__ void act_inplace_kernel(float4* __restrict__ x, int64_t n4, int kind) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        float4 v = x[i];
        if (kind == 0) {
            v.x = max_keep_nan(v.x, 0.f); v.y = max_keep_nan(v.y, 0.f); v.z = max_keep_nan(v.z, 0.f); v.w = max_keep_nan(v.w, 0.f);
        } else {
            v.x = 0.5f * v.x * (1.f + erff(v.x * 0.70710678118654752f)); v.y = 0.5f * v.y * (1.f + erff(v.y * 0.70710678118654752f));
            v.z = 0.5f * v.z * (1.f + erff(v.z * 0.70710678118654752f)); v.w = 0.5f * v.w * (1.f + erff(v.w * 0.70710678118654752f));
        }
        x[i] = v;
    }
}

static inline int blocks_for(int64_t total, int threads = 256) {
    const int64_t cap = (int64_t)sm_count() * 16;
    int64_t b = (total + threads - 1) / threads;
    if (b > cap) b = cap;
    return (int)(b < 1 ? 1 : b);
}

}  // namespace sfb

using namespace sfb;

extern "C" {

int sfb_maxpool3x3s2_nhwc(const float* x, float* y, int NB, int H, int W, int C, void* stream) {
    SFB_REQUIRE(x && y, "maxpool3x3s2: null pointer");
    SFB_REQUIRE(C % 4 == 0, "maxpool3x3s2: C must be a multiple of 4");
    const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
    const int64_t total = (int64_t)NB * Ho * Wo * (C / 4);
    if (total == 0) return SFB_OK;
    maxpool3x3s2_kernel<<<blocks_for(total), 256, 0, as_stream(stream)>>>(reinterpret_cast<const float4*>(x), reinterpret_cast<float4*>(y), H, W, Ho, Wo, C / 4, total);
    return check_launch("maxpool3x3s2");
}

int sfb_resize_bilinear_ac_nhwc(const float* x, int64_t ldx, float* y, int64_t ldo, int NB, int H, int W, int C, int Ho, int Wo, void* stream) {
    SFB_REQUIRE(x && y, "resize_bilinear_ac: null pointer");
    SFB_REQUIRE(C % 4 == 0 && ldx % 4 == 0 && ldo % 4 == 0, "resize_bilinear_ac: channel counts / strides must be multiples of 4");
    const int64_t total = (int64_t)NB * Ho * Wo * (C / 4);
    if (total == 0) return SFB_OK;
    const float sh = Ho > 1 ? (float)(H - 1) / (float)(Ho - 1) : 0.f, sw = Wo > 1 ? (float)(W - 1) / (float)(Wo - 1) : 0.f;
    resize_bilinear_ac_kernel<<<blocks_for(total), 256, 0, as_stream(stream)>>>(x, ldx, y, ldo, H, W, Ho, Wo, C / 4, sh, sw, total);
    return check_launch("resize_bilinear_ac");
}

int sfb_grid_sample_nhwc(const float* x, int64_t ldx, const float* grid, float* out, int64_t ldo, int NB, int H, int W, int C, int64_t M, void* stream) {
    SFB_REQUIRE(x && grid && out, "grid_sample: null pointer");
    const int64_t pts = (int64_t)NB * M;
    if (pts == 0 || C == 0) return SFB_OK;
    grid_sample_kernel<<<(unsigned)ceil_div(pts, (int64_t)8), 256, 0, as_stream(stream)>>>(x, ldx, grid, out, ldo, H, W, C, M, pts);
    return check_launch("grid_sample");
}

int sfb_eft_t1_tokens(const float* cams, const float* origins, const float* directions, const float* lengths, const float* latent, int64_t ldl,
                      int h, int w, int C, const float* images, int64_t ldi, int H, int W, int Ci, float omega0, float* out, int64_t ldo, int V,
                      int NC, int N, int D, void* stream) {
    SFB_REQUIRE(cams && origins && directions && lengths && latent && images && out, "eft_t1_tokens: null pointer");
    SFB_REQUIRE(ldo >= 91 + C + Ci && ldl >= C && ldi >= Ci, "eft_t1_tokens: row stride below 91 + C + Ci, or a channel stride below its channel count");
    SFB_REQUIRE(h >= 1 && w >= 1 && H >= 1 && W >= 1, "eft_t1_tokens: empty latent or image");
    const int64_t rows = (int64_t)NC * V * N * D;
    if (rows == 0) return SFB_OK;
    eft_t1_tokens_kernel<<<(unsigned)ceil_div(rows, (int64_t)8), 256, 0, as_stream(stream)>>>(cams, origins, directions, lengths, latent, ldl, h, w, C,
                                                                                              images, ldi, H, W, Ci, omega0, out, ldo, V, NC, N, D);
    return check_launch("eft_t1_tokens");
}

int sfb_seq_attention(const float* qkv, float* out, int S, int B, int E, void* stream) {
    SFB_REQUIRE(qkv && out, "seq_attention: null pointer");
    SFB_REQUIRE(S >= 1 && S <= kSeqMax && E % 4 == 0, "seq_attention: 1 <= S <= 32 positions, E a multiple of 4");
    const int64_t warps = (int64_t)S * B;
    if (warps == 0) return SFB_OK;
    seq_attention_kernel<<<(unsigned)ceil_div(warps, (int64_t)8), 256, 0, as_stream(stream)>>>(qkv, out, S, B, E, 1.f / sqrtf((float)E));
    return check_launch("seq_attention");
}

int sfb_act_inplace(float* x, int64_t n, int kind, void* stream) {
    SFB_REQUIRE(x && (kind == 0 || kind == 1), "act_inplace: null pointer or unknown activation");
    SFB_REQUIRE(n % 4 == 0, "act_inplace: element count must be a multiple of 4");
    if (n == 0) return SFB_OK;
    act_inplace_kernel<<<blocks_for(n / 4), 256, 0, as_stream(stream)>>>(reinterpret_cast<float4*>(x), n / 4, kind);
    return check_launch("act_inplace");
}
}
