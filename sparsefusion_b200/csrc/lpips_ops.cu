// lpips_ops.cu -- SURVEY.md section 8f row 3: the LPIPS-VGG perceptual term of the fusion loss (sparsefusion/distillation.py:312-314 through
// external/external_utils.py:11-49 -> lpips.LPIPS(net='vgg'), Zhang et al. CVPR 2018), forward AND the gradient w.r.t. the rendered image.
//
// The thirteen 3x3 convolutions (and their data-gradient convolutions, same kernel with transposed / flipped weights) run on the wgmma
// implicit-GEMM engine (conv_wgmma.cu); this file holds what surrounds them, all NHWC fp32:
//   lpips_prep        (2 img - 1 - shift) / scale of both images -> [2,H,W,4] (4th channel zero: TMA wants 16-byte pixels)
//   relu              in place
//   maxpool2x2        forward; backward routes the gradient to the first maximum of each window (torch semantics) and applies the ReLU mask of
//                     the layer below in the same pass
//   add_relu_mask     g = (g + g_head) * (act > 0): joins the gradient arriving from the deeper layers with the LPIPS head's at a tap
//   lpips_head        per tap: channel-unit-normalise both feature maps, sum_c w_c (n0 - n1)^2, spatial mean -> value, and d value / d f0
//   lpips_prep_bwd    back to the NCHW [3,H,W] image in [0,1]
#include "common.cuh"
#include "../../include/sparsefusion_b200.h"

namespace sfb {

__constant__ float c_lpips_shift[3] = {-.030f, -.088f, -.188f};
__constant__ float c_lpips_scale[3] = {.458f, .448f, .450f};

static inline int lp_blocks(int64_t total, int threads = 256) {
    int64_t b = (total + threads - 1) / threads;
    const int64_t cap = (int64_t)sm_count() * 16;
    return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

// x [2][H][W][4]: image 0 = pred, image 1 = target, both given as [3][H][W] planes in [0,1]; normalize = (2 v - 1) first (external_utils.py:37-39)
__global__ void lpips_prep_kernel(const float* __restrict__ pred, const float* __restrict__ target, int HW, int normalize, float4* __restrict__ x) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < 2 * HW; i += gridDim.x * blockDim.x) {
        const int n = i / HW, p = i - n * HW;
        const float* src = n == 0 ? pred : target;
        float v[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            float t = __ldg(src + (size_t)c * HW + p);
            if (normalize) t = 2.f * t - 1.f;
            v[c] = (t - c_lpips_shift[c]) / c_lpips_scale[c];
        }
        x[i] = make_float4(v[0], v[1], v[2], 0.f);
    }
}

// g_pred [3][H][W] = factor * gx[0][p][c] * (normalize ? 2 : 1) / scale[c]
__global__ void lpips_prep_bwd_kernel(const float4* __restrict__ gx, int HW, int normalize, float factor, float* __restrict__ g_pred) {
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += gridDim.x * blockDim.x) {
        const float4 g = gx[p];
        const float m = factor * (normalize ? 2.f : 1.f);
        g_pred[p] = g.x * m / c_lpips_scale[0];
        g_pred[(size_t)HW + p] = g.y * m / c_lpips_scale[1];
        g_pred[2 * (size_t)HW + p] = g.z * m / c_lpips_scale[2];
    }
}

__global__ void relu_kernel(float4* __restrict__ x, int64_t n4) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        float4 v = x[i];
        v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
        x[i] = v;
    }
}

// y [NB][H/2][W/2][C] = max over 2x2 windows of x [NB][H][W][C]
__global__ void maxpool2x2_kernel(const float4* __restrict__ x, float4* __restrict__ y, int H, int W, int C4, int64_t total) {
    const int Ho = H >> 1, Wo = W >> 1;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % C4);
        int64_t t = i / C4;
        const int ox = (int)(t % Wo); t /= Wo;
        const int oy = (int)(t % Ho);
        const int64_t n = t / Ho;
        const float4* b = x + ((n * H + 2 * oy) * (int64_t)W + 2 * ox) * C4 + c;
        const float4 a0 = __ldg(b), a1 = __ldg(b + C4), a2 = __ldg(b + (int64_t)W * C4), a3 = __ldg(b + (int64_t)W * C4 + C4);
        y[i] = make_float4(fmaxf(fmaxf(a0.x, a1.x), fmaxf(a2.x, a3.x)), fmaxf(fmaxf(a0.y, a1.y), fmaxf(a2.y, a3.y)),
                           fmaxf(fmaxf(a0.z, a1.z), fmaxf(a2.z, a3.z)), fmaxf(fmaxf(a0.w, a1.w), fmaxf(a2.w, a3.w)));
    }
}

// gx [H][W][C] of ONE image: the window's gradient goes to its FIRST maximum in row-major order (torch.max_pool2d backward), and only if that
// maximum is positive -- x is a post-ReLU activation, so (x > 0) is the ReLU mask of the layer that produced it.  Every gx element is written.
__global__ void maxpool2x2_relu_bwd_kernel(const float* __restrict__ x, const float* __restrict__ gy, float* __restrict__ gx, int H, int W, int C,
                                           int64_t total) {
    const int Ho = H >> 1, Wo = W >> 1;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        int64_t t = i / C;
        const int ox = (int)(t % Wo);
        const int oy = (int)(t / Wo);
        const int64_t b = ((int64_t)(2 * oy) * W + 2 * ox) * C + c;
        const int64_t off[4] = {0, C, (int64_t)W * C, (int64_t)W * C + C};
        float best = __ldg(x + b);
        int arg = 0;
#pragma unroll
        for (int k = 1; k < 4; ++k) {
            const float v = __ldg(x + b + off[k]);
            if (v > best) { best = v; arg = k; }
        }
        const float g = best > 0.f ? __ldg(gy + i) : 0.f;
#pragma unroll
        for (int k = 0; k < 4; ++k) gx[b + off[k]] = (k == arg) ? g : 0.f;
    }
}

// g = (g + (g_head ? g_head : 0)) * (act > 0)
__global__ void add_relu_mask_kernel(float4* __restrict__ g, const float4* __restrict__ g_head, const float4* __restrict__ act, int64_t n4) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        float4 v = g[i];
        if (g_head != nullptr) {
            const float4 h = __ldg(g_head + i);
            v.x += h.x; v.y += h.y; v.z += h.z; v.w += h.w;
        }
        const float4 a = __ldg(act + i);
        v.x = a.x > 0.f ? v.x : 0.f; v.y = a.y > 0.f ? v.y : 0.f; v.z = a.z > 0.f ? v.z : 0.f; v.w = a.w > 0.f ? v.w : 0.f;
        g[i] = v;
    }
}

__device__ __forceinline__ float warp_sum_f(float v) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// One warp per pixel.  f0, f1 [HW][C]; w [C] >= 0.  n = f / (||f|| + 1e-10); value += sum_c w_c (n0 - n1)^2 / HW (atomicAdd into *value);
// g_f0 [HW][C] = d value / d f0 = (dn - n0 (n0 . dn) * (r0 + eps) / r0 ... ) see below, with dn = 2 w (n0 - n1) / HW.
//   n = f / (r + e), r = ||f||:  dL/df = dn / (r + e) - f (f . dn) / (r (r + e)^2)      (the second term vanishes when r == 0)
__global__ void __launch_bounds__(256) lpips_head_kernel(const float* __restrict__ f0, const float* __restrict__ f1, const float* __restrict__ w, int HW,
                                                        int C, float* __restrict__ value, float* __restrict__ g_f0) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float acc = 0.f;
    for (int p = blockIdx.x * 8 + warp; p < HW; p += gridDim.x * 8) {
        const float* a = f0 + (size_t)p * C;
        const float* b = f1 + (size_t)p * C;
        float s0 = 0.f, s1 = 0.f;
        for (int c = lane * 4; c < C; c += 128) {
            const float4 va = __ldg(reinterpret_cast<const float4*>(a + c)), vb = __ldg(reinterpret_cast<const float4*>(b + c));
            s0 += va.x * va.x + va.y * va.y + va.z * va.z + va.w * va.w;
            s1 += vb.x * vb.x + vb.y * vb.y + vb.z * vb.z + vb.w * vb.w;
        }
        s0 = warp_sum_f(s0);
        s1 = warp_sum_f(s1);
        const float r0 = sqrtf(s0), r1 = sqrtf(s1);
        const float i0 = 1.f / (r0 + 1e-10f), i1 = 1.f / (r1 + 1e-10f);
        float val = 0.f, dot = 0.f;   // dot = f0 . dn
        for (int c = lane * 4; c < C; c += 128) {
            const float4 va = __ldg(reinterpret_cast<const float4*>(a + c)), vb = __ldg(reinterpret_cast<const float4*>(b + c));
            const float4 ww = __ldg(reinterpret_cast<const float4*>(w + c));
            const float fa[4] = {va.x, va.y, va.z, va.w}, fb[4] = {vb.x, vb.y, vb.z, vb.w}, wv[4] = {ww.x, ww.y, ww.z, ww.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float d = fa[e] * i0 - fb[e] * i1;
                val += wv[e] * d * d;
                dot += fa[e] * (2.f * wv[e] * d / HW);
            }
        }
        val = warp_sum_f(val);
        dot = warp_sum_f(dot);
        acc += val;
        const float k2 = r0 > 0.f ? dot * i0 * i0 / r0 : 0.f;
        float* g = g_f0 + (size_t)p * C;
        for (int c = lane * 4; c < C; c += 128) {
            const float4 va = __ldg(reinterpret_cast<const float4*>(a + c)), vb = __ldg(reinterpret_cast<const float4*>(b + c));
            const float4 ww = __ldg(reinterpret_cast<const float4*>(w + c));
            const float fa[4] = {va.x, va.y, va.z, va.w}, fb[4] = {vb.x, vb.y, vb.z, vb.w}, wv[4] = {ww.x, ww.y, ww.z, ww.w};
            float o[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float dn = 2.f * wv[e] * (fa[e] * i0 - fb[e] * i1) / HW;
                o[e] = dn * i0 - fa[e] * k2;
            }
            *reinterpret_cast<float4*>(g + c) = make_float4(o[0], o[1], o[2], o[3]);
        }
    }
    __shared__ float sh[8];
    if (lane == 0) sh[warp] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int k = 0; k < 8; ++k) t += sh[k];
        atomicAdd(value, t / HW);
    }
}

}  // namespace sfb

using namespace sfb;

extern "C" {

int sfb_lpips_prep(const float* pred, const float* target, int H, int W, int normalize, float* x, void* stream) {
    SFB_REQUIRE(pred && target && x, "lpips_prep: null pointer");
    SFB_REQUIRE(H > 0 && W > 0 && ((uintptr_t)x & 15) == 0, "lpips_prep: bad size or alignment");
    lpips_prep_kernel<<<lp_blocks(2 * (int64_t)H * W), 256, 0, as_stream(stream)>>>(pred, target, H * W, normalize, reinterpret_cast<float4*>(x));
    return check_launch("lpips_prep");
}

int sfb_lpips_prep_backward(const float* gx, int H, int W, int normalize, float factor, float* g_pred, void* stream) {
    SFB_REQUIRE(gx && g_pred, "lpips_prep_backward: null pointer");
    lpips_prep_bwd_kernel<<<lp_blocks((int64_t)H * W), 256, 0, as_stream(stream)>>>(reinterpret_cast<const float4*>(gx), H * W, normalize, factor, g_pred);
    return check_launch("lpips_prep_backward");
}

int sfb_relu_nhwc(float* x, int64_t n, void* stream) {
    SFB_REQUIRE(x && n % 4 == 0 && ((uintptr_t)x & 15) == 0, "relu_nhwc: needs a 16-byte aligned buffer of a multiple of 4 floats");
    if (n == 0) return SFB_OK;
    relu_kernel<<<lp_blocks(n / 4), 256, 0, as_stream(stream)>>>(reinterpret_cast<float4*>(x), n / 4);
    return check_launch("relu_nhwc");
}

int sfb_maxpool2x2_nhwc(const float* x, float* y, int NB, int H, int W, int C, void* stream) {
    SFB_REQUIRE(x && y, "maxpool2x2_nhwc: null pointer");
    SFB_REQUIRE(H % 2 == 0 && W % 2 == 0 && C % 4 == 0, "maxpool2x2_nhwc: even H, W and C % 4 == 0");
    const int64_t total = (int64_t)NB * (H / 2) * (W / 2) * (C / 4);
    if (total == 0) return SFB_OK;
    maxpool2x2_kernel<<<lp_blocks(total), 256, 0, as_stream(stream)>>>(reinterpret_cast<const float4*>(x), reinterpret_cast<float4*>(y), H, W, C / 4, total);
    return check_launch("maxpool2x2_nhwc");
}

int sfb_maxpool2x2_relu_backward_nhwc(const float* x, const float* gy, float* gx, int H, int W, int C, void* stream) {
    SFB_REQUIRE(x && gy && gx, "maxpool2x2_relu_backward: null pointer");
    SFB_REQUIRE(H % 2 == 0 && W % 2 == 0, "maxpool2x2_relu_backward: even H and W");
    const int64_t total = (int64_t)(H / 2) * (W / 2) * C;
    if (total == 0) return SFB_OK;
    maxpool2x2_relu_bwd_kernel<<<lp_blocks(total), 256, 0, as_stream(stream)>>>(x, gy, gx, H, W, C, total);
    return check_launch("maxpool2x2_relu_backward");
}

int sfb_add_relu_mask(float* g, const float* g_head, const float* act, int64_t n, void* stream) {
    SFB_REQUIRE(g && act && n % 4 == 0, "add_relu_mask: null pointer or length not a multiple of 4");
    if (n == 0) return SFB_OK;
    add_relu_mask_kernel<<<lp_blocks(n / 4), 256, 0, as_stream(stream)>>>(reinterpret_cast<float4*>(g), reinterpret_cast<const float4*>(g_head),
                                                                           reinterpret_cast<const float4*>(act), n / 4);
    return check_launch("add_relu_mask");
}

int sfb_lpips_head(const float* f0, const float* f1, const float* w, int HW, int C, float* value, float* g_f0, void* stream) {
    SFB_REQUIRE(f0 && f1 && w && value && g_f0, "lpips_head: null pointer");
    SFB_REQUIRE(C % 4 == 0 && HW > 0, "lpips_head: C % 4 == 0");
    const int blocks = min((HW + 7) / 8, sm_count() * 8);
    lpips_head_kernel<<<blocks, 256, 0, as_stream(stream)>>>(f0, f1, w, HW, C, value, g_f0);
    return check_launch("lpips_head");
}
}
