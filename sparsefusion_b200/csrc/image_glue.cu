// image_glue.cu -- SURVEY.md section 8f row 2: ray generation and the image-space glue of a distillation step as fused kernels.
//
// The reference does this with ~50 eager PyTorch launches per sub-step (sparsefusion/distillation.py:201-241, :274-288, :307-344,
// utils/common_utils.py:183-190, utils/render_utils.py:40-47): reshape / permute of the rendered [N,3] image to NCHW, nearest x0.5 of the
// input view, huber, means, opacity regulariser, bilinear x2 up-sampling, L1 * (1 - alpha_bar), and autograd's backward of all of that.
// Here each sub-step's loss is ONE forward kernel (the up-sampled NCHW image for the VAE where needed) and ONE kernel that produces the
// loss value together with d loss / d image and d loss / d weights_sum -- the two tensors the render's backward consumes.
//
// Conventions: rendered image `img` [h*w, 3] (pixel-major, as NeRFRenderer.run returns it), opacity `sil` [h*w]; full-resolution tensors
// are NCHW planes [C][H][W] of ONE view.  huber(x, y) = (sqrt(1 + (x-y)^2 / s^2) - 1) * s with s = 0.1 (common_utils.py:183-190; the clamp
// at 1e-4 never binds because the radicand is >= 1).  F.interpolate(..., scale_factor=0.5) is 'nearest': out[i] = in[2 i].
// F.interpolate(..., scale_factor=2, mode='bilinear') has align_corners=False: src = (dst + 0.5) / 2 - 0.5 clamped at 0.
#include "common.cuh"
#include "../../include/sparsefusion_b200.h"

namespace sfb {

constexpr float kHuberS = 0.1f;

__device__ __forceinline__ float huber_val(float d) { return (sqrtf(1.f + d * d / (kHuberS * kHuberS)) - 1.f) * kHuberS; }
__device__ __forceinline__ float huber_grad(float d) { return d / (kHuberS * sqrtf(1.f + d * d / (kHuberS * kHuberS))); }

__device__ __forceinline__ float block_sum_256(float v, float* sh) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    float t = 0.f;
    if (threadIdx.x < 8) t = sh[threadIdx.x];
    if (threadIdx.x < 32) {
        for (int o = 4; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    }
    __syncthreads();
    return t;   // valid in thread 0
}

// rays of a pixel-centre NDC grid (utils/render_utils.py:40-47; directions un-normalised, plane at depth 1, as pytorch3d's ray sampler):
// d = (x / f, y / f, 1) . R with rows of R = (right, up, forward), o = camera centre.  cam = centre[3] | R[9].
__global__ void rays_from_camera_kernel(const float* __restrict__ cam, int H, int W, float focal, float* __restrict__ rays_o, float* __restrict__ rays_d) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= H * W) return;
    const int py = i / W, px = i - py * W;
    // np.linspace(1 - 1/W, -1 + 1/W, W): start + k * step with step = (stop - start) / (W - 1)
    // evaluated in fp64 and rounded once, like numpy does for a float32 linspace
    const double x0 = 1.0 - 1.0 / W, y0 = 1.0 - 1.0 / H;
    const float xs = (float)(W > 1 ? x0 + px * ((-x0 - x0) / (double)(W - 1)) : x0);
    const float ys = (float)(H > 1 ? y0 + py * ((-y0 - y0) / (double)(H - 1)) : y0);
    const float dx = xs / focal, dy = ys / focal;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        rays_o[i * 3 + k] = cam[k];
        rays_d[i * 3 + k] = dx * cam[3 + k] + dy * cam[6 + k] + cam[9 + k];
    }
}

// Entropy regulariser (distillation.py:236-241, :338-344): a = clamp(s, 1e-5, 1 - 1e-5), H = -a log2 a - (1 - a) log2 (1 - a).
// Returns H and sets dH/ds = log2((1 - a) / a) inside [1e-5, 1 - 1e-5] and 0 outside, as autograd's clamp backward gives (it passes the
// gradient at the bounds themselves).  The bounds are the fp32 values torch compares an fp32 tensor with; a NaN s gives a NaN H.
constexpr float kEntLo = 1e-5f, kEntHi = 0.99999f;

__device__ __forceinline__ float entropy_val_grad(float s, float& grad) {
    const float a = s < kEntLo ? kEntLo : (s > kEntHi ? kEntHi : s);
    const float l0 = log2f(a), l1 = log2f(1.f - a);
    grad = (s >= kEntLo && s <= kEntHi) ? l1 - l0 : 0.f;
    return -a * l0 - (1.f - a) * l1;
}

// Photometric sub-step (distillation.py:210-234): loss = lc * mean huber(img, rgb[::2]) + ls * mean huber(sil, mask[::2]) + lo * mean sqrt(sil^2 + .01)
// (kEnt: + le * mean H(sil), :236-241).  sums[0..2] += (sum huber colour, sum huber silhouette, sum opacity), kEnt: sums[3] += sum H;
// gradients written directly (they do not depend on the sums).
template <bool kEnt>
__global__ void __launch_bounds__(256) photometric_loss_kernel(const float* __restrict__ img, const float* __restrict__ sil, const float* __restrict__ rgb,
                                                              const float* __restrict__ mask, int h, int w, int scale, float lc, float ls, float lo,
                                                              float le, float* __restrict__ sums, float* __restrict__ g_img, float* __restrict__ g_sil) {
    __shared__ float sh[8];
    const int n = h * w, Hf = h * scale, Wf = w * scale;
    float s_c = 0.f, s_s = 0.f, s_o = 0.f, s_e = 0.f;
    for (int i = blockIdx.x * 256 + threadIdx.x; i < n; i += gridDim.x * 256) {
        const int y = i / w, x = i - y * w;
        const int src = (y * scale) * Wf + x * scale;
        float gc[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float d = img[i * 3 + c] - __ldg(rgb + (size_t)c * Hf * Wf + src);
            s_c += huber_val(d);
            gc[c] = lc * huber_grad(d) / (3.f * n);
        }
        const float sv = sil[i];
        const float dm = sv - __ldg(mask + src);
        s_s += huber_val(dm);
        const float op = sqrtf(sv * sv + 0.01f);
        s_o += op;
        g_img[i * 3 + 0] = gc[0]; g_img[i * 3 + 1] = gc[1]; g_img[i * 3 + 2] = gc[2];
        float gs = ls * huber_grad(dm) / n + lo * sv / (op * n);
        if constexpr (kEnt) {
            float dh;
            s_e += entropy_val_grad(sv, dh);
            gs += le * dh / n;
        }
        g_sil[i] = gs;
    }
    const float a = block_sum_256(s_c, sh), b = block_sum_256(s_s, sh), c = block_sum_256(s_o, sh);
    if (threadIdx.x == 0) { atomicAdd(sums + 0, a); atomicAdd(sums + 1, b); atomicAdd(sums + 2, c); }
    if constexpr (kEnt) {
        const float e = block_sum_256(s_e, sh);
        if (threadIdx.x == 0) atomicAdd(sums + 3, e);
    }
}

// bilinear x2 (align_corners = False) source taps of destination index d in a length-n axis: i0, i1, weight of i1
__device__ __forceinline__ void up2_taps(int d, int n, int& i0, int& i1, float& l1) {
    float s = (d + 0.5f) * 0.5f - 0.5f;
    if (s < 0.f) s = 0.f;
    i0 = (int)s;
    i1 = i0 + (i0 < n - 1 ? 1 : 0);
    l1 = s - (float)i0;
}

// up [4][2h][2w] NCHW: channels 0..2 = bilinear x2 of the rendered image, channel 3 = of the opacity   (distillation.py:287-288)
__global__ void upsample2x_render_kernel(const float* __restrict__ img, const float* __restrict__ sil, int h, int w, float* __restrict__ up) {
    const int H2 = 2 * h, W2 = 2 * w;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= H2 * W2) return;
    const int Y = i / W2, X = i - Y * W2;
    int y0, y1, x0, x1;
    float ly, lx;
    up2_taps(Y, h, y0, y1, ly);
    up2_taps(X, w, x0, x1, lx);
    const float w00 = (1.f - ly) * (1.f - lx), w01 = (1.f - ly) * lx, w10 = ly * (1.f - lx), w11 = ly * lx;
    const int p00 = y0 * w + x0, p01 = y0 * w + x1, p10 = y1 * w + x0, p11 = y1 * w + x1;
#pragma unroll
    for (int c = 0; c < 3; ++c)
        up[(size_t)c * H2 * W2 + i] = w00 * img[p00 * 3 + c] + w01 * img[p01 * 3 + c] + w10 * img[p10 * 3 + c] + w11 * img[p11 * 3 + c];
    up[(size_t)3 * H2 * W2 + i] = w00 * sil[p00] + w01 * sil[p01] + w10 * sil[p10] + w11 * sil[p11];
}

// Fusion sub-step loss at full resolution, forward value + gradient w.r.t. the UP-SAMPLED planes (distillation.py:310, :316-329, :336-344):
//   mode 0 (SDS):  loss = wgt * mean |up_rgb - target| + lo * mean sqrt(up_sil^2 + .01)                  (wgt = 1 - alpha_bar)
//   mode 1 (EFT bootstrap): loss = lc * mean huber(up_rgb, target) + ls * mean huber(up_sil, tmask) + lo * mean sqrt(up_sil^2 + .01),
//                           tmask = (mean_c target > 0.1)                                                  (distillation.py:269-271)
//   kEnt: + le * mean H(up_sil) in either mode (:338-344)
// g_up [4][H][W] receives d loss / d up; sums[0..2] += (sum colour term, sum silhouette term, sum opacity term), kEnt: sums[3] += sum H.
template <bool kEnt>
__global__ void __launch_bounds__(256) fusion_loss_kernel(const float* __restrict__ up, const float* __restrict__ target, int HW, int mode, float wgt,
                                                         float lc, float ls, float lo, float le, const float* __restrict__ g_extra,
                                                         float* __restrict__ sums, float* __restrict__ g_up) {
    __shared__ float sh[8];
    float s_c = 0.f, s_s = 0.f, s_o = 0.f, s_e = 0.f;
    for (int i = blockIdx.x * 256 + threadIdx.x; i < HW; i += gridDim.x * 256) {
        const float t0 = __ldg(target + i), t1 = __ldg(target + HW + i), t2 = __ldg(target + 2 * (size_t)HW + i);
        const float tv[3] = {t0, t1, t2};
        const float sv = up[3 * (size_t)HW + i];
        const float op = sqrtf(sv * sv + 0.01f);
        s_o += op;
        float gs = lo * sv / (op * HW);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float d = up[(size_t)c * HW + i] - tv[c];
            const float ge = g_extra != nullptr ? __ldg(g_extra + (size_t)c * HW + i) : 0.f;   // e.g. the perceptual term's gradient
            if (mode == 0) {
                s_c += fabsf(d);
                g_up[(size_t)c * HW + i] = wgt * (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f)) / (3.f * HW) + ge;
            } else {
                s_c += huber_val(d);
                g_up[(size_t)c * HW + i] = lc * huber_grad(d) / (3.f * HW) + ge;
            }
        }
        if (mode == 1) {
            const float m = ((t0 + t1 + t2) / 3.f > 0.1f) ? 1.f : 0.f;
            const float dm = sv - m;
            s_s += huber_val(dm);
            gs += ls * huber_grad(dm) / HW;
        }
        if constexpr (kEnt) {
            float dh;
            s_e += entropy_val_grad(sv, dh);
            gs += le * dh / HW;
        }
        g_up[3 * (size_t)HW + i] = gs;
    }
    const float a = block_sum_256(s_c, sh), b = block_sum_256(s_s, sh), c = block_sum_256(s_o, sh);
    if (threadIdx.x == 0) { atomicAdd(sums + 0, a); atomicAdd(sums + 1, b); atomicAdd(sums + 2, c); }
    if constexpr (kEnt) {
        const float e = block_sum_256(s_e, sh);
        if (threadIdx.x == 0) atomicAdd(sums + 3, e);
    }
}

// adjoint of upsample2x_render_kernel: g_img[p][c] = sum over the <= 16 destination pixels that read p of weight * g_up
__global__ void upsample2x_render_backward_kernel(const float* __restrict__ g_up, int h, int w, float* __restrict__ g_img, float* __restrict__ g_sil) {
    const int H2 = 2 * h, W2 = 2 * w;
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= h * w) return;
    const int y = p / w, x = p - y * w;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int Y = max(0, 2 * y - 2); Y <= min(H2 - 1, 2 * y + 3); ++Y) {
        int y0, y1;
        float ly;
        up2_taps(Y, h, y0, y1, ly);
        const float wy = (y0 == y ? 1.f - ly : 0.f) + (y1 == y ? ly : 0.f);
        if (wy == 0.f) continue;
        for (int X = max(0, 2 * x - 2); X <= min(W2 - 1, 2 * x + 3); ++X) {
            int x0, x1;
            float lx;
            up2_taps(X, w, x0, x1, lx);
            const float wx = (x0 == x ? 1.f - lx : 0.f) + (x1 == x ? lx : 0.f);
            if (wx == 0.f) continue;
            const float ww = wy * wx;
            const int i = Y * W2 + X;
#pragma unroll
            for (int c = 0; c < 4; ++c) acc[c] += ww * __ldg(g_up + (size_t)c * H2 * W2 + i);
        }
    }
    g_img[p * 3 + 0] = acc[0]; g_img[p * 3 + 1] = acc[1]; g_img[p * 3 + 2] = acc[2];
    g_sil[p] = acc[3];
}

}  // namespace sfb

using namespace sfb;

extern "C" {

int sfb_rays_from_camera(const float* cam, int H, int W, float focal_ndc, float* rays_o, float* rays_d, void* stream) {
    SFB_REQUIRE(cam && rays_o && rays_d, "rays_from_camera: null pointer");
    SFB_REQUIRE(H > 0 && W > 0 && focal_ndc > 0.f, "rays_from_camera: bad image size or focal length");
    rays_from_camera_kernel<<<ceil_div(H * W, 256), 256, 0, as_stream(stream)>>>(cam, H, W, focal_ndc, rays_o, rays_d);
    return check_launch("rays_from_camera");
}

int sfb_photometric_loss(const float* img, const float* sil, const float* rgb, const float* mask, int h, int w, int scale, float lambda_color,
                         float lambda_sil, float lambda_opacity, float* sums, float* g_img, float* g_sil, void* stream) {
    SFB_REQUIRE(img && sil && rgb && mask && sums && g_img && g_sil, "photometric_loss: null pointer");
    SFB_REQUIRE(h > 0 && w > 0 && scale >= 1, "photometric_loss: bad sizes");
    cudaStream_t st = as_stream(stream);
    SFB_CUDA(cudaMemsetAsync(sums, 0, 3 * sizeof(float), st));
    const int blocks = min(ceil_div(h * w, 256), sm_count() * 2);
    photometric_loss_kernel<false><<<blocks, 256, 0, st>>>(img, sil, rgb, mask, h, w, scale, lambda_color, lambda_sil, lambda_opacity, 0.f, sums, g_img,
                                                           g_sil);
    return check_launch("photometric_loss");
}

int sfb_photometric_loss_ent(const float* img, const float* sil, const float* rgb, const float* mask, int h, int w, int scale, float lambda_color,
                             float lambda_sil, float lambda_opacity, float lambda_entropy, float* sums, float* g_img, float* g_sil, void* stream) {
    SFB_REQUIRE(img && sil && rgb && mask && sums && g_img && g_sil, "photometric_loss_ent: null pointer");
    SFB_REQUIRE(h > 0 && w > 0 && scale >= 1, "photometric_loss_ent: bad sizes");
    cudaStream_t st = as_stream(stream);
    SFB_CUDA(cudaMemsetAsync(sums, 0, 4 * sizeof(float), st));
    const int blocks = min(ceil_div(h * w, 256), sm_count() * 2);
    photometric_loss_kernel<true><<<blocks, 256, 0, st>>>(img, sil, rgb, mask, h, w, scale, lambda_color, lambda_sil, lambda_opacity, lambda_entropy,
                                                          sums, g_img, g_sil);
    return check_launch("photometric_loss_ent");
}

int sfb_upsample2x_render(const float* img, const float* sil, int h, int w, float* up, void* stream) {
    SFB_REQUIRE(img && sil && up, "upsample2x_render: null pointer");
    SFB_REQUIRE(h > 0 && w > 0, "upsample2x_render: bad sizes");
    upsample2x_render_kernel<<<ceil_div(4 * h * w, 256), 256, 0, as_stream(stream)>>>(img, sil, h, w, up);
    return check_launch("upsample2x_render");
}

int sfb_fusion_loss(const float* up, const float* target, int H, int W, int mode, float weight, float lambda_color, float lambda_sil,
                    float lambda_opacity, float* sums, float* g_up, int h, int w, float* g_img, float* g_sil, void* stream) {
    return sfb_fusion_loss_ex(up, target, H, W, mode, weight, lambda_color, lambda_sil, lambda_opacity, nullptr, sums, g_up, h, w, g_img, g_sil, stream);
}

int sfb_fusion_loss_ex(const float* up, const float* target, int H, int W, int mode, float weight, float lambda_color, float lambda_sil,
                       float lambda_opacity, const float* g_extra, float* sums, float* g_up, int h, int w, float* g_img, float* g_sil, void* stream) {
    SFB_REQUIRE(up && target && sums && g_up && g_img && g_sil, "fusion_loss: null pointer");
    SFB_REQUIRE(H == 2 * h && W == 2 * w && h > 0 && w > 0 && (mode == 0 || mode == 1), "fusion_loss: the full-resolution planes must be 2x the render");
    cudaStream_t st = as_stream(stream);
    SFB_CUDA(cudaMemsetAsync(sums, 0, 3 * sizeof(float), st));
    const int blocks = min(ceil_div(H * W, 256), sm_count() * 2);
    fusion_loss_kernel<false><<<blocks, 256, 0, st>>>(up, target, H * W, mode, weight, lambda_color, lambda_sil, lambda_opacity, 0.f, g_extra, sums,
                                                      g_up);
    if (int rc = check_launch("fusion_loss(value)")) return rc;
    upsample2x_render_backward_kernel<<<ceil_div(h * w, 256), 256, 0, st>>>(g_up, h, w, g_img, g_sil);
    return check_launch("fusion_loss(adjoint)");
}

int sfb_fusion_loss_ent(const float* up, const float* target, int H, int W, int mode, float weight, float lambda_color, float lambda_sil,
                        float lambda_opacity, float lambda_entropy, const float* g_extra, float* sums, float* g_up, int h, int w, float* g_img,
                        float* g_sil, void* stream) {
    SFB_REQUIRE(up && target && sums && g_up && g_img && g_sil, "fusion_loss_ent: null pointer");
    SFB_REQUIRE(H == 2 * h && W == 2 * w && h > 0 && w > 0 && (mode == 0 || mode == 1), "fusion_loss_ent: the full-resolution planes must be 2x the render");
    cudaStream_t st = as_stream(stream);
    SFB_CUDA(cudaMemsetAsync(sums, 0, 4 * sizeof(float), st));
    const int blocks = min(ceil_div(H * W, 256), sm_count() * 2);
    fusion_loss_kernel<true><<<blocks, 256, 0, st>>>(up, target, H * W, mode, weight, lambda_color, lambda_sil, lambda_opacity, lambda_entropy, g_extra,
                                                     sums, g_up);
    if (int rc = check_launch("fusion_loss_ent(value)")) return rc;
    upsample2x_render_backward_kernel<<<ceil_div(h * w, 256), 256, 0, st>>>(g_up, h, w, g_img, g_sil);
    return check_launch("fusion_loss_ent(adjoint)");
}
}
