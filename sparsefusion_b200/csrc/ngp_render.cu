// ngp_render.cu -- the per-ray stages of NeRFRenderer.run (external/nerf/renderer_df.py:310-468), fused for sm_90a.
//
// The reference expresses these as ~120 eager PyTorch launches per render (linspace / rand / cumprod / searchsorted /
// gather / sort / sum ...), all on [N,64] or [N,128] tensors.  Here one WARP owns one ray and keeps the ray's samples in
// registers / a few hundred bytes of shared memory:
//   ray_coarse_z      near/far (slab test) + 64 stratified depths                                  (:328, :356-364)
//   ray_resample      coarse weights -> pdf/cdf (warp scans) -> 64 inverse-CDF samples -> rank-merge with the 64
//                     coarse depths into 128 sorted depths                                         (:381-395, :15-49, :404-405)
//   ray_composite     alpha compositing of the 128 sorted samples: weights, image, depth, opacity  (:414-456)
//   ray_composite_bwd analytic gradient of the compositing w.r.t. sigma and rgb (what autograd derives through
//                     cumprod in the reference), via one forward and one reverse warp scan
// The field itself (grid encode + MLP) is evaluated between these stages by ngp_field.cu directly from the depths
// (x = clamp(o + d*z)), so no [N,128,3] point tensor ever exists.  fp32 throughout; every product/sum that the
// reference performs as separate torch ops is kept un-fused (__fmul_rn/__fadd_rn) where it decides sample positions.
// Every random number the reference draws (torch.rand at :363 and :31) is an INPUT, so parity tests can inject the
// oracle's noise; in production the host module draws them with torch.rand exactly like the reference.
#include "common.cuh"
#include "raymarching.cuh"
#include "../../include/sparsefusion_b200.h"

namespace sfb {

constexpr int kTc = 64;   // coarse samples per ray (opt.num_steps)
constexpr int kTf = 64;   // importance samples per ray (opt.upsample_steps)
constexpr int kT = kTc + kTf;
constexpr int kWarpsPerBlock = 4;

__device__ __forceinline__ float wscan_add(float v, int lane) {  // inclusive warp prefix sum
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const float n = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += n;
    }
    return v;
}
__device__ __forceinline__ float wscan_mul(float v, int lane) {  // inclusive warp prefix product
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const float n = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v *= n;
    }
    return v;
}
__device__ __forceinline__ float wsum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// ------------------------------------------------------------------------------------------------ coarse depths
// one thread per (ray, sample): z = near + (far - near) * lin[t] (+ (noise - 0.5) * (far - near) / Tc)
__global__ void __launch_bounds__(256) ray_coarse_z_kernel(const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                                                          const float* __restrict__ aabb, float min_near, const float* __restrict__ lin,
                                                          const float* __restrict__ noise, uint32_t N, float* __restrict__ nears,
                                                          float* __restrict__ fars, float* __restrict__ z) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N * kTc) return;
    const uint32_t n = i / kTc, t = i - n * kTc;
    float near, far;
    ray_aabb(rays_o + (size_t)n * 3, rays_d + (size_t)n * 3, aabb, min_near, near, far);
    if (t == 0) { nears[n] = near; fars[n] = far; }
    const float span = __fsub_rn(far, near);
    float zz = __fadd_rn(near, __fmul_rn(span, lin[t]));
    if (noise) zz = __fadd_rn(zz, __fmul_rn(__fsub_rn(noise[i], 0.5f), __fdiv_rn(span, (float)kTc)));
    z[i] = zz;
}

// ------------------------------------------------------------------------------------------------ resample + merge
// warp per ray.  lane holds coarse samples 2*lane, 2*lane+1.
__global__ void __launch_bounds__(kWarpsPerBlock * 32) ray_resample_kernel(const float* __restrict__ z_coarse, const float* __restrict__ sigma_c,
                                                                          const float* __restrict__ nears, const float* __restrict__ fars,
                                                                          const float* __restrict__ u_in, int det, uint32_t N,
                                                                          float* __restrict__ z_sorted, float* __restrict__ z_new,
                                                                          uint8_t* __restrict__ src_of) {
    __shared__ float s_zc[kWarpsPerBlock][kTc];
    __shared__ float s_mid[kWarpsPerBlock][kTc];
    __shared__ float s_cdf[kWarpsPerBlock][kTc];
    __shared__ float s_zf[kWarpsPerBlock][kTf];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t n = blockIdx.x * kWarpsPerBlock + warp;
    if (n >= N) return;
    float* zc = s_zc[warp];
    float* mid = s_mid[warp];
    float* cdf = s_cdf[warp];
    float* zf = s_zf[warp];
    const float sample_dist = __fdiv_rn(__fsub_rn(fars[n], nears[n]), (float)kTc);

    const float2 zz = *reinterpret_cast<const float2*>(z_coarse + (size_t)n * kTc + 2 * lane);
    const float2 sg = *reinterpret_cast<const float2*>(sigma_c + (size_t)n * kTc + 2 * lane);
    zc[2 * lane] = zz.x;
    zc[2 * lane + 1] = zz.y;
    __syncwarp();
    // deltas (renderer_df.py:383-384)
    const float d0 = __fsub_rn(zz.y, zz.x);
    const float d1 = (lane < 31) ? __fsub_rn(zc[2 * lane + 2], zz.y) : sample_dist;
    // alphas, transmittance, weights (:386-388)
    const float a0 = 1.f - expf(-d0 * sg.x), a1 = 1.f - expf(-d1 * sg.y);
    const float s0 = 1.f - a0 + 1e-15f, s1 = 1.f - a1 + 1e-15f;
    const float incl = wscan_mul(s0 * s1, lane);                 // prod of shifted alphas up to and including element 2*lane+1
    float excl = __shfl_up_sync(0xffffffffu, incl, 1);
    if (lane == 0) excl = 1.f;                                   // T before element 2*lane
    const float w0 = a0 * excl, w1 = a1 * (excl * s0);
    // bin mid points (:391): z_mid[t] = z[t] + 0.5 * delta[t], t < 63
    mid[2 * lane] = __fadd_rn(zz.x, __fmul_rn(0.5f, d0));
    mid[2 * lane + 1] = __fadd_rn(zz.y, __fmul_rn(0.5f, d1));   // index 63 is never read
    // pdf over weights[1:-1] (62 bins) and its cdf with a leading zero: cdf[0..62]
    const float p0 = (lane >= 1) ? w0 + 1e-5f : 0.f;             // element 2*lane   participates for t in [1,62]
    const float p1 = (lane <= 30) ? w1 + 1e-5f : 0.f;            // element 2*lane+1 participates for t in [1,62]
    const float total = wsum(p0 + p1);
    const float q0 = p0 / total, q1 = p1 / total;
    const float run = wscan_add(q0 + q1, lane);                  // cumulative through element 2*lane+1
    // cdf[k] = sum of pdf[0..k-1], pdf index k-1 <-> weight element k  => cdf[t] = cumulative through element t (t>=1), cdf[0] = 0
    if (lane == 0) cdf[0] = 0.f;
    if (lane >= 1) cdf[2 * lane] = run - q1;                     // through element 2*lane
    if (lane <= 30) cdf[2 * lane + 1] = run;                     // through element 2*lane+1 (t = 63 excluded)
    __syncwarp();
    // inverse CDF (:26-47): two samples per lane
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int j = 2 * lane + r;
        const float u = det ? (0.5f / kTf + j * ((1.f - 1.f / kTf) / (kTf - 1))) : u_in[(size_t)n * kTf + j];
        // searchsorted(cdf, u, right=True): number of entries <= u, over cdf[0..62]
        int lo = 0, hi = kTc - 1;
        while (lo < hi) {
            const int m = (lo + hi) >> 1;
            if (cdf[m] <= u) lo = m + 1; else hi = m;
        }
        const int below = max(lo - 1, 0), above = min(lo, kTc - 2);
        const float cb = cdf[below], ca = cdf[above];
        const float bb = mid[below], ba = mid[above];
        float denom = __fsub_rn(ca, cb);
        if (denom < 1e-5f) denom = 1.f;
        const float tt = __fdiv_rn(__fsub_rn(u, cb), denom);
        zf[j] = __fadd_rn(bb, __fmul_rn(tt, __fsub_rn(ba, bb)));
    }
    __syncwarp();
    // rank merge of the 64 coarse and 64 fine depths (torch.sort at :405; ties: coarse first, then by index)
    float* out = z_sorted + (size_t)n * kT;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int t = 2 * lane + r;
        const float c = zc[t], f = zf[t];
        int pc = t, pf = 0;
        for (int j = 0; j < kTf; ++j) {
            const float fj = zf[j], cj = zc[j];
            pc += (fj < c);
            pf += (cj <= f);
            pf += (fj < f) || (fj == f && j < t);
        }
        out[pc] = c;
        out[pf] = f;
        if (src_of != nullptr) {   // where each sorted slot came from: coarse sample t (< 64) or importance sample t (64 + t)
            src_of[(size_t)n * kT + pc] = (uint8_t)t;
            src_of[(size_t)n * kT + pf] = (uint8_t)(kTc + t);
        }
        if (z_new != nullptr) z_new[(size_t)n * kTf + t] = f;
    }
}

// sigma / rgb of the 128 sorted samples assembled from the coarse pass (64) and the importance pass (64) through src_of: the field is a pure
// function of the sample position, so the values of the coarse samples need not be evaluated a second time (the reference gathers its coarse
// sigmas the same way, renderer_df.py:405-416).  One thread per sorted sample.
__global__ void ray_gather_sorted_kernel(const uint8_t* __restrict__ src_of, const float* __restrict__ sig_c, const float* __restrict__ rgb_c,
                                         const float* __restrict__ sig_n, const float* __restrict__ rgb_n, uint32_t N, float* __restrict__ sigma,
                                         float* __restrict__ rgb) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)N * kT) return;
    const size_t n = i / kT;
    const int s = src_of[i];
    const bool coarse = s < kTc;
    const size_t j = n * (size_t)kTc + (coarse ? s : s - kTc);
    const float* sp = coarse ? sig_c : sig_n;
    const float* cp = coarse ? rgb_c : rgb_n;
    sigma[i] = sp[j];
    rgb[i * 3 + 0] = cp[j * 3 + 0];
    rgb[i * 3 + 1] = cp[j * 3 + 1];
    rgb[i * 3 + 2] = cp[j * 3 + 2];
}

// ------------------------------------------------------------------------------------------------ compositing
struct RaySamples {  // 4 consecutive samples per lane: t = 4*lane + i
    float z[4], delta[4], alpha[4], T[4], w[4];
};

__device__ __forceinline__ void ray_weights(const float* __restrict__ zrow, const float* __restrict__ srow, float sample_dist, int lane,
                                            RaySamples& r, float (&sig)[4]) {
    const float4 z4 = *reinterpret_cast<const float4*>(zrow + 4 * lane);
    const float4 s4 = *reinterpret_cast<const float4*>(srow + 4 * lane);
    r.z[0] = z4.x; r.z[1] = z4.y; r.z[2] = z4.z; r.z[3] = z4.w;
    sig[0] = s4.x; sig[1] = s4.y; sig[2] = s4.z; sig[3] = s4.w;
    const float znext = __shfl_down_sync(0xffffffffu, r.z[0], 1);
    r.delta[0] = __fsub_rn(r.z[1], r.z[0]);
    r.delta[1] = __fsub_rn(r.z[2], r.z[1]);
    r.delta[2] = __fsub_rn(r.z[3], r.z[2]);
    r.delta[3] = (lane < 31) ? __fsub_rn(znext, r.z[3]) : sample_dist;
    float local = 1.f;
    float sh[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        r.alpha[i] = 1.f - expf(-r.delta[i] * sig[i]);
        sh[i] = 1.f - r.alpha[i] + 1e-15f;
        local *= sh[i];
    }
    const float incl = wscan_mul(local, lane);
    float excl = __shfl_up_sync(0xffffffffu, incl, 1);
    if (lane == 0) excl = 1.f;
    float T = excl;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        r.T[i] = T;
        r.w[i] = r.alpha[i] * T;
        T *= sh[i];
    }
}

__global__ void __launch_bounds__(kWarpsPerBlock * 32) ray_composite_kernel(const float* __restrict__ z_sorted, const float* __restrict__ sigma,
                                                                           const float* __restrict__ rgb, const float* __restrict__ nears,
                                                                           const float* __restrict__ fars, float bg, uint32_t N,
                                                                           float* __restrict__ image, float* __restrict__ depth,
                                                                           float* __restrict__ weights_sum) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t n = blockIdx.x * kWarpsPerBlock + warp;
    if (n >= N) return;
    const float near = nears[n], far = fars[n];
    RaySamples r;
    float sig[4];
    ray_weights(z_sorted + (size_t)n * kT, sigma + (size_t)n * kT, __fdiv_rn(__fsub_rn(far, near), (float)kTc), lane, r, sig);
    const float* c = rgb + ((size_t)n * kT + 4 * lane) * 3;
    float ws = 0.f, dp = 0.f, cr = 0.f, cg = 0.f, cb = 0.f;
    const float inv = 1.f / (far - near);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        ws += r.w[i];
        const float oz = fminf(fmaxf((r.z[i] - near) * inv, 0.f), 1.f);
        dp += r.w[i] * oz;
        cr += r.w[i] * c[i * 3];
        cg += r.w[i] * c[i * 3 + 1];
        cb += r.w[i] * c[i * 3 + 2];
    }
    ws = wsum(ws); dp = wsum(dp); cr = wsum(cr); cg = wsum(cg); cb = wsum(cb);
    if (lane == 0) {
        weights_sum[n] = ws;
        depth[n] = dp;
        image[(size_t)n * 3] = cr + (1.f - ws) * bg;
        image[(size_t)n * 3 + 1] = cg + (1.f - ws) * bg;
        image[(size_t)n * 3 + 2] = cb + (1.f - ws) * bg;
    }
}

// d(loss)/d(sigma_t), d(loss)/d(rgb_t) given d(loss)/d(image), d(loss)/d(weights_sum), d(loss)/d(depth)
__global__ void __launch_bounds__(kWarpsPerBlock * 32) ray_composite_bwd_kernel(const float* __restrict__ z_sorted, const float* __restrict__ sigma,
                                                                               const float* __restrict__ rgb, const float* __restrict__ nears,
                                                                               const float* __restrict__ fars, float bg, uint32_t N,
                                                                               const float* __restrict__ g_image, const float* __restrict__ g_ws,
                                                                               const float* __restrict__ g_depth, float* __restrict__ g_sigma,
                                                                               float* __restrict__ g_rgb) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t n = blockIdx.x * kWarpsPerBlock + warp;
    if (n >= N) return;
    const float near = nears[n], far = fars[n];
    RaySamples r;
    float sig[4];
    ray_weights(z_sorted + (size_t)n * kT, sigma + (size_t)n * kT, __fdiv_rn(__fsub_rn(far, near), (float)kTc), lane, r, sig);
    const float gi0 = g_image[(size_t)n * 3], gi1 = g_image[(size_t)n * 3 + 1], gi2 = g_image[(size_t)n * 3 + 2];
    const float gws = g_ws ? g_ws[n] : 0.f, gdp = g_depth ? g_depth[n] : 0.f;
    const float* c = rgb + ((size_t)n * kT + 4 * lane) * 3;
    float* gc = g_rgb + ((size_t)n * kT + 4 * lane) * 3;
    const float inv = 1.f / (far - near);
    // G_t = dL/dw_t ; local sums of G_t * w_t for the suffix scan
    float G[4], gw[4], local = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float oz = fminf(fmaxf((r.z[i] - near) * inv, 0.f), 1.f);
        G[i] = gi0 * (c[i * 3] - bg) + gi1 * (c[i * 3 + 1] - bg) + gi2 * (c[i * 3 + 2] - bg) + gws + gdp * oz;
        gw[i] = G[i] * r.w[i];
        local += gw[i];
        gc[i * 3] = gi0 * r.w[i];
        gc[i * 3 + 1] = gi1 * r.w[i];
        gc[i * 3 + 2] = gi2 * r.w[i];
    }
    const float incl = wscan_add(local, lane);
    const float total = __shfl_sync(0xffffffffu, incl, 31);
    float suffix = total - incl;  // sum over samples of later lanes
    float4 out;
    float o[4];
#pragma unroll
    for (int i = 3; i >= 0; --i) {
        // dL/dalpha_t = G_t T_t - S_t / (1 - alpha_t + 1e-15),  S_t = sum_{u>t} G_u w_u ;  dalpha/dsigma = delta * exp(-delta*sigma)
        const float sh = 1.f - r.alpha[i] + 1e-15f;
        const float dalpha = G[i] * r.T[i] - suffix / sh;
        o[i] = dalpha * r.delta[i] * (1.f - r.alpha[i]);
        suffix += gw[i];
    }
    out.x = o[0]; out.y = o[1]; out.z = o[2]; out.w = o[3];
    *reinterpret_cast<float4*>(g_sigma + (size_t)n * kT + 4 * lane) = out;
}

}  // namespace sfb

using namespace sfb;

extern "C" {

int sfb_ray_coarse_z(const float* rays_o, const float* rays_d, const float* aabb, float min_near, const float* lin, const float* noise, uint32_t N,
                     uint32_t num_steps, float* nears, float* fars, float* z, void* stream) {
    if (N == 0) return SFB_OK;
    SFB_REQUIRE(rays_o && rays_d && aabb && lin && nears && fars && z, "ray_coarse_z: null pointer");
    SFB_REQUIRE(num_steps == (uint32_t)kTc, "ray_coarse_z: the fused renderer is built for num_steps == 64 (get_default_torch_ngp_opt)");
    ray_coarse_z_kernel<<<ceil_div(N * (uint32_t)kTc, 256u), 256, 0, as_stream(stream)>>>(rays_o, rays_d, aabb, min_near, lin, noise, N, nears, fars, z);
    return check_launch("ray_coarse_z");
}

int sfb_ray_resample(const float* z_coarse, const float* sigma_coarse, const float* nears, const float* fars, const float* u, int det, uint32_t N,
                     uint32_t num_steps, uint32_t upsample_steps, float* z_sorted, void* stream) {
    if (N == 0) return SFB_OK;
    SFB_REQUIRE(z_coarse && sigma_coarse && nears && fars && z_sorted && (det || u), "ray_resample: null pointer");
    SFB_REQUIRE(num_steps == (uint32_t)kTc && upsample_steps == (uint32_t)kTf, "ray_resample: built for 64 + 64 samples per ray");
    ray_resample_kernel<<<ceil_div(N, (uint32_t)kWarpsPerBlock), kWarpsPerBlock * 32, 0, as_stream(stream)>>>(z_coarse, sigma_coarse, nears, fars, u, det,
                                                                                                          N, z_sorted, nullptr, nullptr);
    return check_launch("ray_resample");
}

int sfb_ray_resample_ex(const float* z_coarse, const float* sigma_coarse, const float* nears, const float* fars, const float* u, int det, uint32_t N,
                        uint32_t num_steps, uint32_t upsample_steps, float* z_sorted, float* z_new, uint8_t* src_of, void* stream) {
    if (N == 0) return SFB_OK;
    SFB_REQUIRE(z_coarse && sigma_coarse && nears && fars && z_sorted && z_new && src_of && (det || u), "ray_resample_ex: null pointer");
    SFB_REQUIRE(num_steps == (uint32_t)kTc && upsample_steps == (uint32_t)kTf, "ray_resample_ex: built for 64 + 64 samples per ray");
    ray_resample_kernel<<<ceil_div(N, (uint32_t)kWarpsPerBlock), kWarpsPerBlock * 32, 0, as_stream(stream)>>>(z_coarse, sigma_coarse, nears, fars, u, det,
                                                                                                          N, z_sorted, z_new, src_of);
    return check_launch("ray_resample_ex");
}

int sfb_ray_gather_sorted(const uint8_t* src_of, const float* sigma_coarse, const float* rgb_coarse, const float* sigma_new, const float* rgb_new,
                          uint32_t N, uint32_t T, float* sigma, float* rgb, void* stream) {
    if (N == 0) return SFB_OK;
    SFB_REQUIRE(src_of && sigma_coarse && rgb_coarse && sigma_new && rgb_new && sigma && rgb, "ray_gather_sorted: null pointer");
    SFB_REQUIRE(T == (uint32_t)kT, "ray_gather_sorted: built for 128 samples per ray");
    const size_t total = (size_t)N * kT;
    ray_gather_sorted_kernel<<<(unsigned)((total + 255) / 256), 256, 0, as_stream(stream)>>>(src_of, sigma_coarse, rgb_coarse, sigma_new, rgb_new, N, sigma,
                                                                                            rgb);
    return check_launch("ray_gather_sorted");
}

int sfb_ray_composite_forward(const float* z_sorted, const float* sigma, const float* rgb, const float* nears, const float* fars, float bg_color,
                              uint32_t N, uint32_t T, float* image, float* depth, float* weights_sum, void* stream) {
    if (N == 0) return SFB_OK;
    SFB_REQUIRE(z_sorted && sigma && rgb && nears && fars && image && depth && weights_sum, "ray_composite_forward: null pointer");
    SFB_REQUIRE(T == (uint32_t)kT, "ray_composite_forward: built for 128 samples per ray");
    ray_composite_kernel<<<ceil_div(N, (uint32_t)kWarpsPerBlock), kWarpsPerBlock * 32, 0, as_stream(stream)>>>(z_sorted, sigma, rgb, nears, fars, bg_color,
                                                                                                           N, image, depth, weights_sum);
    return check_launch("ray_composite_forward");
}

int sfb_ray_composite_backward(const float* z_sorted, const float* sigma, const float* rgb, const float* nears, const float* fars, float bg_color,
                               uint32_t N, uint32_t T, const float* grad_image, const float* grad_weights_sum, const float* grad_depth,
                               float* grad_sigma, float* grad_rgb, void* stream) {
    if (N == 0) return SFB_OK;
    SFB_REQUIRE(z_sorted && sigma && rgb && nears && fars && grad_image && grad_sigma && grad_rgb, "ray_composite_backward: null pointer");
    SFB_REQUIRE(T == (uint32_t)kT, "ray_composite_backward: built for 128 samples per ray");
    ray_composite_bwd_kernel<<<ceil_div(N, (uint32_t)kWarpsPerBlock), kWarpsPerBlock * 32, 0, as_stream(stream)>>>(
        z_sorted, sigma, rgb, nears, fars, bg_color, N, grad_image, grad_weights_sum, grad_depth, grad_sigma, grad_rgb);
    return check_launch("ray_composite_backward");
}
}
