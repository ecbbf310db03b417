// ngp_render.cu -- the per-ray stages of NeRFRenderer.run (external/nerf/renderer_df.py:310-468), fused for sm_90a.
//
// The reference expresses these as ~120 eager PyTorch launches per render (linspace / rand / cumprod / searchsorted /
// gather / sort / sum ...), all on [N,Tc], [N,Tf] or [N,Tc+Tf] tensors (Tc = num_steps, Tf = upsample_steps).  Here one WARP
// owns one ray and keeps the ray's samples in registers / at most 4 KB of shared memory:
//   ray_coarse_z      near/far (slab test) + Tc stratified depths                                  (:328, :356-364)
//   ray_resample      coarse weights -> pdf/cdf (warp scans) -> Tf inverse-CDF samples -> rank-merge with the Tc
//                     coarse depths into Tc + Tf sorted depths                                     (:381-395, :15-49, :404-405)
//   ray_composite     alpha compositing of the T sorted samples: weights, image, depth, opacity    (:414-456)
//   ray_composite_bwd analytic gradient of the compositing w.r.t. sigma and rgb (what autograd derives through
//                     cumprod in the reference), via one forward and one reverse warp scan
// The counts are run-time arguments; the kernels are templated on K, the samples each lane holds (lane l holds samples
// K*l .. K*l + K-1), so 64 + 64 resamples with K = 2 and composites 128 samples with K = 4.  Tc + Tf <= 256 (kMaxSamples):
// a sorted slot index fits the uint8 src_of.
// The field itself (grid encode + MLP) is evaluated between these stages by ngp_field.cu directly from the depths
// (x = clamp(o + d*z)), so no [N,T,3] point tensor ever exists.  fp32 throughout; every product/sum that the
// reference performs as separate torch ops is kept un-fused (__fmul_rn/__fadd_rn) where it decides sample positions.
// Every random number the reference draws (torch.rand at :363 and :31) is an INPUT, so parity tests can inject the
// oracle's noise; in production the host module draws them with torch.rand exactly like the reference.
#include "common.cuh"
#include "raymarching.cuh"
#include "../../include/sparsefusion_b200.h"

namespace sfb {

constexpr int kMaxSamples = 256;   // num_steps + upsample_steps: src_of is uint8
constexpr int kMaxK = kMaxSamples / 32;
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

// (far - near) / Tc as torch forms it on CUDA tensors: a division by a Python number is a multiplication by its fp32 reciprocal there
// (exact division when Tc is a power of two)
__device__ __forceinline__ float coarse_spacing(float span, int Tc) { return __fmul_rn(span, __frcp_rn((float)Tc)); }

// ------------------------------------------------------------------------------------------------ coarse depths
// one thread per (ray, sample): z = near + (far - near) * lin[t] (+ (noise - 0.5) * (far - near) / Tc)
__global__ void __launch_bounds__(256) ray_coarse_z_kernel(const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                                                          const float* __restrict__ aabb, float min_near, const float* __restrict__ lin,
                                                          const float* __restrict__ noise, uint32_t N, uint32_t Tc, float* __restrict__ nears,
                                                          float* __restrict__ fars, float* __restrict__ z) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N * Tc) return;
    const uint32_t n = i / Tc, t = i - n * Tc;
    float near, far;
    ray_aabb(rays_o + (size_t)n * 3, rays_d + (size_t)n * 3, aabb, min_near, near, far);
    if (t == 0) { nears[n] = near; fars[n] = far; }
    const float span = __fsub_rn(far, near);
    float zz = __fadd_rn(near, __fmul_rn(span, lin[t]));
    if (noise) zz = __fadd_rn(zz, __fmul_rn(__fsub_rn(noise[i], 0.5f), coarse_spacing(span, (int)Tc)));
    z[i] = zz;
}

// ------------------------------------------------------------------------------------------------ resample + merge
// warp per ray, K >= max(Tc, Tf) / 32: lane holds coarse samples K*lane + i and draws importance samples K*lane + i.  Tc >= 2 when Tf > 0.
template <int K>
__global__ void __launch_bounds__(kWarpsPerBlock * 32) ray_resample_kernel(const float* __restrict__ z_coarse, const float* __restrict__ sigma_c,
                                                                          const float* __restrict__ nears, const float* __restrict__ fars,
                                                                          const float* __restrict__ u_in, int det, uint32_t N, int Tc, int Tf,
                                                                          float* __restrict__ z_sorted, float* __restrict__ z_new,
                                                                          uint8_t* __restrict__ src_of) {
    __shared__ float s_zc[kWarpsPerBlock][32 * K];
    __shared__ float s_mid[kWarpsPerBlock][32 * K];
    __shared__ float s_cdf[kWarpsPerBlock][32 * K];
    __shared__ float s_zf[kWarpsPerBlock][32 * K];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t n = blockIdx.x * kWarpsPerBlock + warp;
    if (n >= N) return;
    float* zc = s_zc[warp];
    float* mid = s_mid[warp];
    float* cdf = s_cdf[warp];
    float* zf = s_zf[warp];
    const int T = Tc + Tf;
    const float sample_dist = coarse_spacing(__fsub_rn(fars[n], nears[n]), Tc);

    float zz[K], a[K], s[K], d[K];
#pragma unroll
    for (int i = 0; i < K; ++i) {
        const int t = K * lane + i;
        zz[i] = (t < Tc) ? z_coarse[(size_t)n * Tc + t] : 0.f;
        zc[t] = zz[i];
    }
    __syncwarp();
    // deltas (renderer_df.py:383-384), alphas and the shifted alphas of the transmittance (:386-388); samples t >= Tc are inert
    float local = 1.f;
#pragma unroll
    for (int i = 0; i < K; ++i) {
        const int t = K * lane + i;
        d[i] = (t < Tc - 1) ? __fsub_rn(zc[t + 1], zz[i]) : sample_dist;
        if (t < Tc) {
            a[i] = 1.f - expf(-d[i] * sigma_c[(size_t)n * Tc + t]);
            s[i] = 1.f - a[i] + 1e-15f;
        } else {
            a[i] = 0.f;
            s[i] = 1.f;
        }
        local *= s[i];
    }
    const float incl = wscan_mul(local, lane);                   // prod of shifted alphas up to and including element K*lane + K-1
    float excl = __shfl_up_sync(0xffffffffu, incl, 1);
    if (lane == 0) excl = 1.f;                                   // T before element K*lane
    // weights; bin mid points (:391): z_mid[t] = z[t] + 0.5 * delta[t], t < Tc-1; pdf over weights[1:-1] (Tc-2 bins, possibly none)
    float p[K], Tr = excl, psum = 0.f;
#pragma unroll
    for (int i = 0; i < K; ++i) {
        const int t = K * lane + i;
        const float w = a[i] * Tr;
        Tr *= s[i];
        mid[t] = __fadd_rn(zz[i], __fmul_rn(0.5f, d[i]));       // indices >= Tc-1 are never read
        p[i] = (t >= 1 && t <= Tc - 2) ? w + 1e-5f : 0.f;
        psum += p[i];
    }
    const float total = wsum(psum);
    float q[K], qsum = 0.f;
#pragma unroll
    for (int i = 0; i < K; ++i) {
        q[i] = p[i] / total;
        qsum += q[i];
    }
    // cdf[k] = sum of pdf[0..k-1], pdf index k-1 <-> weight element k  => cdf[t] = cumulative through element t (1 <= t <= Tc-2), cdf[0] = 0
    float run = wscan_add(qsum, lane);                           // cumulative through element K*lane + K-1
    if (lane == 0) cdf[0] = 0.f;
#pragma unroll
    for (int i = K - 1; i >= 0; --i) {
        const int t = K * lane + i;
        if (t >= 1 && t <= Tc - 2) cdf[t] = run;
        run = run - q[i];
    }
    __syncwarp();
    // inverse CDF (:26-47); with no bins (Tc = 2) every sample lands on z_mid[0], as in the reference
#pragma unroll
    for (int r = 0; r < K; ++r) {
        const int j = K * lane + r;
        if (j >= Tf) break;
        const float u = det ? (Tf > 1 ? 0.5f / Tf + j * ((1.f - 1.f / Tf) / (Tf - 1)) : 0.5f) : u_in[(size_t)n * Tf + j];
        // searchsorted(cdf, u, right=True): number of entries <= u, over cdf[0..Tc-2]
        int lo = 0, hi = Tc - 1;
        while (lo < hi) {
            const int m = (lo + hi) >> 1;
            if (cdf[m] <= u) lo = m + 1; else hi = m;
        }
        const int below = max(lo - 1, 0), above = min(lo, Tc - 2);
        const float cb = cdf[below], ca = cdf[above];
        const float bb = mid[below], ba = mid[above];
        float denom = __fsub_rn(ca, cb);
        if (denom < 1e-5f) denom = 1.f;
        const float tt = __fdiv_rn(__fsub_rn(u, cb), denom);
        zf[j] = __fadd_rn(bb, __fmul_rn(tt, __fsub_rn(ba, bb)));
    }
    __syncwarp();
    // rank merge of the Tc coarse and Tf fine depths (torch.sort at :405; ties: coarse first, then by index).  The coarse depths are sorted.
    float* out = z_sorted + (size_t)n * T;
#pragma unroll
    for (int r = 0; r < K; ++r) {
        const int t = K * lane + r;
        if (t < Tc) {
            const float c = zc[t];
            int pc = t;
            for (int j = 0; j < Tf; ++j) pc += (zf[j] < c);
            out[pc] = c;
            if (src_of != nullptr) src_of[(size_t)n * T + pc] = (uint8_t)t;   // where each sorted slot came from: coarse sample t (< Tc) ...
        }
        if (t < Tf) {
            const float f = zf[t];
            int pf = 0;
            for (int j = 0; j < Tc; ++j) pf += (zc[j] <= f);
            for (int j = 0; j < Tf; ++j) {
                const float fj = zf[j];
                pf += (fj < f) || (fj == f && j < t);
            }
            out[pf] = f;
            if (src_of != nullptr) src_of[(size_t)n * T + pf] = (uint8_t)(Tc + t);   // ... or importance sample t (Tc + t)
            if (z_new != nullptr) z_new[(size_t)n * Tf + t] = f;
        }
    }
}

// sigma / rgb of the T sorted samples assembled from the coarse pass (Tc) and the importance pass (Tf) through src_of: the field is a pure
// function of the sample position, so the values of the coarse samples need not be evaluated a second time (the reference gathers its coarse
// sigmas the same way, renderer_df.py:405-416).  One thread per sorted sample.
__global__ void ray_gather_sorted_kernel(const uint8_t* __restrict__ src_of, const float* __restrict__ sig_c, const float* __restrict__ rgb_c,
                                         const float* __restrict__ sig_n, const float* __restrict__ rgb_n, uint32_t N, uint32_t Tc, uint32_t Tf,
                                         float* __restrict__ sigma, float* __restrict__ rgb) {
    const size_t T = Tc + Tf;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)N * T) return;
    const size_t n = i / T;
    const uint32_t s = src_of[i];
    const bool coarse = s < Tc;
    const size_t j = coarse ? n * Tc + s : n * Tf + (s - Tc);
    const float* sp = coarse ? sig_c : sig_n;
    const float* cp = coarse ? rgb_c : rgb_n;
    sigma[i] = sp[j];
    rgb[i * 3 + 0] = cp[j * 3 + 0];
    rgb[i * 3 + 1] = cp[j * 3 + 1];
    rgb[i * 3 + 2] = cp[j * 3 + 2];
}

// ------------------------------------------------------------------------------------------------ compositing
template <int K>
struct RaySamples {  // K consecutive samples per lane: t = K*lane + i; samples t >= T have alpha 0, weight 0
    float z[K], delta[K], alpha[K], T[K], w[K];
};

// row[K*lane .. K*lane + K-1], zero past T; whole rows of a multiple of 4 samples load as float4
template <int K>
__device__ __forceinline__ void load_lane(const float* __restrict__ row, int T, int lane, float (&v)[K]) {
    if constexpr (K % 4 == 0) {
        if (T == 32 * K) {
#pragma unroll
            for (int i = 0; i < K; i += 4) {
                const float4 q = *reinterpret_cast<const float4*>(row + K * lane + i);
                v[i] = q.x; v[i + 1] = q.y; v[i + 2] = q.z; v[i + 3] = q.w;
            }
            return;
        }
    }
#pragma unroll
    for (int i = 0; i < K; ++i) v[i] = (K * lane + i < T) ? row[K * lane + i] : 0.f;
}

template <int K>
__device__ __forceinline__ void ray_weights(const float* __restrict__ zrow, const float* __restrict__ srow, float sample_dist, int T, int lane,
                                            RaySamples<K>& r, float (&sig)[K]) {
    load_lane<K>(zrow, T, lane, r.z);
    load_lane<K>(srow, T, lane, sig);
    const float znext = __shfl_down_sync(0xffffffffu, r.z[0], 1);
#pragma unroll
    for (int i = 0; i < K; ++i) {
        const float next = (i < K - 1) ? r.z[i + 1] : znext;
        r.delta[i] = (K * lane + i < T - 1) ? __fsub_rn(next, r.z[i]) : sample_dist;
    }
    float local = 1.f;
    float sh[K];
#pragma unroll
    for (int i = 0; i < K; ++i) {
        if (K * lane + i < T) {
            r.alpha[i] = 1.f - expf(-r.delta[i] * sig[i]);
            sh[i] = 1.f - r.alpha[i] + 1e-15f;
        } else {
            r.alpha[i] = 0.f;
            sh[i] = 1.f;
        }
        local *= sh[i];
    }
    const float incl = wscan_mul(local, lane);
    float excl = __shfl_up_sync(0xffffffffu, incl, 1);
    if (lane == 0) excl = 1.f;
    float Tr = excl;
#pragma unroll
    for (int i = 0; i < K; ++i) {
        r.T[i] = Tr;
        r.w[i] = r.alpha[i] * Tr;
        Tr *= sh[i];
    }
}

// the last delta is (far - near) / Tc (renderer_df.py:414-415 uses the coarse sample_dist whatever T is)
template <int K>
__global__ void __launch_bounds__(kWarpsPerBlock * 32) ray_composite_kernel(const float* __restrict__ z_sorted, const float* __restrict__ sigma,
                                                                           const float* __restrict__ rgb, const float* __restrict__ nears,
                                                                           const float* __restrict__ fars, float bg, uint32_t N, int Tc, int T,
                                                                           float* __restrict__ image, float* __restrict__ depth,
                                                                           float* __restrict__ weights_sum) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t n = blockIdx.x * kWarpsPerBlock + warp;
    if (n >= N) return;
    const float near = nears[n], far = fars[n];
    RaySamples<K> r;
    float sig[K];
    ray_weights<K>(z_sorted + (size_t)n * T, sigma + (size_t)n * T, coarse_spacing(__fsub_rn(far, near), Tc), T, lane, r, sig);
    const float* c = rgb + ((size_t)n * T + K * lane) * 3;
    float ws = 0.f, dp = 0.f, cr = 0.f, cg = 0.f, cb = 0.f;
    const float inv = 1.f / (far - near);
#pragma unroll
    for (int i = 0; i < K; ++i) {
        if (K * lane + i >= T) break;
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
template <int K>
__global__ void __launch_bounds__(kWarpsPerBlock * 32) ray_composite_bwd_kernel(const float* __restrict__ z_sorted, const float* __restrict__ sigma,
                                                                               const float* __restrict__ rgb, const float* __restrict__ nears,
                                                                               const float* __restrict__ fars, float bg, uint32_t N, int Tc, int T,
                                                                               const float* __restrict__ g_image, const float* __restrict__ g_ws,
                                                                               const float* __restrict__ g_depth, float* __restrict__ g_sigma,
                                                                               float* __restrict__ g_rgb) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t n = blockIdx.x * kWarpsPerBlock + warp;
    if (n >= N) return;
    const float near = nears[n], far = fars[n];
    RaySamples<K> r;
    float sig[K];
    ray_weights<K>(z_sorted + (size_t)n * T, sigma + (size_t)n * T, coarse_spacing(__fsub_rn(far, near), Tc), T, lane, r, sig);
    const float gi0 = g_image[(size_t)n * 3], gi1 = g_image[(size_t)n * 3 + 1], gi2 = g_image[(size_t)n * 3 + 2];
    const float gws = g_ws ? g_ws[n] : 0.f, gdp = g_depth ? g_depth[n] : 0.f;
    const float* c = rgb + ((size_t)n * T + K * lane) * 3;
    float* gc = g_rgb + ((size_t)n * T + K * lane) * 3;
    const float inv = 1.f / (far - near);
    // G_t = dL/dw_t ; local sums of G_t * w_t for the suffix scan
    // (samples t >= T read colour 0 and have weight 0, so they add nothing; the arithmetic is the same for every sample)
    float G[K], gw[K], local = 0.f;
#pragma unroll
    for (int i = 0; i < K; ++i) {
        const bool in = K * lane + i < T;
        const float c0 = in ? c[i * 3] : 0.f, c1 = in ? c[i * 3 + 1] : 0.f, c2 = in ? c[i * 3 + 2] : 0.f;
        const float oz = fminf(fmaxf((r.z[i] - near) * inv, 0.f), 1.f);
        G[i] = gi0 * (c0 - bg) + gi1 * (c1 - bg) + gi2 * (c2 - bg) + gws + gdp * oz;
        gw[i] = G[i] * r.w[i];
        local += gw[i];
        if (in) {
            gc[i * 3] = gi0 * r.w[i];
            gc[i * 3 + 1] = gi1 * r.w[i];
            gc[i * 3 + 2] = gi2 * r.w[i];
        }
    }
    const float incl = wscan_add(local, lane);
    const float total = __shfl_sync(0xffffffffu, incl, 31);
    float suffix = total - incl;  // sum over samples of later lanes
    float o[K];
#pragma unroll
    for (int i = K - 1; i >= 0; --i) {
        // dL/dalpha_t = G_t T_t - S_t / (1 - alpha_t + 1e-15),  S_t = sum_{u>t} G_u w_u ;  dalpha/dsigma = delta * exp(-delta*sigma)
        const float sh = 1.f - r.alpha[i] + 1e-15f;
        const float dalpha = G[i] * r.T[i] - suffix / sh;
        o[i] = dalpha * r.delta[i] * (1.f - r.alpha[i]);
        suffix += gw[i];
    }
    float* gs = g_sigma + (size_t)n * T;
    if constexpr (K % 4 == 0) {
        if (T == 32 * K) {
#pragma unroll
            for (int i = 0; i < K; i += 4) *reinterpret_cast<float4*>(gs + K * lane + i) = make_float4(o[i], o[i + 1], o[i + 2], o[i + 3]);
            return;
        }
    }
#pragma unroll
    for (int i = 0; i < K; ++i)
        if (K * lane + i < T) gs[K * lane + i] = o[i];
}

// the launches, one instantiation per K = ceil(samples / 32) in 1..kMaxK
template <template <int> class Launch, typename... Args>
void dispatch_k(int K, Args... args) {
    switch (K) {
        case 1: Launch<1>::run(args...); break;
        case 2: Launch<2>::run(args...); break;
        case 3: Launch<3>::run(args...); break;
        case 4: Launch<4>::run(args...); break;
        case 5: Launch<5>::run(args...); break;
        case 6: Launch<6>::run(args...); break;
        case 7: Launch<7>::run(args...); break;
        default: Launch<8>::run(args...); break;
    }
}
static_assert(kMaxK == 8, "dispatch_k instantiates K = 1..8");

template <int K>
struct LaunchResample {
    static void run(cudaStream_t st, const float* zc, const float* sc, const float* nears, const float* fars, const float* u, int det, uint32_t N, int Tc,
                    int Tf, float* zs, float* zn, uint8_t* src) {
        ray_resample_kernel<K><<<ceil_div(N, (uint32_t)kWarpsPerBlock), kWarpsPerBlock * 32, 0, st>>>(zc, sc, nears, fars, u, det, N, Tc, Tf, zs, zn, src);
    }
};
template <int K>
struct LaunchComposite {
    static void run(cudaStream_t st, const float* zs, const float* sigma, const float* rgb, const float* nears, const float* fars, float bg, uint32_t N,
                    int Tc, int T, float* image, float* depth, float* ws) {
        ray_composite_kernel<K><<<ceil_div(N, (uint32_t)kWarpsPerBlock), kWarpsPerBlock * 32, 0, st>>>(zs, sigma, rgb, nears, fars, bg, N, Tc, T, image,
                                                                                                     depth, ws);
    }
};
template <int K>
struct LaunchCompositeBwd {
    static void run(cudaStream_t st, const float* zs, const float* sigma, const float* rgb, const float* nears, const float* fars, float bg, uint32_t N,
                    int Tc, int T, const float* gi, const float* gws, const float* gdp, float* gsig, float* grgb) {
        ray_composite_bwd_kernel<K><<<ceil_div(N, (uint32_t)kWarpsPerBlock), kWarpsPerBlock * 32, 0, st>>>(zs, sigma, rgb, nears, fars, bg, N, Tc, T, gi,
                                                                                                         gws, gdp, gsig, grgb);
    }
};

// num_steps >= 1, upsample_steps >= 0, their sum <= 256, and num_steps >= 2 when there are importance samples (their pdf needs the
// coarse bin mid points; the reference's own gather fails at num_steps = 1)
inline bool steps_ok(uint32_t Tc, uint32_t Tf) {
    return Tc >= 1 && Tc <= (uint32_t)kMaxSamples && Tf <= (uint32_t)kMaxSamples && Tc + Tf <= (uint32_t)kMaxSamples && (Tf == 0 || Tc >= 2);
}
inline int lanes_k(uint32_t samples) { return (int)ceil_div(samples, 32u); }

int resample(const char* who, const float* z_coarse, const float* sigma_coarse, const float* nears, const float* fars, const float* u, int det, uint32_t N,
             uint32_t Tc, uint32_t Tf, float* z_sorted, float* z_new, uint8_t* src_of, void* stream) {
    dispatch_k<LaunchResample>(lanes_k(Tc > Tf ? Tc : Tf), as_stream(stream), z_coarse, sigma_coarse, nears, fars, u, det, N, (int)Tc, (int)Tf, z_sorted,
                               z_new, src_of);
    return check_launch(who);
}

int gather_sorted(const char* who, const uint8_t* src_of, const float* sigma_coarse, const float* rgb_coarse, const float* sigma_new,
                  const float* rgb_new, uint32_t N, uint32_t Tc, uint32_t Tf, float* sigma, float* rgb, void* stream) {
    const size_t total = (size_t)N * (Tc + Tf);
    ray_gather_sorted_kernel<<<(unsigned)((total + 255) / 256), 256, 0, as_stream(stream)>>>(src_of, sigma_coarse, rgb_coarse, sigma_new, rgb_new, N, Tc,
                                                                                            Tf, sigma, rgb);
    return check_launch(who);
}

int composite_forward(const char* who, const float* z_sorted, const float* sigma, const float* rgb, const float* nears, const float* fars, float bg,
                      uint32_t N, uint32_t Tc, uint32_t Tf, float* image, float* depth, float* weights_sum, void* stream) {
    const uint32_t T = Tc + Tf;
    dispatch_k<LaunchComposite>(lanes_k(T), as_stream(stream), z_sorted, sigma, rgb, nears, fars, bg, N, (int)Tc, (int)T, image, depth, weights_sum);
    return check_launch(who);
}

int composite_backward(const char* who, const float* z_sorted, const float* sigma, const float* rgb, const float* nears, const float* fars, float bg,
                       uint32_t N, uint32_t Tc, uint32_t Tf, const float* grad_image, const float* grad_weights_sum, const float* grad_depth,
                       float* grad_sigma, float* grad_rgb, void* stream) {
    const uint32_t T = Tc + Tf;
    dispatch_k<LaunchCompositeBwd>(lanes_k(T), as_stream(stream), z_sorted, sigma, rgb, nears, fars, bg, N, (int)Tc, (int)T, grad_image, grad_weights_sum,
                                   grad_depth, grad_sigma, grad_rgb);
    return check_launch(who);
}

}  // namespace sfb

using namespace sfb;

#define SFB_REQUIRE_STEPS(who, Tc, Tf)                                                                                                \
    SFB_REQUIRE(steps_ok(Tc, Tf), who ": needs num_steps >= 1, num_steps + upsample_steps <= 256, and num_steps >= 2 when upsample_steps > 0")

extern "C" {

int sfb_ray_coarse_z(const float* rays_o, const float* rays_d, const float* aabb, float min_near, const float* lin, const float* noise, uint32_t N,
                     uint32_t num_steps, float* nears, float* fars, float* z, void* stream) {
    if (N == 0) return SFB_OK;
    SFB_REQUIRE(rays_o && rays_d && aabb && lin && nears && fars && z, "ray_coarse_z: null pointer");
    SFB_REQUIRE_STEPS("ray_coarse_z", num_steps, 0u);
    ray_coarse_z_kernel<<<ceil_div(N * num_steps, 256u), 256, 0, as_stream(stream)>>>(rays_o, rays_d, aabb, min_near, lin, noise, N, num_steps, nears,
                                                                                     fars, z);
    return check_launch("ray_coarse_z");
}

int sfb_ray_resample(const float* z_coarse, const float* sigma_coarse, const float* nears, const float* fars, const float* u, int det, uint32_t N,
                     uint32_t num_steps, uint32_t upsample_steps, float* z_sorted, void* stream) {
    if (N == 0) return SFB_OK;
    SFB_REQUIRE(z_coarse && sigma_coarse && nears && fars && z_sorted && (det || u || upsample_steps == 0), "ray_resample: null pointer");
    SFB_REQUIRE_STEPS("ray_resample", num_steps, upsample_steps);
    return resample("ray_resample", z_coarse, sigma_coarse, nears, fars, u, det, N, num_steps, upsample_steps, z_sorted, nullptr, nullptr, stream);
}

int sfb_ray_resample_ex(const float* z_coarse, const float* sigma_coarse, const float* nears, const float* fars, const float* u, int det, uint32_t N,
                        uint32_t num_steps, uint32_t upsample_steps, float* z_sorted, float* z_new, uint8_t* src_of, void* stream) {
    if (N == 0) return SFB_OK;
    SFB_REQUIRE(z_coarse && sigma_coarse && nears && fars && z_sorted && (z_new || upsample_steps == 0) && src_of && (det || u || upsample_steps == 0),
                "ray_resample_ex: null pointer");
    SFB_REQUIRE_STEPS("ray_resample_ex", num_steps, upsample_steps);
    return resample("ray_resample_ex", z_coarse, sigma_coarse, nears, fars, u, det, N, num_steps, upsample_steps, z_sorted, z_new, src_of, stream);
}

int sfb_ray_gather_sorted(const uint8_t* src_of, const float* sigma_coarse, const float* rgb_coarse, const float* sigma_new, const float* rgb_new,
                          uint32_t N, uint32_t T, float* sigma, float* rgb, void* stream) {
    if (N == 0) return SFB_OK;
    SFB_REQUIRE(src_of && sigma_coarse && rgb_coarse && sigma_new && rgb_new && sigma && rgb, "ray_gather_sorted: null pointer");
    SFB_REQUIRE(T == 128u, "ray_gather_sorted: takes T = 64 + 64 samples per ray; sfb_ray_gather_sorted_steps takes other counts");
    return gather_sorted("ray_gather_sorted", src_of, sigma_coarse, rgb_coarse, sigma_new, rgb_new, N, 64, 64, sigma, rgb, stream);
}

int sfb_ray_gather_sorted_steps(const uint8_t* src_of, const float* sigma_coarse, const float* rgb_coarse, const float* sigma_new, const float* rgb_new,
                                uint32_t N, uint32_t num_steps, uint32_t upsample_steps, float* sigma, float* rgb, void* stream) {
    if (N == 0) return SFB_OK;
    SFB_REQUIRE(src_of && sigma_coarse && rgb_coarse && sigma && rgb && ((sigma_new && rgb_new) || upsample_steps == 0),
                "ray_gather_sorted_steps: null pointer");
    SFB_REQUIRE_STEPS("ray_gather_sorted_steps", num_steps, upsample_steps);
    return gather_sorted("ray_gather_sorted_steps", src_of, sigma_coarse, rgb_coarse, sigma_new, rgb_new, N, num_steps, upsample_steps, sigma, rgb, stream);
}

int sfb_ray_composite_forward(const float* z_sorted, const float* sigma, const float* rgb, const float* nears, const float* fars, float bg_color,
                              uint32_t N, uint32_t T, float* image, float* depth, float* weights_sum, void* stream) {
    if (N == 0) return SFB_OK;
    SFB_REQUIRE(z_sorted && sigma && rgb && nears && fars && image && depth && weights_sum, "ray_composite_forward: null pointer");
    SFB_REQUIRE(T == 128u, "ray_composite_forward: takes T = 64 + 64 samples per ray; sfb_ray_composite_forward_steps takes other counts");
    return composite_forward("ray_composite_forward", z_sorted, sigma, rgb, nears, fars, bg_color, N, 64, 64, image, depth, weights_sum, stream);
}

int sfb_ray_composite_forward_steps(const float* z_sorted, const float* sigma, const float* rgb, const float* nears, const float* fars, float bg_color,
                                    uint32_t N, uint32_t num_steps, uint32_t upsample_steps, float* image, float* depth, float* weights_sum,
                                    void* stream) {
    if (N == 0) return SFB_OK;
    SFB_REQUIRE(z_sorted && sigma && rgb && nears && fars && image && depth && weights_sum, "ray_composite_forward_steps: null pointer");
    SFB_REQUIRE_STEPS("ray_composite_forward_steps", num_steps, upsample_steps);
    return composite_forward("ray_composite_forward_steps", z_sorted, sigma, rgb, nears, fars, bg_color, N, num_steps, upsample_steps, image, depth,
                             weights_sum, stream);
}

int sfb_ray_composite_backward(const float* z_sorted, const float* sigma, const float* rgb, const float* nears, const float* fars, float bg_color,
                               uint32_t N, uint32_t T, const float* grad_image, const float* grad_weights_sum, const float* grad_depth,
                               float* grad_sigma, float* grad_rgb, void* stream) {
    if (N == 0) return SFB_OK;
    SFB_REQUIRE(z_sorted && sigma && rgb && nears && fars && grad_image && grad_sigma && grad_rgb, "ray_composite_backward: null pointer");
    SFB_REQUIRE(T == 128u, "ray_composite_backward: takes T = 64 + 64 samples per ray; sfb_ray_composite_backward_steps takes other counts");
    return composite_backward("ray_composite_backward", z_sorted, sigma, rgb, nears, fars, bg_color, N, 64, 64, grad_image, grad_weights_sum, grad_depth,
                              grad_sigma, grad_rgb, stream);
}

int sfb_ray_composite_backward_steps(const float* z_sorted, const float* sigma, const float* rgb, const float* nears, const float* fars, float bg_color,
                                     uint32_t N, uint32_t num_steps, uint32_t upsample_steps, const float* grad_image, const float* grad_weights_sum,
                                     const float* grad_depth, float* grad_sigma, float* grad_rgb, void* stream) {
    if (N == 0) return SFB_OK;
    SFB_REQUIRE(z_sorted && sigma && rgb && nears && fars && grad_image && grad_sigma && grad_rgb, "ray_composite_backward_steps: null pointer");
    SFB_REQUIRE_STEPS("ray_composite_backward_steps", num_steps, upsample_steps);
    return composite_backward("ray_composite_backward_steps", z_sorted, sigma, rgb, nears, fars, bg_color, N, num_steps, upsample_steps, grad_image,
                              grad_weights_sum, grad_depth, grad_sigma, grad_rgb, stream);
}
}
