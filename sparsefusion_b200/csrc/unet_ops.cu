// unet_ops.cu -- the non-GEMM operators of the VLDM UNet forward, NHWC fp32, for sm_90a.
//
// They replace the eager PyTorch elementwise / normalisation / tiny-attention launches of the
// reference's Unet (external/imagen_pytorch.py): GroupNorm+FiLM+SiLU of `Block` (:654-662), gain-only
// LayerNorm / ChanLayerNorm (:301-329), GELU of ChanFeedForward (:953-961), the multi-query Attention
// (:511-566) and CrossAttention (:764-805) softmax cores (at most 1+2+H*W keys), GlobalContext pooling
// (:936-941), PixelShuffle(2)+SiLU (:588-592), skip concatenation (:1639), the learned sinusoidal time
// embedding (:634-639) and small-M Linear layers (time MLPs, token projections), which are weight
// streaming GEMVs and stay in full fp32.
// Tensors that feed a wgmma GEMM are rounded to TF32 (cvt.rna) when they are written here, so the
// tensor core's operand truncation never biases the result.
#include "common.cuh"
#include "wgmma.cuh"
#include <cooperative_groups.h>
#include "../../include/sparsefusion_b200.h"

namespace sfb {
namespace cg = cooperative_groups;

__device__ __forceinline__ float silu_f(float x) { return x / (1.f + __expf(-x)); }
__device__ __forceinline__ float sigmoid_f(float x) { return 1.f / (1.f + __expf(-x)); }
__device__ __forceinline__ float gelu_f(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// ------------------------------------------------------------------------------------ layout
// NCHW [NB,C,H,W] -> channel slice [c_off, c_off+C) of NHWC [NB,H,W,ld]; 32x32 smem transpose per (n)
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ src, float* __restrict__ dst, int C, int HW, int64_t ld, int c_off, int round) {
    pdl_sync();
    __shared__ float tile[32][33];
    const int n = blockIdx.z;
    const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    const int tx = threadIdx.x, ty = threadIdx.y;  // 32 x 8
    for (int i = ty; i < 32; i += 8) {
        const int c = c0 + i, p = p0 + tx;
        tile[i][tx] = (c < C && p < HW) ? src[((int64_t)n * C + c) * HW + p] : 0.f;
    }
    __syncthreads();
    for (int i = ty; i < 32; i += 8) {
        const int p = p0 + i, c = c0 + tx;
        if (c < C && p < HW) {
            float v = tile[tx][i];
            if (round) v = tc::round_tf32(v);
            dst[((int64_t)n * HW + p) * ld + c_off + c] = v;
        }
    }
}
__global__ void nhwc_to_nchw_kernel(const float* __restrict__ src, float* __restrict__ dst, int C, int HW, int64_t ld) {
    pdl_sync();
    __shared__ float tile[32][33];
    const int n = blockIdx.z;
    const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    const int tx = threadIdx.x, ty = threadIdx.y;
    for (int i = ty; i < 32; i += 8) {
        const int p = p0 + i, c = c0 + tx;
        tile[i][tx] = (c < C && p < HW) ? src[((int64_t)n * HW + p) * ld + c] : 0.f;
    }
    __syncthreads();
    for (int i = ty; i < 32; i += 8) {
        const int c = c0 + i, p = p0 + tx;
        if (c < C && p < HW) dst[((int64_t)n * C + c) * HW + p] = tile[tx][i];
    }
}

// out[pix][0:C1] = a[pix][0:C1]; out[pix][C1:C1+C2] = b[pix][0:C2] * scale_b   (float4 granularity)
__global__ void concat2_kernel(const float4* __restrict__ a, int C1v, int64_t lda_v, const float4* __restrict__ b, int C2v, int64_t ldb_v,
                               float scale_b, float4* __restrict__ out, int64_t ldo_v, int64_t npix) {
    pdl_sync();
    const int Cv = C1v + C2v;
    const int64_t total = npix * Cv;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t pix = i / Cv;
        const int c = (int)(i - pix * Cv);
        float4 v;
        if (c < C1v) v = __ldg(a + pix * lda_v + c);
        else {
            v = __ldg(b + pix * ldb_v + (c - C1v));
            v.x *= scale_b; v.y *= scale_b; v.z *= scale_b; v.w *= scale_b;
        }
        out[pix * ldo_v + c] = v;
    }
}

// PixelShuffle(2) of silu(y): y [NB,H,W,4*Co] -> out [NB,2H,2W, channel slice of width Co]; y channel = c*4 + i*2 + j
__global__ void pixel_shuffle_silu_kernel(const float* __restrict__ y, float* __restrict__ out, int H, int W, int Co, int64_t ldo, int64_t total) {
    pdl_sync();
    for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        // idx enumerates output elements: ((n*2H + oh)*2W + ow)*Co + c
        const int c = (int)(idx % Co);
        int64_t t = idx / Co;
        const int ow = (int)(t % (2 * W)); t /= (2 * W);
        const int oh = (int)(t % (2 * H));
        const int64_t n = t / (2 * H);
        const int h = oh >> 1, i = oh & 1, w = ow >> 1, j = ow & 1;
        const float v = __ldg(y + ((n * H + h) * W + w) * (int64_t)(4 * Co) + c * 4 + i * 2 + j);
        out[((n * 2 * H + oh) * (int64_t)(2 * W) + ow) * ldo + c] = silu_f(v);
    }
}

// im2col of a FEW-channel NHWC tensor: out[n][h][w][(ky*KW + kx)*C + c] = x[n][h + ky - pad][w + kx - pad][c] (zero outside), row stride ldo >= KH*KW*C
// (the tail up to ldo is zero-filled).  The CrossEmbed init convolutions of the UNet see 4 latent channels next to the cached 256-channel share
// (Unet.precompute_cond): as implicit GEMMs their 32-channel K granularity would spend 8x the work on zero padding (15x15 x 32 instead of 15x15 x 4);
// unfolded, the three kernel sizes become ONE 1x1 convolution with K = 900.  One thread per (pixel, tap): C <= 4 channels as one float4.
__global__ void im2col_small_kernel(const float* __restrict__ x, int64_t ldx, float* __restrict__ out, int64_t ldo, int H, int W, int C, int KH, int KW,
                                    int pad, int64_t total) {
    pdl_sync();
    const int taps = KH * KW;
    const int cols = (int)(ldo / 4);                 // float4 columns per output row (taps first, then zero padding)
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int t = (int)(i % cols);
        int64_t r = i / cols;
        const int w = (int)(r % W); r /= W;
        const int h = (int)(r % H);
        const int n = (int)(r / H);
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (t < taps) {
            const int ky = t / KW, kx = t - ky * KW;
            const int ih = h + ky - pad, iw = w + kx - pad;
            if (ih >= 0 && ih < H && iw >= 0 && iw < W) v = __ldg(reinterpret_cast<const float4*>(x + (((int64_t)n * H + ih) * W + iw) * ldx));
        }
        *reinterpret_cast<float4*>(out + (((int64_t)n * H + h) * W + w) * ldo + (int64_t)t * 4) = v;
    }
}

// ------------------------------------------------------------------------------------ GroupNorm
// Two launches, no atomics: (1) CTAs (group, n, pixel-slab) write fp64 partial (sum, sumsq) per slab; (2) every CTA of the apply kernel
// folds the <= 64 partials of its image's groups into (mean, rstd) in shared memory (one warp per group) and normalises its pixels.
// (The earlier "last CTA finalises" variant cost 5.5-6.6 us per launch in the replayed graph: threadfence + counter atomics.)
__global__ void __launch_bounds__(256) gn_stats_kernel(const float* __restrict__ x, int64_t ldx, int HW, int C, int G, int S,
                                                      double2* __restrict__ partial) {
    pdl_sync();
    const int g = blockIdx.x, n = blockIdx.y, sl = blockIdx.z;
    const int Cg = C / G;
    const int Cg4 = Cg >> 2;
    const int p0 = (int)(((int64_t)HW * sl) / S), p1 = (int)(((int64_t)HW * (sl + 1)) / S);
    const float* base = x + ((int64_t)n * HW + p0) * ldx + g * Cg;
    double s = 0.0, ss = 0.0;
    if ((Cg & 3) == 0) {
        const int64_t total4 = (int64_t)(p1 - p0) * Cg4;
        for (int64_t i = threadIdx.x; i < total4; i += blockDim.x) {
            const int64_t pix = i / Cg4;
            const int c4 = (int)(i - pix * Cg4);
            const float4 v = __ldg(reinterpret_cast<const float4*>(base + pix * ldx) + c4);
            const float a = v.x + v.y + v.z + v.w;
            const float b = v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
            s += (double)a;
            ss += (double)b;
        }
    } else {   // narrow groups (1..3 channels, or not a multiple of 4): scalar loads
        const int64_t total = (int64_t)(p1 - p0) * Cg;
        for (int64_t i = threadIdx.x; i < total; i += blockDim.x) {
            const int64_t pix = i / Cg;
            const float v = __ldg(base + pix * ldx + (int)(i - pix * Cg));
            s += (double)v;
            ss += (double)(v * v);
        }
    }
    __shared__ double sh_s[8], sh_ss[8];
    s = warp_sum_d(s);
    ss = warp_sum_d(ss);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { sh_s[warp] = s; sh_ss[warp] = ss; }
    __syncthreads();
    if (threadIdx.x == 0) {
        const int nw = blockDim.x >> 5;
        s = 0.0; ss = 0.0;
        for (int w = 0; w < nw; ++w) { s += sh_s[w]; ss += sh_ss[w]; }
        partial[((int64_t)n * G + g) * S + sl] = make_double2(s, ss);
    }
}

// Row-coalesced statistics: CTA (slab, n) walks whole pixel rows of its slab, thread t keeps ONE float4 column (so one group) per pass over
// <= 256 columns and sums (sum, sumsq) in fp64; the per-thread sums meet in shared memory, one thread per group folds its columns and
// writes the slab's partial.  Versus the group-major kernel above this reads every 32-byte sector once (with narrow groups -- the VAE's
// GroupNorm(32) over 128 channels -- a group is 16 bytes of each pixel and the group-major CTAs pulled every sector twice).
// Needs 4 | C/G, C/4 a divisor or a multiple of 256, and a group not wider than one pass.
__global__ void __launch_bounds__(256) gn_stats_rows_kernel(const float* __restrict__ x, int64_t ldx, int HW, int C, int G, int S,
                                                           double2* __restrict__ partial) {
    pdl_sync();
    __shared__ double sh_s[256], sh_ss[256];
    const int sl = blockIdx.x, n = blockIdx.y;
    const int C4 = C >> 2, Cg4 = (C / G) >> 2;
    const int cols = C4 < 256 ? C4 : 256, passes = C4 < 256 ? 1 : C4 / 256;
    const int rpi = 256 / cols;                          // pixel rows per block iteration
    const int p0 = (int)(((int64_t)HW * sl) / S), p1 = (int)(((int64_t)HW * (sl + 1)) / S);
    const int tc = threadIdx.x % cols, tr = threadIdx.x / cols;
    const int gpp = cols / Cg4;                          // groups per pass
    for (int pass = 0; pass < passes; ++pass) {
        const float* base = x + (int64_t)n * HW * ldx + (pass * 256 + tc) * 4;
        double s = 0.0, ss = 0.0;
#pragma unroll 8
        for (int p = p0 + tr; p < p1; p += rpi) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(base + (int64_t)p * ldx));
            s += (double)(v.x + v.y + v.z + v.w);
            ss += (double)(v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w);
        }
        sh_s[threadIdx.x] = s;
        sh_ss[threadIdx.x] = ss;
        __syncthreads();
        if (threadIdx.x < gpp) {
            double ts = 0.0, tss = 0.0;
            for (int r = 0; r < rpi; ++r)
                for (int j = 0; j < Cg4; ++j) {
                    const int i = r * cols + threadIdx.x * Cg4 + j;
                    ts += sh_s[i];
                    tss += sh_ss[i];
                }
            const int g = pass * gpp + threadIdx.x;
            partial[((int64_t)n * G + g) * S + sl] = make_double2(ts, tss);
        }
        __syncthreads();
    }
}

constexpr int kGnMaxGroups = 32;
constexpr int kGnMaxSlabs = 256;   // partials per (image, group): sizes the workspace (sfb_groupnorm_ws_floats)
// Single launch: groups are independent, so each (image, group) gets its own thread-block CLUSTER of k CTAs that split the pixels; a CTA keeps
// its slab of the group's channels in registers (<= ITEMS float4 per thread), the k partial (sum, sumsq) pairs meet through distributed shared
// memory at one cluster barrier (a few hundred ns), and every CTA normalises its own slab: 6.0 us per GroupNorm in the replayed batch-1 graph.
// (Round 1 used one launch with a SOFTWARE grid barrier over <= 128 co-resident CTAs -- 8.9 us, and a spin-wait that could hang under MPS /
// green contexts; it is gone.)  Works for any batch size (grid (G k, NB)); deterministic (fixed fold order, fp64 partials).
template <int ITEMS>
__global__ void __launch_bounds__(256) gn_cluster_kernel(const float* __restrict__ x, int64_t ldx, int HW, int C, int G, float eps,
                                                         const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ film,
                                                         int64_t ldf, float* __restrict__ y, int64_t ldy, int act, int round) {
    pdl_sync();
    cg::cluster_group cl = cg::this_cluster();
    __shared__ double red_s[8], red_ss[8];
    __shared__ __align__(16) double part[2];
    __shared__ float2 stat;
    const unsigned k = cl.num_blocks(), rank = cl.block_rank();
    const int g = blockIdx.x / k, n = blockIdx.y;
    const int Cg = C / G, Cg4 = Cg >> 2;
    const int p0 = (int)(((int64_t)HW * rank) / k), p1 = (int)(((int64_t)HW * (rank + 1)) / k);
    const int total = (p1 - p0) * Cg4;
    const float* base = x + ((int64_t)n * HW + p0) * ldx + g * Cg;
    float4 v[ITEMS];
    float s = 0.f, ss = 0.f;
#pragma unroll
    for (int i = 0; i < ITEMS; ++i) {
        const int idx = threadIdx.x + i * 256;
        v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (idx < total) {
            const int pix = idx / Cg4, c4 = idx - pix * Cg4;
            v[i] = __ldg(reinterpret_cast<const float4*>(base + (int64_t)pix * ldx) + c4);
        }
        s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
        ss += (v[i].x * v[i].x + v[i].y * v[i].y) + (v[i].z * v[i].z + v[i].w * v[i].w);
    }
    // affine / FiLM coefficients do not depend on the statistics: fetch them before the cluster barrier so that their L2 round trip overlaps the
    // reduction (small slabs only: ITEMS <= 8 keeps the register budget)
    constexpr bool kPrefetch = ITEMS <= 8;
    float4 pga[kPrefetch ? ITEMS : 1], pbe[kPrefetch ? ITEMS : 1], psc[kPrefetch ? ITEMS : 1], psh[kPrefetch ? ITEMS : 1];
    if (kPrefetch) {
#pragma unroll
        for (int i = 0; i < (kPrefetch ? ITEMS : 1); ++i) {
            const int idx = threadIdx.x + i * 256;
            if (idx < total) {
                const int c = g * Cg + (idx % Cg4) * 4;
                pga[i] = __ldg(reinterpret_cast<const float4*>(gamma + c));
                pbe[i] = __ldg(reinterpret_cast<const float4*>(beta + c));
                if (film) {
                    const float* fr = film + (int64_t)n * ldf;
                    psc[i] = __ldg(reinterpret_cast<const float4*>(fr + c));
                    psh[i] = __ldg(reinterpret_cast<const float4*>(fr + C + c));
                }
            }
        }
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const double ds = warp_sum_d((double)s), dss = warp_sum_d((double)ss);
    if (lane == 0) { red_s[warp] = ds; red_ss[warp] = dss; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double a = 0.0, b = 0.0;
#pragma unroll
        for (int w = 0; w < 8; ++w) { a += red_s[w]; b += red_ss[w]; }
        part[0] = a; part[1] = b;
    }
    cl.sync();                                             // every CTA's partial pair is published
    if (warp == 0) {
        double a = 0.0, b = 0.0;
        if (lane < (int)k) {
            const double* rp = cl.map_shared_rank(part, lane);
            a = rp[0]; b = rp[1];
        }
        a = warp_sum_d(a);                                 // fixed butterfly order: the same value in every CTA of the cluster
        b = warp_sum_d(b);
        if (lane == 0) {
            const double cnt = (double)HW * Cg;
            const double mean = a / cnt;
            double var = b / cnt - mean * mean;
            if (var < 0) var = 0;
            stat = make_float2((float)mean, (float)(1.0 / sqrt(var + (double)eps)));
        }
    }
    __syncthreads();                                       // stat visible to the CTA
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");   // this CTA has finished reading its peers' shared memory ...
    const float2 st = stat;
    float* yb = y + ((int64_t)n * HW + p0) * ldy + g * Cg;
#pragma unroll
    for (int i = 0; i < ITEMS; ++i) {
        const int idx = threadIdx.x + i * 256;
        if (idx < total) {
            const int pix = idx / Cg4, c4 = idx - pix * Cg4;
            const int c = g * Cg + c4 * 4;
            const float4 ga = kPrefetch ? pga[kPrefetch ? i : 0] : __ldg(reinterpret_cast<const float4*>(gamma + c));
            const float4 be = kPrefetch ? pbe[kPrefetch ? i : 0] : __ldg(reinterpret_cast<const float4*>(beta + c));
            float o[4] = {(v[i].x - st.x) * st.y * ga.x + be.x, (v[i].y - st.x) * st.y * ga.y + be.y, (v[i].z - st.x) * st.y * ga.z + be.z,
                          (v[i].w - st.x) * st.y * ga.w + be.w};
            if (film) {
                const float* fr = film + (int64_t)n * ldf;
                const float4 sc = kPrefetch ? psc[kPrefetch ? i : 0] : __ldg(reinterpret_cast<const float4*>(fr + c));
                const float4 sh = kPrefetch ? psh[kPrefetch ? i : 0] : __ldg(reinterpret_cast<const float4*>(fr + C + c));
                o[0] = o[0] * (sc.x + 1.f) + sh.x; o[1] = o[1] * (sc.y + 1.f) + sh.y;
                o[2] = o[2] * (sc.z + 1.f) + sh.z; o[3] = o[3] * (sc.w + 1.f) + sh.w;
            }
            if (act) {
#pragma unroll
                for (int e = 0; e < 4; ++e) o[e] = silu_f(o[e]);
            }
            if (round) {
#pragma unroll
                for (int e = 0; e < 4; ++e) o[e] = tc::round_tf32(o[e]);
            }
            *reinterpret_cast<float4*>(yb + (int64_t)pix * ldy + c4 * 4) = make_float4(o[0], o[1], o[2], o[3]);
        }
    }
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");     // ... and does not exit before every peer has finished reading its own
}

// y = silu( ((x-mean)*rstd*gamma + beta) * (scale+1) + shift ), rounded to tf32.  film [NB, 2C] (scale | shift) or null.  grid (blocks, NB)
__global__ void __launch_bounds__(256) gn_apply_kernel(const float* __restrict__ x, int64_t ldx, const double2* __restrict__ partial, int S, float eps,
                                                      const float* __restrict__ gamma, const float* __restrict__ beta,
                                                      const float* __restrict__ film, int64_t ldf, float* __restrict__ y, int64_t ldy, int HW, int C,
                                                      int G, int act, int round) {
    pdl_sync();
    __shared__ float2 st_sh[kGnMaxGroups];
    const int n = blockIdx.y;
    const int Cg = C / G;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int g = warp; g < G; g += 8) {
        double ts = 0.0, tss = 0.0;
        for (int k = lane; k < S; k += 32) {
            const double2 pr = partial[((int64_t)n * G + g) * S + k];
            ts += pr.x; tss += pr.y;
        }
        ts = warp_sum_d(ts);
        tss = warp_sum_d(tss);
        if (lane == 0) {
            const double cnt = (double)HW * Cg;
            const double mean = ts / cnt;
            double var = tss / cnt - mean * mean;
            if (var < 0) var = 0;
            st_sh[g] = make_float2((float)mean, (float)(1.0 / sqrt(var + (double)eps)));
        }
    }
    __syncthreads();
    const int C4 = C >> 2;
    const int64_t total4 = (int64_t)HW * C4;
    const float* xn = x + (int64_t)n * HW * ldx;
    float* yn = y + (int64_t)n * HW * ldy;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total4; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t pix = i / C4;
        const int c = (int)(i - pix * C4) * 4;
        const float2 s0 = st_sh[c / Cg], s1 = st_sh[(c + 1) / Cg], s2 = st_sh[(c + 2) / Cg], s3 = st_sh[(c + 3) / Cg];   // equal when 4 | Cg
        const float4 v = __ldg(reinterpret_cast<const float4*>(xn + pix * ldx + c));
        const float4 ga = __ldg(reinterpret_cast<const float4*>(gamma + c));
        const float4 be = __ldg(reinterpret_cast<const float4*>(beta + c));
        float o[4] = {(v.x - s0.x) * s0.y * ga.x + be.x, (v.y - s1.x) * s1.y * ga.y + be.y, (v.z - s2.x) * s2.y * ga.z + be.z,
                      (v.w - s3.x) * s3.y * ga.w + be.w};
        if (film) {
            const float4 sc = __ldg(reinterpret_cast<const float4*>(film + (int64_t)n * ldf + c));
            const float4 sh = __ldg(reinterpret_cast<const float4*>(film + (int64_t)n * ldf + C + c));
            o[0] = o[0] * (sc.x + 1.f) + sh.x; o[1] = o[1] * (sc.y + 1.f) + sh.y;
            o[2] = o[2] * (sc.z + 1.f) + sh.z; o[3] = o[3] * (sc.w + 1.f) + sh.w;
        }
        if (act) {
#pragma unroll
            for (int k = 0; k < 4; ++k) o[k] = silu_f(o[k]);
        }
        if (round) {
#pragma unroll
            for (int k = 0; k < 4; ++k) o[k] = tc::round_tf32(o[k]);
        }
        *reinterpret_cast<float4*>(yn + pix * ldy + c) = make_float4(o[0], o[1], o[2], o[3]);
    }
}

// Same contract for C/4 a divisor of 256 (every layer up to 1 024 channels): a thread keeps ONE float4 column, so its group statistics, affine and
// FiLM coefficients are loaded once and the loop is load -> 3 FP ops per element -> store with no index division (the generic kernel above re-reads
// five coefficient vectors and divides a 64-bit index per element: 31 us for the 33.5 MB tensors of the VAE decoder's 256 x 256 stage).
__global__ void __launch_bounds__(256, 3) gn_apply_cols_kernel(const float* __restrict__ x, int64_t ldx, const double2* __restrict__ partial, int S, float eps,
                                                           const float* __restrict__ gamma, const float* __restrict__ beta,
                                                           const float* __restrict__ film, int64_t ldf, float* __restrict__ y, int64_t ldy, int HW, int C,
                                                           int G, int act, int round) {
    pdl_sync();
    __shared__ float2 st_sh[kGnMaxGroups];
    const int n = blockIdx.y;
    const int Cg = C / G;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int C4 = C >> 2, rpi = 256 / C4;
    const int tc = threadIdx.x % C4, tr = threadIdx.x / C4;
    const int c = tc * 4;
    const float* xn = x + (int64_t)n * HW * ldx + c;
    const int step = (int)gridDim.x * rpi;
    const int pfirst = (int)blockIdx.x * rpi + tr;
    // the thread's first eight rows are requested BEFORE the statistics are folded (independent of them): the fold's ~2 us hide under the loads
    float4 v8[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int p = pfirst + i * step;
        v8[i] = p < HW ? __ldg(reinterpret_cast<const float4*>(xn + (int64_t)p * ldx)) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    for (int g = warp; g < G; g += 8) {
        double ts = 0.0, tss = 0.0;
        for (int k = lane; k < S; k += 32) {
            const double2 pr = partial[((int64_t)n * G + g) * S + k];
            ts += pr.x; tss += pr.y;
        }
        ts = warp_sum_d(ts);
        tss = warp_sum_d(tss);
        if (lane == 0) {
            const double cnt = (double)HW * Cg;
            const double mean = ts / cnt;
            double var = tss / cnt - mean * mean;
            if (var < 0) var = 0;
            st_sh[g] = make_float2((float)mean, (float)(1.0 / sqrt(var + (double)eps)));
        }
    }
    __syncthreads();
    float mu[4], a[4], b[4];       // y = (x - mu) a + b with the affine and the FiLM pair folded: a = rstd gamma (s + 1), b = beta (s + 1) + shift
    {
        const float4 ga = __ldg(reinterpret_cast<const float4*>(gamma + c));
        const float4 be = __ldg(reinterpret_cast<const float4*>(beta + c));
        const float gv[4] = {ga.x, ga.y, ga.z, ga.w}, bv[4] = {be.x, be.y, be.z, be.w};
        float fs[4] = {1.f, 1.f, 1.f, 1.f}, fh[4] = {0.f, 0.f, 0.f, 0.f};
        if (film) {
            const float4 sc = __ldg(reinterpret_cast<const float4*>(film + (int64_t)n * ldf + c));
            const float4 sh = __ldg(reinterpret_cast<const float4*>(film + (int64_t)n * ldf + C + c));
            fs[0] = sc.x + 1.f; fs[1] = sc.y + 1.f; fs[2] = sc.z + 1.f; fs[3] = sc.w + 1.f;
            fh[0] = sh.x; fh[1] = sh.y; fh[2] = sh.z; fh[3] = sh.w;
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float2 st = st_sh[(c + k) / Cg];
            mu[k] = st.x;
            a[k] = st.y * gv[k] * fs[k];
            b[k] = bv[k] * fs[k] + fh[k];
        }
    }
    float* yn = y + (int64_t)n * HW * ldy + c;
    auto finish = [&](const float4& v, int p) {
        float o[4] = {(v.x - mu[0]) * a[0] + b[0], (v.y - mu[1]) * a[1] + b[1], (v.z - mu[2]) * a[2] + b[2], (v.w - mu[3]) * a[3] + b[3]};
        if (act) {
#pragma unroll
            for (int k = 0; k < 4; ++k) o[k] = silu_f(o[k]);
        }
        if (round) {
#pragma unroll
            for (int k = 0; k < 4; ++k) o[k] = tc::round_tf32(o[k]);
        }
        *reinterpret_cast<float4*>(yn + (int64_t)p * ldy) = make_float4(o[0], o[1], o[2], o[3]);
    };
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int p = pfirst + i * step;
        if (p < HW) finish(v8[i], p);
    }
#pragma unroll 4
    for (int p = pfirst + 8 * step; p < HW; p += step) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(xn + (int64_t)p * ldx));
        finish(v, p);
    }
}

// ------------------------------------------------------------------------------------ LayerNorm over the last dim
// rows [T, C] (row stride ldx); y = LN(pre(x)) * g (+ b) (+ res); pre: 0 none, 1 GELU.  One 128-thread CTA per row.  eps 1e-5, biased variance.
__device__ __forceinline__ float block_sum_128(float v, float* sh) {
    v = warp_sum(v);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    const float t = sh[0] + sh[1] + sh[2] + sh[3];
    __syncthreads();
    return t;
}
__global__ void __launch_bounds__(128) layernorm_rows_kernel(const float* __restrict__ x, int64_t ldx, const float* __restrict__ g,
                                                            const float* __restrict__ b, const float* __restrict__ res, int64_t ldr,
                                                            float* __restrict__ y, int64_t ldy, int T, int C, int pre, int round) {
    pdl_sync();
    __shared__ float sh[4];
    const int row = blockIdx.x;
    const float* xr = x + (int64_t)row * ldx;
    float s = 0.f;
    for (int c = threadIdx.x; c < C; c += 128) {
        float v = xr[c];
        if (pre == 1) v = gelu_f(v);
        s += v;
    }
    const float mean = block_sum_128(s, sh) / C;
    float ss = 0.f;
    for (int c = threadIdx.x; c < C; c += 128) {
        float v = xr[c];
        if (pre == 1) v = gelu_f(v);
        const float d = v - mean;
        ss += d * d;
    }
    const float rstd = rsqrtf(block_sum_128(ss, sh) / C + 1e-5f);
    float* yr = y + (int64_t)row * ldy;
    for (int c = threadIdx.x; c < C; c += 128) {
        float v = xr[c];
        if (pre == 1) v = gelu_f(v);
        float o = (v - mean) * rstd * g[c] + (b ? b[c] : 0.f);
        if (res) o += res[(int64_t)row * ldr + c];
        if (round) o = tc::round_tf32(o);
        yr[c] = o;
    }
}

// ------------------------------------------------------------------------------------ small-M Linear (fp32 GEMV)
// y[m][o] = post( bias[o] + sum_k pre(x[m][k]) * W[o][k] ) (+ res[m][o]);  M <= 8 rows per pass, one warp per output feature.
// pre: 0 none, 1 SiLU ; post: 0 none, 1 SiLU, 2 sigmoid
template <int MT>
__global__ void __launch_bounds__(256) linear_small_kernel(const float* __restrict__ x, int64_t ldx, const float* __restrict__ Wt,
                                                          const float* __restrict__ bias, const float* __restrict__ res, int64_t ldr,
                                                          float* __restrict__ y, int64_t ldy, int M, int K, int O, int pre, int post, int round) {
    pdl_sync();
    extern __shared__ float xs[];  // [MT][K]
    const int m0 = blockIdx.y * MT;
    const int mrows = min(MT, M - m0);
    for (int i = threadIdx.x; i < MT * K; i += blockDim.x) {
        const int m = i / K, k = i - m * K;
        float v = (m < mrows) ? x[(int64_t)(m0 + m) * ldx + k] : 0.f;
        if (pre == 1) v = silu_f(v);
        xs[i] = v;
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int o = blockIdx.x * (blockDim.x >> 5) + warp;
    if (o >= O) return;
    const float* wr = Wt + (int64_t)o * K;
    float acc[MT];
#pragma unroll
    for (int m = 0; m < MT; ++m) acc[m] = 0.f;
    if ((K & 3) == 0) {
        for (int k = lane * 4; k < K; k += 128) {
            const float4 w = __ldg(reinterpret_cast<const float4*>(wr + k));
#pragma unroll
            for (int m = 0; m < MT; ++m) {
                const float4 xv = *reinterpret_cast<const float4*>(xs + m * K + k);
                acc[m] += w.x * xv.x + w.y * xv.y + w.z * xv.z + w.w * xv.w;
            }
        }
    } else {
        for (int k = lane; k < K; k += 32) {
            const float w = __ldg(wr + k);
#pragma unroll
            for (int m = 0; m < MT; ++m) acc[m] += w * xs[m * K + k];
        }
    }
#pragma unroll
    for (int m = 0; m < MT; ++m) acc[m] = warp_sum(acc[m]);
    if (lane == 0) {
        const float bv = bias ? bias[o] : 0.f;
        for (int m = 0; m < mrows; ++m) {
            float v = acc[m] + bv;
            if (post == 1) v = silu_f(v);
            else if (post == 2) v = sigmoid_f(v);
            if (res) v += res[(int64_t)(m0 + m) * ldr + o];
            if (round) v = tc::round_tf32(v);
            y[(int64_t)(m0 + m) * ldy + o] = v;
        }
    }
}

// ------------------------------------------------------------------------------------ time embedding
// four[b] = [t, sin(2 pi t w_0..), cos(2 pi t w_0..)]   (imagen_pytorch.py:634-639)
__global__ void time_fourier_kernel(const float* __restrict__ t, const float* __restrict__ w, float* __restrict__ out, int B, int half) {
    pdl_sync();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int width = 2 * half + 1;
    if (i >= B * width) return;
    const int b = i / width, j = i - b * width;
    const float tv = t[b];
    float v;
    if (j == 0) v = tv;
    else {
        const int k = (j - 1) % half;
        const float f = tv * w[k] * 2.f * 3.14159265358979323846f;
        v = (j - 1 < half) ? sinf(f) : cosf(f);
    }
    out[i] = v;
}

// ------------------------------------------------------------------------------------ attention cores
// Multi-query self attention (imagen_pytorch.py:511-566): q [B,n,heads*dh] (already scaled? no: scaled here), kv [B,n,2*dh] shared by all
// heads, null_kv [2,dh], optional context kv ckv [B,nc,2*dh].  Key order: context, null, tokens (:523-532).  out [B,n,heads*dh].
// One warp per (b, head, query); dh <= 128.
__global__ void mq_attention_kernel(const float* __restrict__ q, const float* __restrict__ kv, const float* __restrict__ null_kv,
                                    const float* __restrict__ ckv, float* __restrict__ out, int B, int n, int heads, int dh, int nc, float scale, int round) {
    pdl_sync();
    extern __shared__ float sm[];  // per warp: scores[nk]
    const int warps = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int gw = blockIdx.x * warps + warp;
    const int nk = nc + 1 + n;
    float* sc = sm + warp * nk;
    if (gw >= B * heads * n) return;
    const int i = gw % n, h = (gw / n) % heads, b = gw / (n * heads);
    const float* qr = q + ((int64_t)(b * n + i) * heads + h) * dh;
    auto key_ptr = [&](int j, int which) -> const float* {  // which 0 = k, 1 = v
        if (j < nc) return ckv + ((int64_t)(b * nc + j) * 2 + which) * dh;
        if (j == nc) return null_kv + which * dh;
        return kv + ((int64_t)(b * n + (j - nc - 1)) * 2 + which) * dh;
    };
    float mx = -INFINITY;
    for (int j = 0; j < nk; ++j) {
        const float* kr = key_ptr(j, 0);
        float d = 0.f;
        for (int e = lane; e < dh; e += 32) d += qr[e] * scale * kr[e];
        d = warp_sum(d);
        if (lane == 0) sc[j] = d;
        mx = fmaxf(mx, d);
    }
    __syncwarp();
    float den = 0.f;
    for (int j = 0; j < nk; ++j) den += __expf(sc[j] - mx);
    const float inv = 1.f / den;
    float* orow = out + ((int64_t)(b * n + i) * heads + h) * dh;
    for (int e = lane; e < dh; e += 32) {
        float acc = 0.f;
        for (int j = 0; j < nk; ++j) acc += __expf(sc[j] - mx) * inv * key_ptr(j, 1)[e];
        orow[e] = round ? tc::round_tf32(acc) : acc;
    }
}

// Same contract, keys/values staged in shared memory.  All heads share one K/V (multi-query), so a CTA of 8 warps (8 queries of one image) loads
// the nk x 2 x dh block once, coalesced; the per-key dot products and the P.V sums then run at shared-memory latency.  (The global-memory
// kernel above walks the keys with one dependent L2 round trip per key: 28 us for 19 keys in the replayed graph.)
__global__ void __launch_bounds__(256) mq_attention_smem_kernel(const float* __restrict__ q, const float* __restrict__ kv,
                                                                const float* __restrict__ null_kv, const float* __restrict__ ckv,
                                                                float* __restrict__ out, int n, int heads, int dh, int nc, float scale, int round) {
    pdl_sync();
    extern __shared__ float sm[];
    const int nk = nc + 1 + n;
    const int row = 2 * dh;                 // k | v of one key
    float* kvs = sm;                        // [nk][2*dh]
    float* scs = sm + (size_t)nk * row;     // [8][nk]
    const int b = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // stage: context keys, the null key, the image's tokens (imagen_pytorch.py:523-532 key order)
    const int row4 = row >> 2;
    for (int i = threadIdx.x; i < nk * row4; i += 256) {
        const int j = i / row4, e4 = i - j * row4;
        const float* src;
        if (j < nc) src = ckv + ((int64_t)(b * nc + j)) * row;
        else if (j == nc) src = null_kv;
        else src = kv + ((int64_t)(b * n + (j - nc - 1))) * row;
        reinterpret_cast<float4*>(kvs)[i] = __ldg(reinterpret_cast<const float4*>(src) + e4);
    }
    __syncthreads();
    const int qi = blockIdx.x * 8 + warp;   // query index over (head, token)
    if (qi >= heads * n) return;
    const int i = qi % n, h = qi / n;
    const float* qr = q + ((int64_t)(b * n + i) * heads + h) * dh;
    float qv[4];                            // dh <= 128
#pragma unroll
    for (int t = 0; t < 4; ++t) qv[t] = (lane + 32 * t < dh) ? qr[lane + 32 * t] * scale : 0.f;
    float* sc = scs + warp * nk;
    float mx = -INFINITY;
    for (int j = 0; j < nk; ++j) {
        const float* kr = kvs + (size_t)j * row;
        float d = 0.f;
#pragma unroll
        for (int t = 0; t < 4; ++t)
            if (lane + 32 * t < dh) d += qv[t] * kr[lane + 32 * t];
        d = warp_sum(d);
        if (lane == 0) sc[j] = d;
        mx = fmaxf(mx, d);
    }
    __syncwarp();
    float den = 0.f;
    for (int j = lane; j < nk; j += 32) { const float e = __expf(sc[j] - mx); sc[j] = e; den += e; }
    den = warp_sum(den);
    __syncwarp();
    const float inv = 1.f / den;
    float* orow = out + ((int64_t)(b * n + i) * heads + h) * dh;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int j = 0; j < nk; ++j) {
        const float pj = sc[j];
        const float* vr = kvs + (size_t)j * row + dh;
#pragma unroll
        for (int t = 0; t < 4; ++t)
            if (lane + 32 * t < dh) acc[t] += pj * vr[lane + 32 * t];
    }
#pragma unroll
    for (int t = 0; t < 4; ++t)
        if (lane + 32 * t < dh) {
            const float v = acc[t] * inv;
            orow[lane + 32 * t] = round ? tc::round_tf32(v) : v;
        }
}

// Many keys (128 x 128 latents: 256 tokens + null + context at the deepest stage).  Same staging, but a LANE owns a key while scoring (rows
// padded by four floats so the quarter-warps' float4 reads fall on 32 distinct banks), one warp maximum / sum per query instead of one shuffle
// tree per key, and a warp walks `qpw` queries so that the 132 KB of keys and values is staged once per 8 qpw queries.
__global__ void __launch_bounds__(256) mq_attention_keys_kernel(const float* __restrict__ q, const float* __restrict__ kv,
                                                                const float* __restrict__ null_kv, const float* __restrict__ ckv,
                                                                float* __restrict__ out, int n, int heads, int dh, int nc, float scale, int round,
                                                                int qpw) {
    pdl_sync();
    extern __shared__ __align__(16) float sm[];
    const int nk = nc + 1 + n, nkp = (nk + 31) & ~31;
    const int row = 2 * dh, rs = row + 4;
    float* kvs = sm;                              // [nk][rs]
    float* scs = sm + (size_t)nk * rs;            // [8][nkp]
    float* qs = scs + 8 * nkp;                    // [8][dh]
    const int b = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int row4 = row >> 2;
    for (int i = threadIdx.x; i < nk * row4; i += 256) {
        const int j = i / row4, e4 = i - j * row4;
        const float* src;
        if (j < nc) src = ckv + ((int64_t)(b * nc + j)) * row;
        else if (j == nc) src = null_kv;
        else src = kv + ((int64_t)(b * n + (j - nc - 1))) * row;
        *reinterpret_cast<float4*>(kvs + (size_t)j * rs + e4 * 4) = __ldg(reinterpret_cast<const float4*>(src) + e4);
    }
    __syncthreads();
    float* sc = scs + warp * nkp;
    float* qw = qs + warp * dh;
    const int dh4 = dh >> 2;
    for (int t = 0; t < qpw; ++t) {
        const int qi = (blockIdx.x * 8 + warp) * qpw + t;     // query index over (head, token)
        if (qi >= heads * n) break;
        const int i = qi % n, h = qi / n;
        const float* qr = q + ((int64_t)(b * n + i) * heads + h) * dh;
        for (int e = lane; e < dh; e += 32) qw[e] = qr[e] * scale;
        __syncwarp();
        float mx = -INFINITY;
        for (int j = lane; j < nk; j += 32) {
            const float4* kr = reinterpret_cast<const float4*>(kvs + (size_t)j * rs);
            float d0 = 0.f, d1 = 0.f;
#pragma unroll 4
            for (int e4 = 0; e4 < dh4; ++e4) {
                const float4 k4 = kr[e4];
                const float4 q4 = reinterpret_cast<const float4*>(qw)[e4];
                d0 += k4.x * q4.x + k4.y * q4.y;
                d1 += k4.z * q4.z + k4.w * q4.w;
            }
            const float d = d0 + d1;
            sc[j] = d;
            mx = fmaxf(mx, d);
        }
        mx = warp_max(mx);
        float den = 0.f;
        for (int j = lane; j < nk; j += 32) { const float e = __expf(sc[j] - mx); sc[j] = e; den += e; }
        den = warp_sum(den);
        __syncwarp();
        const float inv = 1.f / den;
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 4
        for (int j = 0; j < nk; ++j) {
            const float pj = sc[j];
            const float* vr = kvs + (size_t)j * rs + dh;
#pragma unroll
            for (int u = 0; u < 4; ++u)
                if (lane + 32 * u < dh) acc[u] += pj * vr[lane + 32 * u];
        }
        float* orow = out + ((int64_t)(b * n + i) * heads + h) * dh;
#pragma unroll
        for (int u = 0; u < 4; ++u)
            if (lane + 32 * u < dh) {
                const float v = acc[u] * inv;
                orow[lane + 32 * u] = round ? tc::round_tf32(v) : v;
            }
        __syncwarp();
    }
}

// Cross attention (imagen_pytorch.py:764-805): q [B,n,heads*dh]; kvc [B,nc,2*heads*dh] = (k | v) per context token, per-head slices;
// null_kv [2,dh] shared by heads; keys: null, context.  One warp per (b, head, query).
__global__ void cross_attention_kernel(const float* __restrict__ q, const float* __restrict__ kvc, const float* __restrict__ null_kv,
                                       float* __restrict__ out, int B, int n, int heads, int dh, int nc, float scale, int round) {
    pdl_sync();
    const int warps = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int gw = blockIdx.x * warps + warp;
    if (gw >= B * heads * n) return;
    const int i = gw % n, h = (gw / n) % heads, b = gw / (n * heads);
    const int inner = heads * dh;
    const float* qr = q + ((int64_t)(b * n + i)) * inner + h * dh;
    float scv[9];  // nc <= 8
    float mx = -INFINITY;
    for (int j = 0; j <= nc; ++j) {
        const float* kr = (j == 0) ? null_kv : kvc + ((int64_t)(b * nc + (j - 1))) * 2 * inner + h * dh;
        float d = 0.f;
        for (int e = lane; e < dh; e += 32) d += qr[e] * scale * kr[e];
        d = warp_sum(d);
        scv[j] = d;
        mx = fmaxf(mx, d);
    }
    float den = 0.f;
    for (int j = 0; j <= nc; ++j) { scv[j] = __expf(scv[j] - mx); den += scv[j]; }
    const float inv = 1.f / den;
    float* orow = out + ((int64_t)(b * n + i)) * inner + h * dh;
    for (int e = lane; e < dh; e += 32) {
        float acc = 0.f;
        for (int j = 0; j <= nc; ++j) {
            const float* vr = (j == 0) ? null_kv + dh : kvc + ((int64_t)(b * nc + (j - 1))) * 2 * inner + inner + h * dh;
            acc += scv[j] * inv * vr[e];
        }
        orow[e] = round ? tc::round_tf32(acc) : acc;
    }
}

// ------------------------------------------------------------------------------------ GlobalContext
// logits[n][p] = bias + sum_c x[n][p][c] * wk[c]      (to_k, imagen_pytorch.py:926,937) -- one warp per pixel
__global__ void gca_logits_kernel(const float* __restrict__ x, int64_t ldx, const float* __restrict__ wk, const float* __restrict__ bk,
                                  float* __restrict__ logits, int64_t npix, int C) {
    pdl_sync();
    const int64_t p = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
    if (p >= npix) return;
    const int lane = threadIdx.x & 31;
    const float* xr = x + p * ldx;
    float d = 0.f;
    for (int c = lane * 4; c < C; c += 128) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(xr + c));
        const float4 w = __ldg(reinterpret_cast<const float4*>(wk + c));
        d += v.x * w.x + v.y * w.y + v.z * w.z + v.w * w.w;
    }
    d = warp_sum(d);
    if (lane == 0) logits[p] = d + bk[0];
}
// pooled[n][c] = sum_p softmax(logits[n])[p] * x[n][p][c].  grid (C / 16, NB): a CTA owns 16 channels of one image -- no atomics, no
// zero-init.  Each CTA first turns the image's logits into softmax weights in shared memory (HW floats; redundant across CTAs, trivial),
// then thread (pixel group pg of 64, float4 column q of 4) accumulates pixels pg, pg + 64, ...; the 64 partial rows fold through smem.
constexpr int kGcaCols = 16;
__global__ void __launch_bounds__(256) gca_pool_kernel(const float* __restrict__ x, int64_t ldx, const float* __restrict__ logits,
                                                      float* __restrict__ pooled, int HW, int C) {
    pdl_sync();
    extern __shared__ float gca_sm[];
    float* wts = gca_sm;                       // [HW]
    float* part = gca_sm + ((HW + 3) & ~3);    // [64][16]
    __shared__ float red[8];
    const int n = blockIdx.y, c0 = blockIdx.x * kGcaCols;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float* lg = logits + (int64_t)n * HW;
    float mx = -INFINITY;
    for (int p = threadIdx.x; p < HW; p += 256) { const float v = lg[p]; wts[p] = v; mx = fmaxf(mx, v); }
    mx = warp_max(mx);
    if (lane == 0) red[warp] = mx;
    __syncthreads();
    mx = red[0];
#pragma unroll
    for (int w = 1; w < 8; ++w) mx = fmaxf(mx, red[w]);
    __syncthreads();
    float sm = 0.f;
    for (int p = threadIdx.x; p < HW; p += 256) { const float e = __expf(wts[p] - mx); wts[p] = e; sm += e; }
    sm = warp_sum(sm);
    if (lane == 0) red[warp] = sm;
    __syncthreads();
    float tot = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) tot += red[w];
    const float inv = 1.f / tot;
    const int pg = threadIdx.x >> 2, q = threadIdx.x & 3;
    const int c = c0 + q * 4;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c < C) {
        const float* xb = x + (int64_t)n * HW * ldx + c;
#pragma unroll 4
        for (int p = pg; p < HW; p += 64) {
            const float w = wts[p];
            const float4 v = __ldg(reinterpret_cast<const float4*>(xb + (int64_t)p * ldx));
            acc.x += w * v.x; acc.y += w * v.y; acc.z += w * v.z; acc.w += w * v.w;
        }
    }
    reinterpret_cast<float4*>(part)[pg * 4 + q] = acc;
    __syncthreads();
    if (threadIdx.x < kGcaCols && c0 + threadIdx.x < C) {
        float t = 0.f;
#pragma unroll 8
        for (int g = 0; g < 64; ++g) t += part[g * kGcaCols + threadIdx.x];
        pooled[(int64_t)n * C + c0 + threadIdx.x] = t * inv;
    }
}

// Large images (128 x 128 latents: 16 384 pixels against 8 channel tiles of work): a thread-block CLUSTER of Z CTAs shares one (image, channel
// tile); CTA z soft-maxes and pools its own slab of pixels (local maximum m_z, local sum s_z, local weighted sums a_z[16]) and rank 0 merges
// the Z triples through distributed shared memory:  M = max m_z,  pooled = sum_z a_z e^(m_z - M) / sum_z s_z e^(m_z - M).
__global__ void __launch_bounds__(256) gca_pool_split_kernel(const float* __restrict__ x, int64_t ldx, const float* __restrict__ logits,
                                                            float* __restrict__ pooled, int HW, int C) {
    pdl_sync();
    cg::cluster_group cl = cg::this_cluster();
    extern __shared__ float gca_sm[];
    const unsigned Z = cl.num_blocks(), rank = cl.block_rank();
    const int p0 = (int)(((int64_t)HW * rank) / Z), p1 = (int)(((int64_t)HW * (rank + 1)) / Z), np = p1 - p0;
    float* wts = gca_sm;                       // [np]
    float* part = gca_sm + ((np + 3) & ~3);    // [64][16]
    __shared__ float red[8];
    __shared__ __align__(16) float merged[2 + kGcaCols];     // m_z, s_z, a_z[16]: read by rank 0 through DSMEM
    const int n = blockIdx.y, c0 = (int)(blockIdx.x / Z) * kGcaCols;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float* lg = logits + (int64_t)n * HW + p0;
    float mx = -INFINITY;
    for (int p = threadIdx.x; p < np; p += 256) { const float v = lg[p]; wts[p] = v; mx = fmaxf(mx, v); }
    mx = warp_max(mx);
    if (lane == 0) red[warp] = mx;
    __syncthreads();
    mx = red[0];
#pragma unroll
    for (int w = 1; w < 8; ++w) mx = fmaxf(mx, red[w]);
    __syncthreads();
    float sm = 0.f;
    for (int p = threadIdx.x; p < np; p += 256) { const float e = __expf(wts[p] - mx); wts[p] = e; sm += e; }
    sm = warp_sum(sm);
    if (lane == 0) red[warp] = sm;
    __syncthreads();
    const int pg = threadIdx.x >> 2, q = threadIdx.x & 3;
    const int c = c0 + q * 4;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c < C) {
        const float* xb = x + ((int64_t)n * HW + p0) * ldx + c;
#pragma unroll 4
        for (int p = pg; p < np; p += 64) {
            const float w = wts[p];
            const float4 v = __ldg(reinterpret_cast<const float4*>(xb + (int64_t)p * ldx));
            acc.x += w * v.x; acc.y += w * v.y; acc.z += w * v.z; acc.w += w * v.w;
        }
    }
    reinterpret_cast<float4*>(part)[pg * 4 + q] = acc;
    __syncthreads();
    if (threadIdx.x < kGcaCols) {
        float t = 0.f;
#pragma unroll 8
        for (int g = 0; g < 64; ++g) t += part[g * kGcaCols + threadIdx.x];
        merged[2 + threadIdx.x] = t;
    }
    if (threadIdx.x == 32) {
        float tot = 0.f;
#pragma unroll
        for (int w = 0; w < 8; ++w) tot += red[w];
        merged[0] = mx;
        merged[1] = tot;
    }
    cl.sync();
    if (rank == 0 && threadIdx.x < kGcaCols && c0 + threadIdx.x < C) {
        float M = -INFINITY;
        for (unsigned z = 0; z < Z; ++z) M = fmaxf(M, cl.map_shared_rank(merged, z)[0]);
        float S = 0.f, A = 0.f;
        for (unsigned z = 0; z < Z; ++z) {
            const float* mz = cl.map_shared_rank(merged, z);
            const float f = __expf(mz[0] - M);
            S += mz[1] * f;
            A += mz[2 + threadIdx.x] * f;
        }
        pooled[(int64_t)n * C + c0 + threadIdx.x] = A / S;
    }
    cl.sync();      // no CTA leaves while rank 0 may still read its shared memory
}

// out = h * gate[n][c] + res      (ResnetBlock tail, imagen_pytorch.py:727-729); gate may be null (== 1)
__global__ void gate_residual_kernel(const float4* __restrict__ h, int64_t ldh_v, const float* __restrict__ gate, const float4* __restrict__ res,
                                     int64_t ldr_v, float4* __restrict__ out, int64_t ldo_v, int HW, int Cv, int64_t total) {
    pdl_sync();
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t pix = i / Cv;
        const int c = (int)(i - pix * Cv);
        float4 v = __ldg(h + pix * ldh_v + c);
        if (gate) {
            const int n = (int)(pix / HW);
            const float4 g = __ldg(reinterpret_cast<const float4*>(gate + (int64_t)n * Cv * 4) + c);
            v.x *= g.x; v.y *= g.y; v.z *= g.z; v.w *= g.w;
        }
        const float4 r = __ldg(res + pix * ldr_v + c);
        out[pix * ldo_v + c] = make_float4(v.x + r.x, v.y + r.y, v.z + r.z, v.w + r.w);
    }
}

// GlobalContext tail fused: gate[n][c] = sigmoid(b2[c] + W2[c][:] . hid[n][:]) (Conv2d(hidden, dim_out, 1) + Sigmoid, imagen_pytorch.py:929-933)
// and out = h * gate + res (ResnetBlock tail, :727-729) in one launch.  grid (C / 8, NB, Z): a CTA owns 8 channels of one image -- each warp
// evaluates one gate channel (a 2 KB weight row), then all threads stream the CTA's 32-byte channel slab of the pixels p = 128 z + .., stride
// 128 Z.  Z > 1 (large images: 16 384 pixels at 128 x 128 latents) recomputes the eight gates per CTA -- L2 hits -- to put every SM to work.
__global__ void __launch_bounds__(256) gate_mlp_residual_kernel(const float* __restrict__ h, int64_t ldh, const float* __restrict__ hid,
                                                               const float* __restrict__ W2, const float* __restrict__ b2, int Hd,
                                                               const float* __restrict__ res, int64_t ldr, float* __restrict__ out, int64_t ldo, int HW,
                                                               int C) {
    pdl_sync();
    __shared__ __align__(16) float gate_s[8];
    const int n = blockIdx.y, c0 = blockIdx.x * 8;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    {
        const int c = c0 + warp;
        float acc = 0.f;
        if (c < C) {
            const float* wr = W2 + (int64_t)c * Hd;
            const float* hr = hid + (int64_t)n * Hd;
            if ((Hd & 3) == 0) {
                for (int k = lane * 4; k < Hd; k += 128) {
                    const float4 w = __ldg(reinterpret_cast<const float4*>(wr + k));
                    const float4 x = __ldg(reinterpret_cast<const float4*>(hr + k));
                    acc += w.x * x.x + w.y * x.y + w.z * x.z + w.w * x.w;
                }
            } else {
                for (int k = lane; k < Hd; k += 32) acc += __ldg(wr + k) * __ldg(hr + k);
            }
        }
        acc = warp_sum(acc);
        if (lane == 0) gate_s[warp] = (c < C) ? sigmoid_f(acc + b2[c]) : 0.f;
    }
    __syncthreads();
    const int q = threadIdx.x & 1, pg = threadIdx.x >> 1;
    const int c = c0 + q * 4;
    if (c >= C) return;
    const float4 g = *reinterpret_cast<const float4*>(gate_s + q * 4);
    const float* hb = h + (int64_t)n * HW * ldh + c;
    const float* rb = res + (int64_t)n * HW * ldr + c;
    float* ob = out + (int64_t)n * HW * ldo + c;
    const int pstep = 128 * (int)gridDim.z;
#pragma unroll 4
    for (int p = pg + 128 * (int)blockIdx.z; p < HW; p += pstep) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(hb + (int64_t)p * ldh));
        const float4 r = __ldg(reinterpret_cast<const float4*>(rb + (int64_t)p * ldr));
        *reinterpret_cast<float4*>(ob + (int64_t)p * ldo) = make_float4(v.x * g.x + r.x, v.y * g.y + r.y, v.z * g.z + r.z, v.w * g.w + r.w);
    }
}

// ------------------------------------------------------------------------------------ VAE helpers (ldm AttnBlock / Upsample)
// y[r][:] = softmax(scale * x[r][:]) over `cols` columns; one CTA per row (ldm model.py:183-190: single-head attention over h*w tokens)
__global__ void __launch_bounds__(256) softmax_rows_kernel(const float* __restrict__ x, int64_t ldx, float* __restrict__ y, int64_t ldy, int cols,
                                                          float scale) {
    pdl_sync();
    __shared__ float red[8];
    const float* xr = x + (int64_t)blockIdx.x * ldx;
    float* yr = y + (int64_t)blockIdx.x * ldy;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float mx = -INFINITY;
    for (int c = threadIdx.x; c < cols; c += 256) mx = fmaxf(mx, xr[c] * scale);
    mx = warp_max(mx);
    if (lane == 0) red[warp] = mx;
    __syncthreads();
    mx = red[0];
#pragma unroll
    for (int w = 1; w < 8; ++w) mx = fmaxf(mx, red[w]);
    __syncthreads();
    float sm = 0.f;
    for (int c = threadIdx.x; c < cols; c += 256) sm += expf(xr[c] * scale - mx);
    sm = warp_sum(sm);
    if (lane == 0) red[warp] = sm;
    __syncthreads();
    float tot = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) tot += red[w];
    const float inv = 1.f / tot;
    for (int c = threadIdx.x; c < cols; c += 256) yr[c] = expf(xr[c] * scale - mx) * inv;
}

// nearest-neighbour x2 upsampling, NHWC: out[n][2h+i][2w+j][c] = x[n][h][w][c]   (ldm model.py:44-52)
__global__ void upsample2x_kernel(const float4* __restrict__ x, int64_t ldx_v, float4* __restrict__ out, int64_t ldo_v, int H, int W, int Cv, int64_t total) {
    pdl_sync();
    for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(idx % Cv);
        int64_t t = idx / Cv;
        const int ow = (int)(t % (2 * W)); t /= (2 * W);
        const int oh = (int)(t % (2 * H));
        const int64_t n = t / (2 * H);
        out[((n * 2 * H + oh) * (int64_t)(2 * W) + ow) * ldo_v + c] = __ldg(x + ((n * H + (oh >> 1)) * W + (ow >> 1)) * ldx_v + c);
    }
}

void trace_bind_unet_ops(unsigned long long* buf, unsigned int cap) { trace_bind_this_tu(buf, cap); }

static inline int ew_blocks(int64_t total, int threads = 256) {
    int64_t b = (total + threads - 1) / threads;
    const int64_t cap = (int64_t)sm_count() * 16;
    return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

}  // namespace sfb

using namespace sfb;

extern "C" {

int sfb_nchw_to_nhwc(const float* src, float* dst, int NB, int C, int H, int W, int64_t ld, int c_off, int round_tf32, void* stream) {
    SFB_REQUIRE(src && dst, "nchw_to_nhwc: null pointer");
    dim3 grid(ceil_div(H * W, 32), ceil_div(C, 32), NB), block(32, 8);
    SFB_LAUNCH(nchw_to_nhwc_kernel, grid, block, 0, as_stream(stream), src, dst, C, H * W, ld, c_off, round_tf32 && precision_mode() == 0);
    return check_launch("nchw_to_nhwc");
}

int sfb_nhwc_to_nchw(const float* src, float* dst, int NB, int C, int H, int W, int64_t ld, void* stream) {
    SFB_REQUIRE(src && dst, "nhwc_to_nchw: null pointer");
    dim3 grid(ceil_div(H * W, 32), ceil_div(C, 32), NB), block(32, 8);
    SFB_LAUNCH(nhwc_to_nchw_kernel, grid, block, 0, as_stream(stream), src, dst, C, H * W, ld);
    return check_launch("nhwc_to_nchw");
}

int sfb_concat2_nhwc(const float* a, int C1, int64_t lda, const float* b, int C2, int64_t ldb, float scale_b, float* out, int64_t ldo,
                     int64_t npix, void* stream) {
    SFB_REQUIRE(a && b && out, "concat2_nhwc: null pointer");
    SFB_REQUIRE(C1 % 4 == 0 && C2 % 4 == 0 && lda % 4 == 0 && ldb % 4 == 0 && ldo % 4 == 0, "concat2_nhwc: channel counts must be multiples of 4");
    const int64_t total = npix * ((C1 + C2) / 4);
    SFB_LAUNCH(concat2_kernel, ew_blocks(total), 256, 0, as_stream(stream), reinterpret_cast<const float4*>(a), C1 / 4, lda / 4,
                                                                    reinterpret_cast<const float4*>(b), C2 / 4, ldb / 4, scale_b,
                                                                    reinterpret_cast<float4*>(out), ldo / 4, npix);
    return check_launch("concat2_nhwc");
}

int sfb_pixel_shuffle_silu_nhwc(const float* y, float* out, int NB, int H, int W, int Co, int64_t ldo, void* stream) {
    SFB_REQUIRE(y && out, "pixel_shuffle_silu: null pointer");
    const int64_t total = (int64_t)NB * 4 * H * W * Co;
    SFB_LAUNCH(pixel_shuffle_silu_kernel, ew_blocks(total), 256, 0, as_stream(stream), y, out, H, W, Co, ldo, total);
    return check_launch("pixel_shuffle_silu");
}

int sfb_im2col4_nhwc(const float* x, int64_t ldx, float* out, int64_t ldo, int NB, int H, int W, int KH, int KW, int pad, void* stream) {
    SFB_REQUIRE(x && out, "im2col4: null pointer");
    SFB_REQUIRE(ldx % 4 == 0 && ldo % 4 == 0 && ldo >= (int64_t)KH * KW * 4, "im2col4: 4-channel input (16-byte pixels), ldo >= 4 KH KW, multiples of 4");
    const int64_t total = (int64_t)NB * H * W * (ldo / 4);
    if (total == 0) return SFB_OK;
    SFB_LAUNCH(im2col_small_kernel, ew_blocks(total), 256, 0, as_stream(stream), x, ldx, out, ldo, H, W, 4, KH, KW, pad, total);
    return check_launch("im2col4");
}

int sfb_groupnorm_ws_floats(int NB, int G) { return ((2 * NB * G + 3) / 4) * 4 + NB * G * kGnMaxSlabs * 4; }

int sfb_groupnorm_nhwc(const float* x, int64_t ldx, int NB, int HW, int C, int G, const float* gamma, const float* beta, const float* film,
                       int64_t film_ld, int act_silu, float eps, float* stats_ws, unsigned int* counters, float* y, int64_t ldy, void* stream) {
    SFB_REQUIRE(x && gamma && beta && stats_ws && y, "groupnorm_nhwc: null pointer");
    SFB_REQUIRE(((uintptr_t)stats_ws & 15) == 0, "groupnorm_nhwc: workspace must be 16-byte aligned");
    SFB_REQUIRE(C % G == 0 && C % 4 == 0 && ldx % 4 == 0 && ldy % 4 == 0, "groupnorm_nhwc: C must be a multiple of the group count and of 4");
    cudaStream_t st = as_stream(stream);
    // workspace: 16-byte aligned fp64 partials [NB*G*S][2] (the leading (mean, rstd) slots of the old layout stay unused)
    SFB_REQUIRE(G <= kGnMaxGroups, "groupnorm_nhwc: at most 32 groups");
    double2* partial = reinterpret_cast<double2*>(stats_ws + (((size_t)2 * NB * G + 3) / 4) * 4);
    const int C4 = C / 4, Cg = C / G;
    // ... for batches up to 4 images (<= 256 CTAs): it is a latency optimisation.  From batch 8 on the two-launch path's row-coalesced passes win
    // (batch-16 evaluation 5.87 ms against 6.38 ms)
    // ... and for tensors of at most 1 Mi elements: 64 - 256 CTAs each reading 64-byte runs cannot pull the bandwidth a 64 x 64 x 512 VAE layer needs
    // (35 us in the cluster kernel against ~25 us for the two row-coalesced launches)
    if (gn_cluster_enabled() && (Cg % 16 == 0) && HW >= 1 && NB <= 4 && (int64_t)NB * HW * C <= (1 << 20)) {
        // one cluster of k CTAs per (image, group); a CTA holds ceil(HW/k) * Cg/4 float4 in registers.  Cg >= 16 keeps every pixel's share a
        // multiple of 64 contiguous bytes (full sectors); narrower groups (the VAE's 128-channel layers) stay on the row-coalesced two-launch path
        // always the widest portable cluster: narrower clusters (or a plain CTA per group) for the small stages measured slower (6.96 vs 5.98 us per launch)
        unsigned k = 8;
        while (k > 1 && (int)k > HW) k >>= 1;
        const int64_t per_cta = (int64_t)((HW + (int)k - 1) / (int)k) * (Cg / 4);
        const int items = (int)((per_cta + 255) / 256);
        if (items <= 16) {     // beyond that (128 x 128 latents) 64 CTAs cannot pull the bandwidth: 47.7 us against 25 us for the two row-coalesced launches
            const dim3 grid(G * k, NB);
            const int rnd = (int)(precision_mode() == 0);
            cudaError_t e;
            if (items <= 4) e = SFB_LAUNCH_CLUSTER(gn_cluster_kernel<4>, grid, 256, 0, st, k, x, ldx, HW, C, G, eps, gamma, beta, film, film_ld, y, ldy, act_silu, rnd);
            else if (items <= 8) e = SFB_LAUNCH_CLUSTER(gn_cluster_kernel<8>, grid, 256, 0, st, k, x, ldx, HW, C, G, eps, gamma, beta, film, film_ld, y, ldy, act_silu, rnd);
            else e = SFB_LAUNCH_CLUSTER(gn_cluster_kernel<16>, grid, 256, 0, st, k, x, ldx, HW, C, G, eps, gamma, beta, film, film_ld, y, ldy, act_silu, rnd);
            (void)e;
            return check_launch("groupnorm_nhwc(cluster)");
        }
    }
    // gn_stats_rows_kernel hands each 256-column pass cols / Cg4 whole groups: a group that straddles two passes would mix two groups' columns
    // and leave the last groups' partials unwritten (C = 3072 or 5120 with 8 groups), so such shapes take the group-major kernel
    const bool rows_ok = (Cg % 4 == 0) && (C4 <= 256 ? (256 % C4 == 0) : (C4 % 256 == 0 && 256 % (Cg / 4) == 0));
    int S = 1;
    if (rows_ok) {
        const int rpi = 256 / (C4 < 256 ? C4 : 256);
        const int want = (2 * sm_count() + NB - 1) / NB;                // ~2 CTAs per SM over the batch
        S = HW / (rpi * 2);                                             // two block iterations per slab: the pass is latency bound (measured: 8 -> 5.5 us, 2 -> 3.8 us)
        if (S > want) S = want;
        if (S > kGnMaxSlabs) S = kGnMaxSlabs;
        if (S < 1) S = 1;
        SFB_LAUNCH(gn_stats_rows_kernel, dim3(S, NB), 256, 0, st, x, ldx, HW, C, G, S, partial);
    } else {
        while (S < 64 && G * NB * S * 2 <= sm_count() * 2 && HW / (S * 2) >= 8) S *= 2;
        SFB_LAUNCH(gn_stats_kernel, dim3(G, NB, S), 256, 0, st, x, ldx, HW, C, G, S, partial);
    }
    if (int rc = check_launch("groupnorm_nhwc(stats)")) return rc;
    const int64_t img4 = (int64_t)HW * (C / 4);
    int ab = (int)((img4 + 256 * 4 - 1) / (256 * 4));     // ~4 float4 per thread
    const int cap = (sm_count() * 8) / (NB < 1 ? 1 : NB);
    if (ab > cap) ab = cap < 1 ? 1 : cap;
    if (ab < 1) ab = 1;
    if (C4 <= 256 && 256 % C4 == 0) {
        const int rpi = 256 / C4;
        int cb = (HW + rpi * 8 - 1) / (rpi * 8);          // ~8 rows per thread
        const int cap3 = (cap * 3) / 8 < 1 ? 1 : (cap * 3) / 8;       // three resident CTAs per SM (84 registers: eight rows in flight per thread)
        if (cb > cap3) cb = cap3;
        SFB_LAUNCH(gn_apply_cols_kernel, dim3(cb, NB), 256, 0, st, x, ldx, (const double2*)partial, S, eps, gamma, beta, film, film_ld, y, ldy, HW, C, G,
                   act_silu, (int)(precision_mode() == 0));
        return check_launch("groupnorm_nhwc(apply, columns)");
    }
    SFB_LAUNCH(gn_apply_kernel, dim3(ab, NB), 256, 0, st, x, ldx, (const double2*)partial, S, eps, gamma, beta, film, film_ld, y, ldy, HW, C, G, act_silu,
               (int)(precision_mode() == 0));
    return check_launch("groupnorm_nhwc(apply)");
}

int sfb_layernorm_rows(const float* x, int64_t ldx, const float* g, const float* b, const float* res, int64_t ldr, float* y, int64_t ldy, int T,
                       int C, int pre_gelu, int round_tf32, void* stream) {
    SFB_REQUIRE(x && g && y, "layernorm_rows: null pointer");
    SFB_LAUNCH(layernorm_rows_kernel, T, 128, 0, as_stream(stream), x, ldx, g, b, res, ldr, y, ldy, T, C, pre_gelu, round_tf32 && precision_mode() == 0);
    return check_launch("layernorm_rows");
}

int sfb_linear_small(const float* x, int64_t ldx, const float* w, const float* bias, const float* res, int64_t ldr, float* y, int64_t ldy, int M,
                     int K, int O, int pre, int post, int round_tf32, void* stream) {
    SFB_REQUIRE(x && w && y, "linear_small: null pointer");
    SFB_REQUIRE(K <= 8192, "linear_small: K too large");
    cudaStream_t st = as_stream(stream);
    if (M <= 2) {
        const size_t sm = (size_t)2 * K * 4;
        SFB_ONCE_PER_DEVICE(SFB_CUDA(cudaFuncSetAttribute(linear_small_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * 8192 * 4)));
        SFB_LAUNCH(linear_small_kernel<2>, dim3(ceil_div(O, 8), ceil_div(M, 2)), 256, sm, st, x, ldx, w, bias, res, ldr, y, ldy, M, K, O, pre, post, round_tf32 && precision_mode() == 0);
    } else {
        const size_t sm = (size_t)8 * K * 4;
        SFB_REQUIRE(sm <= 200 * 1024, "linear_small: K too large for 8-row tile");
        SFB_ONCE_PER_DEVICE(SFB_CUDA(cudaFuncSetAttribute(linear_small_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)));
        SFB_LAUNCH(linear_small_kernel<8>, dim3(ceil_div(O, 8), ceil_div(M, 8)), 256, sm, st, x, ldx, w, bias, res, ldr, y, ldy, M, K, O, pre, post, round_tf32 && precision_mode() == 0);
    }
    return check_launch("linear_small");
}

int sfb_time_fourier(const float* t, const float* w, float* out, int B, int half, void* stream) {
    SFB_REQUIRE(t && w && out, "time_fourier: null pointer");
    const int total = B * (2 * half + 1);
    SFB_LAUNCH(time_fourier_kernel, ceil_div(total, 128), 128, 0, as_stream(stream), t, w, out, B, half);
    return check_launch("time_fourier");
}

int sfb_mq_attention(const float* q, const float* kv, const float* null_kv, const float* ckv, float* out, int B, int n, int heads, int dh, int nc,
                     float scale, void* stream) {
    SFB_REQUIRE(q && kv && null_kv && out && (nc == 0 || ckv), "mq_attention: null pointer");
    const int nk = nc + 1 + n;
    if (nk > 64 && dh % 4 == 0 && dh <= 128) {
        const size_t smk = ((size_t)nk * (2 * dh + 4) + (size_t)8 * ((nk + 31) & ~31) + (size_t)8 * dh) * 4;
        if (smk <= 200 * 1024) {
            // queries per warp: about one CTA per SM over the batch
            int qpw = ceil_div(heads * n * B, 8 * sm_count());
            if (qpw < 1) qpw = 1;
            SFB_ONCE_PER_DEVICE(SFB_CUDA(cudaFuncSetAttribute(mq_attention_keys_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)));
            SFB_LAUNCH(mq_attention_keys_kernel, dim3(ceil_div(heads * n, 8 * qpw), B), 256, smk, as_stream(stream), q, kv, null_kv, ckv, out, n, heads, dh, nc,
                       scale, (int)(precision_mode() == 0), qpw);
            return check_launch("mq_attention(keys)");
        }
    }
    {
        const size_t sm2 = ((size_t)nk * 2 * dh + (size_t)8 * nk) * 4;
        if (dh % 4 == 0 && dh <= 128 && sm2 <= 160 * 1024) {
            SFB_ONCE_PER_DEVICE(SFB_CUDA(cudaFuncSetAttribute(mq_attention_smem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024)));
            SFB_LAUNCH(mq_attention_smem_kernel, dim3(ceil_div(heads * n, 8), B), 256, sm2, as_stream(stream), q, kv, null_kv, ckv, out, n, heads, dh, nc, scale,
                       (int)(precision_mode() == 0));
            return check_launch("mq_attention");
        }
    }
    const int warps = 4;
    const size_t sm = (size_t)warps * nk * 4;
    SFB_REQUIRE(sm <= 48 * 1024, "mq_attention: too many keys for the single-pass kernel");
    SFB_LAUNCH(mq_attention_kernel, ceil_div(B * heads * n, warps), warps * 32, sm, as_stream(stream), q, kv, null_kv, ckv, out, B, n, heads, dh, nc, scale, precision_mode() == 0);
    return check_launch("mq_attention");
}

int sfb_cross_attention(const float* q, const float* kvc, const float* null_kv, float* out, int B, int n, int heads, int dh, int nc, float scale,
                        void* stream) {
    SFB_REQUIRE(q && kvc && null_kv && out, "cross_attention: null pointer");
    SFB_REQUIRE(nc <= 8, "cross_attention: at most 8 context tokens");
    SFB_LAUNCH(cross_attention_kernel, ceil_div(B * heads * n, 4), 128, 0, as_stream(stream), q, kvc, null_kv, out, B, n, heads, dh, nc, scale, precision_mode() == 0);
    return check_launch("cross_attention");
}

int sfb_gca_pool(const float* x, int64_t ldx, int NB, int HW, int C, const float* wk, const float* bk, float* logits_ws, float* pooled,
                 void* stream) {
    SFB_REQUIRE(x && wk && bk && logits_ws && pooled, "gca_pool: null pointer");
    SFB_REQUIRE(C % 4 == 0 && ldx % 4 == 0, "gca_pool: unsupported shape");
    cudaStream_t st = as_stream(stream);
    const int64_t npix = (int64_t)NB * HW;
    SFB_LAUNCH(gca_logits_kernel, (unsigned)ceil_div(npix, (int64_t)8), 256, 0, st, x, ldx, wk, bk, logits_ws, npix, C);
    if (int rc = check_launch("gca_pool(logits)")) return rc;
    if (HW >= 4096) {          // pixel-split clusters: 8 CTAs per (image, 16-channel tile)
        const unsigned Z = 8;
        const size_t sms = ((size_t)(((HW + (int)Z - 1) / (int)Z + 4) & ~3) + 64 * kGcaCols) * 4;
        SFB_REQUIRE(sms <= 200 * 1024, "gca_pool: image too large");
        if (sms > 48 * 1024) SFB_ONCE_PER_DEVICE(SFB_CUDA(cudaFuncSetAttribute(gca_pool_split_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)));
        cudaError_t e = SFB_LAUNCH_CLUSTER(gca_pool_split_kernel, dim3(Z * ceil_div(C, kGcaCols), NB), 256, sms, st, Z, x, ldx, (const float*)logits_ws, pooled, HW, C);
        (void)e;
        return check_launch("gca_pool(pool, split)");
    }
    const size_t sm = ((size_t)((HW + 3) & ~3) + 64 * kGcaCols) * 4;
    SFB_REQUIRE(sm <= 200 * 1024, "gca_pool: image too large for the single-pass pooling kernel (softmax weights of one image live in shared memory)");
    if (sm > 48 * 1024) SFB_ONCE_PER_DEVICE(SFB_CUDA(cudaFuncSetAttribute(gca_pool_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)));
    SFB_LAUNCH(gca_pool_kernel, dim3(ceil_div(C, kGcaCols), NB), 256, sm, st, x, ldx, logits_ws, pooled, HW, C);
    return check_launch("gca_pool(pool)");
}

int sfb_gate_mlp_residual_nhwc(const float* h, int64_t ldh, const float* hid, const float* w2, const float* b2, int Hd, const float* res, int64_t ldr,
                               float* out, int64_t ldo, int NB, int HW, int C, void* stream) {
    SFB_REQUIRE(h && hid && w2 && b2 && res && out, "gate_mlp_residual: null pointer");
    SFB_REQUIRE(C % 4 == 0 && ldh % 4 == 0 && ldr % 4 == 0 && ldo % 4 == 0 && Hd > 0, "gate_mlp_residual: channel counts must be multiples of 4");
    if (NB == 0 || HW == 0) return SFB_OK;
    // pixel split: about two CTAs per SM over the batch, at least four 128-pixel passes per CTA
    int Z = (2 * sm_count()) / (ceil_div(C, 8) * NB);
    if (Z > HW / 512) Z = HW / 512;
    if (Z < 1) Z = 1;
    SFB_LAUNCH(gate_mlp_residual_kernel, dim3(ceil_div(C, 8), NB, Z), 256, 0, as_stream(stream), h, ldh, hid, w2, b2, Hd, res, ldr, out, ldo, HW, C);
    return check_launch("gate_mlp_residual");
}

int sfb_softmax_rows(const float* x, int64_t ldx, float* y, int64_t ldy, int rows, int cols, float scale, void* stream) {
    SFB_REQUIRE(x && y && rows >= 0 && cols > 0, "softmax_rows: null pointer or empty row");
    if (rows == 0) return SFB_OK;
    SFB_LAUNCH(softmax_rows_kernel, rows, 256, 0, as_stream(stream), x, ldx, y, ldy, cols, scale);
    return check_launch("softmax_rows");
}

int sfb_upsample2x_nhwc(const float* x, int64_t ldx, float* out, int64_t ldo, int NB, int H, int W, int C, void* stream) {
    SFB_REQUIRE(x && out, "upsample2x_nhwc: null pointer");
    SFB_REQUIRE(C % 4 == 0 && ldx % 4 == 0 && ldo % 4 == 0, "upsample2x_nhwc: channel counts must be multiples of 4");
    const int64_t total = (int64_t)NB * 4 * H * W * (C / 4);
    if (total == 0) return SFB_OK;
    SFB_LAUNCH(upsample2x_kernel, ew_blocks(total), 256, 0, as_stream(stream), reinterpret_cast<const float4*>(x), ldx / 4, reinterpret_cast<float4*>(out),
               ldo / 4, H, W, C / 4, total);
    return check_launch("upsample2x_nhwc");
}

int sfb_gate_residual_nhwc(const float* h, int64_t ldh, const float* gate, const float* res, int64_t ldr, float* out, int64_t ldo, int NB, int HW,
                           int C, void* stream) {
    SFB_REQUIRE(h && res && out, "gate_residual: null pointer");
    SFB_REQUIRE(C % 4 == 0 && ldh % 4 == 0 && ldr % 4 == 0 && ldo % 4 == 0, "gate_residual: channel counts must be multiples of 4");
    const int64_t total = (int64_t)NB * HW * (C / 4);
    SFB_LAUNCH(gate_residual_kernel, ew_blocks(total), 256, 0, as_stream(stream), reinterpret_cast<const float4*>(h), ldh / 4, gate,
                                                                          reinterpret_cast<const float4*>(res), ldr / 4,
                                                                          reinterpret_cast<float4*>(out), ldo / 4, HW, C / 4, total);
    return check_launch("gate_residual");
}
}

// ------------------------------------------------------------------------------------ PLMS sampler update
// One fused pass for PLMSSampler.p_sample's tail (external/plms.py:143-154 + get_model_output :183-212):
//   e' = sum_i coef[i] * eps[i]                                   (Adams-Bashforth combination, :143-152)
//   x0 = clamp((x - sigma * e') / max(alpha, 1e-8), -clip, clip)  (predict_start_from_noise + clamp, :184,:205)
//   x_prev = alpha_next * (x * (1 - c) / alpha + c * x0) + noise_scale * noise     (q_posterior mean + sigma_t * z, :208-212)
// The per-step scalars (alpha, sigma, alpha_next, c, noise_scale = mask * exp(0.5 * log var)) are computed on the host from t, t_next.
// plms_update_rows_kernel is the same element for a batch whose rows sit at different noise levels (scene-batched sampling): row blockIdx.y reads
// its five scalars from a table.  Both kernels run plms_update_element, so a row's result is bit-identical to a separate sfb_plms_update launch.
namespace sfb {
// element i with e0's value already loaded (e0v)
__device__ __forceinline__ void plms_update_value(int64_t i, float e0v, const float* __restrict__ x, const float* __restrict__ e1,
                                                  const float* __restrict__ e2, const float* __restrict__ e3, float c0, float c1, float c2,
                                                  float c3, const float* __restrict__ noise, float alpha, float sigma, float alpha_next, float c,
                                                  float noise_scale, float clip, float* __restrict__ x_prev, float* __restrict__ x0_out,
                                                  float* __restrict__ e_out) {
    float e = c0 * e0v;
    if (e1) e += c1 * e1[i];
    if (e2) e += c2 * e2[i];
    if (e3) e += c3 * e3[i];
    const float xv = x[i];
    float x0 = (xv - sigma * e) / fmaxf(alpha, 1e-8f);
    x0 = clamp_keep_nan(x0, -clip, clip);     // a NaN eps or x gives a NaN x0 and x_prev, as torch.clamp does
    const float mean = alpha_next * (xv * (1.f - c) / alpha + c * x0);
    x_prev[i] = mean + noise_scale * noise[i];
    if (x0_out) x0_out[i] = x0;
    if (e_out) e_out[i] = e;
}

__device__ __forceinline__ void plms_update_element(int64_t i, const float* __restrict__ x, const float* __restrict__ e0,
                                                    const float* __restrict__ e1, const float* __restrict__ e2, const float* __restrict__ e3,
                                                    float c0, float c1, float c2, float c3, const float* __restrict__ noise, float alpha,
                                                    float sigma, float alpha_next, float c, float noise_scale, float clip,
                                                    float* __restrict__ x_prev, float* __restrict__ x0_out, float* __restrict__ e_out) {
    plms_update_value(i, e0[i], x, e1, e2, e3, c0, c1, c2, c3, noise, alpha, sigma, alpha_next, c, noise_scale, clip, x_prev, x0_out, e_out);
}

__global__ void plms_update_kernel(const float* __restrict__ x, const float* __restrict__ e0, const float* __restrict__ e1,
                                   const float* __restrict__ e2, const float* __restrict__ e3, float c0, float c1, float c2, float c3,
                                   const float* __restrict__ noise, float alpha, float sigma, float alpha_next, float c, float noise_scale,
                                   float clip, float* __restrict__ x_prev, float* __restrict__ x0_out, float* __restrict__ e_out, int64_t n) {
    pdl_sync();
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        plms_update_element(i, x, e0, e1, e2, e3, c0, c1, c2, c3, noise, alpha, sigma, alpha_next, c, noise_scale, clip, x_prev, x0_out, e_out);
}

__global__ void plms_update_rows_kernel(const float* __restrict__ x, const float* __restrict__ e0, const float* __restrict__ e1,
                                        const float* __restrict__ e2, const float* __restrict__ e3, float c0, float c1, float c2, float c3,
                                        const float* __restrict__ noise, const float* __restrict__ row_scalars, float clip,
                                        float* __restrict__ x_prev, float* __restrict__ x0_out, int64_t row_len) {
    pdl_sync();
    __shared__ float s[5];
    const int64_t off = (int64_t)blockIdx.y * row_len;
    if (threadIdx.x < 5) s[threadIdx.x] = row_scalars[blockIdx.y * 5 + threadIdx.x];
    __syncthreads();
    const float alpha = s[0], sigma = s[1], alpha_next = s[2], c = s[3], noise_scale = s[4];
    // row-local pointers (NULL stays NULL): element i of the row is element off + i of the batch
    const float* r1 = e1 ? e1 + off : nullptr;
    const float* r2 = e2 ? e2 + off : nullptr;
    const float* r3 = e3 ? e3 + off : nullptr;
    float* rx0 = x0_out ? x0_out + off : nullptr;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < row_len; i += (int64_t)gridDim.x * blockDim.x)
        plms_update_element(i, x + off, e0 + off, r1, r2, r3, c0, c1, c2, c3, noise + off, alpha, sigma, alpha_next, c, noise_scale, clip,
                            x_prev + off, rx0, nullptr);
}

// Classifier-free guidance in front of the same element: e_t = e_null + (e_cond - e_null) * cond_scale (imagen_pytorch.py:572-577) is formed
// in a register, written to e_out (the sampler's eps history holds the guided eps, as the reference's p_sample returns it) and takes e0's place
// in the combination, so the update rounds exactly as plms_update_rows_kernel with e0 = e_out.
__global__ void plms_update_rows_cfg_kernel(const float* __restrict__ x, const float* __restrict__ e_cond, const float* __restrict__ e_null,
                                            float cond_scale, const float* __restrict__ e1, const float* __restrict__ e2,
                                            const float* __restrict__ e3, float c0, float c1, float c2, float c3, const float* __restrict__ noise,
                                            const float* __restrict__ row_scalars, float clip, float* __restrict__ x_prev,
                                            float* __restrict__ e_out, int64_t row_len) {
    pdl_sync();
    __shared__ float s[5];
    const int64_t off = (int64_t)blockIdx.y * row_len;
    if (threadIdx.x < 5) s[threadIdx.x] = row_scalars[blockIdx.y * 5 + threadIdx.x];
    __syncthreads();
    const float alpha = s[0], sigma = s[1], alpha_next = s[2], c = s[3], noise_scale = s[4];
    const float* r1 = e1 ? e1 + off : nullptr;
    const float* r2 = e2 ? e2 + off : nullptr;
    const float* r3 = e3 ? e3 + off : nullptr;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < row_len; i += (int64_t)gridDim.x * blockDim.x) {
        const float en = e_null[off + i];
        const float et = __fadd_rn(en, __fmul_rn(__fsub_rn(e_cond[off + i], en), cond_scale));   // no FMA contraction: the reference's rounding
        if (e_out) e_out[off + i] = et;
        plms_update_value(i, et, x + off, r1, r2, r3, c0, c1, c2, c3, noise + off, alpha, sigma, alpha_next, c, noise_scale, clip, x_prev + off,
                          nullptr, nullptr);
    }
}
}  // namespace sfb

extern "C" int sfb_plms_update(const float* x, const float* e0, const float* e1, const float* e2, const float* e3, float c0, float c1, float c2,
                               float c3, const float* noise, float alpha, float sigma, float alpha_next, float c, float noise_scale, float clip,
                               float* x_prev, float* x0_out, float* e_out, int64_t n, void* stream) {
    if (n == 0) return SFB_OK;
    SFB_REQUIRE(x && e0 && noise && x_prev, "plms_update: null pointer");
    int64_t blocks = (n + 255) / 256;
    if (blocks > 1024) blocks = 1024;
    SFB_LAUNCH(sfb::plms_update_kernel, (unsigned)blocks, 256, 0, sfb::as_stream(stream), x, e0, e1, e2, e3, c0, c1, c2, c3, noise, alpha, sigma, alpha_next, c,
                                                                                 noise_scale, clip, x_prev, x0_out, e_out, n);
    return sfb::check_launch("plms_update");
}

extern "C" int sfb_plms_update_rows(const float* x, const float* e0, const float* e1, const float* e2, const float* e3, float c0, float c1,
                                    float c2, float c3, const float* noise, const float* row_scalars, float clip, float* x_prev, float* x0_out,
                                    int rows, int64_t row_len, void* stream) {
    if (rows == 0 || row_len == 0) return SFB_OK;
    SFB_REQUIRE(x && e0 && noise && row_scalars && x_prev, "plms_update_rows: null pointer");
    SFB_REQUIRE(rows > 0 && rows <= 65535 && row_len > 0, "plms_update_rows: rows must be in [1, 65535]");
    int64_t bx = (row_len + 255) / 256;
    if (bx > 1024) bx = 1024;
    SFB_LAUNCH(sfb::plms_update_rows_kernel, dim3((unsigned)bx, (unsigned)rows), 256, 0, sfb::as_stream(stream), x, e0, e1, e2, e3, c0, c1, c2, c3,
               noise, row_scalars, clip, x_prev, x0_out, row_len);
    return sfb::check_launch("plms_update_rows");
}

extern "C" int sfb_plms_update_rows_cfg(const float* x, const float* e_cond, const float* e_null, float cond_scale, const float* e1, const float* e2,
                                        const float* e3, float c0, float c1, float c2, float c3, const float* noise, const float* row_scalars,
                                        float clip, float* x_prev, float* e_out, int rows, int64_t row_len, void* stream) {
    if (rows == 0 || row_len == 0) return SFB_OK;
    SFB_REQUIRE(x && e_cond && e_null && noise && row_scalars && x_prev, "plms_update_rows_cfg: null pointer");
    SFB_REQUIRE(rows > 0 && rows <= 65535 && row_len > 0, "plms_update_rows_cfg: rows must be in [1, 65535]");
    int64_t bx = (row_len + 255) / 256;
    if (bx > 1024) bx = 1024;
    SFB_LAUNCH(sfb::plms_update_rows_cfg_kernel, dim3((unsigned)bx, (unsigned)rows), 256, 0, sfb::as_stream(stream), x, e_cond, e_null, cond_scale,
               e1, e2, e3, c0, c1, c2, c3, noise, row_scalars, clip, x_prev, e_out, row_len);
    return sfb::check_launch("plms_update_rows_cfg");
}

// ------------------------------------------------------------------------------------ DDPM ancestral step with dynamic thresholding
// One launch per step of DDPM.p_sample (sparsefusion/vldm.py:289-361) when dynamic_thresholding is on.  Per row (one sample of row_len floats):
//   e  = cond_scale * e_cond + (1 - cond_scale) * e_null      (classifier-free guidance; e = e_cond when e_null is NULL)
//   x0 = (x - sigma * e) / max(alpha, 1e-8)
//   s  = max(torch.quantile(|x0|, p, 'linear'), 1);  x0 = clamp(x0, -s, s) / s
//   x_prev = alpha_next * (x * (1 - c) / alpha + c * x0) + noise_scale * noise        (same expression order as plms_update_kernel)
// The quantile is exact: |x0| >= 0, so the order of its uint32 bit patterns is the order of the values, and a 4-pass radix select on 8-bit digits
// finds the value of rank floor(p * (n - 1)) without sorting; the next rank is either the same value (ties) or the least value above it.  A row
// is split over a thread-block cluster of up to 8 CTAs (kDynChunk floats each, held in shared memory); their digit histograms are summed
// through distributed shared memory, as in gn_cluster_kernel.  NaN patterns sort above +inf; torch.quantile returns NaN for a row that holds
// a NaN, so pass 0's histogram has a 257th bin counting them, and such a row gets s = NaN (and an all-NaN x_prev, as clamp / s gives).
namespace sfb {
constexpr int kDynThreads = 1024;
constexpr int kDynChunk = 8192;       // floats of a row per CTA: 32 KB of shared memory
constexpr int kDynMaxCluster = 8;     // portable cluster size: rows up to 65 536 floats (4 x 128 x 128 latents)

template <bool CLUSTER>
__device__ __forceinline__ void dyn_sync() {
    if (CLUSTER) cg::this_cluster().sync();
    else __syncthreads();
}

template <bool CLUSTER>
__global__ void __launch_bounds__(kDynThreads) ddpm_dynamic_step_kernel(
    const float* __restrict__ x, const float* __restrict__ e_cond, const float* __restrict__ e_null, float cond_scale,
    const float* __restrict__ noise, float alpha, float sigma, float alpha_next, float c, float noise_scale, float percentile, int row_len,
    float* __restrict__ x_prev, float* __restrict__ s_out, float* __restrict__ x0_out) {
    pdl_sync();
    extern __shared__ float x0s[];                 // this CTA's slice of the row's x0
    __shared__ unsigned hist[2][257];              // digit histogram (+ NaN count), double-buffered so that one cluster barrier per pass suffices
    __shared__ unsigned tot[257];
    __shared__ unsigned sel[3];                    // selected digit, rank left within it, its count
    __shared__ unsigned vmin;
    unsigned k = 1, crank = 0;
    if (CLUSTER) {
        cg::cluster_group cl = cg::this_cluster();
        k = cl.num_blocks();
        crank = cl.block_rank();
    }
    const int chunk = (row_len + (int)k - 1) / (int)k;
    const int i0 = min(row_len, (int)crank * chunk), len = min(row_len, i0 + chunk) - i0;
    const int64_t base = (int64_t)blockIdx.y * row_len + i0;
    const int lane = threadIdx.x & 31;
    for (int i = threadIdx.x; i < 2 * 257; i += blockDim.x) (&hist[0][0])[i] = 0u;
    if (threadIdx.x == 0) vmin = 0xffffffffu;

    const float cn = 1.f - cond_scale;
    const float alpha_c = fmaxf(alpha, 1e-8f);
    for (int i = threadIdx.x; i < len; i += blockDim.x) {
        float e = cond_scale * e_cond[base + i];
        if (e_null) e += cn * e_null[base + i];
        const float x0 = (x[base + i] - sigma * e) / alpha_c;
        x0s[i] = x0;
        if (x0_out) x0_out[base + i] = x0;
    }

    // torch.quantile(..., interpolation='linear'): rank = q * (n - 1) in fp32, values at floor / ceil of it, lerp (ATen/native/Lerp.h)
    const float rk = percentile * (float)(row_len - 1);
    const int klo = (int)rk, khi = (int)ceilf(rk);
    const float w = rk - (float)klo;
    unsigned prefix = 0u, want = (unsigned)klo, cnt_eq = 0u;
    bool has_nan = false;
    const int iters = (len + blockDim.x - 1) / blockDim.x;
#pragma unroll 1
    for (int pass = 0; pass < 4; ++pass) {
        const int shift = 24 - 8 * pass;
        const unsigned pmask = pass == 0 ? 0u : (0xffffffffu << (shift + 8));
        unsigned* h = hist[pass & 1];
        __syncthreads();                                           // x0s written, h zeroed
        for (int it = 0; it < iters; ++it) {                       // warp-uniform trip count: __match_any_sync below needs full warps
            const int i = it * blockDim.x + threadIdx.x;
            const unsigned u = i < len ? (__float_as_uint(x0s[i]) & 0x7fffffffu) : 0u;
            const bool m = i < len && (u & pmask) == prefix;
            const unsigned d = (u >> shift) & 255u;
            const unsigned peers = __match_any_sync(0xffffffffu, m ? d : 0xffffffffu);   // lanes with the same digit add once
            if (m && lane == __ffs(peers) - 1) atomicAdd(&h[d], (unsigned)__popc(peers));
            if (pass == 0) {
                const unsigned nans = __ballot_sync(0xffffffffu, i < len && u > 0x7f800000u);
                if (nans && lane == 0) atomicAdd(&h[256], (unsigned)__popc(nans));
            }
        }
        dyn_sync<CLUSTER>();                                       // every CTA's histogram of this pass is complete
        for (int b = threadIdx.x; b < 257; b += blockDim.x) {
            unsigned s = 0u;
            if (CLUSTER) {
                cg::cluster_group cl = cg::this_cluster();
                for (unsigned r = 0; r < k; ++r) s += cl.map_shared_rank(h, r)[b];
            } else {
                s = h[b];
            }
            tot[b] = s;
        }
        // every peer finished reading the other buffer before it reached the barrier above: clear it for the next pass
        for (int b = threadIdx.x; b < 257; b += blockDim.x) hist[(pass + 1) & 1][b] = 0u;
        __syncthreads();
        if (threadIdx.x < 32) {                                    // find the digit holding rank `want`: 8 bins per lane, warp prefix sum
            unsigned v[8], sum = 0u;
#pragma unroll
            for (int j = 0; j < 8; ++j) { v[j] = tot[lane * 8 + j]; sum += v[j]; }
            unsigned incl = sum;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned n = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += n;
            }
            unsigned acc = incl - sum;
            if (want >= acc && want < incl) {
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    if (want >= acc && want < acc + v[j]) { sel[0] = lane * 8 + j; sel[1] = want - acc; sel[2] = v[j]; }
                    acc += v[j];
                }
            }
        }
        __syncthreads();
        if (pass == 0) has_nan = tot[256] != 0u;
        prefix |= sel[0] << shift;
        want = sel[1];
        cnt_eq = sel[2];
    }
    const float vlo = __uint_as_float(prefix);
    float vhi = vlo;
    if (khi != klo && want + 1u >= cnt_eq) {                       // rank khi lies above the ties of vlo: the least |x0| greater than vlo
        unsigned m = 0xffffffffu;
        for (int i = threadIdx.x; i < len; i += blockDim.x) {
            const unsigned u = __float_as_uint(x0s[i]) & 0x7fffffffu;
            if (u > prefix) m = min(m, u);
        }
        m = __reduce_min_sync(0xffffffffu, m);
        if (lane == 0) atomicMin(&vmin, m);
        dyn_sync<CLUSTER>();
        if (CLUSTER) {
            cg::cluster_group cl = cg::this_cluster();
            for (unsigned r = 0; r < k; ++r) m = min(m, *cl.map_shared_rank(&vmin, r));
        } else {
            m = vmin;
        }
        vhi = __uint_as_float(m);
    }
    if (CLUSTER) asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");   // done reading the peers' shared memory ...
    const float dv = vhi - vlo;
    // lerp(vlo, vhi, w) exactly as ATen/native/Lerp.h compiles for CUDA (the product and the add contract to one fma)
    const float q = has_nan ? __uint_as_float(0x7fffffffu) : (fabsf(w) < 0.5f ? __fmaf_rn(w, dv, vlo) : __fmaf_rn(-dv, 1.f - w, vhi));
    const float s = q != q ? q : fmaxf(q, 1.f);                    // .clamp(min=1) keeps NaN
    if (s_out && crank == 0 && threadIdx.x == 0) s_out[blockIdx.y] = s;
    for (int i = threadIdx.x; i < len; i += blockDim.x) {
        const float x0 = clamp_keep_nan(x0s[i], -s, s) / s;
        const float xv = x[base + i];
        const float mean = alpha_next * (xv * (1.f - c) / alpha + c * x0);
        x_prev[base + i] = mean + noise_scale * noise[base + i];
    }
    if (CLUSTER) asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");     // ... and stays resident until the peers are too
}
}  // namespace sfb

extern "C" int sfb_ddpm_dynamic_step(const float* x, const float* e_cond, const float* e_null, float cond_scale, const float* noise, float alpha,
                                     float sigma, float alpha_next, float c, float noise_scale, float percentile, int row_len, int B, float* x_prev,
                                     float* s_out, float* x0_out, void* stream) {
    SFB_REQUIRE(B >= 0 && B <= 65535, "ddpm_dynamic_step: B must be 0..65535");
    if (B == 0) return SFB_OK;
    SFB_REQUIRE(x && e_cond && noise && x_prev, "ddpm_dynamic_step: null pointer");
    SFB_REQUIRE(row_len >= 1 && row_len <= sfb::kDynChunk * sfb::kDynMaxCluster, "ddpm_dynamic_step: row_len must be 1..%d", sfb::kDynChunk * sfb::kDynMaxCluster);
    SFB_REQUIRE(percentile >= 0.f && percentile <= 1.f, "ddpm_dynamic_step: percentile must be in [0, 1]");
    const unsigned k = (unsigned)((row_len + sfb::kDynChunk - 1) / sfb::kDynChunk);
    const size_t smem = (size_t)((row_len + (int)k - 1) / (int)k) * sizeof(float);
    cudaStream_t st = sfb::as_stream(stream);
    if (k == 1) {
        SFB_LAUNCH(sfb::ddpm_dynamic_step_kernel<false>, dim3(1, B), sfb::kDynThreads, smem, st, x, e_cond, e_null, cond_scale, noise, alpha, sigma,
                   alpha_next, c, noise_scale, percentile, row_len, x_prev, s_out, x0_out);
    } else {
        SFB_LAUNCH_CLUSTER(sfb::ddpm_dynamic_step_kernel<true>, dim3(k, B), sfb::kDynThreads, smem, st, k, x, e_cond, e_null, cond_scale, noise, alpha,
                           sigma, alpha_next, c, noise_scale, percentile, row_len, x_prev, s_out, x0_out);
    }
    return sfb::check_launch("ddpm_dynamic_step");
}
