// metrics.cu -- SSIM and mean squared error of image pairs with scikit-image's semantics (the scores the reference writes after distilling a
// scene: sparsefusion/distillation.py:391-443, utils/common_utils.py:48-64).
//
// Images are fp32 [B][H][W][3].  Per channel, scikit-image filters a, b, a*a, b*b and a*b with scipy.ndimage.uniform_filter (size 7,
// mode 'reflect'); scipy runs each 1D pass over fp64 line buffers and stores the result as fp32, so the box sums here are fp64 and rounded to
// fp32 after each pass (axis 0, then axis 1).  Everything after the filter is fp32 arithmetic in numpy's operation order, written with
// explicit _rn intrinsics so that nvcc cannot contract it into FMAs: identical images then give an SSIM map of exactly 1.
// One CTA per (image, 32x32 output tile) keeps both images' tile plus a 3-pixel reflected halo in shared memory and writes four fp64
// partial sums (the SSIM map over the cropped interior, per channel, and the squared error over the tile); one CTA per image adds them in a
// fixed order.  No atomics: repeated calls are bit-identical.
#include "common.cuh"

namespace sfb {
namespace {

constexpr int kTile = 32;                 // output pixels per tile side
constexpr int kHalf = 3;                  // window radius (7x7 window)
constexpr int kWin = 2 * kHalf + 1;
constexpr int kIn = kTile + 2 * kHalf;    // tile side with its halo
constexpr int kThreads = 256;
constexpr int kParts = 4;                 // partial sums per tile: SSIM map of channels 0..2, squared error

// scipy.ndimage mode='reflect' (half-sample symmetric: d c b a | a b c d | d c b a), folding as often as needed
__device__ __forceinline__ int reflect_index(int q, int n) {
    if ((unsigned)q < (unsigned)n) return q;
    const int p = 2 * n;
    int m = q % p;
    if (m < 0) m += p;
    return m < n ? m : p - 1 - m;
}

// fixed-order sum of kParts values over the block (warp shuffles, then the warp totals); valid in thread 0
__device__ void block_sum_parts(double (&x)[kParts]) {
    __shared__ double warp_tot[kParts][kThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < kParts; ++k) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) x[k] += __shfl_down_sync(0xffffffffu, x[k], o);
        if (lane == 0) warp_tot[k][warp] = x[k];
    }
    __syncthreads();
    if (warp == 0) {
#pragma unroll
        for (int k = 0; k < kParts; ++k) {
            x[k] = lane < kThreads / 32 ? warp_tot[k][lane] : 0.0;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) x[k] += __shfl_down_sync(0xffffffffu, x[k], o);
        }
    }
}

__device__ __forceinline__ float box_mean(double s) { return (float)(s / (double)kWin); }

__global__ void __launch_bounds__(kThreads) ssim_tile_kernel(const float* __restrict__ a, const float* __restrict__ b, int H, int W, int tiles_x,
                                                             double* __restrict__ part) {
    __shared__ float sa[kIn][kIn], sb[kIn][kIn];
    __shared__ float col[5][kTile][kIn];       // axis-0 pass of the five moments: rows of the tile, columns of tile + halo
    const int tile = blockIdx.x, img = blockIdx.y;
    const int y0 = (tile / tiles_x) * kTile, x0 = (tile % tiles_x) * kTile;
    const float* pa = a + (size_t)img * H * W * 3;
    const float* pb = b + (size_t)img * H * W * 3;
    // numpy's Python-float constants, rounded to fp32 where they meet fp32 arrays
    const float cov_norm = (float)(49.0 / 48.0);
    const float C1 = (float)((0.01 * 1.0) * (0.01 * 1.0)), C2 = (float)((0.03 * 1.0) * (0.03 * 1.0));
    double acc[kParts] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        if (c) __syncthreads();                 // the previous channel's readers are done with sa / sb / col
        for (int q = threadIdx.x; q < kIn * kIn; q += kThreads) {
            const int r = q / kIn, x = q % kIn;
            const size_t off = ((size_t)reflect_index(y0 - kHalf + r, H) * W + reflect_index(x0 - kHalf + x, W)) * 3 + c;
            sa[r][x] = pa[off];
            sb[r][x] = pb[off];
        }
        __syncthreads();
        for (int q = threadIdx.x; q < kTile * kIn; q += kThreads) {
            const int r = q / kIn, x = q % kIn;
            double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0, s4 = 0.0;
#pragma unroll
            for (int k = 0; k < kWin; ++k) {
                const float u = sa[r + k][x], v = sb[r + k][x];
                s0 += (double)u;
                s1 += (double)v;
                s2 += (double)__fmul_rn(u, u);
                s3 += (double)__fmul_rn(v, v);
                s4 += (double)__fmul_rn(u, v);
            }
            col[0][r][x] = box_mean(s0);
            col[1][r][x] = box_mean(s1);
            col[2][r][x] = box_mean(s2);
            col[3][r][x] = box_mean(s3);
            col[4][r][x] = box_mean(s4);
        }
        __syncthreads();
        for (int q = threadIdx.x; q < kTile * kTile; q += kThreads) {
            const int r = q / kTile, x = q % kTile, gy = y0 + r, gx = x0 + x;
            if (gy >= H || gx >= W) continue;
            double s[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll
            for (int k = 0; k < kWin; ++k) {
#pragma unroll
                for (int m = 0; m < 5; ++m) s[m] += (double)col[m][r][x + k];
            }
            const float ux = box_mean(s[0]), uy = box_mean(s[1]), uxx = box_mean(s[2]), uyy = box_mean(s[3]), uxy = box_mean(s[4]);
            // skimage.metrics.structural_similarity, float32 branch, term by term
            const float vx = __fmul_rn(cov_norm, __fsub_rn(uxx, __fmul_rn(ux, ux)));
            const float vy = __fmul_rn(cov_norm, __fsub_rn(uyy, __fmul_rn(uy, uy)));
            const float vxy = __fmul_rn(cov_norm, __fsub_rn(uxy, __fmul_rn(ux, uy)));
            const float A1 = __fadd_rn(__fmul_rn(__fmul_rn(2.f, ux), uy), C1);
            const float A2 = __fadd_rn(__fmul_rn(2.f, vxy), C2);
            const float B1 = __fadd_rn(__fadd_rn(__fmul_rn(ux, ux), __fmul_rn(uy, uy)), C1);
            const float B2 = __fadd_rn(__fadd_rn(vx, vy), C2);
            const float S = __fdiv_rn(__fmul_rn(A1, A2), __fmul_rn(B1, B2));
            if (gy >= kHalf && gy < H - kHalf && gx >= kHalf && gx < W - kHalf) acc[c] += (double)S;
            const float d = __fsub_rn(sa[r + kHalf][x + kHalf], sb[r + kHalf][x + kHalf]);
            acc[3] += (double)__fmul_rn(d, d);
        }
    }
    block_sum_parts(acc);
    if (threadIdx.x == 0) {
        double* p = part + ((size_t)img * gridDim.x + tile) * kParts;
#pragma unroll
        for (int k = 0; k < kParts; ++k) p[k] = acc[k];
    }
}

// one CTA per image: add its tiles' partial sums in a fixed order, then the per-channel means and scikit-image's fp32 mean of the three
__global__ void __launch_bounds__(kThreads) ssim_final_kernel(const double* __restrict__ part, int tiles, int H, int W, double* __restrict__ out) {
    const int img = blockIdx.x;
    double acc[kParts] = {0.0, 0.0, 0.0, 0.0};
    for (int t = threadIdx.x; t < tiles; t += kThreads) {
        const double* p = part + ((size_t)img * tiles + t) * kParts;
#pragma unroll
        for (int k = 0; k < kParts; ++k) acc[k] += p[k];
    }
    block_sum_parts(acc);
    if (threadIdx.x == 0) {
        const double n_in = (double)(H - 2 * kHalf) * (double)(W - 2 * kHalf);
        // mssim = np.empty(3, float32); mssim[ch] = crop(S, 3).mean(dtype=float64); mssim.mean()  (fp32 sum, then / 3)
        const float m0 = (float)(acc[0] / n_in), m1 = (float)(acc[1] / n_in), m2 = (float)(acc[2] / n_in);
        const float sum = __fadd_rn(__fadd_rn(m0, m1), m2);
        out[2 * img] = (double)(float)((double)sum / 3.0);
        out[2 * img + 1] = acc[3] / ((double)H * (double)W * 3.0);
    }
}

bool sizes_ok(int B, int H, int W) {
    return B >= 1 && B <= 65535 && H >= kWin && W >= kWin && (int64_t)ceil_div(H, kTile) * ceil_div(W, kTile) <= (int64_t)INT32_MAX;
}

}  // namespace
}  // namespace sfb

using namespace sfb;

extern "C" {

uint64_t sfb_image_ssim_psnr_work(int B, int H, int W) {
    if (!sizes_ok(B, H, W)) return 0;
    return (uint64_t)B * (uint64_t)ceil_div(H, kTile) * (uint64_t)ceil_div(W, kTile) * kParts;
}

int sfb_image_ssim_psnr(const float* a, const float* b, int B, int H, int W, double* out, double* work, void* stream) {
    SFB_REQUIRE(a && b && out && work, "image_ssim_psnr: null pointer");
    SFB_REQUIRE(B >= 1 && B <= 65535, "image_ssim_psnr: B must be in 1..65535 (got %d)", B);
    SFB_REQUIRE(H >= kWin && W >= kWin, "image_ssim_psnr: images must be at least %d x %d, the SSIM window (got %d x %d)", kWin, kWin, H, W);
    SFB_REQUIRE(sizes_ok(B, H, W), "image_ssim_psnr: image too large (%d x %d)", H, W);
    const int tiles_x = ceil_div(W, kTile);
    const int64_t tiles = (int64_t)ceil_div(H, kTile) * tiles_x;
    const cudaStream_t st = as_stream(stream);
    ssim_tile_kernel<<<dim3((unsigned)tiles, (unsigned)B), kThreads, 0, st>>>(a, b, H, W, tiles_x, work);
    int rc = check_launch("image_ssim_psnr(tiles)");
    if (rc) return rc;
    ssim_final_kernel<<<B, kThreads, 0, st>>>(work, (int)tiles, H, W, out);
    return check_launch("image_ssim_psnr(final)");
}

}  // extern "C"
