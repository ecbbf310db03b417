// palette.cu -- 256-colour GIF palettes of uint8 RGB frames (the quantisation imageio / Pillow run on the host when the reference writes its
// sequence and circle-path gifs: sparsefusion/distillation.py:444-493).  One palette per frame, by median cut over a 32^3 histogram, defined in
// integer arithmetic so that the result is a pure function of the input (header section 11, which the tests' numpy restatement follows).
//
// Three launches:
//   1. histogram over pixels: per cell (r>>3, g>>3, b>>3) the pixel count and the r, g, b sums (uint32).  Renders are mostly black, so one
//      cell receives most of a frame's pixels: a warp whose 32 pixels share one cell keeps a running total for that cell in registers and
//      flushes it once; otherwise the lanes of each cell (__match_any_sync) are summed with shuffles and only the cell's first lane issues
//      the global atomics.
//   2. median cut, one CTA per frame with the box table in shared memory.  Each split scans the chosen box once, slice by slice along the split
//      axis, and gets from that one scan the cut and both halves' bounding boxes, counts and sums.
//   3. map over pixels with the frame's palette in shared memory: nearest entry by integer squared distance, ties to the lowest index (the
//      minimum of distance << 8 | index).  A warp of 32 identical pixels splits the palette over its lanes instead.
// Every reduction is an integer sum, min or max, so atomics leave the result bit-identical from run to run.
#include "common.cuh"

namespace sfb {
namespace {

constexpr int kBits = 5;                              // bits per channel of a histogram cell
constexpr int kSide = 1 << kBits;                     // 32 slices per axis
constexpr int kCells = kSide * kSide * kSide;         // 32^3
constexpr int kMaxColors = 256;
constexpr int kThreads = 256;
constexpr int kWarpIters = 16;                        // histogram: 32-pixel rows per warp
constexpr int kHistPix = kThreads * kWarpIters;       // pixels per histogram CTA
constexpr int kMapIters = 8;                          // map: 32-pixel rows per warp
constexpr int kMapPix = kThreads * kMapIters;
constexpr uint32_t kNone = 0xFFFFFFFFu;               // cell / colour of a lane past the frame's end
constexpr unsigned kFull = 0xFFFFFFFFu;
// H*W * 255 must fit a uint32 channel sum
constexpr int64_t kMaxPixels = 16843009;              // floor((2^32 - 1) / 255)

__device__ __forceinline__ uint32_t cell_of(uint32_t r, uint32_t g, uint32_t b) {
    return ((r >> 3) << (2 * kBits)) | ((g >> 3) << kBits) | (b >> 3);
}

__device__ __forceinline__ void add_cell(uint32_t* h, uint32_t cell, uint32_t n, uint32_t r, uint32_t g, uint32_t b) {
    uint32_t* p = h + (size_t)cell * 4;
    atomicAdd(p + 0, n);
    atomicAdd(p + 1, r);
    atomicAdd(p + 2, g);
    atomicAdd(p + 3, b);
}

// hist [B][kCells][4] = (n, sum r, sum g, sum b), zeroed by the caller
__global__ void __launch_bounds__(kThreads) palette_hist_kernel(const uint8_t* __restrict__ rgb, int HW, uint32_t* __restrict__ hist) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint8_t* px = rgb + (size_t)blockIdx.y * HW * 3;
    uint32_t* h = hist + (size_t)blockIdx.y * kCells * 4;
    const int base = blockIdx.x * kHistPix + warp * (kWarpIters * 32);
    uint32_t run_cell = kNone, run_n = 0, run_r = 0, run_g = 0, run_b = 0;     // warp-uniform running total of whole-warp rows
    for (int it = 0; it < kWarpIters; ++it) {
        const int q = base + it * 32 + lane;
        if (base + it * 32 >= HW) break;                                        // warp-uniform
        uint32_t r = 0, g = 0, b = 0, cell = kNone;
        if (q < HW) {
            r = px[3 * (size_t)q];
            g = px[3 * (size_t)q + 1];
            b = px[3 * (size_t)q + 2];
            cell = cell_of(r, g, b);
        }
        const unsigned peers = __match_any_sync(kFull, cell);
        if (peers == kFull) {                                                   // one cell for the whole row: keep it in registers
            if (cell != run_cell) {
                if (lane == 0 && run_cell != kNone) add_cell(h, run_cell, run_n, run_r, run_g, run_b);
                run_cell = cell;
                run_n = run_r = run_g = run_b = 0;
            }
            run_n += 32;
            run_r += __reduce_add_sync(kFull, r);
            run_g += __reduce_add_sync(kFull, g);
            run_b += __reduce_add_sync(kFull, b);
            continue;
        }
        // sum each cell's lanes: a binary tree over the lanes' ranks within their cell (every lane takes part in every shuffle)
        const unsigned above = peers & ~((2u << lane) - 1u);                    // same-cell lanes after this one (2u << 31 == 0)
        const int rank = __popc(peers & ((1u << lane) - 1u));
        unsigned long long v = (unsigned long long)r | ((unsigned long long)g << 21) | ((unsigned long long)b << 42);   // <= 32 * 255 per field
#pragma unroll
        for (int s = 1; s < 32; s <<= 1) {
            unsigned m = above;                                                 // the s-th same-cell lane after this one
            for (int k = 1; k < s; ++k) m &= m - 1u;
            const unsigned long long o = __shfl_sync(kFull, v, m ? __ffs(m) - 1 : lane);
            if (m && (rank & (2 * s - 1)) == 0) v += o;
        }
        if (rank == 0 && cell != kNone)
            add_cell(h, cell, __popc(peers), (uint32_t)(v & 0x1FFFFF), (uint32_t)((v >> 21) & 0x1FFFFF), (uint32_t)(v >> 42));
    }
    if (lane == 0 && run_cell != kNone) add_cell(h, run_cell, run_n, run_r, run_g, run_b);
}

struct CutSmem {
    int lo[kMaxColors][3], hi[kMaxColors][3];        // inclusive cell range per axis, shrunk to the non-empty cells
    uint32_t n[kMaxColors], sum[kMaxColors][3];
    // per slice of the box being split, along the split axis: pixel count, channel sums, range of the other two axes' non-empty cells
    uint32_t sl_n[kSide], sl_sum[kSide][3], sl_min[kSide][2], sl_max[kSide][2];
    unsigned long long warp_best[kThreads / 32];
    int pick, axis, nboxes;
};

// every thread: fill the slice table of a box along `axis` from the frame's histogram.  The box spans [lo0, hi0] along `axis` and
// [lo1, hi1], [lo2, hi2] along the other two axes in r, g, b order.
__device__ void scan_box(CutSmem& S, const uint4* __restrict__ h, int axis, int lo0, int hi0, int lo1, int hi1, int lo2, int hi2) {
    if (threadIdx.x < kSide) {
        const int s = threadIdx.x;
        S.sl_n[s] = S.sl_sum[s][0] = S.sl_sum[s][1] = S.sl_sum[s][2] = 0;
        S.sl_min[s][0] = S.sl_min[s][1] = kSide;
        S.sl_max[s][0] = S.sl_max[s][1] = 0;
    }
    __syncthreads();
    const int d0 = hi0 - lo0 + 1, d1 = hi1 - lo1 + 1, d2 = hi2 - lo2 + 1;
    const int plane = d1 * d2, vol = d0 * plane;
    // cells of one slice are consecutive in q, so a thread's walk stays in a slice for plane / kThreads steps: accumulate locally, flush on change
    int cur = -1;
    uint32_t n = 0, sr = 0, sg = 0, sb = 0, mn1 = kSide, mx1 = 0, mn2 = kSide, mx2 = 0;
    for (int q = threadIdx.x; q < vol + kThreads; q += kThreads) {
        const bool in = q < vol;
        const int s = in ? q / plane : -2;
        if (s != cur && cur >= 0 && n) {
            atomicAdd(&S.sl_n[cur], n);
            atomicAdd(&S.sl_sum[cur][0], sr);
            atomicAdd(&S.sl_sum[cur][1], sg);
            atomicAdd(&S.sl_sum[cur][2], sb);
            atomicMin(&S.sl_min[cur][0], mn1);
            atomicMax(&S.sl_max[cur][0], mx1);
            atomicMin(&S.sl_min[cur][1], mn2);
            atomicMax(&S.sl_max[cur][1], mx2);
        }
        if (!in) break;
        if (s != cur) {
            cur = s;
            n = sr = sg = sb = 0;
            mn1 = mn2 = kSide;
            mx1 = mx2 = 0;
        }
        const int rem = q - s * plane;
        const uint32_t c0 = lo0 + s, c1 = lo1 + rem / d2, c2 = lo2 + rem % d2;
        const uint32_t cell = axis == 0 ? (c0 << (2 * kBits)) | (c1 << kBits) | c2
                            : axis == 1 ? (c1 << (2 * kBits)) | (c0 << kBits) | c2
                                        : (c1 << (2 * kBits)) | (c2 << kBits) | c0;
        const uint4 v = h[cell];
        if (v.x) {
            n += v.x;
            sr += v.y;
            sg += v.z;
            sb += v.w;
            mn1 = min(mn1, c1);
            mx1 = max(mx1, c1);
            mn2 = min(mn2, c2);
            mx2 = max(mx2, c2);
        }
    }
    __syncthreads();
}

// one thread: box k <- the non-empty cells of slices s0..s1 of the scanned box (lo along `axis`); the range holds at least one pixel
__device__ void gather_slices(CutSmem& S, int k, int lo_axis, int axis, int s0, int s1) {
    const int a1 = axis == 0 ? 1 : 0, a2 = axis == 2 ? 1 : 2;
    uint32_t n = 0, sr = 0, sg = 0, sb = 0, mn1 = kSide, mx1 = 0, mn2 = kSide, mx2 = 0;
    int first = -1, last = -1;
    for (int s = s0; s <= s1; ++s) {
        if (!S.sl_n[s]) continue;
        if (first < 0) first = s;
        last = s;
        n += S.sl_n[s];
        sr += S.sl_sum[s][0];
        sg += S.sl_sum[s][1];
        sb += S.sl_sum[s][2];
        mn1 = min(mn1, S.sl_min[s][0]);
        mx1 = max(mx1, S.sl_max[s][0]);
        mn2 = min(mn2, S.sl_min[s][1]);
        mx2 = max(mx2, S.sl_max[s][1]);
    }
    S.lo[k][axis] = lo_axis + first;
    S.hi[k][axis] = lo_axis + last;
    S.lo[k][a1] = (int)mn1;
    S.hi[k][a1] = (int)mx1;
    S.lo[k][a2] = (int)mn2;
    S.hi[k][a2] = (int)mx2;
    S.n[k] = n;
    S.sum[k][0] = sr;
    S.sum[k][1] = sg;
    S.sum[k][2] = sb;
}

__global__ void __launch_bounds__(kThreads) palette_cut_kernel(const uint32_t* __restrict__ hist, int colors, uint8_t* __restrict__ palette,
                                                               int32_t* __restrict__ ncolors) {
    __shared__ CutSmem S;
    const int f = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint4* h = reinterpret_cast<const uint4*>(hist) + (size_t)f * kCells;
    {   // the first box: every non-empty cell of the frame
        scan_box(S, h, 0, 0, kSide - 1, 0, kSide - 1, 0, kSide - 1);
        if (tid == 0) {
            gather_slices(S, 0, 0, 0, 0, kSide - 1);
            S.nboxes = 1;
        }
        __syncthreads();
    }
    for (;;) {
        const int nb = S.nboxes;
        if (nb >= colors) break;
        // the splittable box with the most pixels, lowest index on ties
        unsigned long long key = 0;
        if (tid < nb && (S.hi[tid][0] > S.lo[tid][0] || S.hi[tid][1] > S.lo[tid][1] || S.hi[tid][2] > S.lo[tid][2]))
            key = ((unsigned long long)S.n[tid] << 32) | (unsigned)(kMaxColors - tid);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) key = max(key, __shfl_xor_sync(kFull, key, o));
        if (lane == 0) S.warp_best[warp] = key;
        __syncthreads();
        if (tid == 0) {
            unsigned long long best = 0;
            for (int w = 0; w < kThreads / 32; ++w) best = max(best, S.warp_best[w]);
            S.pick = best ? kMaxColors - (int)(best & 0xFFFFFFFFu) : -1;
            if (best) {
                const int k = S.pick;
                int ax = 0;
                for (int a = 1; a < 3; ++a)
                    if (S.hi[k][a] - S.lo[k][a] > S.hi[k][ax] - S.lo[k][ax]) ax = a;
                S.axis = ax;
            }
        }
        __syncthreads();
        const int k = S.pick;
        if (k < 0) break;                                                       // nothing left to split
        const int axis = S.axis, a1 = axis == 0 ? 1 : 0, a2 = axis == 2 ? 1 : 2;
        const int lo0 = S.lo[k][axis], last = S.hi[k][axis] - lo0;
        scan_box(S, h, axis, lo0, lo0 + last, S.lo[k][a1], S.hi[k][a1], S.lo[k][a2], S.hi[k][a2]);
        if (tid == 0) {
            const unsigned long long n = S.n[k];
            unsigned long long cum = 0;
            int t = last - 1;
            for (int s = 0; s < last; ++s) {
                cum += S.sl_n[s];
                if (2 * cum >= n) {
                    t = s;
                    break;
                }
            }
            gather_slices(S, k, lo0, axis, 0, t);
            gather_slices(S, nb, lo0, axis, t + 1, last);
            S.nboxes = nb + 1;
        }
        __syncthreads();
    }
    const int nb = S.nboxes;
    for (int i = tid; i < kMaxColors; i += kThreads) {
        uint8_t* p = palette + ((size_t)f * kMaxColors + i) * 3;
        if (i < nb) {
            const unsigned long long N = S.n[i];
#pragma unroll
            for (int c = 0; c < 3; ++c) p[c] = (uint8_t)((2ull * S.sum[i][c] + N) / (2ull * N));
        } else {
            p[0] = p[1] = p[2] = 0;
        }
    }
    if (tid == 0) ncolors[f] = nb;
}

__device__ __forceinline__ uint32_t dist_key(int r, int g, int b, int4 e) {
    const int dr = r - e.x, dg = g - e.y, db = b - e.z;
    return ((uint32_t)(dr * dr + dg * dg + db * db) << 8) | (uint32_t)e.w;
}

__global__ void __launch_bounds__(kThreads) palette_map_kernel(const uint8_t* __restrict__ rgb, int HW, const uint8_t* __restrict__ palette,
                                                               const int32_t* __restrict__ ncolors, uint8_t* __restrict__ indices) {
    __shared__ int4 pal[kMaxColors];
    const int f = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nc = ncolors[f];
    for (int i = tid; i < nc; i += kThreads) {
        const uint8_t* p = palette + ((size_t)f * kMaxColors + i) * 3;
        pal[i] = make_int4(p[0], p[1], p[2], i);
    }
    __syncthreads();
    const uint8_t* px = rgb + (size_t)f * HW * 3;
    uint8_t* out = indices + (size_t)f * HW;
    const int base = blockIdx.x * kMapPix + warp * (kMapIters * 32);
    for (int it = 0; it < kMapIters; ++it) {
        if (base + it * 32 >= HW) break;                                        // warp-uniform
        const int q = base + it * 32 + lane;
        int r = 0, g = 0, b = 0;
        uint32_t colour = kNone;
        if (q < HW) {
            r = px[3 * (size_t)q];
            g = px[3 * (size_t)q + 1];
            b = px[3 * (size_t)q + 2];
            colour = (uint32_t)r | ((uint32_t)g << 8) | ((uint32_t)b << 16);
        }
        uint32_t best = kNone;
        if (__match_any_sync(kFull, colour) == kFull) {                         // one colour for the whole row: the lanes share the palette
            for (int i = lane; i < nc; i += 32) best = min(best, dist_key(r, g, b, pal[i]));
            best = __reduce_min_sync(kFull, best);
        } else {
            int i = 0;
            for (; i + 4 <= nc; i += 4) {
                best = min(best, dist_key(r, g, b, pal[i]));
                best = min(best, dist_key(r, g, b, pal[i + 1]));
                best = min(best, dist_key(r, g, b, pal[i + 2]));
                best = min(best, dist_key(r, g, b, pal[i + 3]));
            }
            for (; i < nc; ++i) best = min(best, dist_key(r, g, b, pal[i]));
        }
        if (q < HW) out[q] = (uint8_t)(best & 0xFFu);
    }
}

bool sizes_ok(int B, int H, int W) {
    return B >= 1 && B <= 65535 && H >= 1 && W >= 1 && (int64_t)H * W <= kMaxPixels;
}

}  // namespace
}  // namespace sfb

using namespace sfb;

extern "C" {

uint64_t sfb_palette_work_bytes(int B, int H, int W) {
    if (!sizes_ok(B, H, W)) return 0;
    return (uint64_t)B * kCells * 4 * sizeof(uint32_t);
}

int sfb_palette_quantize(const uint8_t* rgb, int B, int H, int W, int colors, uint8_t* palette, int32_t* ncolors, uint8_t* indices, void* work,
                         void* stream) {
    SFB_REQUIRE(rgb && palette && ncolors && indices && work, "palette_quantize: null pointer");
    SFB_REQUIRE(B >= 1 && B <= 65535, "palette_quantize: B must be in 1..65535 (got %d)", B);
    SFB_REQUIRE(H >= 1 && W >= 1, "palette_quantize: frames must be at least 1 x 1 (got %d x %d)", H, W);
    SFB_REQUIRE((int64_t)H * W <= kMaxPixels, "palette_quantize: %d x %d frames exceed %lld pixels (the uint32 channel sums)", H, W,
                (long long)kMaxPixels);
    SFB_REQUIRE(colors >= 2 && colors <= kMaxColors, "palette_quantize: colors must be in 2..%d (got %d)", kMaxColors, colors);
    const cudaStream_t st = as_stream(stream);
    const int HW = H * W;
    uint32_t* hist = static_cast<uint32_t*>(work);
    SFB_CUDA(cudaMemsetAsync(hist, 0, sfb_palette_work_bytes(B, H, W), st));
    palette_hist_kernel<<<dim3((unsigned)ceil_div(HW, kHistPix), (unsigned)B), kThreads, 0, st>>>(rgb, HW, hist);
    int rc = check_launch("palette_quantize(histogram)");
    if (rc) return rc;
    palette_cut_kernel<<<B, kThreads, 0, st>>>(hist, colors, palette, ncolors);
    rc = check_launch("palette_quantize(median cut)");
    if (rc) return rc;
    palette_map_kernel<<<dim3((unsigned)ceil_div(HW, kMapPix), (unsigned)B), kThreads, 0, st>>>(rgb, HW, palette, ncolors, indices);
    return check_launch("palette_quantize(map)");
}

}  // extern "C"
