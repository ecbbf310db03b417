// mesh.cu -- geometry out of a density lattice: separable 3D Gaussian filter, fp64 volume statistics, two-phase marching cubes
// (NeRFRenderer.export_mesh; external/nerf/renderer_df.py:121-153 of the reference does the same on the CPU through PyMCubes).
//
// Volumes are fp32 [X][Y][Z], row-major (i slowest, k fastest), axis order (i, j, k) = (x, y, z).
// Marching cubes is deterministic: per lattice point the count phase flags its three owned edges (to +i, +j, +k) that cross the isovalue
// and per cell the triangle count of its case; CUB exclusive scans turn both counts into output offsets; the emit phase writes each crossing
// edge's vertex once at its scanned index (shared by the up to four cells around the edge) and each cell's triangles at theirs.  No atomics,
// so repeated runs are bit-identical.  Triangle table and corner / edge numbering: mc_tables.cuh (tools/gen_mc_tables.py).
#include <cub/device/device_scan.cuh>

#include "common.cuh"
#include "mc_tables.cuh"

namespace sfb {
namespace {

constexpr int kGaussMaxRadius = 32;          // sigma up to 7.9 (radius = int(4 sigma + 0.5))
constexpr int kRowTile = 256;                // outputs per CTA of the contiguous-axis pass
constexpr int kThreads = 256;
constexpr int kStatBlocks = SFB_VOLUME_STATS_WORK;   // partial sums per statistics pass (the caller's work buffer)
constexpr int kMcMaxAxis = SFB_MC_MAX_AXIS;

struct Taps {
    float w[2 * kGaussMaxRadius + 1];
    int r;
};

// scipy.ndimage mode='reflect' (half-sample symmetric: d c b a | a b c d | d c b a), folding as often as needed when the axis is shorter than
// the filter radius
__device__ __forceinline__ int reflect_index(int q, int n) {
    if ((unsigned)q < (unsigned)n) return q;
    const int p = 2 * n;
    int m = q % p;
    if (m < 0) m += p;
    return m < n ? m : p - 1 - m;
}

// pass along the contiguous axis: one CTA filters kRowTile outputs of one row from a shared-memory copy of its window
__global__ void __launch_bounds__(kThreads) gauss_rows_kernel(const float* __restrict__ in, float* __restrict__ out, int L, int tiles,
                                                              const __grid_constant__ Taps tp) {
    __shared__ float s[kRowTile + 2 * kGaussMaxRadius];
    const int64_t row = blockIdx.x / tiles;
    const int t0 = (int)(blockIdx.x % tiles) * kRowTile;
    const int r = tp.r;
    const float* src = in + row * L;
    for (int q = threadIdx.x; q < kRowTile + 2 * r; q += blockDim.x) s[q] = src[reflect_index(t0 - r + q, L)];
    __syncthreads();
    const int k = t0 + threadIdx.x;
    if (k >= L) return;
    float acc = 0.f;
    for (int t = 0; t <= 2 * r; ++t) acc = fmaf(tp.w[t], s[threadIdx.x + t], acc);
    out[row * L + k] = acc;
}

// pass along a strided axis (length L, stride `stride` elements): consecutive threads take consecutive elements of the contiguous axis,
// so every tap is a coalesced row read
__global__ void __launch_bounds__(kThreads) gauss_strided_kernel(const float* __restrict__ in, float* __restrict__ out, int64_t n, int L,
                                                                 int64_t stride, const __grid_constant__ Taps tp) {
    const int r = tp.r;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t inner = e % stride, rest = e / stride;
        const int pos = (int)(rest % L);
        const float* base = in + (rest - pos) * stride + inner;
        float acc = 0.f;
        for (int t = 0; t <= 2 * r; ++t) acc = fmaf(tp.w[t], base[(int64_t)reflect_index(pos + t - r, L) * stride], acc);
        out[e] = acc;
    }
}

// fixed-order block sum (warp shuffles, then the warp totals): the same inputs give the same bits
__device__ double block_sum(double x) {
    __shared__ double warp_tot[32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x += __shfl_down_sync(0xffffffffu, x, o);
    if ((threadIdx.x & 31) == 0) warp_tot[threadIdx.x >> 5] = x;
    __syncthreads();
    x = threadIdx.x < (blockDim.x >> 5) ? warp_tot[threadIdx.x] : 0.0;
    if (threadIdx.x < 32) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) x += __shfl_down_sync(0xffffffffu, x, o);
    }
    return x;   // valid in thread 0
}

// partial[b] = sum over a grid-stride share of v of x (mean == NULL) or of (x - *mean)^2, in fp64
__global__ void __launch_bounds__(kThreads) stats_partial_kernel(const float* __restrict__ v, int64_t n, const double* mean, double* partial) {
    const double m = mean ? *mean : 0.0;
    double acc = 0.0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const double x = (double)v[i] - m;
        acc += mean ? x * x : x;
    }
    acc = block_sum(acc);
    if (threadIdx.x == 0) partial[blockIdx.x] = acc;
}

// one CTA of kStatBlocks threads: out = sum(partial) / n (mean), or sqrt of it (population std)
__global__ void __launch_bounds__(kStatBlocks) stats_final_kernel(const double* partial, int nb, int64_t n, int take_sqrt, double* out) {
    double s = block_sum(threadIdx.x < nb ? partial[threadIdx.x] : 0.0);
    if (threadIdx.x == 0) *out = take_sqrt ? sqrt(s / (double)n) : s / (double)n;
}

struct Lattice {
    int X, Y, Z;
    int64_t N, YZ;
};

__device__ __forceinline__ bool below(const float* v, int64_t p, float iso) { return v[p] <= iso; }

__device__ __forceinline__ int cell_case(const float* __restrict__ v, int64_t p, const Lattice& g, float iso) {
    int c = 0;
#pragma unroll
    for (int q = 0; q < 8; ++q) c |= (int)below(v, p + (q & 1) * g.YZ + ((q >> 1) & 1) * g.Z + ((q >> 2) & 1), iso) << q;
    return c;
}

// per lattice point p (and the sentinel p == N): crossing mask of its owned edges, vertex count, triangle count of the cell it anchors
__global__ void __launch_bounds__(kThreads) mc_count_kernel(const float* __restrict__ v, Lattice g, float iso, int64_t* __restrict__ vo,
                                                            int64_t* __restrict__ to, uint8_t* __restrict__ mask) {
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p <= g.N; p += (int64_t)gridDim.x * blockDim.x) {
        if (p == g.N) {
            vo[p] = 0;
            to[p] = 0;
            continue;
        }
        const int k = (int)(p % g.Z), j = (int)((p / g.Z) % g.Y), i = (int)(p / g.YZ);
        const bool b0 = below(v, p, iso);
        unsigned m = 0;
        if (i + 1 < g.X && below(v, p + g.YZ, iso) != b0) m |= 1u;
        if (j + 1 < g.Y && below(v, p + g.Z, iso) != b0) m |= 2u;
        if (k + 1 < g.Z && below(v, p + 1, iso) != b0) m |= 4u;
        mask[p] = (uint8_t)m;
        vo[p] = __popc(m);
        to[p] = (i + 1 < g.X && j + 1 < g.Y && k + 1 < g.Z) ? (int64_t)c_mc_tri_count[cell_case(v, p, g, iso)] : 0;
    }
}

__global__ void mc_totals_kernel(const int64_t* vo, const int64_t* to, int64_t N, int64_t* counts) {
    counts[0] = vo[N];
    counts[1] = to[N];
}

__global__ void __launch_bounds__(kThreads) mc_emit_kernel(const float* __restrict__ v, Lattice g, float iso, const int64_t* __restrict__ vo,
                                                           const int64_t* __restrict__ to, const uint8_t* __restrict__ mask, float* __restrict__ verts,
                                                           int32_t* __restrict__ tris) {
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < g.N; p += (int64_t)gridDim.x * blockDim.x) {
        const int k = (int)(p % g.Z), j = (int)((p / g.Z) % g.Y), i = (int)(p / g.YZ);
        const unsigned m = mask[p];
        if (m) {
            int64_t out = vo[p];
            const float v0 = v[p];
            const int64_t step[3] = {g.YZ, (int64_t)g.Z, 1};
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                if (!((m >> a) & 1u)) continue;
                const float t = (iso - v0) / (v[p + step[a]] - v0);
                verts[out * 3 + 0] = (float)i + (a == 0 ? t : 0.f);
                verts[out * 3 + 1] = (float)j + (a == 1 ? t : 0.f);
                verts[out * 3 + 2] = (float)k + (a == 2 ? t : 0.f);
                ++out;
            }
        }
        const int64_t t0 = to[p], nt = to[p + 1] - t0;
        if (nt == 0) continue;
        const int c = cell_case(v, p, g, iso);
        for (int s = 0; s < 3 * (int)nt; ++s) {
            const int e = c_mc_tri_table[c][s];
            const int a = e >> 2, r = e & 3;
            // owner corner of edge e: the two coordinates other than `a`, in axis order, are (r & 1, r >> 1)
            const int64_t owner = p + (a == 0 ? (r & 1) * (int64_t)g.Z + (r >> 1)
                                          : a == 1 ? (r & 1) * g.YZ + (r >> 1)
                                                   : (r & 1) * g.YZ + (r >> 1) * (int64_t)g.Z);
            tris[t0 * 3 + s] = (int32_t)(vo[owner] + __popc((unsigned)mask[owner] & ((1u << a) - 1u)));
        }
    }
}

int grid_for(int64_t n) { return (int)std::min<int64_t>(ceil_div<int64_t>(n, kThreads), (int64_t)sm_count() * 16); }

bool lattice_ok(int X, int Y, int Z) { return X >= 1 && Y >= 1 && Z >= 1 && X <= kMcMaxAxis && Y <= kMcMaxAxis && Z <= kMcMaxAxis; }

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

struct McScratch {
    size_t vo, to, mask, cub, cub_bytes, total;
};

// scratch layout for an X*Y*Z lattice: vertex offsets int64[N+1] | triangle offsets int64[N+1] | edge masks uint8[N] | CUB scan storage
cudaError_t mc_layout(int X, int Y, int Z, McScratch* s) {
    const int64_t n1 = (int64_t)X * Y * Z + 1;
    size_t cub_bytes = 0;
    const cudaError_t e = cub::DeviceScan::ExclusiveSum(nullptr, cub_bytes, (int64_t*)nullptr, n1);
    s->vo = 0;
    s->to = align256(n1 * sizeof(int64_t));
    s->mask = s->to + align256(n1 * sizeof(int64_t));
    s->cub = s->mask + align256((size_t)n1);
    s->cub_bytes = cub_bytes;
    s->total = s->cub + align256(cub_bytes);
    return e;
}

}  // namespace
}  // namespace sfb

using namespace sfb;

extern "C" {

int sfb_gaussian_filter3d(const float* in, float* out, float* tmp, int X, int Y, int Z, float sigma, void* stream) {
    SFB_REQUIRE(in && out && tmp, "gaussian_filter3d: null pointer");
    SFB_REQUIRE(in != out && in != tmp && out != tmp, "gaussian_filter3d: in, out and tmp must be distinct buffers");
    SFB_REQUIRE(X >= 1 && Y >= 1 && Z >= 1, "gaussian_filter3d: every axis needs at least one sample (got %d x %d x %d)", X, Y, Z);
    SFB_REQUIRE((int64_t)X * Y * ceil_div(Z, kRowTile) <= (int64_t)INT32_MAX, "gaussian_filter3d: volume too large (%d x %d x %d)", X, Y, Z);
    SFB_REQUIRE(sigma > 0.f && (int)(4.0 * sigma + 0.5) <= kGaussMaxRadius, "gaussian_filter3d: sigma must be in (0, %.2f] (got %g)",
                (kGaussMaxRadius + 0.5) / 4.0 - 1e-6, sigma);
    // scipy.ndimage._gaussian_kernel1d: radius int(truncate * sigma + 0.5) with truncate = 4, exp(-x^2 / 2 sigma^2) normalised to sum 1
    Taps tp{};
    tp.r = (int)(4.0 * (double)sigma + 0.5);
    double w[2 * kGaussMaxRadius + 1], sum = 0.0;
    for (int t = -tp.r; t <= tp.r; ++t) sum += (w[t + tp.r] = exp(-0.5 / ((double)sigma * sigma) * t * t));
    for (int t = 0; t <= 2 * tp.r; ++t) tp.w[t] = (float)(w[t] / sum);
    const cudaStream_t st = as_stream(stream);
    const int64_t n = (int64_t)X * Y * Z;
    const int tiles = ceil_div(Z, kRowTile);
    gauss_rows_kernel<<<(unsigned)((int64_t)X * Y * tiles), kThreads, 0, st>>>(in, out, Z, tiles, tp);
    int rc = check_launch("gaussian_filter3d(k)");
    if (rc) return rc;
    gauss_strided_kernel<<<grid_for(n), kThreads, 0, st>>>(out, tmp, n, Y, (int64_t)Z, tp);
    if ((rc = check_launch("gaussian_filter3d(j)"))) return rc;
    gauss_strided_kernel<<<grid_for(n), kThreads, 0, st>>>(tmp, out, n, X, (int64_t)Y * Z, tp);
    return check_launch("gaussian_filter3d(i)");
}

int sfb_volume_mean_std(const float* v, int64_t n, double* out2, double* work, void* stream) {
    SFB_REQUIRE(v && out2 && work, "volume_mean_std: null pointer");
    SFB_REQUIRE(n >= 1, "volume_mean_std: empty volume");
    const cudaStream_t st = as_stream(stream);
    const int nb = (int)std::min<int64_t>(kStatBlocks, ceil_div<int64_t>(n, kThreads * 8));   // depends on n only: same n, same summation order
    stats_partial_kernel<<<nb, kThreads, 0, st>>>(v, n, nullptr, work);
    stats_final_kernel<<<1, kStatBlocks, 0, st>>>(work, nb, n, 0, out2);
    stats_partial_kernel<<<nb, kThreads, 0, st>>>(v, n, out2, work);
    stats_final_kernel<<<1, kStatBlocks, 0, st>>>(work, nb, n, 1, out2 + 1);
    count_launches(3);
    return check_launch("volume_mean_std");
}

uint64_t sfb_marching_cubes_scratch_bytes(int X, int Y, int Z) {
    if (!lattice_ok(X, Y, Z)) return 0;
    McScratch s;
    if (mc_layout(X, Y, Z, &s) != cudaSuccess) return 0;
    return (uint64_t)s.total;
}

int sfb_marching_cubes_count(const float* v, int X, int Y, int Z, float iso, void* scratch, int64_t* counts, void* stream) {
    SFB_REQUIRE(v && scratch && counts, "marching_cubes_count: null pointer");
    SFB_REQUIRE(lattice_ok(X, Y, Z), "marching_cubes_count: lattice %d x %d x %d outside 1..%d per axis", X, Y, Z, kMcMaxAxis);
    McScratch s;
    SFB_CUDA(mc_layout(X, Y, Z, &s));
    char* base = static_cast<char*>(scratch);
    int64_t* vo = reinterpret_cast<int64_t*>(base + s.vo);
    int64_t* to = reinterpret_cast<int64_t*>(base + s.to);
    const Lattice g{X, Y, Z, (int64_t)X * Y * Z, (int64_t)Y * Z};
    const cudaStream_t st = as_stream(stream);
    mc_count_kernel<<<grid_for(g.N + 1), kThreads, 0, st>>>(v, g, iso, vo, to, reinterpret_cast<uint8_t*>(base + s.mask));
    int rc = check_launch("marching_cubes_count");
    if (rc) return rc;
    size_t bytes = s.cub_bytes;
    SFB_CUDA(cub::DeviceScan::ExclusiveSum(base + s.cub, bytes, vo, g.N + 1, st));
    bytes = s.cub_bytes;
    SFB_CUDA(cub::DeviceScan::ExclusiveSum(base + s.cub, bytes, to, g.N + 1, st));
    count_launches(4);      // two CUB scans of an init and a scan kernel each
    mc_totals_kernel<<<1, 1, 0, st>>>(vo, to, g.N, counts);
    return check_launch("marching_cubes_count(totals)");
}

int sfb_marching_cubes_emit(const float* v, int X, int Y, int Z, float iso, const void* scratch, float* verts, int32_t* tris, void* stream) {
    SFB_REQUIRE(v && scratch, "marching_cubes_emit: null pointer");
    SFB_REQUIRE(lattice_ok(X, Y, Z), "marching_cubes_emit: lattice %d x %d x %d outside 1..%d per axis", X, Y, Z, kMcMaxAxis);
    McScratch s;
    SFB_CUDA(mc_layout(X, Y, Z, &s));
    const char* base = static_cast<const char*>(scratch);
    const Lattice g{X, Y, Z, (int64_t)X * Y * Z, (int64_t)Y * Z};
    mc_emit_kernel<<<grid_for(g.N), kThreads, 0, as_stream(stream)>>>(v, g, iso, reinterpret_cast<const int64_t*>(base + s.vo),
                                                                      reinterpret_cast<const int64_t*>(base + s.to),
                                                                      reinterpret_cast<const uint8_t*>(base + s.mask), verts, tris);
    return check_launch("marching_cubes_emit");
}

}  // extern "C"
