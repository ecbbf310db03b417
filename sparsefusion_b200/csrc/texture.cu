// texture.cu -- albedo texture of an extracted mesh: a per-triangle UV atlas, the surface point under every texel, and the uint8 pack of
// the field's albedo there (NeRFRenderer.export_mesh(texture_size=T); the reference's xatlas / nvdiffrast export, renderer_df.py:166-306,
// is dead code there).  Header section 12 states the contract; every output is a pure function of its inputs (no atomics).
//
// Atlas: triangles 2k and 2k+1 share square cell k of c x c texels (n cells per row).  In cell-local texel coordinates the lower triangle
// is (m, m), (c-m-d, m), (m, c-m-d) and the upper one (c-m, c-m), (m+d, c-m), (c-m, m+d): both are right isosceles triangles of leg
// L = c - 2m - d whose first corner is the right angle.  Texel (i, j) of the cell belongs to the lower triangle when i + j + 1 < c.  With
// m = 1/2 and d = 2, every texel that a bilinear lookup anywhere inside a triangle gives a nonzero weight is owned by that triangle, so
// the texture needs no seam fill.
#include "common.cuh"

namespace sfb {
namespace {

constexpr int kThreads = 256;
constexpr float kMargin = 0.5f;   // m: texels between a triangle's legs and the cell border
constexpr float kGap = 2.0f;      // d: texels between the two hypotenuses of a cell

int64_t ceil_sqrt(int64_t k) {
    int64_t n = (int64_t)sqrt((double)k);
    while (n * n < k) ++n;
    while (n > 0 && (n - 1) * (n - 1) >= k) --n;
    return n;
}

// cells per atlas row: n = ceil(sqrt(ceil(F / 2))), at least 1
int atlas_cols(int F) { return (int)std::max<int64_t>(1, ceil_sqrt(((int64_t)F + 1) / 2)); }

int atlas_cell(int F, int T) {
    if (F < 0 || T < SFB_TEXTURE_MIN || T > SFB_TEXTURE_MAX) return 0;
    const int c = T / atlas_cols(F);
    return c >= SFB_TEXTURE_MIN_CELL ? c : 0;
}

__global__ void __launch_bounds__(kThreads) uv_atlas_kernel(int F, int n, int c, float* __restrict__ uv) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= F) return;
    const int k = t >> 1;
    const float x0 = (float)((k % n) * c), y0 = (float)((k / n) * c), cf = (float)c;
    // corners in tris[t, 0..2] order: the right angle, then along x, then along y
    float u[3], v[3];
    if ((t & 1) == 0) {
        u[0] = kMargin, v[0] = kMargin;
        u[1] = cf - kMargin - kGap, v[1] = kMargin;
        u[2] = kMargin, v[2] = cf - kMargin - kGap;
    } else {
        u[0] = cf - kMargin, v[0] = cf - kMargin;
        u[1] = kMargin + kGap, v[1] = cf - kMargin;
        u[2] = cf - kMargin, v[2] = kMargin + kGap;
    }
    float* o = uv + (int64_t)t * 6;
#pragma unroll
    for (int q = 0; q < 3; ++q) {
        o[2 * q] = x0 + u[q];
        o[2 * q + 1] = y0 + v[q];
    }
}

// one thread per texel of rows [row0, row0 + rows): owner triangle (-1 = none) and the surface point of the owner closest, in the atlas, to
// the texel centre
__global__ void __launch_bounds__(kThreads) texel_points_kernel(const float* __restrict__ verts, const int32_t* __restrict__ tris, int F, int T,
                                                                int n, int c, int row0, int64_t count, int32_t* __restrict__ owner,
                                                                float* __restrict__ xyz) {
    const float L = (float)c - 2.f * kMargin - kGap;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < count; e += (int64_t)gridDim.x * blockDim.x) {
        const int x = (int)(e % T), y = row0 + (int)(e / T);
        const int cx = x / c, cy = y / c;
        const int i = x - cx * c, j = y - cy * c;
        const int t = 2 * (cy * n + cx) + ((2 * i + 1) + (2 * j + 1) < 2 * c ? 0 : 1);
        if (cx >= n || cy >= n || t >= F) {
            owner[e] = -1;
            xyz[3 * e] = xyz[3 * e + 1] = xyz[3 * e + 2] = 0.f;
            continue;
        }
        // texel centre in the triangle's leg frame, legs scaled to 1: (s, r) = (0, 0), (1, 0), (0, 1) at corners 0, 1, 2.  The upper
        // triangle's legs run toward -x and -y, so its frame is the lower one's turned by 180 degrees; both maps are similarities, so the
        // closest point in the frame is the closest point in texel units.
        float s, r;
        if ((t & 1) == 0) {
            s = ((float)i + 0.5f - kMargin) / L;
            r = ((float)j + 0.5f - kMargin) / L;
        } else {
            s = ((float)c - kMargin - ((float)i + 0.5f)) / L;
            r = ((float)c - kMargin - ((float)j + 0.5f)) / L;
        }
        // closest point of the triangle s, r >= 0, s + r <= 1: beyond the hypotenuse, the clamped projection onto it; otherwise the
        // clamp onto the unit square, which lands on a leg or a corner
        if (s + r > 1.f) {
            s = fminf(fmaxf(0.5f * (1.f + s - r), 0.f), 1.f);
            r = 1.f - s;
        } else {
            s = fminf(fmaxf(s, 0.f), 1.f);
            r = fminf(fmaxf(r, 0.f), 1.f);
        }
        const float l0 = 1.f - s - r;
        const float* a = verts + 3 * (int64_t)tris[3 * t];
        const float* b = verts + 3 * (int64_t)tris[3 * t + 1];
        const float* d = verts + 3 * (int64_t)tris[3 * t + 2];
        owner[e] = t;
#pragma unroll
        for (int q = 0; q < 3; ++q) xyz[3 * e + q] = fmaf(l0, a[q], fmaf(s, b[q], r * d[q]));
    }
}

__global__ void __launch_bounds__(kThreads) texture_pack_kernel(const int32_t* __restrict__ owner, const float* __restrict__ rgb, int64_t count,
                                                                uint8_t* __restrict__ out) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < count; e += (int64_t)gridDim.x * blockDim.x) {
        const bool own = owner[e] >= 0;
#pragma unroll
        for (int q = 0; q < 3; ++q) out[3 * e + q] = own ? (uint8_t)__float2uint_rz(255.f * rgb[3 * e + q]) : (uint8_t)0;
    }
}

int grid_for(int64_t count) { return (int)std::min<int64_t>(ceil_div<int64_t>(count, kThreads), (int64_t)sm_count() * 16); }

}  // namespace
}  // namespace sfb

using namespace sfb;

extern "C" {

int sfb_mesh_atlas_cell(int F, int T) { return atlas_cell(F, T); }

int sfb_mesh_uv_atlas(int F, int T, float* uv, void* stream) {
    SFB_REQUIRE(F >= 0, "mesh_uv_atlas: negative triangle count %d", F);
    const int c = atlas_cell(F, T);
    SFB_REQUIRE(c > 0, "mesh_uv_atlas: a %d x %d texture has no atlas for %d triangles", T, T, F);
    if (F == 0) return SFB_OK;
    SFB_REQUIRE(uv, "mesh_uv_atlas: null pointer");
    uv_atlas_kernel<<<ceil_div(F, kThreads), kThreads, 0, as_stream(stream)>>>(F, atlas_cols(F), c, uv);
    return check_launch("mesh_uv_atlas");
}

int sfb_mesh_texel_points(const float* verts, const int32_t* tris, int F, int T, int row0, int rows, int32_t* owner, float* xyz, void* stream) {
    SFB_REQUIRE(F >= 0, "mesh_texel_points: negative triangle count %d", F);
    const int c = atlas_cell(F, T);
    SFB_REQUIRE(c > 0, "mesh_texel_points: a %d x %d texture has no atlas for %d triangles", T, T, F);
    SFB_REQUIRE(row0 >= 0 && rows >= 0 && (int64_t)row0 + rows <= T, "mesh_texel_points: rows [%d, %d + %d) outside 0..%d", row0, row0, rows, T);
    if (rows == 0) return SFB_OK;
    SFB_REQUIRE(owner && xyz && (F == 0 || (verts && tris)), "mesh_texel_points: null pointer");
    const int64_t count = (int64_t)rows * T;
    texel_points_kernel<<<grid_for(count), kThreads, 0, as_stream(stream)>>>(verts, tris, F, T, atlas_cols(F), c, row0, count, owner, xyz);
    return check_launch("mesh_texel_points");
}

int sfb_mesh_texture_pack(const int32_t* owner, const float* rgb, int64_t n, uint8_t* out, void* stream) {
    SFB_REQUIRE(n >= 0, "mesh_texture_pack: negative texel count");
    if (n == 0) return SFB_OK;
    SFB_REQUIRE(owner && rgb && out, "mesh_texture_pack: null pointer");
    texture_pack_kernel<<<grid_for(n), kThreads, 0, as_stream(stream)>>>(owner, rgb, n, out);
    return check_launch("mesh_texture_pack");
}

}  // extern "C"
