// scene_ops.cu -- ray grids of the per-scene preparation of a distillation (sparsefusion/distillation.py:85-86, :201-204, :395-402, :463-469),
// sm_90a.
//
// The reference builds every ray bundle of a scene with pytorch3d's GridRaysampler (utils/render_utils.py:16-65): the pixel-centre NDC grid
// of the image, each pixel unprojected at depths 1 and 2 by the camera, direction = p2 - p1 (not normalised), origin = p1 - direction.  One
// launch here covers all cameras of a bundle (scene views, circle views, EFT query views): one thread per (camera, pixel).
#include "common.cuh"
#include "../../include/sparsefusion_b200.h"

namespace sfb {

// torch.linspace(start, end, steps)[i]: the first half counts up from start, the second half down from end
__device__ __forceinline__ float linspace_at(float start, float end, int steps, int i) {
    if (steps == 1) return start;
    const float step = (end - start) / (float)(steps - 1);
    return i < steps / 2 ? start + step * (float)i : end - step * (float)(steps - 1 - i);
}

// cams [V][16] = R (9, row-major) | T (3) | focal (2) | principal point (2); NDC row-vector convention: x_view = x_world R + T,
// x_ndc = f x_view / z + p.  Unprojection of NDC (x, y) at depth z: x_view = ((x - px) z / fx, (y - py) z / fy, z), x_world = (x_view - T) R^T.
__global__ void grid_rays_kernel(const float* __restrict__ cams, int V, int H, int W, float min_x, float max_x, float min_y, float max_y,
                                 float* __restrict__ rays_o, float* __restrict__ rays_d) {
    const int64_t HW = (int64_t)H * W;
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= (int64_t)V * HW) return;
    const int v = (int)(i / HW);
    const int pix = (int)(i % HW);
    const float* cam = cams + (int64_t)v * 16;
    const float x = linspace_at(min_x, max_x, W, pix % W), y = linspace_at(min_y, max_y, H, pix / W);
    const float fx = __ldg(cam + 12), fy = __ldg(cam + 13), px = __ldg(cam + 14), py = __ldg(cam + 15);
    const float ux = (x - px) / fx, uy = (y - py) / fy;
    float p1[3], p2[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        const float r0 = __ldg(cam + j * 3 + 0), r1 = __ldg(cam + j * 3 + 1), r2 = __ldg(cam + j * 3 + 2);   // row j of R = column j of R^T
        const float t0 = __ldg(cam + 9), t1 = __ldg(cam + 10), t2 = __ldg(cam + 11);
        p1[j] = (ux - t0) * r0 + (uy - t1) * r1 + (1.f - t2) * r2;
        p2[j] = (2.f * ux - t0) * r0 + (2.f * uy - t1) * r1 + (2.f - t2) * r2;
    }
    float* o = rays_o + i * 3;
    float* d = rays_d + i * 3;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        const float dj = p2[j] - p1[j];
        d[j] = dj;
        o[j] = p1[j] - dj;
    }
}

}  // namespace sfb

using namespace sfb;

extern "C" {

int sfb_grid_rays(const float* cams, int V, int H, int W, float min_x, float max_x, float min_y, float max_y, float* rays_o, float* rays_d,
                  void* stream) {
    SFB_REQUIRE(cams && rays_o && rays_d, "grid_rays: null pointer");
    SFB_REQUIRE(V >= 0 && H >= 1 && W >= 1, "grid_rays: V >= 0 cameras of an H x W >= 1 x 1 grid");
    const int64_t total = (int64_t)V * H * W;
    if (total == 0) return SFB_OK;
    grid_rays_kernel<<<(unsigned)ceil_div(total, (int64_t)256), 256, 0, as_stream(stream)>>>(cams, V, H, W, min_x, max_x, min_y, max_y, rays_o, rays_d);
    return check_launch("grid_rays");
}
}
