// raymarching.cu -- ray/aabb, morton, bit-packing, occupancy-grid marching and compositing operators
// for sm_90a.  Drop-in for the reference's `_raymarching` pybind module
// (raymarching/src/bindings.cpp:5-18): same argument order, layouts and in-place conventions, fp32.
//
// Integer contract kept bit-identical to raymarching/src/raymarching.cu: morton codes (:56-81), mip
// level from frexpf (:42-54), nearest occupancy cell through the double-precision 0.5*(x/mip+1)*H
// truncation (:374-376), step counts per ray.  Point ranges are claimed with atomics in arrival order
// exactly like the reference (:405-406), so point layout is not deterministic -- consumers go through
// the `rays` table.
//
// H100 notes: one thread per ray is kept for the marchers (divergent DDA loops); they are bound by the
// 786 KB occupancy bitfield which stays in L1/L2.  The compositing kernels read three streams
// (sigma 4 B, rgb 12 B, delta 8 B per point) -- HBM-bound, so each thread walks its ray's contiguous
// point range with independent loads in flight.
#include "common.cuh"
#include "raymarching.cuh"
#include "../../include/sparsefusion_b200.h"
#include <float.h>

namespace sfb {

__global__ void __launch_bounds__(256) near_far_kernel(const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                                                      const float* __restrict__ aabb, uint32_t N, float min_near,
                                                      float* __restrict__ nears, float* __restrict__ fars) {
    const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    float near, far;
    ray_aabb(rays_o + (size_t)n * 3, rays_d + (size_t)n * 3, aabb, min_near, near, far);
    nears[n] = near;
    fars[n] = far;
}

__global__ void __launch_bounds__(256) sph_from_ray_kernel(const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                                                          float radius, uint32_t N, float* __restrict__ coords) {
    const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    const float ox = rays_o[n * 3], oy = rays_o[n * 3 + 1], oz = rays_o[n * 3 + 2];
    const float dx = rays_d[n * 3], dy = rays_d[n * 3 + 1], dz = rays_d[n * 3 + 2];
    const float A = dx * dx + dy * dy + dz * dz;
    const float Bh = ox * dx + oy * dy + oz * dz;
    const float Cc = ox * ox + oy * oy + oz * oz - radius * radius;
    const float t = (-Bh + sqrtf(Bh * Bh - A * Cc)) / A;
    const float x = ox + t * dx, y = oy + t * dy, z = oz + t * dz;
    const float theta = atan2(sqrtf(x * x + z * z), y);
    const float phi = atan2(z, x);
    const float RPI = 0.3183098861837907f;
    coords[n * 2] = 2 * theta * RPI - 1;
    coords[n * 2 + 1] = phi * RPI;
}

__global__ void __launch_bounds__(256) morton3D_kernel(const int32_t* __restrict__ coords, uint32_t N, int32_t* __restrict__ indices) {
    const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    indices[n] = (int32_t)morton3D_encode((uint32_t)coords[n * 3], (uint32_t)coords[n * 3 + 1], (uint32_t)coords[n * 3 + 2]);
}

__global__ void __launch_bounds__(256) morton3D_invert_kernel(const int32_t* __restrict__ indices, uint32_t N, int32_t* __restrict__ coords) {
    const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    const int32_t ind = indices[n];
    coords[n * 3] = (int32_t)morton3D_decode((uint32_t)(ind >> 0));
    coords[n * 3 + 1] = (int32_t)morton3D_decode((uint32_t)(ind >> 1));
    coords[n * 3 + 2] = (int32_t)morton3D_decode((uint32_t)(ind >> 2));
}

// 8 floats -> 1 byte; two float4 loads per thread
__global__ void __launch_bounds__(256) packbits_kernel(const float* __restrict__ grid, uint32_t N, float thresh, uint8_t* __restrict__ bitfield) {
    const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    const float4 a = __ldg(reinterpret_cast<const float4*>(grid) + 2 * (size_t)n);
    const float4 b = __ldg(reinterpret_cast<const float4*>(grid) + 2 * (size_t)n + 1);
    uint32_t bits = 0;
    bits |= (a.x > thresh) ? 1u : 0u;
    bits |= (a.y > thresh) ? 2u : 0u;
    bits |= (a.z > thresh) ? 4u : 0u;
    bits |= (a.w > thresh) ? 8u : 0u;
    bits |= (b.x > thresh) ? 16u : 0u;
    bits |= (b.y > thresh) ? 32u : 0u;
    bits |= (b.z > thresh) ? 64u : 0u;
    bits |= (b.w > thresh) ? 128u : 0u;
    bitfield[n] = (uint8_t)bits;
}

__global__ void __launch_bounds__(128) march_rays_train_kernel(const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                                                              const uint8_t* __restrict__ grid, float bound, float dt_gamma,
                                                              uint32_t max_steps, uint32_t N, uint32_t C, uint32_t H, uint32_t M,
                                                              const float* __restrict__ nears, const float* __restrict__ fars,
                                                              float* __restrict__ xyzs, float* __restrict__ dirs, float* __restrict__ deltas,
                                                              int32_t* __restrict__ rays, int32_t* __restrict__ counter,
                                                              const float* __restrict__ noises) {
    const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    Marcher m(rays_o + (size_t)n * 3, rays_d + (size_t)n * 3, grid, bound, dt_gamma, max_steps, C, H);
    const float far = fars[n];
    float t0 = nears[n];
    t0 += clampf(t0 * dt_gamma, m.dt_min, m.dt_max) * noises[n];

    // pass 1: count occupied samples
    float t = t0;
    uint32_t num_steps = 0;
    while (t < far && num_steps < max_steps) {
        MarchSample s;
        if (m.probe(t, s)) { num_steps++; t += s.dt; }
        else m.skip(t, s);
    }
    const uint32_t point_index = atomicAdd((unsigned int*)counter, num_steps);
    const uint32_t ray_index = atomicAdd((unsigned int*)counter + 1, 1u);
    rays[ray_index * 3] = (int32_t)n;
    rays[ray_index * 3 + 1] = (int32_t)point_index;
    rays[ray_index * 3 + 2] = (int32_t)num_steps;
    if (num_steps == 0 || point_index + num_steps > M) return;

    // pass 2: emit
    float* px = xyzs + (size_t)point_index * 3;
    float* pd = dirs + (size_t)point_index * 3;
    float* pl = deltas + (size_t)point_index * 2;
    t = t0;
    float last_t = t;
    uint32_t step = 0;
    while (t < far && step < num_steps) {
        MarchSample s;
        if (m.probe(t, s)) {
            px[0] = s.x; px[1] = s.y; px[2] = s.z;
            pd[0] = m.dx; pd[1] = m.dy; pd[2] = m.dz;
            t += s.dt;
            pl[0] = s.dt;
            pl[1] = t - last_t;
            last_t = t;
            px += 3; pd += 3; pl += 2;
            step++;
        } else m.skip(t, s);
    }
}

__global__ void __launch_bounds__(128) composite_train_fwd_kernel(const float* __restrict__ sigmas, const float* __restrict__ rgbs,
                                                                 const float* __restrict__ deltas, const int32_t* __restrict__ rays,
                                                                 uint32_t M, uint32_t N, float T_thresh, float* __restrict__ weights_sum,
                                                                 float* __restrict__ depth, float* __restrict__ image) {
    const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    const uint32_t index = (uint32_t)rays[n * 3], offset = (uint32_t)rays[n * 3 + 1], num_steps = (uint32_t)rays[n * 3 + 2];
    if (num_steps == 0 || offset + num_steps > M) {
        weights_sum[index] = 0; depth[index] = 0;
        image[index * 3] = 0; image[index * 3 + 1] = 0; image[index * 3 + 2] = 0;
        return;
    }
    const float* s = sigmas + offset;
    const float* c = rgbs + (size_t)offset * 3;
    const float* dl = deltas + (size_t)offset * 2;
    float T = 1.0f, r = 0, g = 0, b = 0, ws = 0, t = 0, d = 0;
    for (uint32_t step = 0; step < num_steps; ++step) {
        const float alpha = 1.0f - __expf(-s[0] * dl[0]);
        const float weight = alpha * T;
        r += weight * c[0]; g += weight * c[1]; b += weight * c[2];
        t += dl[1];
        d += weight * t;
        ws += weight;
        T *= 1.0f - alpha;
        if (T < T_thresh) break;
        s++; c += 3; dl += 2;
    }
    weights_sum[index] = ws; depth[index] = d;
    image[index * 3] = r; image[index * 3 + 1] = g; image[index * 3 + 2] = b;
}

__global__ void __launch_bounds__(128) composite_train_bwd_kernel(const float* __restrict__ grad_weights_sum, const float* __restrict__ grad_image,
                                                                 const float* __restrict__ sigmas, const float* __restrict__ rgbs,
                                                                 const float* __restrict__ deltas, const int32_t* __restrict__ rays,
                                                                 const float* __restrict__ weights_sum, const float* __restrict__ image,
                                                                 uint32_t M, uint32_t N, float T_thresh, float* __restrict__ grad_sigmas,
                                                                 float* __restrict__ grad_rgbs) {
    const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    const uint32_t index = (uint32_t)rays[n * 3], offset = (uint32_t)rays[n * 3 + 1], num_steps = (uint32_t)rays[n * 3 + 2];
    if (num_steps == 0 || offset + num_steps > M) return;
    const float gws = grad_weights_sum[index];
    const float gi0 = grad_image[index * 3], gi1 = grad_image[index * 3 + 1], gi2 = grad_image[index * 3 + 2];
    const float r_final = image[index * 3], g_final = image[index * 3 + 1], b_final = image[index * 3 + 2];
    const float ws_final = weights_sum[index];
    const float* s = sigmas + offset;
    const float* c = rgbs + (size_t)offset * 3;
    const float* dl = deltas + (size_t)offset * 2;
    float* gs = grad_sigmas + offset;
    float* gc = grad_rgbs + (size_t)offset * 3;
    float T = 1.0f, r = 0, g = 0, b = 0, ws = 0;
    for (uint32_t step = 0; step < num_steps; ++step) {
        const float alpha = 1.0f - __expf(-s[0] * dl[0]);
        const float weight = alpha * T;
        r += weight * c[0]; g += weight * c[1]; b += weight * c[2];
        ws += weight;
        T *= 1.0f - alpha;
        gc[0] = gi0 * weight; gc[1] = gi1 * weight; gc[2] = gi2 * weight;
        gs[0] = dl[0] * (gi0 * (T * c[0] - (r_final - r)) + gi1 * (T * c[1] - (g_final - g)) + gi2 * (T * c[2] - (b_final - b)) +
                         gws * (1 - ws_final));
        if (T < T_thresh) break;
        s++; c += 3; dl += 2; gs++; gc += 3;
    }
}

__global__ void __launch_bounds__(128) march_rays_kernel(uint32_t n_alive, uint32_t n_step, const int32_t* __restrict__ rays_alive,
                                                        const float* __restrict__ rays_t, const float* __restrict__ rays_o,
                                                        const float* __restrict__ rays_d, float bound, float dt_gamma, uint32_t max_steps,
                                                        uint32_t C, uint32_t H, const uint8_t* __restrict__ grid,
                                                        const float* __restrict__ nears, const float* __restrict__ fars,
                                                        float* __restrict__ xyzs, float* __restrict__ dirs, float* __restrict__ deltas,
                                                        const float* __restrict__ noises) {
    const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= n_alive) return;
    const int32_t index = rays_alive[n];
    Marcher m(rays_o + (size_t)index * 3, rays_d + (size_t)index * 3, grid, bound, dt_gamma, max_steps, C, H);
    float* px = xyzs + (size_t)n * n_step * 3;
    float* pd = dirs + (size_t)n * n_step * 3;
    float* pl = deltas + (size_t)n * n_step * 2;
    float t = rays_t[index];
    const float far = fars[index];
    t += clampf(t * dt_gamma, m.dt_min, m.dt_max) * noises[n];
    float last_t = t;
    uint32_t step = 0;
    while (t < far && step < n_step) {
        MarchSample s;
        if (m.probe(t, s)) {
            px[0] = s.x; px[1] = s.y; px[2] = s.z;
            pd[0] = m.dx; pd[1] = m.dy; pd[2] = m.dz;
            t += s.dt;
            pl[0] = s.dt;
            pl[1] = t - last_t;
            last_t = t;
            px += 3; pd += 3; pl += 2;
            step++;
        } else m.skip(t, s);
    }
}

__global__ void __launch_bounds__(128) composite_rays_kernel(uint32_t n_alive, uint32_t n_step, float T_thresh, int32_t* __restrict__ rays_alive,
                                                            float* __restrict__ rays_t, const float* __restrict__ sigmas,
                                                            const float* __restrict__ rgbs, const float* __restrict__ deltas,
                                                            float* __restrict__ weights_sum, float* __restrict__ depth, float* __restrict__ image) {
    const uint32_t n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= n_alive) return;
    const int32_t index = rays_alive[n];
    const float* s = sigmas + (size_t)n * n_step;
    const float* c = rgbs + (size_t)n * n_step * 3;
    const float* dl = deltas + (size_t)n * n_step * 2;
    float t = rays_t[index], ws = weights_sum[index], d = depth[index];
    float r = image[index * 3], g = image[index * 3 + 1], b = image[index * 3 + 2];
    uint32_t step = 0;
    while (step < n_step) {
        if (dl[0] == 0) break;
        const float alpha = 1.0f - __expf(-s[0] * dl[0]);
        const float T = 1 - ws;
        const float weight = alpha * T;
        ws += weight;
        t += dl[1];
        d += weight * t;
        r += weight * c[0]; g += weight * c[1]; b += weight * c[2];
        if (T < T_thresh) break;
        s++; c += 3; dl += 2;
        step++;
    }
    if (step < n_step) rays_alive[n] = -1;
    else rays_t[index] = t;
    weights_sum[index] = ws; depth[index] = d;
    image[index * 3] = r; image[index * 3 + 1] = g; image[index * 3 + 2] = b;
}

}  // namespace sfb

using namespace sfb;

extern "C" {

int sfb_near_far_from_aabb(const float* rays_o, const float* rays_d, const float* aabb, uint32_t N, float min_near, float* nears,
                           float* fars, void* stream) {
    if (N == 0) return SFB_OK;  // empty problem: nothing to do, pointers may be null
    SFB_REQUIRE(rays_o && rays_d && aabb && nears && fars, "near_far_from_aabb: null pointer");
    near_far_kernel<<<ceil_div(N, 256u), 256, 0, as_stream(stream)>>>(rays_o, rays_d, aabb, N, min_near, nears, fars);
    return check_launch("near_far_from_aabb");
}

int sfb_sph_from_ray(const float* rays_o, const float* rays_d, float radius, uint32_t N, float* coords, void* stream) {
    if (N == 0) return SFB_OK;  // empty problem: nothing to do, pointers may be null
    SFB_REQUIRE(rays_o && rays_d && coords, "sph_from_ray: null pointer");
    sph_from_ray_kernel<<<ceil_div(N, 256u), 256, 0, as_stream(stream)>>>(rays_o, rays_d, radius, N, coords);
    return check_launch("sph_from_ray");
}

int sfb_morton3D(const int32_t* coords, uint32_t N, int32_t* indices, void* stream) {
    if (N == 0) return SFB_OK;  // empty problem: nothing to do, pointers may be null
    SFB_REQUIRE(coords && indices, "morton3D: null pointer");
    morton3D_kernel<<<ceil_div(N, 256u), 256, 0, as_stream(stream)>>>(coords, N, indices);
    return check_launch("morton3D");
}

int sfb_morton3D_invert(const int32_t* indices, uint32_t N, int32_t* coords, void* stream) {
    if (N == 0) return SFB_OK;  // empty problem: nothing to do, pointers may be null
    SFB_REQUIRE(coords && indices, "morton3D_invert: null pointer");
    morton3D_invert_kernel<<<ceil_div(N, 256u), 256, 0, as_stream(stream)>>>(indices, N, coords);
    return check_launch("morton3D_invert");
}

int sfb_packbits(const float* grid, uint32_t N, float density_thresh, uint8_t* bitfield, void* stream) {
    if (N == 0) return SFB_OK;  // empty problem: nothing to do, pointers may be null
    SFB_REQUIRE(grid && bitfield, "packbits: null pointer");
    SFB_REQUIRE((reinterpret_cast<uintptr_t>(grid) & 15) == 0, "packbits: grid must be 16-byte aligned");
    packbits_kernel<<<ceil_div(N, 256u), 256, 0, as_stream(stream)>>>(grid, N, density_thresh, bitfield);
    return check_launch("packbits");
}

int sfb_march_rays_train(const float* rays_o, const float* rays_d, const uint8_t* grid, float bound, float dt_gamma, uint32_t max_steps,
                         uint32_t N, uint32_t C, uint32_t H, uint32_t M, const float* nears, const float* fars, float* xyzs, float* dirs,
                         float* deltas, int32_t* rays, int32_t* counter, const float* noises, void* stream) {
    if (N == 0) return SFB_OK;  // empty problem: nothing to do, pointers may be null
    SFB_REQUIRE(rays_o && rays_d && grid && nears && fars && xyzs && dirs && deltas && rays && counter && noises, "march_rays_train: null pointer");
    SFB_REQUIRE(C >= 1 && C <= 8 && H >= 1 && H <= 1024, "march_rays_train: cascade/grid size out of range");
    march_rays_train_kernel<<<ceil_div(N, 128u), 128, 0, as_stream(stream)>>>(rays_o, rays_d, grid, bound, dt_gamma, max_steps, N, C, H, M, nears,
                                                                             fars, xyzs, dirs, deltas, rays, counter, noises);
    return check_launch("march_rays_train");
}

int sfb_composite_rays_train_forward(const float* sigmas, const float* rgbs, const float* deltas, const int32_t* rays, uint32_t M, uint32_t N,
                                     float T_thresh, float* weights_sum, float* depth, float* image, void* stream) {
    if (N == 0) return SFB_OK;  // empty problem: nothing to do, pointers may be null
    SFB_REQUIRE(sigmas && rgbs && deltas && rays && weights_sum && depth && image, "composite_rays_train_forward: null pointer");
    composite_train_fwd_kernel<<<ceil_div(N, 128u), 128, 0, as_stream(stream)>>>(sigmas, rgbs, deltas, rays, M, N, T_thresh, weights_sum, depth, image);
    return check_launch("composite_rays_train_forward");
}

int sfb_composite_rays_train_backward(const float* grad_weights_sum, const float* grad_image, const float* sigmas, const float* rgbs,
                                      const float* deltas, const int32_t* rays, const float* weights_sum, const float* image, uint32_t M,
                                      uint32_t N, float T_thresh, float* grad_sigmas, float* grad_rgbs, void* stream) {
    if (N == 0) return SFB_OK;  // empty problem: nothing to do, pointers may be null
    SFB_REQUIRE(grad_weights_sum && grad_image && sigmas && rgbs && deltas && rays && weights_sum && image && grad_sigmas && grad_rgbs,
                "composite_rays_train_backward: null pointer");
    composite_train_bwd_kernel<<<ceil_div(N, 128u), 128, 0, as_stream(stream)>>>(grad_weights_sum, grad_image, sigmas, rgbs, deltas, rays,
                                                                                weights_sum, image, M, N, T_thresh, grad_sigmas, grad_rgbs);
    return check_launch("composite_rays_train_backward");
}

int sfb_march_rays(uint32_t n_alive, uint32_t n_step, const int32_t* rays_alive, const float* rays_t, const float* rays_o, const float* rays_d,
                   float bound, float dt_gamma, uint32_t max_steps, uint32_t C, uint32_t H, const uint8_t* grid, const float* nears,
                   const float* fars, float* xyzs, float* dirs, float* deltas, const float* noises, void* stream) {
    if (n_alive == 0 || n_step == 0) return SFB_OK;  // empty problem: nothing to do, pointers may be null
    SFB_REQUIRE(rays_alive && rays_t && rays_o && rays_d && grid && nears && fars && xyzs && dirs && deltas && noises, "march_rays: null pointer");
    march_rays_kernel<<<ceil_div(n_alive, 128u), 128, 0, as_stream(stream)>>>(n_alive, n_step, rays_alive, rays_t, rays_o, rays_d, bound, dt_gamma,
                                                                             max_steps, C, H, grid, nears, fars, xyzs, dirs, deltas, noises);
    return check_launch("march_rays");
}

int sfb_composite_rays(uint32_t n_alive, uint32_t n_step, float T_thresh, int32_t* rays_alive, float* rays_t, const float* sigmas,
                       const float* rgbs, const float* deltas, float* weights_sum, float* depth, float* image, void* stream) {
    if (n_alive == 0) return SFB_OK;  // empty problem: nothing to do, pointers may be null
    SFB_REQUIRE(rays_alive && rays_t && sigmas && rgbs && deltas && weights_sum && depth && image, "composite_rays: null pointer");
    composite_rays_kernel<<<ceil_div(n_alive, 128u), 128, 0, as_stream(stream)>>>(n_alive, n_step, T_thresh, rays_alive, rays_t, sigmas, rgbs,
                                                                                 deltas, weights_sum, depth, image);
    return check_launch("composite_rays");
}
}
