// gridencoder.cu -- multi-resolution tiled/hash grid encoder operators for sm_90a.
//
// Drop-in for the reference's `_gridencoder` pybind module (external/gridencoder/src/bindings.cpp:5-8):
// same argument order and layouts ([L,B,C] level-major outputs, [B,L,D,C] dy_dx, pre-zeroed gradient
// table), fp32, launched on the caller's stream.  Index arithmetic is kept bit-identical to the
// reference kernels (gridencoder.cu:54-72 index, :124-137 scale / cell / fraction) -- including the
// tiled-index quirk that drops trailing coordinates once the running stride exceeds the level's row
// count -- so that embeddings trained by either implementation are interchangeable.
//
// H100 notes: the whole live table is 7.1 MB and lives in the 50 MB L2, so these kernels are L2-gather
// bound; what matters is (a) one 8-byte gather per corner for C == 2 (float2), (b) coalesced [L,B,C]
// stores, (c) for the backward, one vector reduction (red.global.add.v2.f32) per corner instead of C
// scalar atomics.  The fused field kernels in ngp_field.cu are the hot path; these operators exist for
// API parity and as their building blocks (grid_locate / grid_row are shared through gridencoder.cuh).
#include "common.cuh"
#include "gridencoder.cuh"
#include "../../include/sparsefusion_b200.h"

namespace sfb {

template <uint32_t D, uint32_t C>
__global__ void __launch_bounds__(256) grid_forward_kernel(const float* __restrict__ inputs, const float* __restrict__ table,
                                                          const int32_t* __restrict__ offsets, float* __restrict__ outputs,
                                                          uint32_t B, uint32_t L, float S, uint32_t H, float* __restrict__ dy_dx,
                                                          uint32_t gridtype, bool align_corners) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const uint32_t level = blockIdx.y;

    float x[D];
#pragma unroll
    for (uint32_t d = 0; d < D; ++d) x[d] = inputs[b * D + d];
    float* out = outputs + ((size_t)level * B + b) * C;

    if (grid_out_of_range<D>(x)) {
#pragma unroll
        for (uint32_t c = 0; c < C; ++c) out[c] = 0.f;
        if (dy_dx) {
            float* dy = dy_dx + (size_t)b * D * L * C + level * D * C;
#pragma unroll
            for (uint32_t i = 0; i < D * C; ++i) dy[i] = 0.f;
        }
        return;
    }

    const GridLevel lv = grid_level(level, S, H, offsets);
    const float* grid = table + (size_t)lv.offset * C;
    float frac[D];
    uint32_t cell[D];
    grid_locate<D>(x, lv.scale, align_corners, frac, cell);

    float acc[C];
#pragma unroll
    for (uint32_t c = 0; c < C; ++c) acc[c] = 0.f;

#pragma unroll
    for (uint32_t corner = 0; corner < (1u << D); ++corner) {
        float w = 1.f;
        uint32_t cl[D];
#pragma unroll
        for (uint32_t d = 0; d < D; ++d) {
            if ((corner & (1u << d)) == 0) { w *= 1 - frac[d]; cl[d] = cell[d]; }
            else { w *= frac[d]; cl[d] = cell[d] + 1; }
        }
        const uint32_t row = grid_row<D>(gridtype, align_corners, lv.rows, lv.resolution, cl);
        float v[C];
        grid_load_row<C>(grid, row, v);
#pragma unroll
        for (uint32_t c = 0; c < C; ++c) acc[c] += w * v[c];
    }
    grid_store_row<C>(out, acc);

    if (dy_dx) {
        float* dy = dy_dx + (size_t)b * D * L * C + level * D * C;
#pragma unroll
        for (uint32_t gd = 0; gd < D; ++gd) {
            float g[C];
#pragma unroll
            for (uint32_t c = 0; c < C; ++c) g[c] = 0.f;
#pragma unroll
            for (uint32_t idx = 0; idx < (1u << (D - 1)); ++idx) {
                float w = lv.scale;
                uint32_t cl[D];
#pragma unroll
                for (uint32_t nd = 0; nd < D - 1; ++nd) {
                    const uint32_t d = (nd >= gd) ? nd + 1 : nd;
                    if ((idx & (1u << nd)) == 0) { w *= 1 - frac[d]; cl[d] = cell[d]; }
                    else { w *= frac[d]; cl[d] = cell[d] + 1; }
                }
                cl[gd] = cell[gd];
                const uint32_t rl = grid_row<D>(gridtype, align_corners, lv.rows, lv.resolution, cl);
                cl[gd] = cell[gd] + 1;
                const uint32_t rr = grid_row<D>(gridtype, align_corners, lv.rows, lv.resolution, cl);
                float vl[C], vr[C];
                grid_load_row<C>(grid, rl, vl);
                grid_load_row<C>(grid, rr, vr);
#pragma unroll
                for (uint32_t c = 0; c < C; ++c) g[c] += w * (vr[c] - vl[c]);
            }
#pragma unroll
            for (uint32_t c = 0; c < C; ++c) dy[gd * C + c] = g[c];
        }
    }
}

// One thread per (point, level): all C channels of a corner go out as one vector reduction.
template <uint32_t D, uint32_t C>
__global__ void __launch_bounds__(256) grid_backward_kernel(const float* __restrict__ grad, const float* __restrict__ inputs,
                                                           const int32_t* __restrict__ offsets, float* __restrict__ grad_table,
                                                           uint32_t B, uint32_t L, float S, uint32_t H, uint32_t gridtype,
                                                           bool align_corners) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const uint32_t level = blockIdx.y;
    float x[D];
#pragma unroll
    for (uint32_t d = 0; d < D; ++d) x[d] = inputs[b * D + d];
    if (grid_out_of_range<D>(x)) return;  // gradient table is pre-zeroed

    const GridLevel lv = grid_level(level, S, H, offsets);
    float* gt = grad_table + (size_t)lv.offset * C;
    float frac[D];
    uint32_t cell[D];
    grid_locate<D>(x, lv.scale, align_corners, frac, cell);

    float g[C];
    grid_load_row<C>(grad + (size_t)level * B * C, b, g);

#pragma unroll
    for (uint32_t corner = 0; corner < (1u << D); ++corner) {
        float w = 1.f;
        uint32_t cl[D];
#pragma unroll
        for (uint32_t d = 0; d < D; ++d) {
            if ((corner & (1u << d)) == 0) { w *= 1 - frac[d]; cl[d] = cell[d]; }
            else { w *= frac[d]; cl[d] = cell[d] + 1; }
        }
        const uint32_t row = grid_row<D>(gridtype, align_corners, lv.rows, lv.resolution, cl);
        float wg[C];
#pragma unroll
        for (uint32_t c = 0; c < C; ++c) wg[c] = w * g[c];
        grid_red_add_row<C>(gt, row, wg);
    }
}

template <uint32_t D, uint32_t C>
__global__ void __launch_bounds__(256) grid_input_backward_kernel(const float* __restrict__ grad, const float* __restrict__ dy_dx,
                                                                 float* __restrict__ grad_inputs, uint32_t B, uint32_t L) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= B * D) return;
    const uint32_t b = t / D, d = t - b * D;
    const float* dy = dy_dx + (size_t)b * L * D * C;
    float r = 0.f;
    for (uint32_t l = 0; l < L; ++l) {
#pragma unroll
        for (uint32_t c = 0; c < C; ++c) r += grad[((size_t)l * B + b) * C + c] * dy[l * D * C + d * C + c];
    }
    grad_inputs[t] = r;
}

template <uint32_t D>
__global__ void grid_rows_kernel(const float* __restrict__ inputs, const int32_t* __restrict__ offsets, int32_t* __restrict__ rows,
                                 uint32_t B, uint32_t L, float S, uint32_t H, uint32_t gridtype, bool align_corners) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const uint32_t level = blockIdx.y;
    float x[D];
#pragma unroll
    for (uint32_t d = 0; d < D; ++d) x[d] = inputs[b * D + d];
    int32_t* out = rows + ((size_t)level * B + b) * (1u << D);
    if (grid_out_of_range<D>(x)) {
        for (uint32_t i = 0; i < (1u << D); ++i) out[i] = -1;
        return;
    }
    const GridLevel lv = grid_level(level, S, H, offsets);
    float frac[D];
    uint32_t cell[D];
    grid_locate<D>(x, lv.scale, align_corners, frac, cell);
    for (uint32_t corner = 0; corner < (1u << D); ++corner) {
        uint32_t cl[D];
#pragma unroll
        for (uint32_t d = 0; d < D; ++d) cl[d] = cell[d] + ((corner >> d) & 1u);
        out[corner] = (int32_t)(lv.offset + grid_row<D>(gridtype, align_corners, lv.rows, lv.resolution, cl));
    }
}

__global__ void grid_scales_kernel(uint32_t L, float S, uint32_t H, float* scales) {
    const uint32_t l = threadIdx.x;
    if (l < L) scales[l] = grid_level_scale(l, S, H);
}

template <uint32_t D, uint32_t C>
static int launch_forward(const float* inputs, const float* emb, const int32_t* offsets, float* out, uint32_t B, uint32_t L, float S,
                          uint32_t H, float* dy_dx, uint32_t gridtype, bool ac, cudaStream_t st) {
    dim3 grid(ceil_div(B, 256u), L);
    grid_forward_kernel<D, C><<<grid, 256, 0, st>>>(inputs, emb, offsets, out, B, L, S, H, dy_dx, gridtype, ac);
    return check_launch("grid_encode_forward");
}

template <uint32_t D, uint32_t C>
static int launch_backward(const float* grad, const float* inputs, const int32_t* offsets, float* ge, uint32_t B, uint32_t L, float S,
                           uint32_t H, const float* dy_dx, float* gi, uint32_t gridtype, bool ac, cudaStream_t st) {
    dim3 grid(ceil_div(B, 256u), L);
    grid_backward_kernel<D, C><<<grid, 256, 0, st>>>(grad, inputs, offsets, ge, B, L, S, H, gridtype, ac);
    if (int rc = check_launch("grid_encode_backward")) return rc;
    if (dy_dx && gi) {
        grid_input_backward_kernel<D, C><<<ceil_div(B * D, 256u), 256, 0, st>>>(grad, dy_dx, gi, B, L);
        return check_launch("grid_encode_backward(inputs)");
    }
    return SFB_OK;
}

#define SFB_DISPATCH_DC(D, C, FN, ...)                                                               \
    [&]() -> int {                                                                                   \
        switch ((D) * 16 + (C)) {                                                                    \
            case 1 * 16 + 1: return FN<1, 1>(__VA_ARGS__); case 1 * 16 + 2: return FN<1, 2>(__VA_ARGS__); \
            case 1 * 16 + 4: return FN<1, 4>(__VA_ARGS__); case 1 * 16 + 8: return FN<1, 8>(__VA_ARGS__); \
            case 2 * 16 + 1: return FN<2, 1>(__VA_ARGS__); case 2 * 16 + 2: return FN<2, 2>(__VA_ARGS__); \
            case 2 * 16 + 4: return FN<2, 4>(__VA_ARGS__); case 2 * 16 + 8: return FN<2, 8>(__VA_ARGS__); \
            case 3 * 16 + 1: return FN<3, 1>(__VA_ARGS__); case 3 * 16 + 2: return FN<3, 2>(__VA_ARGS__); \
            case 3 * 16 + 4: return FN<3, 4>(__VA_ARGS__); case 3 * 16 + 8: return FN<3, 8>(__VA_ARGS__); \
            case 4 * 16 + 1: return FN<4, 1>(__VA_ARGS__); case 4 * 16 + 2: return FN<4, 2>(__VA_ARGS__); \
            case 4 * 16 + 4: return FN<4, 4>(__VA_ARGS__); case 4 * 16 + 8: return FN<4, 8>(__VA_ARGS__); \
            case 5 * 16 + 1: return FN<5, 1>(__VA_ARGS__); case 5 * 16 + 2: return FN<5, 2>(__VA_ARGS__); \
            case 5 * 16 + 4: return FN<5, 4>(__VA_ARGS__); case 5 * 16 + 8: return FN<5, 8>(__VA_ARGS__); \
            default: return fail(SFB_ERR_ARG, "GridEncoding: D must be 1..5 and C must be 1, 2, 4, or 8 (got D=%u C=%u)", (unsigned)(D), (unsigned)(C)); \
        }                                                                                            \
    }()

}  // namespace sfb

using namespace sfb;

extern "C" {

int sfb_grid_encode_forward(const float* inputs, const float* embeddings, const int32_t* offsets, float* outputs, uint32_t B,
                            uint32_t D, uint32_t C, uint32_t L, float S, uint32_t H, float* dy_dx, uint32_t gridtype,
                            int align_corners, void* stream) {
    if (B == 0 || L == 0) return SFB_OK;  // empty problem: nothing to do, pointers may be null
    SFB_REQUIRE(inputs && embeddings && offsets && outputs, "grid_encode_forward: null pointer");
    SFB_REQUIRE(gridtype <= 1, "grid_encode_forward: gridtype must be 0 (hash) or 1 (tiled)");
    return SFB_DISPATCH_DC(D, C, launch_forward, inputs, embeddings, offsets, outputs, B, L, S, H, dy_dx, gridtype, align_corners != 0,
                           as_stream(stream));
}

int sfb_grid_encode_backward(const float* grad, const float* inputs, const float* embeddings, const int32_t* offsets,
                             float* grad_embeddings, uint32_t B, uint32_t D, uint32_t C, uint32_t L, float S, uint32_t H,
                             const float* dy_dx, float* grad_inputs, uint32_t gridtype, int align_corners, void* stream) {
    if (B == 0 || L == 0) return SFB_OK;  // empty problem: nothing to do, pointers may be null
    (void)embeddings;
    SFB_REQUIRE(grad && inputs && offsets && grad_embeddings, "grid_encode_backward: null pointer");
    SFB_REQUIRE(gridtype <= 1, "grid_encode_backward: gridtype must be 0 (hash) or 1 (tiled)");
    return SFB_DISPATCH_DC(D, C, launch_backward, grad, inputs, offsets, grad_embeddings, B, L, S, H, dy_dx, grad_inputs, gridtype,
                           align_corners != 0, as_stream(stream));
}

int sfb_grid_level_scales(uint32_t L, float S, uint32_t H, float* scales, void* stream) {
    SFB_REQUIRE(scales && L <= 32, "grid_level_scales: null pointer or L > 32");
    grid_scales_kernel<<<1, 32, 0, as_stream(stream)>>>(L, S, H, scales);
    return check_launch("grid_level_scales");
}

int sfb_grid_corner_rows(const float* inputs, const int32_t* offsets, int32_t* rows, uint32_t B, uint32_t D, uint32_t L, float S,
                         uint32_t H, uint32_t gridtype, int align_corners, void* stream) {
    if (B == 0 || L == 0) return SFB_OK;  // empty problem: nothing to do, pointers may be null
    SFB_REQUIRE(inputs && offsets && rows, "grid_corner_rows: null pointer");
    dim3 grid(ceil_div(B, 256u), L);
    cudaStream_t st = as_stream(stream);
    // every D the encoder accepts, so that the rows of each instantiation can be checked
    switch (D) {
        case 1: grid_rows_kernel<1><<<grid, 256, 0, st>>>(inputs, offsets, rows, B, L, S, H, gridtype, align_corners != 0); break;
        case 2: grid_rows_kernel<2><<<grid, 256, 0, st>>>(inputs, offsets, rows, B, L, S, H, gridtype, align_corners != 0); break;
        case 3: grid_rows_kernel<3><<<grid, 256, 0, st>>>(inputs, offsets, rows, B, L, S, H, gridtype, align_corners != 0); break;
        case 4: grid_rows_kernel<4><<<grid, 256, 0, st>>>(inputs, offsets, rows, B, L, S, H, gridtype, align_corners != 0); break;
        case 5: grid_rows_kernel<5><<<grid, 256, 0, st>>>(inputs, offsets, rows, B, L, S, H, gridtype, align_corners != 0); break;
        default: return fail(SFB_ERR_ARG, "grid_corner_rows: D must be 1..5");
    }
    return check_launch("grid_corner_rows");
}
}
