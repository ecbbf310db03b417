// ngp_field.cu -- the Instant-NGP field query of SparseFusion's NeRFNetwork, fused, for sm_90a:
//     xyz -> tiled-grid encode (16 levels x 2) -> MLP 32-64-64-4 (ReLU) -> sigma = exp(h0 + blob(x)), albedo = sigmoid(h1:4)
// (external/nerf/network_grid.py:69-88 common_forward; external/gridencoder/grid.py:138-154; ngp_activation.py:10-21).
// The reference runs this as ~12 eager launches per call (kernel_grid + permute + 3 cuBLAS GEMMs + elementwise) and
// calls it three times per render; here one kernel evaluates a point once, and one kernel pair back-propagates.
//
// fp32 SIMT by design (the 1e-3 RGB contract and bit-exact grid indexing rule out reduced precision here):
//   * one thread per point; the 7.1 MB embedding table stays L2-resident, corners fetched as 8-byte float2;
//   * MLP weights live in shared memory TRANSPOSED ([k][j]) so that one broadcast LDS.128 feeds 4 FMAs; the
//     per-thread activation vector lives in a conflict-free shared-memory column (hs[k][tid]), so the k loop is a
//     real loop (small code, no register-indexed arrays);
//   * backward recomputes the forward (no activation tape through HBM for the data path), scatters grid gradients
//     with red.global.add.v2.f32, and writes feature-major activation / pre-activation-gradient tapes that the
//     weight-gradient kernel reduces with a register-tiled outer-product GEMM (one red per weight per CTA).
// Points are addressed either explicitly (xyz [B,3]) or implicitly as rays: x = clamp(o + d*z, aabb) with separate
// fp32 multiply and add, which is bit-identical to the reference's torch expression (renderer_df.py:367-368).
#include "common.cuh"
#include "gridencoder.cuh"
#include "../../include/sparsefusion_b200.h"

namespace sfb {

constexpr int kL = 16, kC = 2, kIn = 32, kHid = 64, kOut = 4;
constexpr int kFieldThreads = 128;

struct FieldGeom {
    float S;
    uint32_t H;
    float bound;
};

struct PointSource {  // either xyz != null, or rays (o, d, z) with T samples per ray
    const float* xyz;
    const float* rays_o;
    const float* rays_d;
    const float* z;
    uint32_t T;
    float aabb_lo[3], aabb_hi[3];
};

__device__ __forceinline__ void fetch_point(const PointSource& ps, uint32_t p, float (&x)[3]) {
    if (ps.xyz) {
        x[0] = ps.xyz[(size_t)p * 3]; x[1] = ps.xyz[(size_t)p * 3 + 1]; x[2] = ps.xyz[(size_t)p * 3 + 2];
    } else {
        const uint32_t ray = p / ps.T;
        const float zz = ps.z[p];
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            const float v = __fadd_rn(ps.rays_o[(size_t)ray * 3 + d], __fmul_rn(ps.rays_d[(size_t)ray * 3 + d], zz));
            x[d] = fminf(fmaxf(v, ps.aabb_lo[d]), ps.aabb_hi[d]);
        }
    }
}

// encode one point: 16 levels x (8 corners, float2) -> hs[2*l + c][tid]
__device__ __forceinline__ void encode_point(const float (&x)[3], const float* __restrict__ table, const int32_t* __restrict__ offsets,
                                             const FieldGeom& g, float* __restrict__ hs, int tid) {
    float u[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) u[d] = __fdiv_rn(__fadd_rn(x[d], g.bound), 2 * g.bound);  // grid.py:142
    const bool oob = grid_out_of_range<3>(u);
#pragma unroll 1
    for (uint32_t level = 0; level < kL; ++level) {
        float a0 = 0.f, a1 = 0.f;
        if (!oob) {
            const GridLevel lv = grid_level(level, g.S, g.H, offsets);
            const float* grid = table + (size_t)lv.offset * kC;
            float frac[3];
            uint32_t cell[3];
            grid_locate<3>(u, lv.scale, false, frac, cell);
#pragma unroll
            for (uint32_t corner = 0; corner < 8; ++corner) {
                float w = 1.f;
                uint32_t cl[3];
#pragma unroll
                for (uint32_t d = 0; d < 3; ++d) {
                    if ((corner & (1u << d)) == 0) { w *= 1 - frac[d]; cl[d] = cell[d]; }
                    else { w *= frac[d]; cl[d] = cell[d] + 1; }
                }
                const uint32_t row = grid_row<3>(1u, false, lv.rows, lv.resolution, cl);
                const float2 v = __ldg(reinterpret_cast<const float2*>(grid) + row);
                a0 += w * v.x;
                a1 += w * v.y;
            }
        }
        hs[(2 * level) * kFieldThreads + tid] = a0;
        hs[(2 * level + 1) * kFieldThreads + tid] = a1;
    }
}

// acc[j] = bias[j] + sum_k WT[k][j] * hs[k][tid]      (WT transposed weights in smem, K in {32, 64}, 64 outputs)
template <int K>
__device__ __forceinline__ void dense64(const float* __restrict__ WT, const float* __restrict__ bias, const float* __restrict__ hs, int tid,
                                        float (&acc)[kHid]) {
#pragma unroll
    for (int j = 0; j < kHid; ++j) acc[j] = bias[j];
#pragma unroll 2
    for (int k = 0; k < K; ++k) {
        const float hk = hs[k * kFieldThreads + tid];
        const float4* w = reinterpret_cast<const float4*>(WT + k * kHid);
#pragma unroll
        for (int j4 = 0; j4 < kHid / 4; ++j4) {
            const float4 wv = w[j4];
            acc[4 * j4 + 0] += wv.x * hk; acc[4 * j4 + 1] += wv.y * hk;
            acc[4 * j4 + 2] += wv.z * hk; acc[4 * j4 + 3] += wv.w * hk;
        }
    }
}

struct FieldSmem {
    float WT0[kIn * kHid];   // [k][j]
    float WT1[kHid * kHid];  // [k][j]
    float WT2[kHid * kOut];  // [k][j]
    float b0[kHid], b1[kHid], b2[kOut];
};

__device__ __forceinline__ void load_weights_T(FieldSmem& s, const float* W0, const float* b0, const float* W1, const float* b1, const float* W2,
                                               const float* b2) {
    for (int i = threadIdx.x; i < kHid * kIn; i += blockDim.x) { const int j = i / kIn, k = i - j * kIn; s.WT0[k * kHid + j] = W0[i]; }
    for (int i = threadIdx.x; i < kHid * kHid; i += blockDim.x) { const int j = i / kHid, k = i - j * kHid; s.WT1[k * kHid + j] = W1[i]; }
    for (int i = threadIdx.x; i < kOut * kHid; i += blockDim.x) { const int j = i / kHid, k = i - j * kHid; s.WT2[k * kOut + j] = W2[i]; }
    for (int i = threadIdx.x; i < kHid; i += blockDim.x) { s.b0[i] = b0[i]; s.b1[i] = b1[i]; }
    if (threadIdx.x < kOut) s.b2[threadIdx.x] = b2[threadIdx.x];
}

__device__ __forceinline__ float density_blob(const float (&x)[3]) {  // network_grid.py:69-75
    const float d = x[0] * x[0] + x[1] * x[1] + x[2] * x[2];
    return 5.f * expf(-d / 0.08f);
}

// ------------------------------------------------------------------------------------------------ forward
__global__ void __launch_bounds__(kFieldThreads) field_forward_kernel(PointSource ps, uint32_t B, const float* __restrict__ table,
                                                                     const int32_t* __restrict__ offsets, FieldGeom g,
                                                                     const float* __restrict__ W0, const float* __restrict__ b0,
                                                                     const float* __restrict__ W1, const float* __restrict__ b1,
                                                                     const float* __restrict__ W2, const float* __restrict__ b2,
                                                                     float* __restrict__ sigma, float* __restrict__ rgb) {
    extern __shared__ __align__(16) uint8_t smraw[];
    FieldSmem& s = *reinterpret_cast<FieldSmem*>(smraw);
    float* hs = reinterpret_cast<float*>(smraw + sizeof(FieldSmem));
    load_weights_T(s, W0, b0, W1, b1, W2, b2);
    __syncthreads();
    const int tid = threadIdx.x;
    for (uint32_t base = blockIdx.x * kFieldThreads; base < B; base += gridDim.x * kFieldThreads) {
        const uint32_t p = base + tid;
        if (p >= B) continue;  // no block-level sync inside the loop
        float x[3];
        fetch_point(ps, p, x);
        encode_point(x, table, offsets, g, hs, tid);
        float acc[kHid];
        dense64<kIn>(s.WT0, s.b0, hs, tid, acc);
#pragma unroll
        for (int j = 0; j < kHid; ++j) hs[j * kFieldThreads + tid] = fmaxf(acc[j], 0.f);
        dense64<kHid>(s.WT1, s.b1, hs, tid, acc);
#pragma unroll
        for (int j = 0; j < kHid; ++j) hs[j * kFieldThreads + tid] = fmaxf(acc[j], 0.f);
        float o0 = s.b2[0], o1 = s.b2[1], o2 = s.b2[2], o3 = s.b2[3];
#pragma unroll 4
        for (int k = 0; k < kHid; ++k) {
            const float hk = hs[k * kFieldThreads + tid];
            const float4 w = *reinterpret_cast<const float4*>(s.WT2 + k * kOut);
            o0 += w.x * hk; o1 += w.y * hk; o2 += w.z * hk; o3 += w.w * hk;
        }
        sigma[p] = expf(o0 + density_blob(x));
        if (rgb) {
            rgb[(size_t)p * 3] = 1.f / (1.f + expf(-o1));
            rgb[(size_t)p * 3 + 1] = 1.f / (1.f + expf(-o2));
            rgb[(size_t)p * 3 + 2] = 1.f / (1.f + expf(-o3));
        }
    }
}

// ------------------------------------------------------------------------------------------------ backward (data path)
// tapes (feature-major, Bp = padded point count): H0 [32][Bp], H1 [64][Bp], H2 [64][Bp], D1 [64][Bp], D2 [64][Bp], D3 [4][Bp]
struct FieldSmemBwd {
    FieldSmem f;  // the transposed weights serve both directions: d_in[k] = dot(WT[k][:], d_out[:])
};

// d_in[k] = sum_j WT[k][j] * dreg[j]  for k < K (K inputs, 64 outputs): one row of the transposed weights per k
template <int K>
__device__ __forceinline__ float backprop_row(const float* __restrict__ WT, int k, const float (&dreg)[kHid]) {
    const float4* w = reinterpret_cast<const float4*>(WT + k * kHid);
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll
    for (int j4 = 0; j4 < kHid / 4; ++j4) {
        const float4 wv = w[j4];
        a0 += wv.x * dreg[4 * j4 + 0]; a1 += wv.y * dreg[4 * j4 + 1]; a2 += wv.z * dreg[4 * j4 + 2]; a3 += wv.w * dreg[4 * j4 + 3];
    }
    return (a0 + a1) + (a2 + a3);
}

__global__ void __launch_bounds__(kFieldThreads) field_backward_kernel(PointSource ps, uint32_t B, uint32_t Bp, const float* __restrict__ table,
                                                                      const int32_t* __restrict__ offsets, FieldGeom g,
                                                                      const float* __restrict__ W0, const float* __restrict__ b0,
                                                                      const float* __restrict__ W1, const float* __restrict__ b1,
                                                                      const float* __restrict__ W2, const float* __restrict__ b2,
                                                                      const float* __restrict__ g_sigma, const float* __restrict__ g_rgb,
                                                                      float* __restrict__ grad_table, float* __restrict__ H0,
                                                                      float* __restrict__ H1, float* __restrict__ H2, float* __restrict__ D1,
                                                                      float* __restrict__ D2, float* __restrict__ D3) {
    extern __shared__ __align__(16) uint8_t smraw[];
    FieldSmemBwd& s = *reinterpret_cast<FieldSmemBwd*>(smraw);
    float* hs = reinterpret_cast<float*>(smraw + sizeof(FieldSmemBwd));  // [64][128] activations
    float* ds = hs + kHid * kFieldThreads;                                // [64][128] pre-activation gradients
    load_weights_T(s.f, W0, b0, W1, b1, W2, b2);
    __syncthreads();
    const int tid = threadIdx.x;
    for (uint32_t base = blockIdx.x * kFieldThreads; base < Bp; base += gridDim.x * kFieldThreads) {
        const uint32_t p = base + tid;
        if (p >= Bp) continue;
        if (p >= B) {  // padding rows of the tapes contribute nothing
            for (int k = 0; k < kIn; ++k) H0[(size_t)k * Bp + p] = 0.f;
            for (int k = 0; k < kHid; ++k) { H1[(size_t)k * Bp + p] = 0.f; H2[(size_t)k * Bp + p] = 0.f; D1[(size_t)k * Bp + p] = 0.f; D2[(size_t)k * Bp + p] = 0.f; }
            for (int k = 0; k < kOut; ++k) D3[(size_t)k * Bp + p] = 0.f;
            continue;
        }
        float x[3];
        fetch_point(ps, p, x);
        encode_point(x, table, offsets, g, hs, tid);
#pragma unroll 4
        for (int k = 0; k < kIn; ++k) H0[(size_t)k * Bp + p] = hs[k * kFieldThreads + tid];
        float acc[kHid];
        uint64_t mask1 = 0, mask2 = 0;
        dense64<kIn>(s.f.WT0, s.f.b0, hs, tid, acc);
#pragma unroll
        for (int j = 0; j < kHid; ++j) {
            const float a = fmaxf(acc[j], 0.f);
            mask1 |= (uint64_t)(acc[j] > 0.f) << j;
            hs[j * kFieldThreads + tid] = a;
            H1[(size_t)j * Bp + p] = a;
        }
        dense64<kHid>(s.f.WT1, s.f.b1, hs, tid, acc);
#pragma unroll
        for (int j = 0; j < kHid; ++j) {
            const float a = fmaxf(acc[j], 0.f);
            mask2 |= (uint64_t)(acc[j] > 0.f) << j;
            hs[j * kFieldThreads + tid] = a;
            H2[(size_t)j * Bp + p] = a;
        }
        float o[4] = {s.f.b2[0], s.f.b2[1], s.f.b2[2], s.f.b2[3]};
#pragma unroll 4
        for (int k = 0; k < kHid; ++k) {
            const float hk = hs[k * kFieldThreads + tid];
            const float4 w = *reinterpret_cast<const float4*>(s.f.WT2 + k * kOut);
            o[0] += w.x * hk; o[1] += w.y * hk; o[2] += w.z * hk; o[3] += w.w * hk;
        }
        // output activations: trunc_exp backward clamps the exponent to +-15 (ngp_activation.py:19-21)
        float d3[4];
        const float pre = o[0] + density_blob(x);
        d3[0] = g_sigma[p] * expf(fminf(fmaxf(pre, -15.f), 15.f));
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float sg = 1.f / (1.f + expf(-o[c + 1]));
            d3[c + 1] = g_rgb ? g_rgb[(size_t)p * 3 + c] * sg * (1.f - sg) : 0.f;
        }
#pragma unroll
        for (int c = 0; c < 4; ++c) D3[(size_t)c * Bp + p] = d3[c];
        // d2 = (W2^T d3) * relu'(a2)
#pragma unroll 4
        for (int k = 0; k < kHid; ++k) {
            const float4 w = *reinterpret_cast<const float4*>(s.f.WT2 + k * kOut);
            float v = w.x * d3[0] + w.y * d3[1] + w.z * d3[2] + w.w * d3[3];
            v = ((mask2 >> k) & 1ull) ? v : 0.f;
            ds[k * kFieldThreads + tid] = v;
            D2[(size_t)k * Bp + p] = v;
        }
        // d1 = (W1^T d2) * relu'(a1)
#pragma unroll
        for (int j = 0; j < kHid; ++j) acc[j] = ds[j * kFieldThreads + tid];  // d2 into registers
#pragma unroll 1
        for (int k = 0; k < kHid; ++k) {
            float v = backprop_row<kHid>(s.f.WT1, k, acc);
            v = ((mask1 >> k) & 1ull) ? v : 0.f;
            ds[k * kFieldThreads + tid] = v;  // own column; d2 is already in registers
            D1[(size_t)k * Bp + p] = v;
        }
        // d0[k] = sum_j W0[j][k] d1[j]   (32 encoder features)
#pragma unroll
        for (int j = 0; j < kHid; ++j) acc[j] = ds[j * kFieldThreads + tid];  // d1 into registers
        float d0[kIn];
#pragma unroll
        for (int k = 0; k < kIn; ++k) d0[k] = backprop_row<kIn>(s.f.WT0, k, acc);
        // scatter into the embedding gradient (kernel_grid_backward, gridencoder.cu:226-313)
        float u[3];
#pragma unroll
        for (int d = 0; d < 3; ++d) u[d] = __fdiv_rn(__fadd_rn(x[d], g.bound), 2 * g.bound);
        if (!grid_out_of_range<3>(u)) {
#pragma unroll
            for (uint32_t level = 0; level < kL; ++level) {
                const GridLevel lv = grid_level(level, g.S, g.H, offsets);
                float* gt = grad_table + (size_t)lv.offset * kC;
                float frac[3];
                uint32_t cell[3];
                grid_locate<3>(u, lv.scale, false, frac, cell);
                const float g0 = d0[2 * level], g1 = d0[2 * level + 1];
#pragma unroll
                for (uint32_t corner = 0; corner < 8; ++corner) {
                    float w = 1.f;
                    uint32_t cl[3];
#pragma unroll
                    for (uint32_t d = 0; d < 3; ++d) {
                        if ((corner & (1u << d)) == 0) { w *= 1 - frac[d]; cl[d] = cell[d]; }
                        else { w *= frac[d]; cl[d] = cell[d] + 1; }
                    }
                    const uint32_t row = grid_row<3>(1u, false, lv.rows, lv.resolution, cl);
                    const float wg[2] = {w * g0, w * g1};
                    grid_red_add_row<2>(gt, row, wg);
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ weight gradients
// db[j] += sum_p D[j][p] for the rows of D1 | D2 | D3 (contiguous [2*kHid + kOut][Bp]); grid (chunks, rows)
__global__ void __launch_bounds__(256) tape_rowsum_kernel(const float* __restrict__ D, uint32_t Bp, float* __restrict__ gb0, float* __restrict__ gb1,
                                                         float* __restrict__ gb2) {
    const int row = blockIdx.y;
    const float4* r4 = reinterpret_cast<const float4*>(D + (size_t)row * Bp);
    const uint32_t n4 = Bp >> 2;   // Bp is a multiple of 64
    float s = 0.f;
    for (uint32_t i = blockIdx.x * 256u + threadIdx.x; i < n4; i += gridDim.x * 256u) {
        const float4 v = __ldg(r4 + i);
        s += (v.x + v.y) + (v.z + v.w);
    }
    __shared__ float sh[8];
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int w = 0; w < 8; ++w) t += sh[w];
        float* dst = row < kHid ? gb0 + row : (row < 2 * kHid ? gb1 + (row - kHid) : gb2 + (row - 2 * kHid));
        atomicAdd(dst, t);
    }
}

// dW[j][k] += sum_p D[j][p] * H[k][p];  db[j] += sum_p D[j][p].   D [J][Bp], H [K][Bp] feature-major.
// CTA = 256 threads as a 16x16 grid of (J/16 x K/16) register tiles; points staged through smem 64 at a time.
template <int J, int K>
__global__ void __launch_bounds__(256) mlp_wgrad_kernel(const float* __restrict__ D, const float* __restrict__ H, uint32_t Bp,
                                                       float* __restrict__ gW, float* __restrict__ gb) {
    constexpr int TJ = (J + 15) / 16, TK = (K + 15) / 16, PT = 64;
    __shared__ float Ds[J][PT + 1];
    __shared__ float Hs[K][PT + 1];
    const int tj = threadIdx.x / 16, tk = threadIdx.x % 16;
    float acc[TJ][TK];
    float accb[TJ];
#pragma unroll
    for (int a = 0; a < TJ; ++a) {
        accb[a] = 0.f;
#pragma unroll
        for (int b = 0; b < TK; ++b) acc[a][b] = 0.f;
    }
    const uint32_t chunks = Bp / PT;
    for (uint32_t ch = blockIdx.x; ch < chunks; ch += gridDim.x) {
        const uint32_t p0 = ch * PT;
        for (int i = threadIdx.x; i < J * PT; i += 256) { const int j = i / PT, q = i % PT; Ds[j][q] = D[(size_t)j * Bp + p0 + q]; }
        for (int i = threadIdx.x; i < K * PT; i += 256) { const int k = i / PT, q = i % PT; Hs[k][q] = H[(size_t)k * Bp + p0 + q]; }
        __syncthreads();
#pragma unroll 4
        for (int q = 0; q < PT; ++q) {
            float dv[TJ], hv[TK];
#pragma unroll
            for (int a = 0; a < TJ; ++a) dv[a] = (tj * TJ + a < J) ? Ds[tj * TJ + a][q] : 0.f;
#pragma unroll
            for (int b = 0; b < TK; ++b) hv[b] = (tk * TK + b < K) ? Hs[tk * TK + b][q] : 0.f;
#pragma unroll
            for (int a = 0; a < TJ; ++a) {
                if (tk == 0) accb[a] += dv[a];
#pragma unroll
                for (int b = 0; b < TK; ++b) acc[a][b] += dv[a] * hv[b];
            }
        }
        __syncthreads();
    }
#pragma unroll
    for (int a = 0; a < TJ; ++a) {
        const int j = tj * TJ + a;
        if (j >= J) continue;
        if (tk == 0) atomicAdd(gb + j, accb[a]);
#pragma unroll
        for (int b = 0; b < TK; ++b) {
            const int k = tk * TK + b;
            if (k < K) atomicAdd(gW + (size_t)j * K + k, acc[a][b]);
        }
    }
}

// ------------------------------------------------------------------------------------------------ Adam
// torch.optim.Adam semantics (no amsgrad, no weight decay): one fused pass over a parameter group
__global__ void adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, int64_t n, float lr,
                            float beta1, float beta2, float eps, float bc1, float bc2_sqrt, float grad_scale) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float gi = g[i] * grad_scale;
        const float mi = beta1 * m[i] + (1.f - beta1) * gi;
        const float vi = beta2 * v[i] + (1.f - beta2) * gi * gi;
        m[i] = mi;
        v[i] = vi;
        const float denom = sqrtf(vi) / bc2_sqrt + eps;
        p[i] -= (lr / bc1) * (mi / denom);
    }
}

// ================================================================================================ v2: tiled field kernels
// Round 2.  The kernels above evaluate the MLP one point per thread: every FMA quartet costs a broadcast LDS.128 of weights plus the activation
// load, which makes them LSU-bound (forward 193 clk / point / SM, of which the 128 grid gathers are ~128), and the backward writes 1.4 KB / point
// of activation tapes to HBM for separate weight-gradient GEMMs.  v2 treats a TILE of 128 points as a small GEMM problem per layer:
//   * activations live feature-major in shared memory ([feature][point], row stride 132 floats) -- E (32), H1, H2 (64 rows) and, in the
//     backward, D2, D1, D0; a thread owns an 8-output x 8-point register tile (64 accumulators), so one k-step is 2 + 2 LDS.128 for 64 FMA
//     (the v1 loop: 17 shared-memory loads for 64 FMA);
//   * the backward accumulates dW / db of the tile IN REGISTERS across the CTA's whole grid-stride loop (per-thread 4x8 / 4x4 tiles of
//     dW1 / dW0, reduction over the points vectorised 4 wide) and reduces once per CTA -- no tape, no second pass over HBM;
//   * encode gathers and gradient scatters are issued two levels (16 requests) at a time per thread; index arithmetic is the shared one
//     (gridencoder.cuh), so rows stay bit-identical to the reference.
// Bound: LSU (128 gathers + 128 red.v2 per point), then FP32 FMA.
constexpr int kPT = 128;          // points per tile == threads per CTA
constexpr int kLd = 132;          // row stride of the activation tiles (floats): rows 4 banks apart -> conflict-free 128-bit row walks

// 2 levels x 8 corners of one point: rows and interpolation weights
struct Corner2 {
    uint32_t row[16];
    float w[16];
    uint32_t off[2];
};
__device__ __forceinline__ void locate_2levels(const float (&u)[3], uint32_t level0, const int32_t* __restrict__ offsets, const FieldGeom& g, Corner2& c) {
#pragma unroll
    for (uint32_t l = 0; l < 2; ++l) {
        const GridLevel lv = grid_level(level0 + l, g.S, g.H, offsets);
        c.off[l] = lv.offset;
        float frac[3];
        uint32_t cell[3];
        grid_locate<3>(u, lv.scale, false, frac, cell);
#pragma unroll
        for (uint32_t corner = 0; corner < 8; ++corner) {
            float w = 1.f;
            uint32_t cl[3];
#pragma unroll
            for (uint32_t d = 0; d < 3; ++d) {
                if ((corner & (1u << d)) == 0) { w *= 1 - frac[d]; cl[d] = cell[d]; }
                else { w *= frac[d]; cl[d] = cell[d] + 1; }
            }
            c.row[l * 8 + corner] = grid_row<3>(1u, false, lv.rows, lv.resolution, cl);
            c.w[l * 8 + corner] = w;
        }
    }
}

// encode one point into column `col` of E ([32][kLd]); the accumulation order per level equals encode_point's (corner 0..7)
__device__ __forceinline__ void encode_point_tile(const float (&x)[3], bool valid, const float* __restrict__ table, const int32_t* __restrict__ offsets,
                                                  const FieldGeom& g, float* __restrict__ E, int col) {
    float u[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) u[d] = __fdiv_rn(__fadd_rn(x[d], g.bound), 2 * g.bound);  // grid.py:142
    const bool live = valid && !grid_out_of_range<3>(u);
#pragma unroll 1
    for (uint32_t level = 0; level < kL; level += 2) {
        float a[4] = {0.f, 0.f, 0.f, 0.f};
        if (live) {
            Corner2 c;
            locate_2levels(u, level, offsets, g, c);
            float2 v[16];
#pragma unroll
            for (int m = 0; m < 8; ++m) {
                // corners 2m / 2m+1 differ in x only: their rows are neighbours unless the level's index wraps between them; an even first row makes
                // the pair one aligned 16-byte element (level offsets are multiples of 8 rows) -> one request instead of two for ~half of the pairs
                const int i0 = 2 * m, i1 = i0 + 1;
                const float* base = table + (size_t)c.off[m >> 2] * kC;
                if (c.row[i1] == c.row[i0] + 1u && (c.row[i0] & 1u) == 0u) {
                    const float4 t = __ldg(reinterpret_cast<const float4*>(base) + (c.row[i0] >> 1));
                    v[i0] = make_float2(t.x, t.y);
                    v[i1] = make_float2(t.z, t.w);
                } else {
                    v[i0] = __ldg(reinterpret_cast<const float2*>(base) + c.row[i0]);
                    v[i1] = __ldg(reinterpret_cast<const float2*>(base) + c.row[i1]);
                }
            }
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                a[(i >> 3) * 2] += c.w[i] * v[i].x;
                a[(i >> 3) * 2 + 1] += c.w[i] * v[i].y;
            }
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) E[(2 * level + q) * kLd + col] = a[q];
    }
}

// Out[j][p] = epi(bias[j] + sum_k WT[k][j] * A[k][p]) for a 64-output x 128-point tile; WT is [K][64] (reduction index major), A and Out are
// [.][kLd].  128 threads: thread (tp = t & 15, tj = t >> 4) owns outputs 8 tj .. 8 tj + 7 of points {4 tp .. 4 tp + 3} u {64 + 4 tp .. 64 + 4 tp + 3}.
// EPI: 0 = ReLU, 1 = multiply by (G[j][p] > 0) (ReLU backward through the activation G)
template <int K, int EPI>
__device__ __forceinline__ void dense_tile64(const float* __restrict__ WT, const float* __restrict__ bias, const float* __restrict__ A,
                                             float* __restrict__ Out, const float* __restrict__ G) {
    const int tp = threadIdx.x & 15, tj = threadIdx.x >> 4;
    float acc[8][8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const float b = bias ? bias[tj * 8 + j] : 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[j][i] = b;
    }
#pragma unroll 2
    for (int k = 0; k < K; ++k) {
        const float4 a0 = *reinterpret_cast<const float4*>(A + k * kLd + tp * 4);
        const float4 a1 = *reinterpret_cast<const float4*>(A + k * kLd + 64 + tp * 4);
        const float4 w0 = *reinterpret_cast<const float4*>(WT + k * kHid + tj * 8);
        const float4 w1 = *reinterpret_cast<const float4*>(WT + k * kHid + tj * 8 + 4);
        const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        const float w[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[j][i] += w[j] * a[i];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int row = (tj * 8 + j) * kLd;
        float o[8];
        if (EPI == 0) {
#pragma unroll
            for (int i = 0; i < 8; ++i) o[i] = fmaxf(acc[j][i], 0.f);
        } else {
            const float4 g0 = *reinterpret_cast<const float4*>(G + row + tp * 4);
            const float4 g1 = *reinterpret_cast<const float4*>(G + row + 64 + tp * 4);
            const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i) o[i] = gg[i] > 0.f ? acc[j][i] : 0.f;
        }
        *reinterpret_cast<float4*>(Out + row + tp * 4) = make_float4(o[0], o[1], o[2], o[3]);
        *reinterpret_cast<float4*>(Out + row + 64 + tp * 4) = make_float4(o[4], o[5], o[6], o[7]);
    }
}

// D0[k][p] = sum_j W0[j][k] * D1[j][p]: 32 outputs x 128 points, reduction over 64; W0 row-major [64][32].  Thread (tp = t & 15, tk = t >> 4) owns
// outputs 4 tk .. 4 tk + 3 of the same 8 points as above.
__device__ __forceinline__ void dense_tile32(const float* __restrict__ W0, const float* __restrict__ A, float* __restrict__ Out) {
    const int tp = threadIdx.x & 15, tk = threadIdx.x >> 4;
    float acc[4][8];
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[j][i] = 0.f;
#pragma unroll 2
    for (int k = 0; k < kHid; ++k) {
        const float4 a0 = *reinterpret_cast<const float4*>(A + k * kLd + tp * 4);
        const float4 a1 = *reinterpret_cast<const float4*>(A + k * kLd + 64 + tp * 4);
        const float4 w0 = *reinterpret_cast<const float4*>(W0 + k * kIn + tk * 4);
        const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        const float w[4] = {w0.x, w0.y, w0.z, w0.w};
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[j][i] += w[j] * a[i];
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int row = (tk * 4 + j) * kLd;
        *reinterpret_cast<float4*>(Out + row + tp * 4) = make_float4(acc[j][0], acc[j][1], acc[j][2], acc[j][3]);
        *reinterpret_cast<float4*>(Out + row + 64 + tp * 4) = make_float4(acc[j][4], acc[j][5], acc[j][6], acc[j][7]);
    }
}

// acc[jr][r] += sum_p D[j0 + jr][p] * H[tk + 8 r][p] over the tile's 128 points (4 at a time): the thread's share of dW = D H^T.
// Thread (tk = t & 7, tj = t >> 3): rows j0 = 4 tj of D, rows {tk, tk + 8, ...} (NR of them) of H -- a quarter-warp walks 8 consecutive H rows
// (conflict-free with the 132-float stride) and shares its D rows (broadcast).
template <int NR>
__device__ __forceinline__ void wgrad_tile(const float* __restrict__ D, const float* __restrict__ H, float (&acc)[4][NR]) {
    const int tk = threadIdx.x & 7, tj = threadIdx.x >> 3;
#pragma unroll 2
    for (int p = 0; p < kPT; p += 4) {
        float4 d[4], h[NR];
#pragma unroll
        for (int jr = 0; jr < 4; ++jr) d[jr] = *reinterpret_cast<const float4*>(D + (tj * 4 + jr) * kLd + p);
#pragma unroll
        for (int r = 0; r < NR; ++r) h[r] = *reinterpret_cast<const float4*>(H + (tk + 8 * r) * kLd + p);
#pragma unroll
        for (int jr = 0; jr < 4; ++jr)
#pragma unroll
            for (int r = 0; r < NR; ++r) {      // four chained FFMAs (a pairwise tree costs 2 FMUL + 2 FFMA + 2 FADD: a third more issue slots)
                float t = acc[jr][r];
                t = fmaf(d[jr].x, h[r].x, t);
                t = fmaf(d[jr].y, h[r].y, t);
                t = fmaf(d[jr].z, h[r].z, t);
                acc[jr][r] = fmaf(d[jr].w, h[r].w, t);
            }
    }
}

struct FieldSmemV2 {
    float WT0[kIn * kHid];    // [k][j]  forward layer 0
    float WT1[kHid * kHid];   // [k][j]  forward layer 1
    float WT2[kHid * kOut];   // [k][c]  forward layer 2 and D2 = W2^T d3
    float b0[kHid], b1[kHid], b2[kOut];
};
struct FieldSmemV2Bwd {
    FieldSmemV2 f;
    float W1[kHid * kHid];    // [j][k] row-major (as stored): D1 = W1^T D2
    float W0[kHid * kIn];     // [j][k] row-major: D0 = W0^T D1
    float d3[kOut * kLd];     // output-layer gradients of the tile, feature-major
};

__device__ __forceinline__ void load_weights_v2(FieldSmemV2& s, const float* W0, const float* b0, const float* W1, const float* b1, const float* W2,
                                                const float* b2) {
    for (int i = threadIdx.x; i < kHid * kIn; i += blockDim.x) { const int j = i / kIn, k = i - j * kIn; s.WT0[k * kHid + j] = W0[i]; }
    for (int i = threadIdx.x; i < kHid * kHid; i += blockDim.x) { const int j = i / kHid, k = i - j * kHid; s.WT1[k * kHid + j] = W1[i]; }
    for (int i = threadIdx.x; i < kOut * kHid; i += blockDim.x) { const int j = i / kHid, k = i - j * kHid; s.WT2[k * kOut + j] = W2[i]; }
    for (int i = threadIdx.x; i < kHid; i += blockDim.x) { s.b0[i] = b0[i]; s.b1[i] = b1[i]; }
    if (threadIdx.x < kOut) s.b2[threadIdx.x] = b2[threadIdx.x];
}

__global__ void __launch_bounds__(kPT) field_forward_v2_kernel(PointSource ps, uint32_t B, const float* __restrict__ table, const int32_t* __restrict__ offsets,
                                                              FieldGeom g, const float* __restrict__ W0, const float* __restrict__ b0,
                                                              const float* __restrict__ W1, const float* __restrict__ b1, const float* __restrict__ W2,
                                                              const float* __restrict__ b2, float* __restrict__ sigma, float* __restrict__ rgb) {
    extern __shared__ __align__(16) uint8_t smraw[];
    FieldSmemV2& s = *reinterpret_cast<FieldSmemV2*>(smraw);
    float* bufA = reinterpret_cast<float*>(smraw + sizeof(FieldSmemV2));      // E (rows 0..31), then H2
    float* bufB = bufA + kHid * kLd;                                         // H1
    load_weights_v2(s, W0, b0, W1, b1, W2, b2);
    __syncthreads();
    const int tid = threadIdx.x;
    const uint32_t tiles = (B + kPT - 1) / kPT;
    for (uint32_t tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const uint32_t p = tile * kPT + tid;
        const bool valid = p < B;
        float x[3] = {0.f, 0.f, 0.f};
        if (valid) fetch_point(ps, p, x);
        encode_point_tile(x, valid, table, offsets, g, bufA, tid);
        __syncthreads();
        dense_tile64<kIn, 0>(s.WT0, s.b0, bufA, bufB, nullptr);
        __syncthreads();
        dense_tile64<kHid, 0>(s.WT1, s.b1, bufB, bufA, nullptr);
        __syncthreads();
        if (valid) {
            float o0 = s.b2[0], o1 = s.b2[1], o2 = s.b2[2], o3 = s.b2[3];
#pragma unroll 8
            for (int k = 0; k < kHid; ++k) {
                const float hk = bufA[k * kLd + tid];
                const float4 w = *reinterpret_cast<const float4*>(s.WT2 + k * kOut);
                o0 += w.x * hk; o1 += w.y * hk; o2 += w.z * hk; o3 += w.w * hk;
            }
            sigma[p] = expf(o0 + density_blob(x));
            if (rgb) {
                rgb[(size_t)p * 3] = 1.f / (1.f + expf(-o1));
                rgb[(size_t)p * 3 + 1] = 1.f / (1.f + expf(-o2));
                rgb[(size_t)p * 3 + 2] = 1.f / (1.f + expf(-o3));
            }
        }
        __syncthreads();     // bufA is overwritten by the next tile's encode
    }
}

// ---- backward: 64-point tiles, 128 threads (two per point), three activation buffers -> 94 KB of shared memory, TWO CTAs per SM, so that one
// CTA's gather / scatter phases (latency bound) overlap the other's FFMA phases.  (Round-2 history: 128-point tiles with one CTA per SM ran every
// phase of the tile back to back on 4 or 8 warps: 4.57 / 4.36 ms for the 2.1 M points of a render.)
constexpr int kPB = 64;           // points per backward tile
constexpr int kLdB = kPB + 4;     // feature-major row stride (floats): 16-byte aligned rows, conflict-free float4 column reads
constexpr int kBT = 128;          // threads of the backward CTA

// Out[j][p] = epi(sum_k WT[k][j] * A[k][p]): thread (tp = t & 7, tj = t >> 3) owns outputs 4 tj .. 4 tj + 3 of points {4 tp ..} u {32 + 4 tp ..}.
// EPI 0: + bias, ReLU.  EPI 1: masked by the sign of what Out held before (the forward activation it overwrites) -- in place.
template <int K, int EPI>
__device__ __forceinline__ void dense64_p64(const float* __restrict__ WT, const float* __restrict__ bias, const float* __restrict__ A, float* Out) {
    const int tp = threadIdx.x & 7, tj = threadIdx.x >> 3;
    float acc[4][8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float b = EPI == 0 ? bias[tj * 4 + j] : 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[j][i] = b;
    }
#pragma unroll 8
    for (int k = 0; k < K; ++k) {
        const float4 a0 = *reinterpret_cast<const float4*>(A + k * kLdB + tp * 4);
        const float4 a1 = *reinterpret_cast<const float4*>(A + k * kLdB + 32 + tp * 4);
        const float4 w0 = *reinterpret_cast<const float4*>(WT + k * kHid + tj * 4);
        const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        const float w[4] = {w0.x, w0.y, w0.z, w0.w};
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[j][i] += w[j] * a[i];
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        float* row = Out + (tj * 4 + j) * kLdB;
        float o[8];
        if (EPI == 0) {
#pragma unroll
            for (int i = 0; i < 8; ++i) o[i] = fmaxf(acc[j][i], 0.f);
        } else {
            const float4 g0 = *reinterpret_cast<const float4*>(row + tp * 4);
            const float4 g1 = *reinterpret_cast<const float4*>(row + 32 + tp * 4);
            const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i) o[i] = gg[i] > 0.f ? acc[j][i] : 0.f;
        }
        *reinterpret_cast<float4*>(row + tp * 4) = make_float4(o[0], o[1], o[2], o[3]);
        *reinterpret_cast<float4*>(row + 32 + tp * 4) = make_float4(o[4], o[5], o[6], o[7]);
    }
}

// D0[k][p] = sum_j W0[j][k] * D1[j][p] (32 x 64, reduction 64): thread (tp = t & 7, tk = t >> 3) owns outputs 2 tk, 2 tk + 1
__device__ __forceinline__ void dense32_p64(const float* __restrict__ W0, const float* __restrict__ A, float* __restrict__ Out) {
    const int tp = threadIdx.x & 7, tk = threadIdx.x >> 3;
    float acc[2][8];
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[j][i] = 0.f;
#pragma unroll 8
    for (int k = 0; k < kHid; ++k) {
        const float4 a0 = *reinterpret_cast<const float4*>(A + k * kLdB + tp * 4);
        const float4 a1 = *reinterpret_cast<const float4*>(A + k * kLdB + 32 + tp * 4);
        const float2 w0 = *reinterpret_cast<const float2*>(W0 + k * kIn + tk * 2);
        const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
#pragma unroll
        for (int i = 0; i < 8; ++i) { acc[0][i] += w0.x * a[i]; acc[1][i] += w0.y * a[i]; }
    }
#pragma unroll
    for (int j = 0; j < 2; ++j) {
        float* row = Out + (tk * 2 + j) * kLdB;
        *reinterpret_cast<float4*>(row + tp * 4) = make_float4(acc[j][0], acc[j][1], acc[j][2], acc[j][3]);
        *reinterpret_cast<float4*>(row + 32 + tp * 4) = make_float4(acc[j][4], acc[j][5], acc[j][6], acc[j][7]);
    }
}

// acc[jr][r] += sum_p D[4 tj + jr][p] * H[tk + 8 r][p]: thread (tk = t & 7, tj = t >> 3 in 0..15)
template <int NR>
__device__ __forceinline__ void wgrad_p64(const float* __restrict__ D, const float* __restrict__ H, float (&acc)[4][NR]) {
    const int tk = threadIdx.x & 7, tj = threadIdx.x >> 3;
#pragma unroll 2
    for (int p = 0; p < kPB; p += 4) {
        float4 d[4], h[NR];
#pragma unroll
        for (int jr = 0; jr < 4; ++jr) d[jr] = *reinterpret_cast<const float4*>(D + (tj * 4 + jr) * kLdB + p);
#pragma unroll
        for (int r = 0; r < NR; ++r) h[r] = *reinterpret_cast<const float4*>(H + (tk + 8 * r) * kLdB + p);
#pragma unroll
        for (int jr = 0; jr < 4; ++jr)
#pragma unroll
            for (int r = 0; r < NR; ++r) {      // four chained FFMAs (a pairwise tree costs 2 FMUL + 2 FFMA + 2 FADD: a third more issue slots)
                float t = acc[jr][r];
                t = fmaf(d[jr].x, h[r].x, t);
                t = fmaf(d[jr].y, h[r].y, t);
                t = fmaf(d[jr].z, h[r].z, t);
                acc[jr][r] = fmaf(d[jr].w, h[r].w, t);
            }
    }
}

// sum of one 64-float row
__device__ __forceinline__ float row_sum_p64(const float* __restrict__ row) {
    float t = 0.f;
#pragma unroll 4
    for (int q = 0; q < kPB; q += 4) {
        const float4 v = *reinterpret_cast<const float4*>(row + q);
        t += (v.x + v.y) + (v.z + v.w);
    }
    return t;
}

// encode levels [l0, l0 + nl) of one point into column `col` of E (row stride kLdB)
__device__ __forceinline__ void encode_levels_p64(const float (&x)[3], bool valid, const float* __restrict__ table, const int32_t* __restrict__ offsets,
                                                  const FieldGeom& g, float* __restrict__ E, int col, uint32_t l0, uint32_t nl) {
    float u[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) u[d] = __fdiv_rn(__fadd_rn(x[d], g.bound), 2 * g.bound);
    const bool live = valid && !grid_out_of_range<3>(u);
#pragma unroll 1
    for (uint32_t level = l0; level < l0 + nl; level += 2) {
        float a[4] = {0.f, 0.f, 0.f, 0.f};
        if (live) {
            Corner2 c;
            locate_2levels(u, level, offsets, g, c);
            float2 v[16];
#pragma unroll
            for (int m = 0; m < 8; ++m) {
                const int i0 = 2 * m, i1 = i0 + 1;
                const float* base = table + (size_t)c.off[m >> 2] * kC;
                if (c.row[i1] == c.row[i0] + 1u && (c.row[i0] & 1u) == 0u) {
                    const float4 t = __ldg(reinterpret_cast<const float4*>(base) + (c.row[i0] >> 1));
                    v[i0] = make_float2(t.x, t.y);
                    v[i1] = make_float2(t.z, t.w);
                } else {
                    v[i0] = __ldg(reinterpret_cast<const float2*>(base) + c.row[i0]);
                    v[i1] = __ldg(reinterpret_cast<const float2*>(base) + c.row[i1]);
                }
            }
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                a[(i >> 3) * 2] += c.w[i] * v[i].x;
                a[(i >> 3) * 2 + 1] += c.w[i] * v[i].y;
            }
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) E[(2 * level + q) * kLdB + col] = a[q];
    }
}

// The rows the tiled backward walks.  PointRows: one row per field point, upstream gradients dL/dsigma [B] and dL/drgb [B,3] (or NULL).
// (StencilRows, below with the normal kernels, generates the six finite-difference rows of each point instead.)
struct PointRows {
    PointSource ps;
    uint32_t B;
    const float* g_sigma;
    const float* g_rgb;
    __device__ __forceinline__ uint32_t tiles() const { return (B + kPB - 1) / kPB; }
    // row `pt` of backward tile `tile`: its point x and row index r; false for padding rows
    __device__ __forceinline__ bool fetch(uint32_t tile, int pt, float (&x)[3], uint32_t& r) const {
        r = tile * kPB + pt;
        if (r >= B) return false;
        fetch_point(ps, r, x);
        return true;
    }
    __device__ __forceinline__ float grad_sigma(uint32_t r) const { return g_sigma[r]; }
    __device__ __forceinline__ bool has_rgb() const { return g_rgb != nullptr; }
    __device__ __forceinline__ float grad_rgb(uint32_t r, int c) const { return g_rgb[(size_t)r * 3 + c]; }
};

template <class Rows>
__global__ void __launch_bounds__(kBT, 2) field_backward_v2_kernel(Rows rows, const float* __restrict__ table, const int32_t* __restrict__ offsets,
                                                                  FieldGeom g, const float* __restrict__ W0, const float* __restrict__ b0,
                                                                  const float* __restrict__ W1, const float* __restrict__ b1, const float* __restrict__ W2,
                                                                  const float* __restrict__ b2, float* __restrict__ grad_table, float* __restrict__ gW0,
                                                                  float* __restrict__ gb0, float* __restrict__ gW1, float* __restrict__ gb1,
                                                                  float* __restrict__ gW2, float* __restrict__ gb2) {
    extern __shared__ __align__(16) uint8_t smraw[];
    FieldSmemV2Bwd& s = *reinterpret_cast<FieldSmemV2Bwd*>(smraw);
    float* bufA = reinterpret_cast<float*>(smraw + sizeof(FieldSmemV2Bwd));   // E (32 rows)
    float* bufB = bufA + kIn * kLdB;                                          // H1, then D1 in place
    float* bufC = bufB + kHid * kLdB;                                         // H2, then D2 in place, then D0 (rows 0..31)
    load_weights_v2(s.f, W0, b0, W1, b1, W2, b2);
    for (int i = threadIdx.x; i < kHid * kHid; i += blockDim.x) s.W1[i] = W1[i];
    for (int i = threadIdx.x; i < kHid * kIn; i += blockDim.x) s.W0[i] = W0[i];
    __syncthreads();
    const int tid = threadIdx.x;
    const int pt = tid & (kPB - 1), half = tid >> 6;       // two threads per point: levels [8 half, 8 half + 8), hidden units [32 half, 32 half + 32)
    // per-thread shares of the weight gradients, kept in registers over all tiles of this CTA
    float aW1[4][8], aW0[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a) {
#pragma unroll
        for (int r = 0; r < 8; ++r) aW1[a][r] = 0.f;
#pragma unroll
        for (int r = 0; r < 4; ++r) aW0[a][r] = 0.f;
    }
    float aW2[2] = {0.f, 0.f};      // dW2[c][k]: k = tid & 63, c = (tid >> 6) + 2 i
    float ab1 = 0.f;                // tid < 64: db1[tid]; tid >= 64: db0[tid - 64]
    float ab2 = 0.f;                // tid < 4: db2[tid]
    const uint32_t tiles = rows.tiles();
    for (uint32_t tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        uint32_t p;
        float x[3] = {0.f, 0.f, 0.f};
        const bool valid = rows.fetch(tile, pt, x, p);
        // ---- forward recompute: E -> H1 -> H2
        encode_levels_p64(x, valid, table, offsets, g, bufA, pt, half * 8, 8);
        __syncthreads();
        dense64_p64<kIn, 0>(s.f.WT0, s.f.b0, bufA, bufB);
        __syncthreads();
        dense64_p64<kHid, 0>(s.f.WT1, s.f.b1, bufB, bufC);
        __syncthreads();
        // ---- output layer and its gradient d3 (one thread per point)
        if (half == 0) {
            float d3[4] = {0.f, 0.f, 0.f, 0.f};
            if (valid) {
                float o[4] = {s.f.b2[0], s.f.b2[1], s.f.b2[2], s.f.b2[3]};
#pragma unroll 8
                for (int k = 0; k < kHid; ++k) {
                    const float hk = bufC[k * kLdB + pt];
                    const float4 w = *reinterpret_cast<const float4*>(s.f.WT2 + k * kOut);
                    o[0] += w.x * hk; o[1] += w.y * hk; o[2] += w.z * hk; o[3] += w.w * hk;
                }
                const float pre = o[0] + density_blob(x);
                d3[0] = rows.grad_sigma(p) * expf(fminf(fmaxf(pre, -15.f), 15.f));       // trunc_exp backward (ngp_activation.py:19-21)
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    const float sg = 1.f / (1.f + expf(-o[c + 1]));
                    d3[c + 1] = rows.has_rgb() ? rows.grad_rgb(p, c) * sg * (1.f - sg) : 0.f;
                }
            }
#pragma unroll
            for (int c = 0; c < 4; ++c) s.d3[c * kLdB + pt] = d3[c];
        }
        __syncthreads();
        // ---- dW2 += d3 H2^T, db2
        {
            const int k = tid & 63, c = tid >> 6;
            float s0 = 0.f, s1 = 0.f;
#pragma unroll 4
            for (int q = 0; q < kPB; q += 4) {
                const float4 h = *reinterpret_cast<const float4*>(bufC + k * kLdB + q);
                const float4 da = *reinterpret_cast<const float4*>(s.d3 + c * kLdB + q);
                const float4 db = *reinterpret_cast<const float4*>(s.d3 + (c + 2) * kLdB + q);
                s0 = fmaf(da.w, h.w, fmaf(da.z, h.z, fmaf(da.y, h.y, fmaf(da.x, h.x, s0))));
                s1 = fmaf(db.w, h.w, fmaf(db.z, h.z, fmaf(db.y, h.y, fmaf(db.x, h.x, s1))));
            }
            aW2[0] += s0;
            aW2[1] += s1;
            if (tid < 4) ab2 += row_sum_p64(s.d3 + tid * kLdB);
        }
        __syncthreads();     // every reader of H2 is done before D2 overwrites it
        // ---- D2 = relu'(H2) (W2^T d3), in place (two threads per point)
        {
            const float d0 = s.d3[pt], d1 = s.d3[kLdB + pt], d2 = s.d3[2 * kLdB + pt], d3v = s.d3[3 * kLdB + pt];
#pragma unroll 8
            for (int k = half * 32; k < half * 32 + 32; ++k) {
                const float4 w = *reinterpret_cast<const float4*>(s.f.WT2 + k * kOut);
                const float v = w.x * d0 + w.y * d1 + w.z * d2 + w.w * d3v;
                bufC[k * kLdB + pt] = bufC[k * kLdB + pt] > 0.f ? v : 0.f;
            }
        }
        __syncthreads();
        // ---- dW1 += D2 H1^T, db1
        wgrad_p64<8>(bufC, bufB, aW1);
        if (tid < 64) ab1 += row_sum_p64(bufC + tid * kLdB);
        __syncthreads();     // every reader of H1 is done before D1 overwrites it
        // ---- D1 = relu'(H1) (W1^T D2), in place over H1
        dense64_p64<kHid, 1>(s.W1, nullptr, bufC, bufB);
        __syncthreads();
        // ---- D0 = W0^T D1 -> bufC rows 0..31 (D2 is dead) ; dW0 += D1 E^T ; db0
        dense32_p64(s.W0, bufB, bufC);
        wgrad_p64<4>(bufB, bufA, aW0);
        if (tid >= 64) ab1 += row_sum_p64(bufB + (tid - 64) * kLdB);
        __syncthreads();
        // ---- scatter D0 into the embedding gradient (kernel_grid_backward, gridencoder.cu:226-313): two threads per point, two levels per batch
        if (valid) {
            float u[3];
#pragma unroll
            for (int d = 0; d < 3; ++d) u[d] = __fdiv_rn(__fadd_rn(x[d], g.bound), 2 * g.bound);
            if (!grid_out_of_range<3>(u)) {
#pragma unroll 1
                for (uint32_t level = half * 8; level < (uint32_t)half * 8 + 8; level += 2) {
                    Corner2 c;
                    locate_2levels(u, level, offsets, g, c);
                    float gq[4];
#pragma unroll
                    for (int q = 0; q < 4; ++q) gq[q] = bufC[(2 * level + q) * kLdB + pt];
#pragma unroll
                    for (int m = 0; m < 8; ++m) {
                        const int i0 = 2 * m, i1 = i0 + 1;
                        float* base = grad_table + (size_t)c.off[m >> 2] * kC;
                        const float g0 = gq[(m >> 2) * 2], g1 = gq[(m >> 2) * 2 + 1];
                        if (c.row[i1] == c.row[i0] + 1u && (c.row[i0] & 1u) == 0u) {      // neighbouring rows, 16-byte aligned: one vector reduction
                            float* q = base + (size_t)c.row[i0] * kC;
                            asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(q), "f"(c.w[i0] * g0), "f"(c.w[i0] * g1), "f"(c.w[i1] * g0),
                                         "f"(c.w[i1] * g1)
                                         : "memory");
                        } else {
                            const float wa[2] = {c.w[i0] * g0, c.w[i0] * g1}, wb[2] = {c.w[i1] * g0, c.w[i1] * g1};
                            grid_red_add_row<2>(base, c.row[i0], wa);
                            grid_red_add_row<2>(base, c.row[i1], wb);
                        }
                    }
                }
            }
        }
        __syncthreads();     // the buffers are rewritten by the next tile
    }
    // ---- one reduction per CTA
    {
        const int tk = tid & 7, tj = tid >> 3;
#pragma unroll
        for (int a = 0; a < 4; ++a) {
#pragma unroll
            for (int r = 0; r < 8; ++r) atomicAdd(gW1 + (size_t)(tj * 4 + a) * kHid + tk + 8 * r, aW1[a][r]);
#pragma unroll
            for (int r = 0; r < 4; ++r) atomicAdd(gW0 + (size_t)(tj * 4 + a) * kIn + tk + 8 * r, aW0[a][r]);
        }
        atomicAdd(gW2 + (size_t)(tid >> 6) * kHid + (tid & 63), aW2[0]);
        atomicAdd(gW2 + (size_t)((tid >> 6) + 2) * kHid + (tid & 63), aW2[1]);
        if (tid < 64) atomicAdd(gb1 + tid, ab1);
        else atomicAdd(gb0 + (tid - 64), ab1);
        if (tid < 4) atomicAdd(gb2 + tid, ab2);
    }
}

// ================================================================================================ finite-difference normals
// NeRFNetwork.finite_difference_normal / _smooth / common_forward_smooth / normal (external/nerf/network_grid.py:91-164) as stencils on
// the tiled field kernels.  The rows of a tile are (point, slot, sample): slot s in 0..5 shifts component s / 2 by +eps (even s) or -eps
// (odd s) and clamps to [-bound, bound] (:93-98, :139-144); sample j adds the jitter (u radius) 2 - radius with no clamp after it
// (:112-114).  The blob is evaluated at the un-jittered (shifted, clamped) point (:123).  Only output row 0 (and, for the centre-only
// stencil, rows 1..3) of the last layer is computed, and a segmented reduction in shared memory turns each point's rows into
// fd [B,3] = 0.5 (mean sigma+ - mean sigma-) / eps and normal = safe_normalize(fd) with NaN -> 0 (:155-164, utils.py:41-42).
//
// Jitter: Philox4x32-10 (Salmon et al., SC'11; the Random123 constants), counter (point, slot, sample, 0), key = the 64-bit value at
// `key` (low word first).  Lanes 0..2 give the three components' uniforms u = (r >> 8) 2^-24.
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
    for (int i = 0; i < 10; ++i) {
        const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
        const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
        c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
        k.x += 0x9E3779B9u;
        k.y += 0xBB67AE85u;
    }
    return c;
}

// x + eps e_{slot/2} (even slot) or x - eps e_{slot/2} (odd slot), clamped to [-bound, bound]; no register-indexed arrays
__device__ __forceinline__ void shift_clamp(float (&x)[3], uint32_t slot, float eps, float bound) {
    const float e = (slot & 1) ? -eps : eps;
#pragma unroll
    for (uint32_t d = 0; d < 3; ++d) {
        const float v = d == (slot >> 1) ? __fadd_rn(x[d], e) : x[d];
        x[d] = fminf(fmaxf(v, -bound), bound);
    }
}

struct StencilSpec {
    uint32_t slots;     // 6: the finite-difference stencil; 1: the centre only (common_forward_smooth)
    uint32_t k;         // jitter samples per slot (1 and no key: the plain stencil)
    uint32_t R;         // rows per point = slots * k (<= kPT)
    uint32_t ppt;       // points per 128-row tile = kPT / R
    float eps, radius, bound;
    const int64_t* key; // device-resident Philox key, or NULL: no jitter
};

// the stencil point of row (q, slot, sample): x is what the grid sees, xb where the blob is evaluated
__device__ __forceinline__ void stencil_point(const PointSource& ps, const StencilSpec& st, uint2 key, uint32_t q, uint32_t slot, uint32_t smp,
                                              float (&x)[3], float (&xb)[3]) {
    fetch_point(ps, q, x);
    if (st.slots == 6) shift_clamp(x, slot, st.eps, st.bound);
#pragma unroll
    for (int d = 0; d < 3; ++d) xb[d] = x[d];
    if (st.key) {
        const uint4 r = philox4x32_10(make_uint4(q, slot, smp, 0u), key);
        const uint32_t rr[3] = {r.x, r.y, r.z};
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            const float u = __uint2float_rn(rr[d] >> 8) * 0x1p-24f;
            x[d] = __fadd_rn(x[d], __fsub_rn(__fmul_rn(__fmul_rn(u, st.radius), 2.f), st.radius));    // x + (rand * radius * 2 - radius)
        }
    }
}

__device__ __forceinline__ uint2 load_key(const int64_t* key) {
    if (!key) return make_uint2(0u, 0u);
    const uint64_t k = (uint64_t)*key;
    return make_uint2((uint32_t)k, (uint32_t)(k >> 32));
}

// safe_normalize(fd) (utils.py:41-42: the clamp is on the squared norm) with NaN -> 0 (network_grid.py:161-162)
__device__ __forceinline__ void safe_normalize_nan0(const float (&fd)[3], float (&n)[3]) {
    const float r = sqrtf(fmaxf(fd[0] * fd[0] + fd[1] * fd[1] + fd[2] * fd[2], 1e-20f));
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float v = fd[a] / r;
        n[a] = isnan(v) ? 0.f : v;
    }
}

__global__ void __launch_bounds__(kPT) field_stencil_forward_kernel(PointSource ps, uint32_t B, StencilSpec st, const float* __restrict__ table,
                                                                   const int32_t* __restrict__ offsets, FieldGeom g, const float* __restrict__ W0,
                                                                   const float* __restrict__ b0, const float* __restrict__ W1, const float* __restrict__ b1,
                                                                   const float* __restrict__ W2, const float* __restrict__ b2, float* __restrict__ fd_out,
                                                                   float* __restrict__ normal_out, float* __restrict__ sigma_out,
                                                                   float* __restrict__ albedo_out) {
    extern __shared__ __align__(16) uint8_t smraw[];
    FieldSmemV2& s = *reinterpret_cast<FieldSmemV2*>(smraw);
    float* bufA = reinterpret_cast<float*>(smraw + sizeof(FieldSmemV2));      // E (rows 0..31), then H2
    float* bufB = bufA + kHid * kLd;                                         // H1, then the rows' sigma (row 0) and albedo (rows 1..3)
    load_weights_v2(s, W0, b0, W1, b1, W2, b2);
    const uint2 key = load_key(st.key);
    __syncthreads();
    const int tid = threadIdx.x;
    const bool centre = st.slots == 1;
    const uint32_t lp = tid / st.R, rr = tid - lp * st.R, slot = rr / st.k, smp = rr - slot * st.k;
    const uint32_t tiles = (B + st.ppt - 1) / st.ppt;
    for (uint32_t tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const uint32_t q = tile * st.ppt + lp;
        const bool valid = lp < st.ppt && q < B;
        float x[3] = {0.f, 0.f, 0.f}, xb[3] = {0.f, 0.f, 0.f};
        if (valid) stencil_point(ps, st, key, q, slot, smp, x, xb);
        encode_point_tile(x, valid, table, offsets, g, bufA, tid);
        __syncthreads();
        dense_tile64<kIn, 0>(s.WT0, s.b0, bufA, bufB, nullptr);
        __syncthreads();
        dense_tile64<kHid, 0>(s.WT1, s.b1, bufB, bufA, nullptr);
        __syncthreads();
        if (valid) {
            float o0 = s.b2[0], o1 = s.b2[1], o2 = s.b2[2], o3 = s.b2[3];
#pragma unroll 8
            for (int k = 0; k < kHid; ++k) {
                const float hk = bufA[k * kLd + tid];
                const float4 w = *reinterpret_cast<const float4*>(s.WT2 + k * kOut);
                o0 += w.x * hk;
                if (centre) { o1 += w.y * hk; o2 += w.z * hk; o3 += w.w * hk; }
            }
            bufB[tid] = expf(o0 + density_blob(xb));
            if (centre) {
                bufB[kLd + tid] = 1.f / (1.f + expf(-o1));
                bufB[2 * kLd + tid] = 1.f / (1.f + expf(-o2));
                bufB[3 * kLd + tid] = 1.f / (1.f + expf(-o3));
            }
        }
        __syncthreads();
        // segmented reduction: one thread per point over its R rows (slot-major, samples in order, then / k as torch's mean does)
        const uint32_t qo = tile * st.ppt + tid;
        if ((uint32_t)tid < st.ppt && qo < B) {
            const float* row = bufB + tid * st.R;
            const float kf = (float)st.k;
            if (centre) {
#pragma unroll 1
                for (int c = 0; c < 4; ++c) {
                    float t = 0.f;
                    for (uint32_t j = 0; j < st.k; ++j) t += row[c * kLd + j];
                    if (c == 0) sigma_out[qo] = t / kf;
                    else if (albedo_out) albedo_out[(size_t)qo * 3 + c - 1] = t / kf;
                }
            } else {
                float m[6];
#pragma unroll
                for (int sl = 0; sl < 6; ++sl) {
                    float t = 0.f;
                    for (uint32_t j = 0; j < st.k; ++j) t += row[sl * st.k + j];
                    m[sl] = t / kf;
                }
                float fd[3], n[3];
#pragma unroll
                for (int a = 0; a < 3; ++a) fd[a] = __fdiv_rn(__fmul_rn(0.5f, __fsub_rn(m[2 * a], m[2 * a + 1])), st.eps);   // 0.5 * (pos - neg) / eps
                safe_normalize_nan0(fd, n);
#pragma unroll
                for (int a = 0; a < 3; ++a) {
                    if (fd_out) fd_out[(size_t)qo * 3 + a] = fd[a];
                    if (normal_out) normal_out[(size_t)qo * 3 + a] = n[a];
                }
            }
        }
        __syncthreads();     // bufA / bufB are rewritten by the next tile
    }
}

// Backward rows of the plain stencil (no jitter): 10 points x 6 slots = 60 of a 64-row backward tile.  dL/dsigma of slot s of point q is
// +-0.5 g_fd / eps, with g_fd = grad_fd [B,3] directly, or the safe_normalize backward of grad_normal [B,3] at fd [B,3]: zero in the
// components whose normal was NaN (network_grid.py:162 writes 0 there), and zero for a point whose fd is not finite.
constexpr int kStencilPB = kPB / 6;
struct StencilRows {
    PointSource ps;
    uint32_t B;
    float eps, bound;
    const float* fd;
    const float* g_normal;
    const float* g_fd;
    __host__ __device__ __forceinline__ uint32_t tiles() const { return (B + kStencilPB - 1) / kStencilPB; }
    __device__ __forceinline__ bool fetch(uint32_t tile, int pt, float (&x)[3], uint32_t& r) const {
        const uint32_t q = tile * kStencilPB + pt / 6, slot = pt % 6;
        if (pt >= kStencilPB * 6 || q >= B) return false;
        r = q * 6 + slot;
        fetch_point(ps, q, x);
        shift_clamp(x, slot, eps, bound);
        return true;
    }
    __device__ __forceinline__ float grad_sigma(uint32_t r) const {
        const uint32_t q = r / 6, slot = r - q * 6, a = slot >> 1;
        float gfd;
        if (g_fd) {
            gfd = g_fd[(size_t)q * 3 + a];
        } else {
            const float f0 = fd[(size_t)q * 3], f1 = fd[(size_t)q * 3 + 1], f2 = fd[(size_t)q * 3 + 2];
            const float ss = f0 * f0 + f1 * f1 + f2 * f2;
            if (!isfinite(ss)) return 0.f;
            const float rn = sqrtf(fmaxf(ss, 1e-20f));
            // dL/dfd = (g - n (n . g)) / r over the components that were not NaN (none is, once ss is finite)
            const float g0 = g_normal[(size_t)q * 3], g1 = g_normal[(size_t)q * 3 + 1], g2 = g_normal[(size_t)q * 3 + 2];
            const float dot = g0 * f0 + g1 * f1 + g2 * f2;
            const float fa = a == 0 ? f0 : (a == 1 ? f1 : f2), ga = a == 0 ? g0 : (a == 1 ? g1 : g2);
            gfd = ga / rn;
            if (ss > 1e-20f) gfd -= fa * (dot / (rn * rn * rn));
        }
        const float gd = 0.5f * (gfd / eps);
        return (slot & 1) ? -gd : gd;
    }
    __device__ __forceinline__ bool has_rgb() const { return false; }
    __device__ __forceinline__ float grad_rgb(uint32_t, int) const { return 0.f; }
};

static int field_args_ok(const float* table, const int32_t* offsets, const float* W0, const float* b0, const float* W1, const float* b1,
                         const float* W2, const float* b2) {
    return table && offsets && W0 && b0 && W1 && b1 && W2 && b2;
}

static PointSource make_source(const float* xyz, const float* rays_o, const float* rays_d, const float* z, uint32_t T, float bound) {
    PointSource ps;
    ps.xyz = xyz; ps.rays_o = rays_o; ps.rays_d = rays_d; ps.z = z; ps.T = T ? T : 1;
    for (int d = 0; d < 3; ++d) { ps.aabb_lo[d] = -bound; ps.aabb_hi[d] = bound; }
    return ps;
}

}  // namespace sfb

using namespace sfb;

extern "C" {

int sfb_ngp_field_forward(const float* xyz, const float* rays_o, const float* rays_d, const float* z, uint32_t T, uint32_t B,
                          const float* embeddings, const int32_t* offsets, float S, uint32_t H, float bound, const float* W0, const float* b0,
                          const float* W1, const float* b1, const float* W2, const float* b2, float* sigma, float* rgb, void* stream) {
    if (B == 0) return SFB_OK;
    SFB_REQUIRE(field_args_ok(embeddings, offsets, W0, b0, W1, b1, W2, b2) && sigma, "ngp_field_forward: null pointer");
    SFB_REQUIRE(xyz || (rays_o && rays_d && z && T > 0), "ngp_field_forward: give xyz or (rays_o, rays_d, z, T)");
    if (B == 0) return SFB_OK;
    if (field_v2_enabled()) {
        const size_t smem2 = sizeof(FieldSmemV2) + (size_t)2 * kHid * kLd * 4;
        SFB_ONCE_PER_DEVICE(SFB_CUDA(cudaFuncSetAttribute(field_forward_v2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2)));
        const uint32_t tiles = ceil_div(B, (uint32_t)kPT);
        const uint32_t blocks2 = min(tiles, (uint32_t)sm_count() * 2);
        field_forward_v2_kernel<<<blocks2, kPT, smem2, as_stream(stream)>>>(make_source(xyz, rays_o, rays_d, z, T, bound), B, embeddings, offsets,
                                                                           FieldGeom{S, H, bound}, W0, b0, W1, b1, W2, b2, sigma, rgb);
        return check_launch("ngp_field_forward(v2)");
    }
    const size_t smem = sizeof(FieldSmem) + (size_t)kHid * kFieldThreads * 4;
    SFB_ONCE_PER_DEVICE(SFB_CUDA(cudaFuncSetAttribute(field_forward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)));
    const uint32_t blocks = min(ceil_div(B, (uint32_t)kFieldThreads), (uint32_t)sm_count() * 3);
    field_forward_kernel<<<blocks, kFieldThreads, smem, as_stream(stream)>>>(make_source(xyz, rays_o, rays_d, z, T, bound), B, embeddings, offsets,
                                                                            FieldGeom{S, H, bound}, W0, b0, W1, b1, W2, b2, sigma, rgb);
    return check_launch("ngp_field_forward");
}

uint32_t sfb_ngp_field_tape_points(uint32_t B) { return (B + 63) / 64 * 64; }

int sfb_ngp_field_backward(const float* xyz, const float* rays_o, const float* rays_d, const float* z, uint32_t T, uint32_t B,
                           const float* embeddings, const int32_t* offsets, float S, uint32_t H, float bound, const float* W0, const float* b0,
                           const float* W1, const float* b1, const float* W2, const float* b2, const float* grad_sigma, const float* grad_rgb,
                           float* grad_embeddings, float* gW0, float* gb0, float* gW1, float* gb1, float* gW2, float* gb2, float* tape,
                           void* stream) {
    if (B == 0) return SFB_OK;
    SFB_REQUIRE(field_args_ok(embeddings, offsets, W0, b0, W1, b1, W2, b2) && grad_sigma && grad_embeddings && gW0 && gb0 && gW1 && gb1 && gW2 &&
                    gb2 && (tape || field_v2_enabled()),
                "ngp_field_backward: null pointer");
    SFB_REQUIRE(xyz || (rays_o && rays_d && z && T > 0), "ngp_field_backward: give xyz or (rays_o, rays_d, z, T)");
    if (B == 0) return SFB_OK;
    if (field_v2_enabled()) {
        // tiled kernel: activations stay in shared memory, weight gradients accumulate in registers per CTA -- `tape` is not touched
        const size_t smem2 = sizeof(FieldSmemV2Bwd) + (size_t)(kIn + 2 * kHid) * kLdB * 4;
        SFB_ONCE_PER_DEVICE(SFB_CUDA(cudaFuncSetAttribute(field_backward_v2_kernel<PointRows>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2)));
        const uint32_t tiles = ceil_div(B, (uint32_t)kPB);
        const uint32_t blocks2 = min(tiles, (uint32_t)sm_count() * 2);
        const PointRows rows{make_source(xyz, rays_o, rays_d, z, T, bound), B, grad_sigma, grad_rgb};
        field_backward_v2_kernel<<<blocks2, kBT, smem2, as_stream(stream)>>>(rows, embeddings, offsets, FieldGeom{S, H, bound}, W0, b0, W1, b1, W2, b2,
                                                                            grad_embeddings, gW0, gb0, gW1, gb1, gW2, gb2);
        return check_launch("ngp_field_backward(v2)");
    }
    const uint32_t Bp = sfb_ngp_field_tape_points(B);
    float* H0 = tape;
    float* H1 = H0 + (size_t)kIn * Bp;
    float* H2 = H1 + (size_t)kHid * Bp;
    float* D1 = H2 + (size_t)kHid * Bp;
    float* D2 = D1 + (size_t)kHid * Bp;
    float* D3 = D2 + (size_t)kHid * Bp;
    const size_t smem = sizeof(FieldSmemBwd) + (size_t)2 * kHid * kFieldThreads * 4;
    SFB_ONCE_PER_DEVICE(SFB_CUDA(cudaFuncSetAttribute(field_backward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)));
    cudaStream_t st = as_stream(stream);
    const uint32_t blocks = min(ceil_div(Bp, (uint32_t)kFieldThreads), (uint32_t)sm_count() * 2);
    field_backward_kernel<<<blocks, kFieldThreads, smem, st>>>(make_source(xyz, rays_o, rays_d, z, T, bound), B, Bp, embeddings, offsets,
                                                              FieldGeom{S, H, bound}, W0, b0, W1, b1, W2, b2, grad_sigma, grad_rgb,
                                                              grad_embeddings, H0, H1, H2, D1, D2, D3);
    if (int rc = check_launch("ngp_field_backward(data)")) return rc;
    if (wgrad_tc_enabled()) {
        // dW = D . H^T with the point index as the GEMM's K dimension: the feature-major tapes are exactly the K-major operands the wgmma
        // implicit-GEMM kernel streams (rows of D = "pixels", rows of H = "output channels", 1x1 tap), 3xTF32, split-K over the 2.1 M points
        // with fp32 reductions into the gradient buffers (accumulate = 1).  Bias gradients are row sums of D.
        const int old = set_precision_override(1);
        int rc = sfb_conv2d_nhwc_tf32(D1, 1, 1, kHid, (int)Bp, (int64_t)Bp, H0, kIn, 1, 1, 1, 0, nullptr, nullptr, 0, gW0, kIn, 1, 0, 0, stream);
        if (!rc) rc = sfb_conv2d_nhwc_tf32(D2, 1, 1, kHid, (int)Bp, (int64_t)Bp, H1, kHid, 1, 1, 1, 0, nullptr, nullptr, 0, gW1, kHid, 1, 0, 0, stream);
        if (!rc) rc = sfb_conv2d_nhwc_tf32(D3, 1, 1, kOut, (int)Bp, (int64_t)Bp, H2, kHid, 1, 1, 1, 0, nullptr, nullptr, 0, gW2, kHid, 1, 0, 0, stream);
        set_precision_override(old);
        if (rc) return rc;
        // D1, D2, D3 are contiguous in the tape: one launch sums all 2*kHid + kOut rows
        const int rows = 2 * kHid + kOut;
        const uint32_t chunks = min(ceil_div(Bp, 4096u), 64u);
        tape_rowsum_kernel<<<dim3(chunks, rows), 256, 0, st>>>(D1, Bp, gb0, gb1, gb2);
        return check_launch("ngp_field_backward(bias)");
    }
    const uint32_t wb = min(Bp / 64, (uint32_t)sm_count() * 2);
    mlp_wgrad_kernel<kHid, kIn><<<wb, 256, 0, st>>>(D1, H0, Bp, gW0, gb0);
    mlp_wgrad_kernel<kHid, kHid><<<wb, 256, 0, st>>>(D2, H1, Bp, gW1, gb1);
    mlp_wgrad_kernel<kOut, kHid><<<wb, 256, 0, st>>>(D3, H2, Bp, gW2, gb2);
    count_launches(2);
    return check_launch("ngp_field_backward(weights)");
}

int sfb_ngp_field_normal_forward(const float* xyz, const float* rays_o, const float* rays_d, const float* z, uint32_t T, uint32_t B,
                                 const float* embeddings, const int32_t* offsets, float S, uint32_t H, float bound, const float* W0, const float* b0,
                                 const float* W1, const float* b1, const float* W2, const float* b2, uint32_t slots, uint32_t k, float eps,
                                 float radius, const int64_t* key, float* fd, float* normal, float* sigma, float* albedo, void* stream) {
    if (B == 0) return SFB_OK;
    SFB_REQUIRE(field_args_ok(embeddings, offsets, W0, b0, W1, b1, W2, b2), "ngp_field_normal_forward: null pointer");
    SFB_REQUIRE(xyz || (rays_o && rays_d && z && T > 0), "ngp_field_normal_forward: give xyz or (rays_o, rays_d, z, T)");
    SFB_REQUIRE((slots == 6 && (fd || normal) && eps != 0.f) || (slots == 1 && sigma), "ngp_field_normal_forward: slots must be 6 (fd / normal) or 1 (sigma)");
    SFB_REQUIRE(k >= 1 && slots * k <= (uint32_t)kPT && (k == 1 || key), "ngp_field_normal_forward: need 1 <= slots * k <= 128, and a key when k > 1");
    const StencilSpec st{slots, k, slots * k, kPT / (slots * k), eps, radius, bound, key};
    const size_t smem = sizeof(FieldSmemV2) + (size_t)2 * kHid * kLd * 4;
    SFB_ONCE_PER_DEVICE(SFB_CUDA(cudaFuncSetAttribute(field_stencil_forward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)));
    const uint32_t blocks = min(ceil_div(B, st.ppt), (uint32_t)sm_count() * 2);
    field_stencil_forward_kernel<<<blocks, kPT, smem, as_stream(stream)>>>(make_source(xyz, rays_o, rays_d, z, T, bound), B, st, embeddings, offsets,
                                                                          FieldGeom{S, H, bound}, W0, b0, W1, b1, W2, b2, fd, normal, sigma, albedo);
    return check_launch("ngp_field_normal_forward");
}

int sfb_ngp_field_normal_backward(const float* xyz, const float* rays_o, const float* rays_d, const float* z, uint32_t T, uint32_t B,
                                  const float* embeddings, const int32_t* offsets, float S, uint32_t H, float bound, const float* W0, const float* b0,
                                  const float* W1, const float* b1, const float* W2, const float* b2, float eps, const float* fd,
                                  const float* grad_normal, const float* grad_fd, float* grad_embeddings, float* gW0, float* gb0, float* gW1,
                                  float* gb1, float* gW2, float* gb2, void* stream) {
    if (B == 0) return SFB_OK;
    SFB_REQUIRE(field_args_ok(embeddings, offsets, W0, b0, W1, b1, W2, b2) && grad_embeddings && gW0 && gb0 && gW1 && gb1 && gW2 && gb2,
                "ngp_field_normal_backward: null pointer");
    SFB_REQUIRE(xyz || (rays_o && rays_d && z && T > 0), "ngp_field_normal_backward: give xyz or (rays_o, rays_d, z, T)");
    SFB_REQUIRE((grad_fd && !grad_normal) || (grad_normal && fd && !grad_fd), "ngp_field_normal_backward: give grad_fd, or grad_normal and fd");
    SFB_REQUIRE(eps != 0.f, "ngp_field_normal_backward: eps must not be 0");
    const size_t smem = sizeof(FieldSmemV2Bwd) + (size_t)(kIn + 2 * kHid) * kLdB * 4;
    SFB_ONCE_PER_DEVICE(SFB_CUDA(cudaFuncSetAttribute(field_backward_v2_kernel<StencilRows>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)));
    const StencilRows rows{make_source(xyz, rays_o, rays_d, z, T, bound), B, eps, bound, fd, grad_normal, grad_fd};
    const uint32_t blocks = min(rows.tiles(), (uint32_t)sm_count() * 2);
    field_backward_v2_kernel<<<blocks, kBT, smem, as_stream(stream)>>>(rows, embeddings, offsets, FieldGeom{S, H, bound}, W0, b0, W1, b1, W2, b2,
                                                                      grad_embeddings, gW0, gb0, gW1, gb1, gW2, gb2);
    return check_launch("ngp_field_normal_backward");
}

uint64_t sfb_ngp_field_tape_floats(uint32_t B) {
    if (field_v2_enabled()) return 0;      // the tiled backward keeps every activation in shared memory
    return (uint64_t)sfb_ngp_field_tape_points(B) * (kIn + 4 * kHid + kOut);
}

int sfb_adam_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n, float lr, float beta1, float beta2, float eps,
                  int step, float grad_scale, void* stream) {
    SFB_REQUIRE(param && grad && exp_avg && exp_avg_sq && step >= 1, "adam_step: null pointer or step < 1");
    if (n == 0) return SFB_OK;
    const float bc1 = 1.f - powf(beta1, (float)step);
    const float bc2_sqrt = sqrtf(1.f - powf(beta2, (float)step));
    int64_t blocks = (n + 255) / 256;
    if (blocks > (int64_t)sm_count() * 8) blocks = (int64_t)sm_count() * 8;
    adam_kernel<<<(unsigned)blocks, 256, 0, as_stream(stream)>>>(param, grad, exp_avg, exp_avg_sq, n, lr, beta1, beta2, eps, bc1, bc2_sqrt, grad_scale);
    return check_launch("adam_step");
}
}
