// conv_wgmma.cu -- NHWC convolution / linear layers of the VLDM UNet (and the VAE, LPIPS-VGG, EFT and NGP weight-gradient GEMMs)
// as implicit GEMM on the Hopper tensor cores: wgmma.mma_async with tf32 inputs and fp32 accumulators in registers, operands staged
// by TMA into 128B-swizzled shared memory.  Replaces the cuDNN/cuBLAS calls behind nn.Conv2d / nn.Linear in the reference's Unet
// (external/imagen_pytorch.py:641-662 Block.project, :708 res_conv, :608-610 Downsample, :578-606 PixelShuffleUpsample conv,
// :1017-1042 CrossEmbedLayer, :953-961 ChanFeedForward, :1386 final_conv), which the reference GPU build runs in TF32 (torch 1.11
// default, SURVEY.md §0.6).
//
// GEMM view:   D[pixel, cout] = sum_{tap, c} X[pixel shifted by tap, c] * W[cout, tap, c]
//   No im2col buffer exists: for every filter tap the producer issues one 4-D TMA box load {32 ch, TW, TH, TN} from the NHWC tensor at
//   the tap's spatial offset; out-of-bounds rows/columns/channels are zero-filled by the TMA unit, which implements the convolution
//   padding and the K tail.  Stride-2 convolutions read four parity-plane views (separate tensor maps over the same buffer).
//   Weights are pre-packed as [Cout][tap][Cin rounded up to 32] (K-major), so both operands are K-major, as tf32 wgmma requires.
//   M side = 128 rows per CTA (two consumer warpgroups of 64), read from shared memory into registers (the wgmma A operand);
//   N side = BN rows, read by the tensor core through a shared-memory descriptor.
//   Normal mode: M = 128 output pixels, N = BN output channels.  SWAP mode (<= 64 output pixels per launch: the 4x4 / 8x8 stages at
//   batch 1, which hold most of the UNet's weights): M = 128 output channels, N = the 16/32/64 pixels, so the tensor core does no work
//   on padding rows and a stage is 20-24 KB: eight stages of weights in flight per SM keep the weight stream at HBM bandwidth.
// 3xTF32 (NP = 3): every operand x is split into hi = x with the 13 low mantissa bits cleared and lo = x - hi; D accumulates
//   hi*hi + lo*hi + hi*lo, which restores fp32-class accuracy (rel. error ~2^-21 per product).  The M-side split happens in registers
//   on the way to the A fragments; the N-side tile is split in shared memory by the producer warpgroup (hi in place, lo to a second
//   buffer), unless the weights arrive pre-split (sfb_conv2d_nhwc_tf32_ex).  NP = 1: single-pass TF32 on the raw words.
// Warp roles (384 threads): warps 0-7 = two consumer warpgroups (A fragments, wgmma, epilogue), warp 8 = TMA producer, warps 9-11 =
// N-side hi/lo splitter.  The producer warpgroup gives its registers to the consumers (setmaxnreg).
// Epilogue: bias, optional residual, fp32 stores -- or red.global.add when the K range is split across CTAs / the output accumulates
// several convolutions.  The swap-mode accumulator is transposed through the idle stages so that global traffic runs along channels.
// Programmatic dependent launch: the first ring of weight tiles streams in before griddepcontrol.wait, the activations after it.
#include "common.cuh"
#include "wgmma.cuh"
#include "../../include/sparsefusion_b200.h"
#include <mutex>
#include <unordered_map>
#include <vector>
#include <string.h>

namespace sfb {

constexpr int kBM = 128;            // M-side rows per CTA
constexpr int kBK = 32;             // fp32 elements per k-step: one 128-byte swizzle row
constexpr int kABytes = kBM * 128;  // M-side tile of one stage: 16 KB
constexpr int kConsumers = 256;     // two consumer warpgroups
constexpr int kThreads = 384;       // + the producer warpgroup
constexpr int kSplitters = 96;      // warps 9-11

struct alignas(64) ConvGemmParams {
    CUtensorMap tmA[4];     // activations (4 parity planes for stride 2)
    CUtensorMap tmB;        // weights (hi when presplit)
    CUtensorMap tmBlo;      // pre-split weights (normal mode only): tmB = hi = w & 0xFFFFE000, tmBlo = lo = w - hi
    float* out;
    const float* bias;
    const float* residual;  // optional [pixel][ldr] tensor added to the result (by split 0)
    int64_t ldo;            // floats between consecutive output pixels
    int64_t ldr;
    int32_t NB, Ho, Wo;
    int32_t TW, TH, TN;
    int32_t tiles_w, tiles_h;
    int32_t Cout, cin_chunks;
    int32_t KH, KW, pad, stride;
    int32_t k_iters, splits;
    int32_t accumulate;
    int32_t presplit;       // tmB / tmBlo hold (hi, lo) of the weights: the N-side tile needs no split
    int32_t w_dynamic;      // the "weight" operand was produced by an earlier kernel of this stream (attention GEMMs): no prefetch before griddepcontrol.wait
    int32_t raw_hi;         // variant 3: feed the un-masked fp32 word as the "hi" tensor-core operand (is the hardware's tf32 read a truncation?)
};

template <int BN, int NP>
struct ConvCfg {
    static constexpr int kNBytes = BN * 128;                                   // N-side tile (raw == hi after the split)
    static constexpr int kStageBytes = kABytes + kNBytes * (NP == 3 ? 2 : 1);  // M raw | N hi | (NP == 3) N lo
    static constexpr int kStagesFit = (200 * 1024) / kStageBytes;
    static constexpr int kStages = kStagesFit < 8 ? kStagesFit : 8;
    static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align*/ + 512 /*barriers*/ + 1024 /*bias*/ + 256 /*pixel index*/;
};

// Phase tracer (sfb_conv_phase_trace): CTA (0,0,0) of every launch stamps %globaltimer at 7 points into buf[1 + 8*launch + phase]:
//   0 kernel entry, 1 prologue done (barriers, bias), 2 griddepcontrol.wait returned, 3 first stage ready (MMA can start),
//   4 last MMA complete (warpgroup 0), 5 epilogue starts, 6 epilogue done.
static __device__ unsigned long long* t_phase_buf = nullptr;
static __device__ unsigned int t_phase_cap = 0;
__device__ __forceinline__ void phase_mark(unsigned int slot, int phase) {
    if (slot != 0xffffffffu) {
        unsigned long long t;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        t_phase_buf[1 + (size_t)slot * 8 + phase] = t;
    }
}

// SWAP == false: M side = 128 output pixels (tmA), N side = BN output channels (tmB).
// SWAP == true : M side = 128 output channels (tmB), N side = BN output pixels (tmA, box {32, TW, TH, TN} with TW*TH*TN == BN).
template <int BN, bool SWAP, int NP>
__global__ void __launch_bounds__(kThreads, 1) conv_gemm_kernel(const __grid_constant__ ConvGemmParams p) {
    using Cfg = ConvCfg<BN, NP>;
    constexpr int S = Cfg::kStages;
    extern __shared__ uint8_t smem_raw[];
    // 1024-byte alignment by OFFSET from the __shared__ symbol, so the compiler keeps the shared address space (LDS/STS, not generic LD/ST)
    uint8_t* smem = smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* tail = smem + S * Cfg::kStageBytes;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(tail);    // TMA bytes of the stage landed
    uint64_t* split_bar = full_bar + S;                        // N-side tile split into hi / lo
    uint64_t* empty_bar = split_bar + S;                       // every consumer warp is done with the stage
    uint32_t* phase_slot = reinterpret_cast<uint32_t*>(empty_bar + S);
    float* bias_s = reinterpret_cast<float*>(tail + 512);      // up to 256 floats
    int* pix_s = reinterpret_cast<int*>(tail + 512 + 1024);    // SWAP: linear output pixel of tile column j, or -1

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tile = blockIdx.x;
    const int tw_i = tile % p.tiles_w, th_i = (tile / p.tiles_w) % p.tiles_h, tn_i = tile / (p.tiles_w * p.tiles_h);
    const int w0 = tw_i * p.TW, h0 = th_i * p.TH, n0 = tn_i * p.TN;
    const int cout0 = blockIdx.y * (SWAP ? kBM : BN);
    const int kb = (int)(((int64_t)p.k_iters * blockIdx.z) / p.splits);
    const int ke = (int)(((int64_t)p.k_iters * (blockIdx.z + 1)) / p.splits);
    const int niter = ke - kb;
    const bool split_n = NP == 3 && (SWAP || !p.presplit);

    if (threadIdx.x == 0) {
        unsigned int slot = 0xffffffffu;
        if (t_phase_buf != nullptr && (blockIdx.x | blockIdx.y | blockIdx.z) == 0) {
            const unsigned long long sidx = atomicAdd(t_phase_buf, 1ull);
            if (sidx < t_phase_cap) slot = (unsigned int)sidx;
        }
        *phase_slot = slot;
        phase_mark(slot, 0);
        for (int i = 0; i < S; ++i) {
            tc::mbar_init(&full_bar[i], 1); tc::mbar_init(&split_bar[i], kSplitters / 32); tc::mbar_init(&empty_bar[i], kConsumers / 32);
        }
        tc::fence_mbar_init();
    }
    if (threadIdx.x == kConsumers) {
        tc::prefetch_tensormap(&p.tmA[0]);
        tc::prefetch_tensormap(&p.tmB);
    }
    if (threadIdx.x < kConsumers) {
        const int nb = SWAP ? kBM : BN;
        for (int i = threadIdx.x; i < nb; i += kConsumers) {
            const int c = cout0 + i;
            bias_s[i] = (p.bias != nullptr && blockIdx.z == 0 && c < p.Cout) ? p.bias[c] : 0.f;
        }
        if (SWAP && threadIdx.x < BN) {
            const int j = threadIdx.x;
            const int tw = j % p.TW, th = (j / p.TW) % p.TH, tn = j / (p.TW * p.TH);
            const int n = n0 + tn, h = h0 + th, w = w0 + tw;
            pix_s[j] = (n < p.NB && h < p.Ho && w < p.Wo) ? (n * p.Ho + h) * p.Wo + w : -1;
        }
    }
    __syncthreads();
    const uint32_t pslot = *phase_slot;

    if (warp >= kConsumers / 32) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
        if (warp == kConsumers / 32) {
            // ------------------------------------------------------------ TMA producer
            if (lane == 0) {
                const bool presplit = !SWAP && p.presplit != 0;
                const uint32_t w_tx = SWAP ? (uint32_t)kABytes : (uint32_t)(Cfg::kNBytes * (presplit ? 2 : 1));
                const uint32_t a_tx = SWAP ? (uint32_t)Cfg::kNBytes : (uint32_t)kABytes;
                auto load_weights = [&](int it) {
                    const int s = it % S;
                    uint8_t* st = smem + s * Cfg::kStageBytes;
                    tc::tma_load_2d(SWAP ? st : st + kABytes, &p.tmB, &full_bar[s], (kb + it) * kBK, cout0);
                    if (presplit) tc::tma_load_2d(st + kABytes + Cfg::kNBytes, &p.tmBlo, &full_bar[s], (kb + it) * kBK, cout0);
                };
                auto load_acts = [&](int it) {
                    const int s = it % S;
                    const int i = kb + it;
                    const int tap = i / p.cin_chunks, cc = i - tap * p.cin_chunks;
                    const int ky = tap / p.KW, kx = tap - ky * p.KW;
                    int oy = ky - p.pad, ox = kx - p.pad, map = 0;
                    if (p.stride == 2) {
                        const int py = oy & 1, px = ox & 1;
                        map = py * 2 + px;
                        oy = (oy - py) >> 1;
                        ox = (ox - px) >> 1;
                    }
                    uint8_t* st = smem + s * Cfg::kStageBytes;
                    tc::tma_load_4d(SWAP ? st + kABytes : st, &p.tmA[map], &full_bar[s], cc * kBK, w0 + ox, h0 + oy, n0);
                };
                // PDL: the weights do not depend on the previous kernel -- the first S stages of weight tiles stream in while it drains;
                // the activation tiles of those stages follow once griddepcontrol.wait returns.
                const int pre = niter < S ? niter : S;
                phase_mark(pslot, 1);
                pdl_trigger();
                // ... unless the "weights" are themselves the output of an earlier kernel (q k^T, P v of the VAE's attention): prologues of a PDL chain
                // run arbitrarily far ahead of the bodies, so such an operand may not exist yet -- wait first
                if (p.w_dynamic) pdl_wait();
                for (int it = 0; it < pre; ++it) {
                    tc::mbar_expect_tx(&full_bar[it], w_tx + a_tx);
                    load_weights(it);
                }
                pdl_wait();
                phase_mark(pslot, 2);
                trace_mark();
                for (int it = 0; it < pre; ++it) load_acts(it);
                for (int it = pre; it < niter; ++it) {
                    const int s = it % S;
                    tc::mbar_wait(&empty_bar[s], ((uint32_t)(it / S) & 1u) ^ 1u);
                    tc::mbar_expect_tx(&full_bar[s], w_tx + a_tx);
                    load_acts(it);
                    load_weights(it);
                }
            }
        } else if (split_n) {
            // ------------------------------------------------------------ N-side splitter: hi in place, lo to the second buffer (same offsets =>
            // the swizzled layout is preserved); the hi words are written back explicitly, so the result does not depend on how the tensor core
            // reduces a full fp32 word
            const int et = threadIdx.x - (kConsumers + 32);
            for (int it = 0; it < niter; ++it) {
                const int s = it % S;
                tc::mbar_wait(&full_bar[s], (uint32_t)(it / S) & 1u);
                uint8_t* st = smem + s * Cfg::kStageBytes;
                float4* nraw = reinterpret_cast<float4*>(st + kABytes);
                float4* nlo = reinterpret_cast<float4*>(st + kABytes + Cfg::kNBytes);
#pragma unroll 2
                for (int i = et; i < BN * 8; i += kSplitters) {
                    const float4 v = nraw[i];
                    float4 h, l;
                    h.x = __uint_as_float(__float_as_uint(v.x) & 0xFFFFE000u); l.x = v.x - h.x;
                    h.y = __uint_as_float(__float_as_uint(v.y) & 0xFFFFE000u); l.y = v.y - h.y;
                    h.z = __uint_as_float(__float_as_uint(v.z) & 0xFFFFE000u); l.z = v.z - h.z;
                    h.w = __uint_as_float(__float_as_uint(v.w) & 0xFFFFE000u); l.w = v.w - h.w;
                    if (!p.raw_hi) nraw[i] = h;
                    nlo[i] = l;
                }
                tc::fence_proxy_async();  // generic-proxy stores -> visible to the tensor core's async-proxy reads
                __syncwarp();
                if (lane == 0) tc::mbar_arrive(&split_bar[s]);
            }
        }
        return;
    }

    // ---------------------------------------------------------------- consumers (warps 0-7)
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
    const int g = lane >> 2, t = lane & 3;
    const int r0 = (warp >> 2) * 64 + (warp & 3) * 16 + g;   // this thread's M-side rows: r0 and r0 + 8 (both == g mod 8)
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;

    for (int it = 0; it < niter; ++it) {
        const int s = it % S;
        const uint32_t ph = (uint32_t)(it / S) & 1u;
        tc::mbar_wait(&full_bar[s], ph);
        if (split_n) tc::mbar_wait(&split_bar[s], ph);
        if (it == 0 && threadIdx.x == 0) phase_mark(pslot, 3);
        const uint8_t* mt = smem + s * Cfg::kStageBytes;
        // A fragments of the 4 k-steps: element (row, col) of the swizzled tile sits at row*128 + ((col/4) ^ (row%8))*16 + (col%4)*4
        uint32_t ah[kBK / 8][4], al[kBK / 8][4];
#pragma unroll
        for (int k = 0; k < kBK / 8; ++k) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int row = r0 + (e & 1) * 8, chunk = 2 * k + (e >> 1);
                const uint32_t x = *reinterpret_cast<const uint32_t*>(mt + row * 128 + ((chunk ^ g) << 4) + t * 4);
                if (NP == 3) {
                    const uint32_t h = x & 0xFFFFE000u;
                    ah[k][e] = p.raw_hi ? x : h;
                    al[k][e] = __float_as_uint(__uint_as_float(x) - __uint_as_float(h));
                } else {
                    ah[k][e] = x;
                }
            }
        }
        const uint32_t b_hi = tc::smem_u32(mt + kABytes), b_lo = b_hi + Cfg::kNBytes;
        tc::fence_regs(acc);
        tc::wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBK / 8; ++k) {  // wgmma K = 8 tf32 = 32 bytes inside the 128-byte swizzle row
            const uint64_t dbh = tc::wgmma_desc_k_sw128(b_hi + k * 32);
            tc::Wgmma<BN>::mma(acc, ah[k], dbh, (it > 0 || k > 0) ? 1u : 0u);
            if (NP == 3) {
                const uint64_t dbl = tc::wgmma_desc_k_sw128(b_lo + k * 32);
                tc::Wgmma<BN>::mma(acc, al[k], dbh, 1u);
                tc::Wgmma<BN>::mma(acc, ah[k], dbl, 1u);
            }
        }
        tc::wgmma_commit();
        tc::fence_regs(acc);
        tc::wgmma_wait_all();
        tc::fence_regs(acc);
        __syncwarp();
        if (lane == 0) tc::mbar_arrive(&empty_bar[s]);   // frees the slot: this warp's LDS and MMAs have read it
    }
    if (threadIdx.x == 0) phase_mark(pslot, 4);

    // ---------------------------------------------------------------- epilogue
    const bool use_red = (p.splits > 1) || (p.accumulate != 0);
    pdl_wait();   // residual reads / output writes below must see the previous kernel's results (returns at once: the activations are in)
    if (threadIdx.x == 0) phase_mark(pslot, 5);
    if (!SWAP) {
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const int r = r0 + half * 8;
            const int tw = r % p.TW, th = (r / p.TW) % p.TH, tn = r / (p.TW * p.TH);
            const int n = n0 + tn, h = h0 + th, w = w0 + tw;
            if ((n < p.NB) && (h < p.Ho) && (w < p.Wo)) {
                const int64_t pix = (int64_t)((int64_t)n * p.Ho + h) * p.Wo + w;
                float* orow = p.out + pix * p.ldo + cout0;
                const float* rrow = (p.residual != nullptr && blockIdx.z == 0) ? p.residual + pix * p.ldr + cout0 : nullptr;
#pragma unroll
                for (int j = 0; j < BN / 8; ++j) {
                    const int c = j * 8 + t * 2;
                    if (cout0 + c < p.Cout) {   // Cout % 4 == 0 and c even: c + 1 is in range too
                        float x0 = acc[4 * j + 2 * half] + bias_s[c];
                        float x1 = acc[4 * j + 2 * half + 1] + bias_s[c + 1];
                        if (rrow) {
                            const float2 rv = __ldg(reinterpret_cast<const float2*>(rrow + c));
                            x0 += rv.x; x1 += rv.y;
                        }
                        if (use_red) {
                            asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(orow + c), "f"(x0), "f"(x1) : "memory");
                        } else {
                            *reinterpret_cast<float2*>(orow + c) = make_float2(x0, x1);
                        }
                    }
                }
            }
        }
    } else {
        // rows = output channels, columns = the BN pixels of the tile.  Transposed through shared memory (the stages are idle once both
        // warpgroups are past their last MMA) so that one warp writes the 128 channels of one pixel = 512 contiguous bytes per instruction.
        constexpr int kLd = 132;   // floats per staged pixel row (16-byte aligned)
        float* stg = reinterpret_cast<float*>(smem);
        asm volatile("bar.sync 1, 256;" ::: "memory");
#pragma unroll
        for (int half = 0; half < 2; ++half) {
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                const int col = j * 8 + t * 2;
                stg[col * kLd + r0 + half * 8] = acc[4 * j + 2 * half];
                stg[(col + 1) * kLd + r0 + half * 8] = acc[4 * j + 2 * half + 1];
            }
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
        const bool add_res = (p.residual != nullptr && blockIdx.z == 0);
        for (int idx = threadIdx.x; idx < BN * 32; idx += kConsumers) {
            const int pj = idx >> 5, c4 = idx & 31;
            const int pix = pix_s[pj];
            const int c = cout0 + c4 * 4;
            if (pix >= 0 && c < p.Cout) {
                float4 a = *reinterpret_cast<const float4*>(stg + pj * kLd + c4 * 4);
                const float4 bv = *reinterpret_cast<const float4*>(bias_s + c4 * 4);
                a.x += bv.x; a.y += bv.y; a.z += bv.z; a.w += bv.w;
                if (add_res) {
                    const float4 rv = __ldg(reinterpret_cast<const float4*>(p.residual + (int64_t)pix * p.ldr + c));
                    a.x += rv.x; a.y += rv.y; a.z += rv.z; a.w += rv.w;
                }
                float* dst = p.out + (int64_t)pix * p.ldo + c;
                if (use_red) {
                    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "f"(a.x), "f"(a.y), "f"(a.z), "f"(a.w) : "memory");
                } else {
                    *reinterpret_cast<float4*>(dst) = a;
                }
            }
        }
    }
    if (threadIdx.x == 0) phase_mark(pslot, 6);
}

// ---------------------------------------------------------------------------------- host side
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
    static PFN_encodeTiled fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_encodeTiled>(p);
    });
    return fn;
}

static int g_tma_tf32_type = 0;   // 0: FLOAT32 loads; 1: TFLOAT32 tensor-map type
static int g_variant = 2;         // 1 = no swap-AB and no pre-split weights, 2 = both where they apply, 3 = 2 with un-masked hi operands

struct MapKey {
    uint64_t v[12];
    bool operator==(const MapKey& o) const { return memcmp(v, o.v, sizeof(v)) == 0; }
};
struct MapKeyHash {
    size_t operator()(const MapKey& k) const {
        uint64_t h = 1469598103934665603ull;
        for (uint64_t x : k.v) { h ^= x; h *= 1099511628211ull; }
        return (size_t)h;
    }
};
static std::unordered_map<MapKey, CUtensorMap, MapKeyHash>& map_cache() {
    static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> c;
    return c;
}
static std::mutex g_map_mutex;

// rank-4 fp32 tensor map: dims {d0..d3} (d0 innermost), byte strides for d1..d3, box {b0..b3}
static int make_map(CUtensorMap* out, const void* base, const uint64_t dims[4], const uint64_t strides[3], const uint32_t box[4], int rank) {
    MapKey key{};
    key.v[0] = reinterpret_cast<uint64_t>(base);
    for (int i = 0; i < 4; ++i) key.v[1 + i] = dims[i];
    for (int i = 0; i < 3; ++i) key.v[5 + i] = strides[i];
    key.v[8] = ((uint64_t)box[0] << 32) | box[1];
    key.v[9] = ((uint64_t)box[2] << 32) | box[3];
    key.v[10] = (uint64_t)rank;
    key.v[11] = (uint64_t)g_tma_tf32_type;
    std::lock_guard<std::mutex> lock(g_map_mutex);
    auto it = map_cache().find(key);
    if (it != map_cache().end()) { *out = it->second; return SFB_OK; }
    PFN_encodeTiled enc = get_encode();
    if (!enc) return fail(SFB_ERR_CUDA, "cuTensorMapEncodeTiled is not available from the driver");
    cuuint64_t gd[4] = {dims[0], dims[1], dims[2], dims[3]};
    cuuint64_t gs[3] = {strides[0], strides[1], strides[2]};
    cuuint32_t bx[4] = {box[0], box[1], box[2], box[3]};
    cuuint32_t es[4] = {1, 1, 1, 1};
    CUresult r = enc(out, g_tma_tf32_type ? CU_TENSOR_MAP_DATA_TYPE_TFLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank,
                     const_cast<void*>(base), gd, gs, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS)
        return fail(SFB_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d) rank=%d dims=[%llu,%llu,%llu,%llu] box=[%u,%u,%u,%u] stride1=%llu", (int)r,
                    rank, (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)dims[2], (unsigned long long)dims[3],
                    box[0], box[1], box[2], box[3], (unsigned long long)strides[0]);
    if (map_cache().size() > 65536) map_cache().clear();
    map_cache()[key] = *out;
    return SFB_OK;
}

// optional per-launch timing of the conv kernel (CUDA events on the launch stream) for bench.py's roofline line
static bool g_prof = false;
static std::vector<std::pair<cudaEvent_t, cudaEvent_t>> g_prof_events;
static double g_prof_bytes = 0.0, g_prof_flops = 0.0;

static int conv_prof_begin(cudaStream_t st) {
    if (!g_prof) return SFB_OK;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    SFB_CUDA(cudaEventCreate(&e0));
    SFB_CUDA(cudaEventCreate(&e1));
    SFB_CUDA(cudaEventRecord(e0, st));
    g_prof_events.emplace_back(e0, e1);
    return SFB_OK;
}
static int conv_prof_end(cudaStream_t st) {
    if (!g_prof) return SFB_OK;
    SFB_CUDA(cudaEventRecord(g_prof_events.back().second, st));
    return SFB_OK;
}

template <int BN, bool SWAP, int NP>
static int launch_conv(const ConvGemmParams& p, dim3 grid, cudaStream_t st) {
    constexpr int smem = ConvCfg<BN, NP>::kSmemBytes;
    SFB_ONCE_PER_DEVICE(SFB_CUDA(cudaFuncSetAttribute(conv_gemm_kernel<BN, SWAP, NP>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem)));
    conv_prof_begin(st);
    trace_name(SWAP ? (BN == 16 ? "conv<16,swap>" : BN == 32 ? "conv<32,swap>" : "conv<64,swap>")
                    : (BN == 32 ? "conv<32>" : BN == 64 ? "conv<64>" : BN == 128 ? "conv<128>" : "conv<256>"));
    launch_pdl(conv_gemm_kernel<BN, SWAP, NP>, grid, dim3(kThreads), smem, st, p);
    conv_prof_end(st);
    return check_launch("conv2d_nhwc_tf32");
}

void trace_bind_conv(unsigned long long* buf, unsigned int cap) { trace_bind_this_tu(buf, cap); }
void phase_bind_conv(unsigned long long* buf, unsigned int cap) {
    cudaMemcpyToSymbol(t_phase_buf, &buf, sizeof(buf));
    cudaMemcpyToSymbol(t_phase_cap, &cap, sizeof(cap));
}

static inline int pow2_floor(int v) {
    int r = 1;
    while (r * 2 <= v) r *= 2;
    return r;
}

}  // namespace sfb

using namespace sfb;

extern "C" {

int sfb_conv_set_tma_tf32(int enable) {
    g_tma_tf32_type = enable ? 1 : 0;
    return SFB_OK;
}

int sfb_conv_prof_enable(int on) {
    g_prof = on != 0;
    if (on) { g_prof_bytes = 0.0; g_prof_flops = 0.0; }
    return SFB_OK;
}

/* sums the recorded conv launches: kernel time (ms), launch count, algorithmic weight bytes and FLOPs (2*MAC); clears the record */
int sfb_conv_prof_collect(double* total_ms, int* launches, double* weight_bytes, double* flops) {
    double t = 0.0;
    for (auto& pr : g_prof_events) {
        SFB_CUDA(cudaEventSynchronize(pr.second));
        float ms = 0.f;
        SFB_CUDA(cudaEventElapsedTime(&ms, pr.first, pr.second));
        t += ms;
        cudaEventDestroy(pr.first);
        cudaEventDestroy(pr.second);
    }
    if (total_ms) *total_ms = t;
    if (launches) *launches = (int)g_prof_events.size();
    if (weight_bytes) *weight_bytes = g_prof_bytes;
    if (flops) *flops = g_prof_flops;
    g_prof_events.clear();
    g_prof_bytes = 0.0; g_prof_flops = 0.0;
    return SFB_OK;
}

int sfb_conv_set_variant(int v) {
    if (v < 1 || v > 3) return fail(SFB_ERR_ARG, "conv_set_variant: 1, 2 or 3 (3 = 2 with un-masked hi operands, experiment)");
    g_variant = v;
    return SFB_OK;
}

int sfb_conv_weight_k(int Cin, int KH, int KW) { return KH * KW * ((Cin + 31) / 32) * 32; }

int sfb_conv2d_nhwc_tf32(const float* x, int NB, int H, int W, int Cin, int64_t ldx, const float* w_packed, int Cout, int KH, int KW, int stride,
                         int pad, const float* bias, const float* residual, int64_t ldr, float* out, int64_t ldo, int accumulate, int splits, int bn,
                         void* stream) {
    return sfb_conv2d_nhwc_tf32_pad(x, NB, H, W, Cin, ldx, w_packed, Cout, KH, KW, stride, pad, pad, bias, residual, ldr, out, ldo, accumulate, splits, bn,
                                    stream);
}

int sfb_conv2d_nhwc_tf32_pad(const float* x, int NB, int H, int W, int Cin, int64_t ldx, const float* w_packed, int Cout, int KH, int KW, int stride,
                             int pad, int pad_after, const float* bias, const float* residual, int64_t ldr, float* out, int64_t ldo, int accumulate,
                             int splits, int bn, void* stream) {
    return sfb_conv2d_nhwc_tf32_ex(x, NB, H, W, Cin, ldx, w_packed, nullptr, Cout, KH, KW, stride, pad, pad_after, bias, residual, ldr, out, ldo, accumulate,
                                   splits, bn, stream);
}

static thread_local int t_w_dynamic = 0;
int sfb_conv2d_nhwc_tf32_dyn(const float* x, int NB, int H, int W, int Cin, int64_t ldx, const float* w, int Cout, int KH, int KW, int stride, int pad,
                             int pad_after, const float* bias, const float* residual, int64_t ldr, float* out, int64_t ldo, int accumulate, int splits,
                             int bn, void* stream) {
    t_w_dynamic = 1;
    const int rc = sfb_conv2d_nhwc_tf32_ex(x, NB, H, W, Cin, ldx, w, nullptr, Cout, KH, KW, stride, pad, pad_after, bias, residual, ldr, out, ldo, accumulate,
                                           splits, bn, stream);
    t_w_dynamic = 0;
    return rc;
}

int sfb_conv2d_nhwc_tf32_ex(const float* x, int NB, int H, int W, int Cin, int64_t ldx, const float* w_packed, const float* w_hi_lo, int Cout, int KH, int KW,
                            int stride, int pad, int pad_after, const float* bias, const float* residual, int64_t ldr, float* out, int64_t ldo,
                            int accumulate, int splits, int bn, void* stream) {
    SFB_REQUIRE(x && w_packed && out, "conv2d_nhwc_tf32: null pointer");
    SFB_REQUIRE(NB > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0, "conv2d_nhwc_tf32: empty shape");
    SFB_REQUIRE(stride == 1 || stride == 2, "conv2d_nhwc_tf32: stride must be 1 or 2");
    SFB_REQUIRE(Cin % 4 == 0 && ldx % 4 == 0 && ldx >= Cin, "conv2d_nhwc_tf32: Cin and ldx must be multiples of 4 floats (TMA 16-byte strides)");
    SFB_REQUIRE(Cout % 4 == 0 && ldo % 4 == 0, "conv2d_nhwc_tf32: Cout and ldo must be multiples of 4");
    SFB_REQUIRE(((uintptr_t)x & 15) == 0 && ((uintptr_t)w_packed & 15) == 0 && ((uintptr_t)out & 15) == 0, "conv2d_nhwc_tf32: pointers must be 16-byte aligned");
    SFB_REQUIRE(pad >= 0 && pad_after >= 0, "conv2d_nhwc_tf32: negative padding");
    // `pad` zeros before row/column 0, `pad_after` after the last one; both are TMA out-of-bounds zero fill, only the output extent differs
    const int Ho = (H + pad + pad_after - KH) / stride + 1, Wo = (W + pad + pad_after - KW) / stride + 1;
    SFB_REQUIRE(Ho > 0 && Wo > 0, "conv2d_nhwc_tf32: empty output");
    if (stride == 2) SFB_REQUIRE(H % 2 == 0 && W % 2 == 0, "conv2d_nhwc_tf32: stride 2 needs even H and W");

    ConvGemmParams p;
    memset(&p, 0, sizeof(p));
    // pixel tile.  Normal: TW x TH x TN = 128 output pixels on the M side.  Swap-AB (<= 64 output pixels in total): the pixels
    // are the N side (16 / 32 / 64 of them) and 128 output channels the M side.
    const int planeW = (stride == 2) ? W / 2 : W, planeH = (stride == 2) ? H / 2 : H;
    const int64_t P_total = (int64_t)NB * Ho * Wo;
    const bool v2 = (precision_mode() == 1 && g_variant >= 2);
    const bool swap = v2 && P_total <= 64 && bn <= 0;
    int tile_pix = kBM;
    if (swap) { tile_pix = 16; while (tile_pix < P_total) tile_pix *= 2; }
    p.TW = Wo >= tile_pix ? tile_pix : pow2_floor(Wo);
    p.TH = tile_pix / p.TW;
    if (p.TH > Ho) p.TH = pow2_floor(Ho);
    p.TN = tile_pix / (p.TW * p.TH);
    p.tiles_w = ceil_div(Wo, p.TW);
    p.tiles_h = ceil_div(Ho, p.TH);
    const int tiles_n = ceil_div(NB, p.TN);
    const int tiles_m = p.tiles_w * p.tiles_h * tiles_n;

    const int cin_pad = ((Cin + 31) / 32) * 32;
    p.cin_chunks = cin_pad / 32;
    p.KH = KH; p.KW = KW; p.pad = pad; p.stride = stride;
    p.k_iters = KH * KW * p.cin_chunks;
    p.NB = NB; p.Ho = Ho; p.Wo = Wo; p.Cout = Cout;
    p.out = out; p.bias = bias; p.ldo = ldo; p.accumulate = accumulate;
    p.raw_hi = (g_variant == 3) ? 1 : 0;
    p.w_dynamic = t_w_dynamic;
    p.residual = residual; p.ldr = ldr;
    SFB_REQUIRE(residual == nullptr || (ldr % 4 == 0 && ((uintptr_t)residual & 15) == 0), "conv2d_nhwc_tf32: residual must be 16-byte aligned");

    // N tile
    int BN = bn;
    if (BN <= 0) {
        BN = Cout >= 256 ? 256 : (Cout >= 128 ? 128 : (Cout >= 64 ? 64 : 32));
        const int sms = sm_count();
        while (BN > 128 && tiles_m * ceil_div(Cout, BN) < sms) BN /= 2;  // prefer more CTAs when the grid is small
        if (v2 && BN > 128) BN = 128;
    }
    SFB_REQUIRE(BN == 32 || BN == 64 || BN == 128 || BN == 256, "conv2d_nhwc_tf32: bn must be 32, 64, 128 or 256");
    const int tiles_c = swap ? ceil_div(Cout, kBM) : ceil_div(Cout, BN);
    if (splits <= 0) {
        const int ctas = tiles_m * tiles_c;
        splits = 1;
        if (ctas < sm_count()) {
            splits = sm_count() / ctas;
            const int max_by_k = p.k_iters / 4 > 0 ? p.k_iters / 4 : 1;  // keep >= 4 k-steps per split
            if (splits > max_by_k) splits = max_by_k;
            if (splits < 1) splits = 1;
        }
    }
    if (precision_mode() == 1) {
        // the tensor core's fp32 accumulation is not exactly rounded: the error of one accumulator grows ~linearly with the number of
        // MMAs chained into it.  Bound the chain; partial sums meet in fp32 reds.
        const int min_splits = ceil_div(p.k_iters, 96);
        if (splits < min_splits) splits = min_splits;
    }
    if (splits > p.k_iters) splits = p.k_iters;
    p.splits = splits;

    // tensor maps: activations (1 map, or 4 parity planes for stride 2) and packed weights
    cudaStream_t st = as_stream(stream);
    const uint32_t boxA[4] = {32u, (uint32_t)p.TW, (uint32_t)p.TH, (uint32_t)p.TN};
    const int w_rows = swap ? kBM : BN;   // rows of the weight box
    if (stride == 1) {
        const uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)W, (uint64_t)H, (uint64_t)NB};
        const uint64_t strides[3] = {(uint64_t)ldx * 4, (uint64_t)W * ldx * 4, (uint64_t)H * W * ldx * 4};
        if (int rc = make_map(&p.tmA[0], x, dims, strides, boxA, 4)) return rc;
        p.tmA[1] = p.tmA[2] = p.tmA[3] = p.tmA[0];
    } else {
        for (int py = 0; py < 2; ++py)
            for (int px = 0; px < 2; ++px) {
                const uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)planeW, (uint64_t)planeH, (uint64_t)NB};
                const uint64_t strides[3] = {(uint64_t)2 * ldx * 4, (uint64_t)2 * W * ldx * 4, (uint64_t)H * W * ldx * 4};
                if (int rc = make_map(&p.tmA[py * 2 + px], x + ((int64_t)py * W + px) * ldx, dims, strides, boxA, 4)) return rc;
            }
    }
    {
        const uint64_t ktot = (uint64_t)KH * KW * cin_pad;
        const uint64_t dims[4] = {ktot, (uint64_t)Cout, 1, 1};
        const uint64_t strides[3] = {ktot * 4, 0, 0};
        const uint32_t boxB[4] = {32u, (uint32_t)w_rows, 1, 1};
        const bool presplit = (w_hi_lo != nullptr) && v2 && !swap;
        p.presplit = presplit ? 1 : 0;
        if (presplit) {
            SFB_REQUIRE(((uintptr_t)w_hi_lo & 15) == 0, "conv2d_nhwc_tf32: w_hi_lo must be 16-byte aligned");
            if (int rc = make_map(&p.tmB, w_hi_lo, dims, strides, boxB, 2)) return rc;
            if (int rc = make_map(&p.tmBlo, w_hi_lo + (size_t)Cout * ktot, dims, strides, boxB, 2)) return rc;
        } else {
            if (int rc = make_map(&p.tmB, w_packed, dims, strides, boxB, 2)) return rc;
            p.tmBlo = p.tmB;
        }
    }

    if (splits > 1 && !accumulate) {
        // partial sums are reduced with red.global.add: the destination slice must start from zero
        SFB_CUDA(cudaMemset2DAsync(out, (size_t)ldo * 4, 0, (size_t)Cout * 4, (size_t)NB * Ho * Wo, st));
    }
    dim3 grid(tiles_m, tiles_c, splits);
    if (g_prof) {
        g_prof_bytes += (double)Cout * KH * KW * Cin * 4.0;
        g_prof_flops += 2.0 * NB * Ho * Wo * (double)Cout * KH * KW * Cin;
    }
    if (swap) {
        switch (tile_pix) {
            case 16: return launch_conv<16, true, 3>(p, grid, st);
            case 32: return launch_conv<32, true, 3>(p, grid, st);
            default: return launch_conv<64, true, 3>(p, grid, st);
        }
    }
    if (precision_mode() == 1) {
        switch (BN) {
            case 32: return launch_conv<32, false, 3>(p, grid, st);
            case 64: return launch_conv<64, false, 3>(p, grid, st);
            case 128: return launch_conv<128, false, 3>(p, grid, st);
            default: return launch_conv<256, false, 3>(p, grid, st);
        }
    }
    switch (BN) {
        case 32: return launch_conv<32, false, 1>(p, grid, st);
        case 64: return launch_conv<64, false, 1>(p, grid, st);
        case 128: return launch_conv<128, false, 1>(p, grid, st);
        default: return launch_conv<256, false, 1>(p, grid, st);
    }
}
}
