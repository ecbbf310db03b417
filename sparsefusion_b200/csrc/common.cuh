// common.cuh -- shared helpers for the sm_90a kernels behind the C-ABI (include/sparsefusion_b200.h)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>
#include "../../include/sparsefusion_b200.h"  // SFB_OK / SFB_ERR_* codes

namespace sfb {

// last error message, per host thread; read through sfb_last_error()
std::string& last_error();
int fail(int code, const char* fmt, ...);


static inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

template <typename T>
static inline __host__ __device__ T ceil_div(T a, T b) { return (a + b - 1) / b; }

int check_launch(const char* what);   // also counts one kernel launch (sfb_launch_count)
void count_launches(int n);            // extra launches made under a single check_launch

// tensor-core operand precision of the UNet GEMMs: 0 = TF32 single pass, 1 = 3xTF32 (error compensated)
int precision_mode();
void set_precision_mode(int m);
int set_precision_override(int m);   // per host thread; -1 = none.  Returns the previous override (NGP weight gradients always use 3xTF32)

// Programmatic dependent launch (PDL).  The UNet evaluation is ~350 short kernels replayed from one CUDA graph; each of them
// (a) is launched with programmatic stream serialisation, so its CTAs may become resident while the previous kernel drains, and
// (b) starts with pdl_sync(): signal that the NEXT kernel may be scheduled, then wait until every kernel before this one has completed
// and flushed its memory.  All global reads and writes of a kernel come after that wait, so ordering is unchanged.
bool pdl_enabled();
// Every PDL-launched kernel asks for the maximum shared-memory carve-out, whether it needs it or not: the wgmma convolutions use ~200 KB of
// smem, and a dependent kernel can only become resident next to the draining CTAs of its predecessor (the point of PDL) when both want the
// same L1/shared split of the SM.
void prefer_smem(const void* kernel);
size_t pad_smem(const void* kernel, size_t smem);   // experiment (sfb_set_pdl bit 2): every PDL kernel requests a conv-sized dynamic smem block
void trace_name(const char* kernel);   // host side of the tracer: kernel names in launch order while a trace is open
void trace_bind_unet_ops(unsigned long long* buf, unsigned int cap);
void trace_bind_conv(unsigned long long* buf, unsigned int cap);
void phase_bind_conv(unsigned long long* buf, unsigned int cap);
// optional paths (sfb_set_fusion): bit 0 = NGP MLP weight gradients as wgmma GEMMs (off: the SIMT outer-product kernel)
int fusion_mask();
static inline bool wgrad_tc_enabled() { return (fusion_mask() & 1) != 0; }
static inline bool field_v2_enabled() { return (fusion_mask() & 16) != 0; }    // tiled NGP field kernels (128-point GEMM tiles in shared memory, no tape)
static inline bool gn_grid_enabled() { return (fusion_mask() & 2) != 0; }
static inline bool gn_cluster_enabled() { return (fusion_mask() & 4) != 0; }
static inline bool gn_cluster_adaptive() { return (fusion_mask() & 8) != 0; }  // cluster width by tensor size (1 = a plain CTA per group) instead of always 8   // single-launch GroupNorm: one thread-block cluster per (image, group)
static inline bool gca_cluster_enabled() { return (fusion_mask() & 8) != 0; }  // GlobalContext + gate + residual as one cluster kernel
static inline bool gca_cluster_wide() { return (fusion_mask() & 16) != 0; }    // ... with 16-CTA (non-portable) clusters where the slab allows, else 8   // single-launch GroupNorm with a software grid barrier (batch 1)
#ifdef __CUDACC__
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
// In-situ tracer (sfb_trace_begin): when bound, CTA (0,0,0) of every kernel appends %globaltimer to a device buffer right after its
// griddepcontrol.wait, i.e. at the moment all earlier kernels have completed.  Consecutive stamps are the chain cost of each kernel inside a
// replayed graph (launch gap included) -- what ncu's serialised, cache-flushed durations cannot show.  buf[0] = count, buf[1..] = stamps.
static __device__ unsigned long long* t_trace_buf = nullptr;
static __device__ unsigned int t_trace_cap = 0;
__device__ __forceinline__ void trace_mark() {
    unsigned long long* b = t_trace_buf;
    if (b != nullptr && (blockIdx.x | blockIdx.y | blockIdx.z | threadIdx.x | threadIdx.y | threadIdx.z) == 0) {
        const unsigned long long slot = atomicAdd(b, 1ull);
        unsigned long long t;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        if (slot < t_trace_cap) b[1 + slot] = t;
    }
}
static inline void trace_bind_this_tu(unsigned long long* buf, unsigned int cap) {
    cudaMemcpyToSymbol(t_trace_buf, &buf, sizeof(buf));
    cudaMemcpyToSymbol(t_trace_cap, &cap, sizeof(cap));
}
__device__ __forceinline__ void pdl_sync() { pdl_trigger(); pdl_wait(); trace_mark(); }

// torch.clamp, max pooling and relu keep a NaN operand; fminf / fmaxf return the other operand instead.  On operands that are not NaN
// these are fminf / fmaxf, bit for bit (signed zeros included).
__device__ __forceinline__ float clamp_keep_nan(float x, float lo, float hi) { return x != x ? x : fminf(fmaxf(x, lo), hi); }
__device__ __forceinline__ float max_keep_nan(float a, float b) { return (a != a || b != b) ? a + b : fmaxf(a, b); }

// cluster_x > 1 launches thread-block clusters of (cluster_x, 1, 1); grid.x must be a multiple of it
template <typename... KA, typename... A>
static inline cudaError_t launch_pdl_cluster(void (*kernel)(KA...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, unsigned cluster_x,
                                             A&&... args) {
    prefer_smem((const void*)kernel);
    smem = pad_smem((const void*)kernel, smem);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
    cfg.numAttrs = 1;
    if (cluster_x > 1) {
        attr[1].id = cudaLaunchAttributeClusterDimension;
        attr[1].val.clusterDim.x = cluster_x;
        attr[1].val.clusterDim.y = 1;
        attr[1].val.clusterDim.z = 1;
        cfg.numAttrs = 2;
    }
    cfg.attrs = attr;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KA>(args)...);
}
template <typename... KA, typename... A>
static inline cudaError_t launch_pdl(void (*kernel)(KA...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, A&&... args) {
    return launch_pdl_cluster(kernel, grid, block, smem, st, 1u, static_cast<A&&>(args)...);
}
#define SFB_LAUNCH(kernel, ...) (sfb::trace_name(#kernel), sfb::launch_pdl(kernel, __VA_ARGS__))
#define SFB_LAUNCH_CLUSTER(kernel, ...) (sfb::trace_name(#kernel), sfb::launch_pdl_cluster(kernel, __VA_ARGS__))
#endif


// number of SMs of the current device (cached per device)
int sm_count();
// index of the current CUDA device (cudaGetDevice)
int current_device();

}  // namespace sfb
#include <atomic>
// run `stmt` once per DEVICE (function attributes such as cudaFuncAttributeMaxDynamicSharedMemorySize are per device: a process that
// touches a second GPU must set them there too).  One bit per device ordinal (mod 64) in a per-site mask.
#define SFB_ONCE_PER_DEVICE(stmt)                                                         \
    do {                                                                                  \
        static std::atomic<unsigned long long> done__{0};                                 \
        const unsigned long long bit__ = 1ull << (sfb::current_device() & 63);            \
        if (!(done__.load(std::memory_order_acquire) & bit__)) {                          \
            stmt;                                                                         \
            done__.fetch_or(bit__, std::memory_order_release);                            \
        }                                                                                 \
    } while (0)
namespace sfb {

}  // namespace sfb

#define SFB_REQUIRE(cond, ...)                                   \
    do {                                                         \
        if (!(cond)) return sfb::fail(SFB_ERR_ARG, __VA_ARGS__); \
    } while (0)

#define SFB_CUDA(call)                                                                                  \
    do {                                                                                                \
        cudaError_t e__ = (call);                                                                       \
        if (e__ != cudaSuccess) return sfb::fail(SFB_ERR_CUDA, "%s: %s", #call, cudaGetErrorString(e__)); \
    } while (0)
