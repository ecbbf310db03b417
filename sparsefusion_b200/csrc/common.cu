// common.cu -- error reporting and device queries shared by every translation unit
#include "common.cuh"
#include <stdarg.h>
#include <atomic>
#include <cstring>
#include <mutex>
#include <unordered_set>
#include <cstdint>
#include "../../include/sparsefusion_b200.h"

namespace sfb {

std::string& last_error() {
    static thread_local std::string msg;
    return msg;
}

int fail(int code, const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    last_error() = buf;
    return code;
}

static std::atomic<unsigned long long> g_launches{0};
void count_launches(int n) { g_launches += (unsigned long long)n; }

int check_launch(const char* what) {
    g_launches += 1;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(SFB_ERR_CUDA, "%s: launch failed: %s", what, cudaGetErrorString(e));
    return SFB_OK;
}

static int g_precision = 1;  // 0: single-pass TF32 (operands rounded on write); 1: error-compensated 3xTF32 (default)
static thread_local int t_precision_override = -1;
int precision_mode() { return t_precision_override >= 0 ? t_precision_override : g_precision; }
int set_precision_override(int m) { const int old = t_precision_override; t_precision_override = m; return old; }
void set_precision_mode(int m) { g_precision = m; }

static std::atomic<int> g_carveout{1};
static inline unsigned long long dev_key(const void* kernel) { return (unsigned long long)(uintptr_t)kernel * 64ull + (unsigned)(current_device() & 63); }
void prefer_smem(const void* kernel) {
    static std::unordered_set<unsigned long long> done;     // keyed on (kernel, device): function attributes are per device
    static std::mutex mu;
    if (!g_carveout.load()) return;
    std::lock_guard<std::mutex> lock(mu);
    if (done.insert(dev_key(kernel)).second) cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
}
static std::atomic<int> g_pad_smem{0};
size_t pad_smem(const void* kernel, size_t smem) {
    constexpr size_t kPad = 150 * 1024;
    if (!g_pad_smem.load() || smem >= kPad) return smem;
    static std::unordered_set<unsigned long long> done;
    static std::mutex mu;
    std::lock_guard<std::mutex> lock(mu);
    if (done.insert(dev_key(kernel)).second) cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kPad);
    return kPad;
}
static std::atomic<int> g_pdl{1};
bool pdl_enabled() { return g_pdl.load() != 0; }
void set_pdl(int on) { g_pdl.store(on != 0); }
static std::mutex g_trace_mu;
static bool g_trace_open = false;
static std::string g_trace_names;
void trace_name(const char* kernel) {
    if (!g_trace_open) return;
    std::lock_guard<std::mutex> lock(g_trace_mu);
    g_trace_names += kernel;
    g_trace_names += '\n';
}
static std::atomic<int> g_fusion{0x7fffffff};
int fusion_mask() { return g_fusion.load(); }
void set_fusion_mask(int m) { g_fusion.store(m); }

int current_device() {
    int dev = 0;
    cudaGetDevice(&dev);
    return dev;
}

int sm_count() {
    static std::atomic<int> cache[64];     // per device ordinal (zero-initialised)
    const int dev = current_device();
    int n = cache[dev & 63].load(std::memory_order_relaxed);
    if (n == 0) {
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        if (n <= 0) n = 132;
        cache[dev & 63].store(n, std::memory_order_relaxed);
    }
    return n;
}

}  // namespace sfb

extern "C" {

const char* sfb_last_error(void) { return sfb::last_error().c_str(); }

int sfb_abi_version(void) { return SFB_ABI_VERSION; }

int sfb_set_precision(int mode) {
    if (mode != 0 && mode != 1) return sfb::fail(SFB_ERR_ARG, "set_precision: mode must be 0 (tf32) or 1 (tf32x3)");
    sfb::set_precision_mode(mode);
    return SFB_OK;
}
int sfb_get_precision(void) { return sfb::precision_mode(); }
int sfb_set_pdl(int on) { sfb::set_pdl(on & 1); sfb::g_carveout.store((on & 2) ? 0 : 1); sfb::g_pad_smem.store((on & 4) ? 1 : 0); return SFB_OK; }
int sfb_trace_begin(unsigned long long* device_buf, unsigned int capacity) {
    {
        std::lock_guard<std::mutex> lock(sfb::g_trace_mu);
        sfb::g_trace_names.clear();
        sfb::g_trace_open = device_buf != nullptr;
    }
    sfb::trace_bind_unet_ops(device_buf, capacity);
    sfb::trace_bind_conv(device_buf, capacity);
    SFB_CUDA(cudaGetLastError());
    return SFB_OK;
}
int sfb_trace_end(void) {
    {
        std::lock_guard<std::mutex> lock(sfb::g_trace_mu);
        sfb::g_trace_open = false;
    }
    sfb::trace_bind_unet_ops(nullptr, 0);
    sfb::trace_bind_conv(nullptr, 0);
    SFB_CUDA(cudaGetLastError());
    return SFB_OK;
}
int sfb_conv_phase_trace(unsigned long long* device_buf, unsigned int capacity) {
    sfb::phase_bind_conv(device_buf, capacity);
    SFB_CUDA(cudaGetLastError());
    return SFB_OK;
}
int sfb_trace_names(char* out, int capacity) {
    std::lock_guard<std::mutex> lock(sfb::g_trace_mu);
    const int n = (int)sfb::g_trace_names.size();
    if (out != nullptr && capacity > 0) {
        const int m = n < capacity - 1 ? n : capacity - 1;
        memcpy(out, sfb::g_trace_names.data(), m);
        out[m] = 0;
    }
    return n;
}
int sfb_set_fusion(int mask) { sfb::set_fusion_mask(mask); return SFB_OK; }
uint64_t sfb_launch_count(void) { return (uint64_t)sfb::g_launches.load(); }

int sfb_device_info(int* sm_count, int* cc_major, int* cc_minor) {
    int dev = 0;
    SFB_CUDA(cudaGetDevice(&dev));
    cudaDeviceProp p;
    SFB_CUDA(cudaGetDeviceProperties(&p, dev));
    if (sm_count) *sm_count = p.multiProcessorCount;
    if (cc_major) *cc_major = p.major;
    if (cc_minor) *cc_minor = p.minor;
    return SFB_OK;
}
}
