// checksum.cu -- 64-bit digest of a device buffer: the check that a resumed distillation runs on the scene cache it was saved with
// (distillation.cache_digest).  Word i of the buffer contributes mix(w_i ^ mix(i + phi)) and the contributions are summed modulo 2^64,
// so the result does not depend on the launch geometry or on the order the atomics land in: equal bits give an equal digest on any
// device and any run, and a changed, moved or missing word changes it.
#include "common.cuh"

namespace {

__device__ __forceinline__ uint64_t mix64(uint64_t x) {      // splitmix64's finaliser
    x ^= x >> 30;
    x *= 0xBF58476D1CE4E5B9ull;
    x ^= x >> 27;
    x *= 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}

__global__ void digest_kernel(const uint32_t* __restrict__ w, int64_t n, unsigned long long* __restrict__ out) {
    uint64_t acc = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        acc += mix64((uint64_t)w[i] ^ mix64((uint64_t)i + 0x9E3779B97F4A7C15ull));
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) atomicAdd(out, (unsigned long long)acc);
}

}  // namespace

extern "C" int sfb_digest_u32(const void* data, int64_t n_words, uint64_t* out, void* stream) {
    using namespace sfb;
    SFB_REQUIRE(out && (data || n_words == 0) && n_words >= 0, "digest_u32: null pointer or n_words < 0");
    SFB_CUDA(cudaMemsetAsync(out, 0, sizeof(uint64_t), as_stream(stream)));
    if (n_words == 0) return SFB_OK;
    int64_t blocks = ceil_div<int64_t>(n_words, 256);
    if (blocks > (int64_t)sm_count() * 8) blocks = (int64_t)sm_count() * 8;
    digest_kernel<<<(unsigned)blocks, 256, 0, as_stream(stream)>>>(static_cast<const uint32_t*>(data), n_words,
                                                                     reinterpret_cast<unsigned long long*>(out));
    return check_launch("digest_u32");
}
