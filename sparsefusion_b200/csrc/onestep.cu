// onestep.cu -- the latent math of DDPM.forward_noloss (sparsefusion/vldm.py:632-709), the one-step denoising target, as two per-row kernels.
//
// Row r of a batch sits at its own noise level, given as the fp32 log-SNR ls[r] the UNet is conditioned on (a device array: nothing is read
// back to the host).  alpha = sqrt(sigmoid(ls)), sigma = sqrt(sigmoid(-ls)) (log_snr_to_alpha_sigma, imagen_pytorch.py:198-199):
//   q_sample (:260-269)                 x_noisy = alpha * x_start + sigma * noise,      alpha_cumprod[r] = sigmoid(ls)
//   predict_start_from_noise (:293-297) x0 = clamp((x_noisy - sigma * eps) / max(alpha, 1e-8), +-clip)       (vldm.py:700-701)
// Every product, sum and quotient is rounded on its own (no FMA contraction) and sigmoid is 1 / (1 + expf(-x)), the operation order of
// the reference's eager fp32 expressions.
#include "common.cuh"
#include "../../include/sparsefusion_b200.h"

namespace sfb {

__device__ __forceinline__ float sigmoid_rn(float x) { return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x))); }

__global__ void ddpm_q_sample_rows_kernel(const float* __restrict__ x_start, const float* __restrict__ noise, const float* __restrict__ log_snr,
                                          int64_t row_len, float* __restrict__ x_noisy, float* __restrict__ alpha_cumprod) {
    pdl_sync();
    const float ls = log_snr[blockIdx.y];
    const float alpha = __fsqrt_rn(sigmoid_rn(ls)), sigma = __fsqrt_rn(sigmoid_rn(-ls));
    if (alpha_cumprod && blockIdx.x == 0 && threadIdx.x == 0) alpha_cumprod[blockIdx.y] = sigmoid_rn(ls);
    const int64_t off = (int64_t)blockIdx.y * row_len;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < row_len; i += (int64_t)gridDim.x * blockDim.x)
        x_noisy[off + i] = __fadd_rn(__fmul_rn(alpha, x_start[off + i]), __fmul_rn(sigma, noise[off + i]));
}

// Classifier-free guidance (e_null given): eps = e_null + (e_cond - e_null) * cond_scale (imagen_pytorch.py:1468), rounded as
// plms_update_rows_cfg_kernel forms it.  The clamp keeps NaN, as torch.clamp does.
__global__ void ddpm_predict_x0_rows_kernel(const float* __restrict__ x_noisy, const float* __restrict__ e_cond, const float* __restrict__ e_null,
                                            float cond_scale, const float* __restrict__ log_snr, float clip, int64_t row_len,
                                            float* __restrict__ eps_out, float* __restrict__ x0_out) {
    pdl_sync();
    const float ls = log_snr[blockIdx.y];
    const float alpha = fmaxf(__fsqrt_rn(sigmoid_rn(ls)), 1e-8f), sigma = __fsqrt_rn(sigmoid_rn(-ls));
    const int64_t off = (int64_t)blockIdx.y * row_len;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < row_len; i += (int64_t)gridDim.x * blockDim.x) {
        float e = e_cond[off + i];
        if (e_null) {
            const float en = e_null[off + i];
            e = __fadd_rn(en, __fmul_rn(__fsub_rn(e, en), cond_scale));
        }
        if (eps_out) eps_out[off + i] = e;
        x0_out[off + i] = clamp_keep_nan(__fdiv_rn(__fsub_rn(x_noisy[off + i], __fmul_rn(sigma, e)), alpha), -clip, clip);
    }
}

static inline dim3 rows_grid(int rows, int64_t row_len) {
    int64_t bx = (row_len + 255) / 256;
    if (bx > 1024) bx = 1024;
    return dim3((unsigned)bx, (unsigned)rows);
}
}  // namespace sfb

extern "C" int sfb_ddpm_q_sample_rows(const float* x_start, const float* noise, const float* log_snr, int rows, int64_t row_len, float* x_noisy,
                                      float* alpha_cumprod, void* stream) {
    SFB_REQUIRE(rows >= 0 && rows <= 65535 && row_len >= 0, "ddpm_q_sample_rows: rows must be in [0, 65535] and row_len >= 0");
    if (rows == 0) return SFB_OK;
    SFB_REQUIRE(log_snr, "ddpm_q_sample_rows: null pointer");
    if (row_len == 0 && !alpha_cumprod) return SFB_OK;
    SFB_REQUIRE(row_len == 0 || (x_start && noise && x_noisy), "ddpm_q_sample_rows: null pointer");
    SFB_LAUNCH(sfb::ddpm_q_sample_rows_kernel, sfb::rows_grid(rows, row_len), 256, 0, sfb::as_stream(stream), x_start, noise, log_snr, row_len,
               x_noisy, alpha_cumprod);
    return sfb::check_launch("ddpm_q_sample_rows");
}

extern "C" int sfb_ddpm_predict_x0_rows(const float* x_noisy, const float* e_cond, const float* e_null, float cond_scale, const float* log_snr,
                                        float clip, int rows, int64_t row_len, float* eps_out, float* x0_out, void* stream) {
    SFB_REQUIRE(rows >= 0 && rows <= 65535 && row_len >= 0, "ddpm_predict_x0_rows: rows must be in [0, 65535] and row_len >= 0");
    if (rows == 0 || row_len == 0) return SFB_OK;
    SFB_REQUIRE(x_noisy && e_cond && log_snr && x0_out, "ddpm_predict_x0_rows: null pointer");
    SFB_LAUNCH(sfb::ddpm_predict_x0_rows_kernel, sfb::rows_grid(rows, row_len), 256, 0, sfb::as_stream(stream), x_noisy, e_cond, e_null, cond_scale,
               log_snr, clip, row_len, eps_out, x0_out);
    return sfb::check_launch("ddpm_predict_x0_rows");
}
