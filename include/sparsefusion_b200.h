/*
 * sparsefusion_b200.h -- C ABI of libsparsefusion_b200.so
 *
 * The drop-in boundary of the H100-native SparseFusion hot path.  Every entry point takes plain
 * DEVICE pointers (fp32 / int32 / uint8, contiguous), sizes and a CUDA stream handle
 * (`void* stream` == cudaStream_t; NULL == the legacy default stream); there are no torch types in
 * any signature.  Each function replaces one binding of the reference's pybind operator modules
 * or one nn.Module hot loop; the comment above each declaration cites the reference interface
 * (file:line relative to zhizdev/sparsefusion) it stands in for.
 *
 * Conventions (same as the reference operators, raymarching/src/bindings.cpp, gridencoder/src/bindings.cpp):
 *   - the CALLER allocates every output and passes it in; nothing is allocated or freed inside;
 *   - launches are asynchronous on `stream`; errors that CUDA reports at launch time are returned,
 *     asynchronous faults surface at the caller's next synchronisation, as with the reference;
 *   - return value 0 == success; non-zero == SFB_ERR_* and sfb_last_error() holds a message
 *     (the Python host raises RuntimeError with it, mirroring TORCH_CHECK in gridencoder.cu:425-441);
 *   - dtype is fp32 only: the reference dispatches half/double too but never calls them
 *     (custom_fwd(cast_inputs=float32), raymarching.py:21 and SURVEY.md §2.3).
 */
#ifndef SPARSEFUSION_B200_H
#define SPARSEFUSION_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SFB_ABI_VERSION 3

#define SFB_OK 0
#define SFB_ERR_ARG 1
#define SFB_ERR_CUDA 2
#define SFB_ERR_UNSUPPORTED 3

const char* sfb_last_error(void);
int sfb_abi_version(void);
int sfb_device_info(int* sm_count, int* cc_major, int* cc_minor);
/* Tensor-core operand precision of the UNet GEMMs.  1 (default) = error-compensated 3xTF32: operands stay fp32 in HBM, every
 * stage is split hi/lo in shared memory and hi*hi + lo*hi + hi*lo is accumulated -- fp32-class accuracy, needed for the 1e-3
 * contract on the predicted noise.  0 = single-pass TF32 (what the reference GPU build's cuDNN/cuBLAS did): operands are rounded
 * to TF32 where they are produced; ~1.5e-3 relative error on the UNet output, ~1/3 of the tensor-pipe work. */
int sfb_set_precision(int mode);
int sfb_get_precision(void);
/* programmatic dependent launch of the UNet kernels (default on): each kernel may be scheduled while its predecessor drains and
 * waits (griddepcontrol.wait) before touching global memory.  Bit 0 clear restores plain stream-ordered launches; bit 1 set stops requesting
 * the maximum shared-memory carve-out for kernels launched for the first time afterwards (A/B measurement). */
int sfb_set_pdl(int on);
/* in-situ tracer for the UNet kernels: while a trace is open every traced kernel appends %globaltimer (ns) to device_buf right after its
 * griddepcontrol.wait (device_buf[0] = number of stamps, device_buf[1..capacity] = stamps; zero it before each run) and the host records
 * the kernel names in launch order (sfb_trace_names: newline separated, returns the full length).  sfb_trace_end() unbinds.
 * sfb_trace_end keeps the recorded names readable until the next sfb_trace_begin. */
int sfb_trace_begin(unsigned long long* device_buf, unsigned int capacity);
int sfb_trace_end(void);
int sfb_trace_names(char* out, int capacity);
/* phase stamps inside the wgmma convolution (CTA 0 of every launch): device_buf[0] = launches seen, device_buf[1 + 8*i + p] = %globaltimer
 * of phase p (0 entry, 1 prologue done, 2 dependency wait returned, 3 first stage converted, 4 last MMA committed, 5 accumulator complete,
 * 6 epilogue done) of launch i < capacity.  NULL unbinds. */
int sfb_conv_phase_trace(unsigned long long* device_buf, unsigned int capacity);
/* optional code paths (default all on): bit 0 = the NGP MLP weight gradients run as 3xTF32 wgmma GEMMs over the feature-major tapes
 * (cleared: the fp32 SIMT outer-product kernel); bit 1 = batch-1 GroupNorm as ONE launch with a software grid barrier between the statistics
 * and the normalisation (cleared: statistics kernel + apply kernel).  Variants agree to fp32 rounding; the switch exists for A/B measurement and tests. */
int sfb_set_fusion(int mask);
/* number of kernels this library has launched so far in this process (bench.py's "gpu_launches") */
uint64_t sfb_launch_count(void);

/* ============================================================================================
 * 1. `_gridencoder` operator module      (external/gridencoder/src/bindings.cpp:5-8)
 * ========================================================================================== */

/* grid_encode_forward  -- gridencoder.h:12, gridencoder.cu:424-447 (kernel_grid :75-223).
 * inputs [B,D] in [0,1]; embeddings [rows,C]; offsets [L+1] int32; outputs [L,B,C] (pre-allocated);
 * S = log2(per_level_scale); H = base resolution; dy_dx [B,L*D*C] or NULL;
 * gridtype 0 = hash, 1 = tiled.  D in 1..5, C in {1,2,4,8} as in the reference. */
int sfb_grid_encode_forward(const float* inputs, const float* embeddings, const int32_t* offsets, float* outputs,
                            uint32_t B, uint32_t D, uint32_t C, uint32_t L, float S, uint32_t H, float* dy_dx,
                            uint32_t gridtype, int align_corners, void* stream);

/* grid_encode_backward -- gridencoder.h:13, gridencoder.cu:449-479 (kernel_grid_backward :226-313,
 * kernel_input_backward :316-342).  grad [L,B,C]; grad_embeddings [rows,C] must be pre-ZEROED by the
 * caller (grid.py:72); dy_dx / grad_inputs [B,D] may both be NULL. */
int sfb_grid_encode_backward(const float* grad, const float* inputs, const float* embeddings, const int32_t* offsets,
                             float* grad_embeddings, uint32_t B, uint32_t D, uint32_t C, uint32_t L, float S,
                             uint32_t H, const float* dy_dx, float* grad_inputs, uint32_t gridtype,
                             int align_corners, void* stream);

/* Parity instrumentation (no reference counterpart): the per-level scale exactly as the device
 * computes it (gridencoder.cu:125, device exp2f) -> scales[L]; and the absolute embedding-row index of
 * every interpolation corner -> rows [L,B,2^D] int32 (-1 for out-of-range points), so that the
 * "bit-exact grid indexing" contract can be tested directly against the oracle. */
int sfb_grid_level_scales(uint32_t L, float S, uint32_t H, float* scales, void* stream);
int sfb_grid_corner_rows(const float* inputs, const int32_t* offsets, int32_t* rows, uint32_t B, uint32_t D,
                         uint32_t L, float S, uint32_t H, uint32_t gridtype, int align_corners, void* stream);

/* ============================================================================================
 * 2. `_raymarching` operator module      (raymarching/src/bindings.cpp:5-18, raymarching.h:7-17)
 *    Argument order is the reference's, with tensors replaced by device pointers.
 * ========================================================================================== */

/* raymarching.cu:148-156 (kernel :91-145).  rays_o/d [N,3], aabb [6] -> nears/fars [N]; misses get FLT_MAX */
int sfb_near_far_from_aabb(const float* rays_o, const float* rays_d, const float* aabb, uint32_t N, float min_near,
                           float* nears, float* fars, void* stream);
/* raymarching.cu:201-209 (kernel :162-198).  -> coords [N,2] */
int sfb_sph_from_ray(const float* rays_o, const float* rays_d, float radius, uint32_t N, float* coords, void* stream);
/* raymarching.cu:229-232 (kernel :214-226).  coords [N,3] int32 -> indices [N] int32 */
int sfb_morton3D(const int32_t* coords, uint32_t N, int32_t* indices, void* stream);
/* raymarching.cu:257-260 (kernel :237-254) */
int sfb_morton3D_invert(const int32_t* indices, uint32_t N, int32_t* coords, void* stream);
/* raymarching.cu:292-300 (kernel :267-289).  grid [N*8] floats -> bitfield [N] bytes */
int sfb_packbits(const float* grid, uint32_t N, float density_thresh, uint8_t* bitfield, void* stream);
/* raymarching.cu:482-490 (kernel :311-480).  grid = density bitfield [C*H^3/8]; xyzs/dirs [M,3], deltas [M,2],
 * rays [N,3] int32 (ray id, point offset, count), counter [2] int32 (points, rays; caller zeroes), noises [N] */
int sfb_march_rays_train(const float* rays_o, const float* rays_d, const uint8_t* grid, float bound, float dt_gamma,
                         uint32_t max_steps, uint32_t N, uint32_t C, uint32_t H, uint32_t M, const float* nears,
                         const float* fars, float* xyzs, float* dirs, float* deltas, int32_t* rays, int32_t* counter,
                         const float* noises, void* stream);
/* raymarching.cu:580-588 (kernel :500-577) */
int sfb_composite_rays_train_forward(const float* sigmas, const float* rgbs, const float* deltas, const int32_t* rays,
                                     uint32_t M, uint32_t N, float T_thresh, float* weights_sum, float* depth,
                                     float* image, void* stream);
/* raymarching.cu:685-693 (kernel :601-682).  grad_sigmas [M] / grad_rgbs [M,3] pre-zeroed by the caller */
int sfb_composite_rays_train_backward(const float* grad_weights_sum, const float* grad_image, const float* sigmas,
                                      const float* rgbs, const float* deltas, const int32_t* rays,
                                      const float* weights_sum, const float* image, uint32_t M, uint32_t N,
                                      float T_thresh, float* grad_sigmas, float* grad_rgbs, void* stream);
/* raymarching.cu:808-815 (kernel :700-805) */
int sfb_march_rays(uint32_t n_alive, uint32_t n_step, const int32_t* rays_alive, const float* rays_t,
                   const float* rays_o, const float* rays_d, float bound, float dt_gamma, uint32_t max_steps, uint32_t C,
                   uint32_t H, const uint8_t* grid, const float* nears, const float* fars, float* xyzs, float* dirs,
                   float* deltas, const float* noises, void* stream);
/* raymarching.cu:908-914 (kernel :818-905); in place on rays_alive / rays_t / weights_sum / depth / image */
int sfb_composite_rays(uint32_t n_alive, uint32_t n_step, float T_thresh, int32_t* rays_alive, float* rays_t,
                       const float* sigmas, const float* rgbs, const float* deltas, float* weights_sum, float* depth,
                       float* image, void* stream);

/* ============================================================================================
 * 3. VLDM UNet forward operators        (external/imagen_pytorch.py Unet, :1078-1671)
 *    Activations are NHWC fp32 ([NB,H,W,ld] with a channel stride `ld` so that a call can read or
 *    write a channel slice of a wider tensor).  The reference runs these as ~600 eager PyTorch
 *    launches per forward (cuDNN / cuBLAS in TF32); here they are the operators the host-side
 *    `Unet` module (sparsefusion_b200/imagen_pytorch.py) strings together.
 * ========================================================================================== */

/* nn.Conv2d / nn.Linear as implicit GEMM on wgmma tensor cores (tf32 inputs, fp32 accumulate), TMA-fed.
 * Stands in for Block.project (:652), res_conv (:708), Downsample (:608-610), PixelShuffleUpsample conv
 * (:586), CrossEmbedLayer convs (:1038), ChanFeedForward 1x1 convs (:957,:960), final_conv (:1386) and the
 * token projections of Attention / CrossAttention when there are many tokens.
 *   x        [NB,H,W,ldx] NHWC, Cin channels used          w_packed [Cout][KH*KW][ceil32(Cin)] (sfb_conv_weight_k floats per
 *   row; TF32-rounded, zero padded; tap-major then channel)          bias [Cout] or NULL          residual [NB,Ho,Wo,ldr] or NULL
 *   out      [NB,Ho,Wo,ldo]; accumulate != 0 adds into `out` (red.global.add) instead of storing
 *   splits   K-range split across CTAs (0 = choose so that ~all SMs stream weights); bn: N tile (0 = auto; 32/64/128/256)
 * stride 1 or 2, any odd/even kernel with symmetric `pad`.  Cin, Cout, ldx, ldo multiples of 4. */
int sfb_conv2d_nhwc_tf32(const float* x, int NB, int H, int W, int Cin, int64_t ldx, const float* w_packed, int Cout, int KH, int KW,
                         int stride, int pad, const float* bias, const float* residual, int64_t ldr, float* out, int64_t ldo,
                         int accumulate, int splits, int bn, void* stream);
/* same with `pad` zeros before the first and `pad_after` after the last row / column: ldm's Downsample pads (0,1,0,1) in front of a
 * stride-2 3x3 convolution (external/ldm/modules/diffusionmodules/model.py:73-75) */
int sfb_conv2d_nhwc_tf32_pad(const float* x, int NB, int H, int W, int Cin, int64_t ldx, const float* w_packed, int Cout, int KH, int KW,
                             int stride, int pad, int pad_after, const float* bias, const float* residual, int64_t ldr, float* out, int64_t ldo,
                             int accumulate, int splits, int bn, void* stream);
/* same with an optional pre-split copy of the weights: w_hi_lo = [2][Cout][sfb_conv_weight_k] with hi = bits & 0xFFFFE000 and lo = w - hi, or
 * NULL.  Used by the tensor-bound launches (more than 64 output pixels) in 3xTF32 mode: hi and lo tiles are TMA-loaded side by side and the
 * operand converter only handles the activation tile.  Weight-streaming launches (swap-AB) keep reading w_packed: they are HBM-bound and the
 * split copy would double their traffic. */
int sfb_conv2d_nhwc_tf32_ex(const float* x, int NB, int H, int W, int Cin, int64_t ldx, const float* w_packed, const float* w_hi_lo, int Cout, int KH,
                            int KW, int stride, int pad, int pad_after, const float* bias, const float* residual, int64_t ldr, float* out, int64_t ldo,
                            int accumulate, int splits, int bn, void* stream);
/* same kernel as a general GEMM whose K-major "weight" operand w [Cout][KH*KW*ceil32(Cin)] is NOT a parameter but the output of an earlier launch on the
 * same stream (q k^T and P v of the VAE's attention, ldm model.py:183-199): the kernel then does not prefetch it ahead of the programmatic-dependent-
 * launch wait.  With sfb_conv2d_nhwc_tf32_ex such an operand may be read before the kernel that produces it has run. */
int sfb_conv2d_nhwc_tf32_dyn(const float* x, int NB, int H, int W, int Cin, int64_t ldx, const float* w, int Cout, int KH, int KW, int stride, int pad,
                             int pad_after, const float* bias, const float* residual, int64_t ldr, float* out, int64_t ldo, int accumulate, int splits,
                             int bn, void* stream);
int sfb_conv_weight_k(int Cin, int KH, int KW);
/* per-launch CUDA-event timing of the conv kernel for the roofline line of bench.py (off by default; do not enable under graph capture) */
int sfb_conv_prof_enable(int on);
int sfb_conv_prof_collect(double* total_ms, int* launches, double* weight_bytes, double* flops);
/* 3xTF32 kernel generation: 2 (default) = swap-AB for <= 64 output pixels and pre-split weights where given; 1 = neither */
int sfb_conv_set_variant(int v);
/* experiment switch: encode activation/weight tensor maps as TFLOAT32 instead of FLOAT32 */
int sfb_conv_set_tma_tf32(int enable);

/* layout at the module boundary (the reference API is NCHW): NCHW [NB,C,H,W] <-> channel slice of NHWC */
int sfb_nchw_to_nhwc(const float* src, float* dst, int NB, int C, int H, int W, int64_t ld, int c_off, int round_tf32, void* stream);
int sfb_nhwc_to_nchw(const float* src, float* dst, int NB, int C, int H, int W, int64_t ld, void* stream);
/* torch.cat((x, skip * scale), dim=1) of the up path (:1639) */
int sfb_concat2_nhwc(const float* a, int C1, int64_t lda, const float* b, int C2, int64_t ldb, float scale_b, float* out, int64_t ldo,
                     int64_t npix, void* stream);
/* im2col of a 4-channel NHWC tensor (16-byte pixels): out[pixel][(ky*KW + kx)*4 + c] = x[pixel + (ky - pad, kx - pad)][c], zero outside and in the
 * tail up to ldo.  Turns the 4-latent-channel share of the CrossEmbed init convolutions (3x3 | 7x7 | 15x15, imagen_pytorch.py:1017-1042) into one
 * 1x1 convolution with K = 900 instead of three implicit GEMMs padded to 32 channels per tap. */
int sfb_im2col4_nhwc(const float* x, int64_t ldx, float* out, int64_t ldo, int NB, int H, int W, int KH, int KW, int pad, void* stream);
/* nn.SiLU + nn.PixelShuffle(2) of PixelShuffleUpsample (:588-592): y [NB,H,W,4*Co] -> out [NB,2H,2W,ldo] */
int sfb_pixel_shuffle_silu_nhwc(const float* y, float* out, int NB, int H, int W, int Co, int64_t ldo, void* stream);
/* Block: GroupNorm(G) -> optional FiLM (x*(scale+1)+shift, film rows [scale(C)|shift(C)] with row stride film_ld) -> optional SiLU (:654-661).
 * stats_ws: sfb_groupnorm_ws_floats(NB, G) floats of 16-byte aligned scratch (fp64 partial statistics per pixel slab).
 * Groups of >= 16 channels, batches of <= 4 images, tensors of <= 1 Mi elements, per-CTA slab of <= 16 float4 per thread: ONE launch, one
 * thread-block cluster of <= 8 CTAs per (image, group), partial sums exchanged through distributed shared memory.  Otherwise two launches
 * (row-coalesced statistics kernel + apply kernel; the apply pass keeps one float4 column per thread when C/4 divides 256).
 * counters: unused since ABI 3 (round 1's single-launch variant met at a software grid barrier through these words); pass NULL.
 * Output is TF32-rounded in single-pass mode (it feeds the conv). */
int sfb_groupnorm_nhwc(const float* x, int64_t ldx, int NB, int HW, int C, int G, const float* gamma, const float* beta, const float* film,
                       int64_t film_ld, int act_silu, float eps, float* stats_ws, unsigned int* counters, float* y, int64_t ldy,
                       void* stream);
int sfb_groupnorm_ws_floats(int NB, int G);
/* LayerNorm / ChanLayerNorm (:301-329; gain g, optional bias b for nn.LayerNorm) over the last dim of [T,C] rows,
 * optionally of GELU(x) (ChanFeedForward :958-959), optionally + res (the `attn(x) + x` of :986) */
int sfb_layernorm_rows(const float* x, int64_t ldx, const float* g, const float* b, const float* res, int64_t ldr, float* y, int64_t ldy, int T,
                       int C, int pre_gelu, int round_tf32, void* stream);
/* nn.Linear for few rows (time MLPs :683-686, to_time_* :1175-1190, GlobalContext.net :929-934, token projections at 4x4):
 * y = post(bias + pre(x) W^T) + res; pre 0|1(SiLU), post 0|1(SiLU)|2(sigmoid); W [O,K] row-major (nn.Linear layout) */
int sfb_linear_small(const float* x, int64_t ldx, const float* w, const float* bias, const float* res, int64_t ldr, float* y, int64_t ldy,
                     int M, int K, int O, int pre, int post, int round_tf32, void* stream);
/* LearnedSinusoidalPosEmb (:634-639): out [B, 2*half+1] */
int sfb_time_fourier(const float* t, const float* w, float* out, int B, int half, void* stream);
/* softmax(QK^T)V cores: multi-query self attention with null and context keys (:517-566) and cross attention (:770-805).
 * sfb_mq_attention stages the keys / values of an image in shared memory (one warp per query up to 64 keys, a lane per key beyond: the 259 keys
 * of the 128x128-latent configuration); key sets that do not fit 200 KB fall back to a global-memory kernel. */
int sfb_mq_attention(const float* q, const float* kv, const float* null_kv, const float* ckv, float* out, int B, int n, int heads, int dh,
                     int nc, float scale, void* stream);
int sfb_cross_attention(const float* q, const float* kvc, const float* null_kv, float* out, int B, int n, int heads, int dh, int nc,
                        float scale, void* stream);
/* GlobalContext (:936-940): pooled[n][c] = sum_p softmax_p(to_k(x))[p] x[n][p][c]; logits_ws NB*HW + 2*NB + 2 floats.
 * From 4 096 pixels per image on, the pixels of a 16-channel slice are split over an 8-CTA cluster and merged through distributed shared memory. */
int sfb_gca_pool(const float* x, int64_t ldx, int NB, int HW, int C, const float* wk, const float* bk, float* logits_ws, float* pooled,
                 void* stream);
/* the same tail with GlobalContext's last layer folded in: gate[n][c] = sigmoid(b2[c] + w2[c][:] . hid[n][:]) (Conv2d(hidden, dim_out, 1) +
 * Sigmoid, :929-933), out = h * gate + res.  hid [NB][Hd], w2 [C][Hd]. */
int sfb_gate_mlp_residual_nhwc(const float* h, int64_t ldh, const float* hid, const float* w2, const float* b2, int Hd, const float* res, int64_t ldr,
                               float* out, int64_t ldo, int NB, int HW, int C, void* stream);
/* VAE (SURVEY section 8f row 1) helpers.  softmax over the columns of every row of scale * x (ldm AttnBlock, model.py:183-190);
 * nearest-neighbour x2 upsampling in NHWC (ldm Upsample, model.py:44-52). */
int sfb_softmax_rows(const float* x, int64_t ldx, float* y, int64_t ldy, int rows, int cols, float scale, void* stream);
int sfb_upsample2x_nhwc(const float* x, int64_t ldx, float* out, int64_t ldo, int NB, int H, int W, int C, void* stream);
/* ResnetBlock tail (:727-729): out = h * gate[n][c] + res (gate NULL == 1) */
int sfb_gate_residual_nhwc(const float* h, int64_t ldh, const float* gate, const float* res, int64_t ldr, float* out, int64_t ldo, int NB,
                           int HW, int C, void* stream);

/* PLMSSampler.p_sample tail (external/plms.py:143-154, :183-212) as one elementwise pass over the latent:
 *   e' = c0*e0 + c1*e1 + c2*e2 + c3*e3 (e1..e3 may be NULL);  x0 = clamp((x - sigma*e') / max(alpha,1e-8), +-clip);
 *   x_prev = alpha_next * (x*(1-c)/alpha + c*x0) + noise_scale * noise.   x0_out / e_out may be NULL.
 * The clamp keeps NaN, as torch.clamp does: a NaN eps or x gives a NaN x0 and x_prev, never a value at +-clip. */
int sfb_plms_update(const float* x, const float* e0, const float* e1, const float* e2, const float* e3, float c0, float c1, float c2,
                    float c3, const float* noise, float alpha, float sigma, float alpha_next, float c, float noise_scale, float clip,
                    float* x_prev, float* x0_out, float* e_out, int64_t n, void* stream);
/* sfb_plms_update for a batch whose rows follow their own noise schedules (scene-batched sampling, PLMSSampler.sample_rows):
 * row_scalars [rows][5] = (alpha, sigma, alpha_next, c, noise_scale) of each row's own (t, t_next); every other argument as
 * sfb_plms_update, with x / eps / noise / outputs holding `rows` contiguous rows of row_len floats (rows <= 65535).  Row r's result is
 * bit-identical to sfb_plms_update on that row with its scalars. */
int sfb_plms_update_rows(const float* x, const float* e0, const float* e1, const float* e2, const float* e3, float c0, float c1, float c2,
                         float c3, const float* noise, const float* row_scalars, float clip, float* x_prev, float* x0_out,
                         int rows, int64_t row_len, void* stream);
/* sfb_plms_update_rows with classifier-free guidance (PLMSSampler.sample with cond_scale != 1): the step's new eps is
 *   e_t = e_null + (e_cond - e_null) * cond_scale   (imagen_pytorch.py:572-577, rounded without contraction)
 * and takes e0's place in e' = c0*e_t + c1*e1 + c2*e2 + c3*e3.  e_out (may be NULL) receives e_t, the eps the sampler keeps in its history.
 * e_cond / e_null hold `rows` contiguous rows each (the conditional and null halves of one batch-2*rows UNet evaluation). */
int sfb_plms_update_rows_cfg(const float* x, const float* e_cond, const float* e_null, float cond_scale, const float* e1, const float* e2,
                             const float* e3, float c0, float c1, float c2, float c3, const float* noise, const float* row_scalars, float clip,
                             float* x_prev, float* e_out, int rows, int64_t row_len, void* stream);

/* DDPM.forward_noloss (sparsefusion/vldm.py:632-709, the one-step target) for `rows` contiguous rows of row_len floats (rows <= 65535), each
 * at its own noise level: log_snr [rows] is the DEVICE array of the rows' fp32 log-SNR (alpha_cosine_log_snr of their times, evaluated by
 * torch, the value the UNet is conditioned on), so nothing is read back to the host.  alpha = sqrt(sigmoid(ls)), sigma = sqrt(sigmoid(-ls)).
 * Products, sums and quotients are rounded one by one, as torch evaluates these expressions.
 * q_sample (imagen_pytorch.py:260-269): x_noisy = alpha*x_start + sigma*noise;  alpha_cumprod [rows] (may be NULL) = sigmoid(ls). */
int sfb_ddpm_q_sample_rows(const float* x_start, const float* noise, const float* log_snr, int rows, int64_t row_len, float* x_noisy,
                           float* alpha_cumprod, void* stream);
/* predict_start_from_noise + clamp (imagen_pytorch.py:293-297, vldm.py:700-701): eps = e_cond, or with e_null given (classifier-free
 * guidance: e_cond / e_null are the conditional and null halves of one batch-2*rows UNet evaluation)
 *   eps = e_null + (e_cond - e_null) * cond_scale   (rounded without contraction, as sfb_plms_update_rows_cfg);
 * eps_out (may be NULL) receives eps;  x0_out = clamp((x_noisy - sigma*eps) / max(alpha, 1e-8), +-clip), keeping NaN as torch.clamp does. */
int sfb_ddpm_predict_x0_rows(const float* x_noisy, const float* e_cond, const float* e_null, float cond_scale, const float* log_snr, float clip,
                             int rows, int64_t row_len, float* eps_out, float* x0_out, void* stream);

/* One step of DDPM.p_sample with dynamic thresholding (sparsefusion/vldm.py:289-361), B rows of row_len floats (row_len <= 65536):
 *   e = cond_scale*e_cond + (1-cond_scale)*e_null (e_null may be NULL: e = e_cond);  x0 = (x - sigma*e) / max(alpha,1e-8);
 *   s = max(torch.quantile(|x0|, percentile, 'linear'), 1) per row, computed exactly;  x0 = clamp(x0, +-s) / s;
 *   x_prev = alpha_next * (x*(1-c)/alpha + c*x0) + noise_scale * noise.
 * NaN follows torch: a row whose x0 holds a NaN has s = NaN and an all-NaN x_prev.
 * s_out [B] receives s, x0_out the unthresholded x0; either may be NULL.  x_prev must not alias the inputs. */
int sfb_ddpm_dynamic_step(const float* x, const float* e_cond, const float* e_null, float cond_scale, const float* noise, float alpha,
                          float sigma, float alpha_next, float c, float noise_scale, float percentile, int row_len, int B, float* x_prev,
                          float* s_out, float* x0_out, void* stream);

/* ============================================================================================
 * 4. Fused Instant-NGP field and optimiser   (external/nerf/network_grid.py NeRFNetwork, torch.optim.Adam)
 * ========================================================================================== */

/* NeRFNetwork.common_forward (network_grid.py:77-88) = GridEncoder (grid.py:138-154, the live tiled geometry: D=3, C=2, L=16)
 * + MLP 32-64-64-4 (:14-33) + trunc_exp(h0 + density blob) (:69-75, ngp_activation.py:10-21) + sigmoid(h1:4), in ONE kernel.
 * Points are either explicit (xyz [B,3], world coordinates in [-bound, bound]) or implicit ray samples: xyz == NULL and
 * rays_o/rays_d [N,3], z [N*T] -> x = clamp(o + d*z, -bound, bound) exactly as renderer_df.py:367-368 computes it.
 * W0 [64,32], W1 [64,64], W2 [4,64] are nn.Linear weights (row-major [out,in]).  sigma [B]; rgb [B,3] or NULL. */
int sfb_ngp_field_forward(const float* xyz, const float* rays_o, const float* rays_d, const float* z, uint32_t T, uint32_t B,
                          const float* embeddings, const int32_t* offsets, float S, uint32_t H, float bound, const float* W0,
                          const float* b0, const float* W1, const float* b1, const float* W2, const float* b2, float* sigma, float* rgb,
                          void* stream);
/* Backward of the above w.r.t. every parameter (autograd through common_forward in the reference): grad_embeddings [rows,2]
 * and gW*, gb* are ACCUMULATED into (caller zeroes them, like grid.py:72); grad_rgb may be NULL.  `tape` is scratch of
 * sfb_ngp_field_tape_floats(B) floats (feature-major activation / pre-activation-gradient tapes for the weight gradients). */
int sfb_ngp_field_backward(const float* xyz, const float* rays_o, const float* rays_d, const float* z, uint32_t T, uint32_t B,
                           const float* embeddings, const int32_t* offsets, float S, uint32_t H, float bound, const float* W0,
                           const float* b0, const float* W1, const float* b1, const float* W2, const float* b2, const float* grad_sigma,
                           const float* grad_rgb, float* grad_embeddings, float* gW0, float* gb0, float* gW1, float* gb1, float* gW2,
                           float* gb2, float* tape, void* stream);
uint32_t sfb_ngp_field_tape_points(uint32_t B);
uint64_t sfb_ngp_field_tape_floats(uint32_t B);
/* Finite-difference normals of the field (network_grid.py:91-164) as stencils on the tiled field kernel: the stencil rows
 * (point, slot, jitter sample) are generated and reduced inside the kernel, so no 6B or 60B point array exists in memory.
 *   slots = 6: slot s shifts component s/2 by +eps (even s) or -eps (odd s) and clamps to [-bound, bound]; each slot is the mean
 *              of k samples.  fd [B,3] = 0.5 (sigma+ - sigma-) / eps and normal [B,3] = safe_normalize(fd), NaN -> 0 (either
 *              may be NULL).  k = 1 without a key: finite_difference_normal(x, eps); k = 10, eps = radius = 0.3:
 *              finite_difference_normal_smooth.
 *   slots = 1: common_forward_smooth(x, radius, k): sigma [B] and albedo [B,3] (or NULL), the means over k samples.
 * A sample adds the jitter (u radius) 2 - radius, not clamped, with u from Philox4x32-10 (counter (point, slot, sample, 0),
 * key = *key as two 32-bit words, low first; u = (r >> 8) 2^-24 of lanes 0..2); the blob is evaluated at the un-jittered point.
 * key is device memory (NULL: no jitter; required when k > 1).  slots * k <= 128.  Always the tiled kernels. */
int sfb_ngp_field_normal_forward(const float* xyz, const float* rays_o, const float* rays_d, const float* z, uint32_t T, uint32_t B,
                                 const float* embeddings, const int32_t* offsets, float S, uint32_t H, float bound, const float* W0,
                                 const float* b0, const float* W1, const float* b1, const float* W2, const float* b2, uint32_t slots,
                                 uint32_t k, float eps, float radius, const int64_t* key, float* fd, float* normal, float* sigma,
                                 float* albedo, void* stream);
/* Backward of the plain stencil (slots = 6, k = 1) w.r.t. every parameter, ACCUMULATED into caller-zeroed buffers like
 * sfb_ngp_field_backward.  Give grad_fd [B,3] (dL/dfd), or grad_normal [B,3] with the forward's fd [B,3]: the safe_normalize
 * backward, zero in components whose normal was NaN and for points whose fd is not finite. */
int sfb_ngp_field_normal_backward(const float* xyz, const float* rays_o, const float* rays_d, const float* z, uint32_t T, uint32_t B,
                                  const float* embeddings, const int32_t* offsets, float S, uint32_t H, float bound, const float* W0,
                                  const float* b0, const float* W1, const float* b1, const float* W2, const float* b2, float eps,
                                  const float* fd, const float* grad_normal, const float* grad_fd, float* grad_embeddings, float* gW0,
                                  float* gb0, float* gW1, float* gb1, float* gW2, float* gb2, void* stream);
/* The per-ray stages of NeRFRenderer.run (external/nerf/renderer_df.py:310-468), one warp per ray, for Tc = num_steps coarse and
 * Tf = upsample_steps importance samples per ray: num_steps >= 1, num_steps + upsample_steps <= 256 (a sorted slot index fits a uint8),
 * num_steps >= 2 when upsample_steps > 0.  Counts outside that return SFB_ERR_ARG.  get_default_torch_ngp_opt uses 64 + 64.
 * All random draws of the reference are inputs: noise [N,Tc] U(0,1) or NULL (perturb=False, :363); u [N,Tf] (torch.rand at :31, or the
 * deterministic linspace of :28 in eval mode).  lin = torch.linspace(0,1,Tc) (:356), passed in so depths are bit-identical to torch's
 * on CUDA tensors, where (far - near) / Tc is a multiplication by the fp32 reciprocal of Tc. */
/* :328 near/far + :356-364 stratified depths -> nears [N], fars [N], z [N,Tc] */
int sfb_ray_coarse_z(const float* rays_o, const float* rays_d, const float* aabb, float min_near, const float* lin, const float* noise,
                     uint32_t N, uint32_t num_steps, float* nears, float* fars, float* z, void* stream);
/* :381-395 (+ sample_pdf :15-49) + :404-405: coarse weights -> inverse-CDF samples -> merged, sorted depths z_sorted [N,Tc+Tf]
 * (ties: coarse first, then by index).  The pdf is over weights[1:-1] (Tc-2 bins); at Tc = 2 it has none and every importance sample
 * is z_mid[0], as in the reference.  Tf = 0 copies the coarse depths. */
int sfb_ray_resample(const float* z_coarse, const float* sigma_coarse, const float* nears, const float* fars, const float* u, int det,
                     uint32_t N, uint32_t num_steps, uint32_t upsample_steps, float* z_sorted, void* stream);
/* same, also returning the Tf importance depths in draw order (z_new [N,Tf]) and, per sorted slot, where it came from (src_of [N,Tc+Tf]
 * uint8: t < Tc = coarse sample t, Tc + t = importance sample t).  With sfb_ray_gather_sorted_steps the renderer evaluates the field once
 * per sample: coarse pass (sigma, rgb at the Tc stratified depths), importance pass (the Tf new depths), then this gather into sorted order. */
int sfb_ray_resample_ex(const float* z_coarse, const float* sigma_coarse, const float* nears, const float* fars, const float* u, int det, uint32_t N,
                        uint32_t num_steps, uint32_t upsample_steps, float* z_sorted, float* z_new, uint8_t* src_of, void* stream);
/* sigma [N,Tc+Tf], rgb [N,Tc+Tf,3] in sorted order from the coarse pass (sigma_coarse [N,Tc], rgb_coarse [N,Tc,3]) and the importance
 * pass (sigma_new [N,Tf], rgb_new [N,Tf,3]; may be NULL when Tf = 0) through src_of */
int sfb_ray_gather_sorted_steps(const uint8_t* src_of, const float* sigma_coarse, const float* rgb_coarse, const float* sigma_new, const float* rgb_new,
                                uint32_t N, uint32_t num_steps, uint32_t upsample_steps, float* sigma, float* rgb, void* stream);
/* the 64 + 64 case of sfb_ray_gather_sorted_steps: T must be 128 */
int sfb_ray_gather_sorted(const uint8_t* src_of, const float* sigma_coarse, const float* rgb_coarse, const float* sigma_new, const float* rgb_new,
                          uint32_t N, uint32_t T, float* sigma, float* rgb, void* stream);
/* :414-456 over T = Tc + Tf sorted samples, the last delta (far - near) / Tc: weights = alpha * cumprod(1 - alpha + 1e-15);
 * image [N,3] (+ (1-ws)*bg_color), depth [N], weights_sum [N].  Rays with near = far (missed) get depth 0. */
int sfb_ray_composite_forward_steps(const float* z_sorted, const float* sigma, const float* rgb, const float* nears, const float* fars,
                                    float bg_color, uint32_t N, uint32_t num_steps, uint32_t upsample_steps, float* image, float* depth,
                                    float* weights_sum, void* stream);
/* the 64 + 64 case of sfb_ray_composite_forward_steps: T must be 128 */
int sfb_ray_composite_forward(const float* z_sorted, const float* sigma, const float* rgb, const float* nears, const float* fars,
                              float bg_color, uint32_t N, uint32_t T, float* image, float* depth, float* weights_sum, void* stream);
/* what autograd derives for :414-456: grad_sigma [N,Tc+Tf], grad_rgb [N,Tc+Tf,3] from grad_image [N,3], grad_weights_sum / grad_depth [N]
 * or NULL; zero for missed rays */
int sfb_ray_composite_backward_steps(const float* z_sorted, const float* sigma, const float* rgb, const float* nears, const float* fars,
                                     float bg_color, uint32_t N, uint32_t num_steps, uint32_t upsample_steps, const float* grad_image,
                                     const float* grad_weights_sum, const float* grad_depth, float* grad_sigma, float* grad_rgb, void* stream);
/* the 64 + 64 case of sfb_ray_composite_backward_steps: T must be 128 */
int sfb_ray_composite_backward(const float* z_sorted, const float* sigma, const float* rgb, const float* nears, const float* fars,
                               float bg_color, uint32_t N, uint32_t T, const float* grad_image, const float* grad_weights_sum,
                               const float* grad_depth, float* grad_sigma, float* grad_rgb, void* stream);

/* torch.optim.Adam.step for one parameter tensor (sparsefusion/distillation.py:165,246,352): no weight decay / amsgrad.
 * grad is multiplied by grad_scale first (1/world_size after a sum all-reduce). step >= 1 is the step count after increment. */
int sfb_adam_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n, float lr, float beta1, float beta2,
                  float eps, int step, float grad_scale, void* stream);

/* ==========================================================================================
 * section 6 -- ray generation and image-space glue of a distillation step (SURVEY.md section 8f row 2)
 *    Replaces ~50 eager launches per sub-step of sparsefusion/distillation.py:201-241, :274-288, :307-344 (+ utils/common_utils.py:183-190,
 *    utils/render_utils.py:40-47) and autograd's backward of them.  img [h*w, 3] pixel-major rendered colours, sil [h*w] opacity;
 *    full-resolution tensors are planes [C][H][W] of one view.
 * ========================================================================================== */
/* rays of the pixel-centre NDC grid (x, y from 1 - 1/W to -1 + 1/W), un-normalised directions on the plane at depth 1 (pytorch3d ray sampler
 * semantics, SURVEY section 8c): cam = centre[3] | R[9] with rows (right, up, forward); rays_o / rays_d [H*W, 3]. */
int sfb_rays_from_camera(const float* cam, int H, int W, float focal_ndc, float* rays_o, float* rays_d, void* stream);
/* photometric sub-step (distillation.py:210-234): value and gradient in one launch.  rgb [3][h*scale][w*scale], mask [1][h*scale][w*scale]
 * (sampled 'nearest' at stride `scale`); sums[3] <- (sum huber colour, sum huber silhouette, sum sqrt(sil^2 + .01)) so that
 * loss = lc * sums[0] / (3 h w) + ls * sums[1] / (h w) + lo * sums[2] / (h w); g_img [h*w,3] and g_sil [h*w] = d loss / d (img, sil). */
int sfb_photometric_loss(const float* img, const float* sil, const float* rgb, const float* mask, int h, int w, int scale, float lambda_color,
                         float lambda_sil, float lambda_opacity, float* sums, float* g_img, float* g_sil, void* stream);
/* up [4][2h][2w]: bilinear x2 (align_corners = False) of the three colour planes and of the opacity (distillation.py:287-288), NCHW for the VAE */
int sfb_upsample2x_render(const float* img, const float* sil, int h, int w, float* up, void* stream);
/* fusion sub-step loss on the up-sampled planes and its gradient back at render resolution (through the adjoint of the bilinear x2).
 * mode 0 (SDS, :310): weight * mean |up_rgb - target| + lo * mean sqrt(up_sil^2 + .01); mode 1 (EFT bootstrap, :316-329): lc * mean huber(up_rgb,
 * target) + ls * mean huber(up_sil, mean_c target > .1) + the same opacity term.  sums[3] as above (colour, silhouette, opacity sums over H*W
 * resp. 3*H*W elements); g_up [4][H][W] scratch; g_img [h*w,3], g_sil [h*w] outputs. */
int sfb_fusion_loss(const float* up, const float* target, int H, int W, int mode, float weight, float lambda_color, float lambda_sil,
                    float lambda_opacity, float* sums, float* g_up, int h, int w, float* g_img, float* g_sil, void* stream);
/* same, with an extra gradient g_extra [3][H][W] w.r.t. the up-sampled colour planes (the perceptual term's, already scaled by its lambda) added
 * before the adjoint of the bilinear up-sampling */
int sfb_fusion_loss_ex(const float* up, const float* target, int H, int W, int mode, float weight, float lambda_color, float lambda_sil,
                       float lambda_opacity, const float* g_extra, float* sums, float* g_up, int h, int w, float* g_img, float* g_sil, void* stream);
/* the two sub-steps' losses with the entropy regulariser (distillation.py:236-241, :338-344): + lambda_entropy * mean H(a), a = clamp(sil,
 * 1e-5, 1 - 1e-5), H(a) = -a log2 a - (1 - a) log2 (1 - a), over the render's opacity (photometric) or the up-sampled one (fusion, its
 * gradient through the same bilinear adjoint).  sums[4]: the three sums above and sums[3] = sum H.  d/dsil of the term is zero where the
 * clamp moves sil (outside [1e-5, 1 - 1e-5]), as autograd's clamp backward.  Otherwise as sfb_photometric_loss / sfb_fusion_loss_ex. */
int sfb_photometric_loss_ent(const float* img, const float* sil, const float* rgb, const float* mask, int h, int w, int scale, float lambda_color,
                             float lambda_sil, float lambda_opacity, float lambda_entropy, float* sums, float* g_img, float* g_sil, void* stream);
int sfb_fusion_loss_ent(const float* up, const float* target, int H, int W, int mode, float weight, float lambda_color, float lambda_sil,
                        float lambda_opacity, float lambda_entropy, const float* g_extra, float* sums, float* g_up, int h, int w, float* g_img,
                        float* g_sil, void* stream);

/* ==========================================================================================
 * section 7 -- LPIPS-VGG perceptual term of the fusion loss (SURVEY.md section 8f row 3)
 *    sparsefusion/distillation.py:161, :312-314 -> external/external_utils.py:11-49 -> lpips.LPIPS(net='vgg') (third party, un-vendored:
 *    algorithm restated in oracle/lpips_oracle.py).  The 13 convolutions and their data-gradient convolutions use sfb_conv2d_nhwc_tf32_ex;
 *    these are the NHWC fp32 operators around them.  sparsefusion_b200/lpips_vgg.py strings them together (value + gradient w.r.t. pred).
 * ========================================================================================== */
/* x [2][H][W][4] <- ((2 v - 1 if normalize) - shift) / scale of pred (image 0) and target (image 1), both [3][H][W] planes; channel 3 = 0 */
int sfb_lpips_prep(const float* pred, const float* target, int H, int W, int normalize, float* x, void* stream);
/* g_pred [3][H][W] <- factor * gx[pixel][c] * (2 if normalize) / scale[c]: adjoint of sfb_lpips_prep for image 0 (gx [H][W][4]) */
int sfb_lpips_prep_backward(const float* gx, int H, int W, int normalize, float factor, float* g_pred, void* stream);
int sfb_relu_nhwc(float* x, int64_t n, void* stream);
int sfb_maxpool2x2_nhwc(const float* x, float* y, int NB, int H, int W, int C, void* stream);
/* one image: gx [H][W][C] <- gy [H/2][W/2][C] routed to the first maximum of each 2x2 window of x (torch semantics), zero where that maximum is
 * not positive (x is a post-ReLU activation: this is the ReLU mask of the layer below) */
int sfb_maxpool2x2_relu_backward_nhwc(const float* x, const float* gy, float* gx, int H, int W, int C, void* stream);
/* g <- (g + g_head) * (act > 0), n floats; g_head may be NULL */
int sfb_add_relu_mask(float* g, const float* g_head, const float* act, int64_t n, void* stream);
/* one tap: f0, f1 [HW][C] feature maps of pred / target, w [C] the non-negative 1x1 `lin` weights.  *value += mean_p sum_c w_c (n0 - n1)^2 with
 * n = f / (||f||_2 + 1e-10) over channels; g_f0 [HW][C] <- d value / d f0 */
int sfb_lpips_head(const float* f0, const float* f1, const float* w, int HW, int C, float* value, float* g_f0, void* stream);

/* ==========================================================================================
 * section 8 -- Epipolar Feature Transformer operators (SURVEY.md section 8f row 4: the per-scene EFT feature cache)
 *    sparsefusion/eft.py:155-470 (encode / index / forward), called from sparsefusion/distillation.py:92-127 through
 *    utils/eft_renderer.py.  ResNet-18 convolutions (BatchNorm folded) and every nn.Linear of the three transformer encoders use
 *    sfb_conv2d_nhwc_tf32_ex; these are the NHWC fp32 operators around them.  sparsefusion_b200/eft.py strings them together.
 * ========================================================================================== */
/* torchvision resnet maxpool: 3x3 window, stride 2, padding 1; y [NB][(H+1)/2][(W+1)/2][C]; a NaN in a window gives NaN (F.max_pool2d) */
int sfb_maxpool3x3s2_nhwc(const float* x, float* y, int NB, int H, int W, int C, void* stream);
/* F.interpolate(mode='bilinear', align_corners=True) to (Ho, Wo), written with channel stride ldo (eft.py:194-202 pyramid concatenation) */
int sfb_resize_bilinear_ac_nhwc(const float* x, int64_t ldx, float* y, int64_t ldo, int NB, int H, int W, int C, int Ho, int Wo, void* stream);
/* F.grid_sample(mode='bilinear', padding_mode='border', align_corners=True) (eft.py:248-275): x [NB][H][W][C] (channel stride ldx),
 * grid [NB][M][2] = (x, y) in [-1, 1], out [NB][M][C] (row stride ldo) */
int sfb_grid_sample_nhwc(const float* x, int64_t ldx, const float* grid, float* out, int64_t ldo, int NB, int H, int W, int C, int64_t M, void* stream);
/* single-head attention core of nn.TransformerEncoderLayer(d_model E, nhead 1), sequence-first: qkv [S][B][3E] = in_proj(x) (q | k | v),
 * out [S][B][E] = softmax(q k^T / sqrt(E)) v over the S <= 32 positions of each batch element (eft.py:30-33: S = input views or depth samples) */
int sfb_seq_attention(const float* qkv, float* out, int S, int B, int E, void* stream);
/* in place over n floats (n % 4 == 0): kind 0 ReLU (NaN stays NaN, as F.relu), 1 GELU (erf) */
int sfb_act_inplace(float* x, int64_t n, int kind, void* stream);
/* the T1 token rows of the view-batched feature cache (eft.py:215-327, what EpipolarFeatureTransformer.forward assembles in eager passes), for
 * V query views with their own NC input cameras each: cams [V][NC][16] = R row-major (9) | T (3) | focal (2) | principal point (2) in pytorch3d's
 * NDC row-vector convention; origins / directions [V][N][3], lengths [V][N][D]; latent [NC][h][w] (channel stride ldl, C channels) and images
 * [NC][H][W] (channel stride ldi, Ci channels) NHWC.  Row (c, v, n, d) of out [NC][V*N*D][ldo] (ldo >= 91 + C + Ci) gets, for the point
 * x = o + l d: the reference Pluecker harmonic embedding (78) of (u, centre_c x u), u = normalize(x - centre_c); the depth harmonic embedding
 * (13) of l; the bilinear look-ups (sfb_grid_sample_nhwc semantics) of the latent and the images at minus the NDC projection of x by camera
 * (v, c); zeros up to ldo.  Harmonics: [sin(x f_k), cos(x f_k), x], f_k = omega0 2^k, k < 6. */
int sfb_eft_t1_tokens(const float* cams, const float* origins, const float* directions, const float* lengths, const float* latent, int64_t ldl,
                      int h, int w, int C, const float* images, int64_t ldi, int H, int W, int Ci, float omega0, float* out, int64_t ldo, int V,
                      int NC, int N, int D, void* stream);

/* ==========================================================================================
 * section 8b -- ray grids of the per-scene preparation (sparsefusion/distillation.py:85-86 through utils/render_utils.py:16-65)
 * ========================================================================================== */
/* pytorch3d GridRaysampler rays of V cameras in one launch: cams [V][16] as for sfb_eft_t1_tokens; the H x W NDC grid x_j = linspace(min_x,
 * max_x, W)[j], y_i = linspace(min_y, max_y, H)[i]; p1, p2 = the pixel unprojected at depths 1 and 2; rays_d = p2 - p1 (not normalised),
 * rays_o = p1 - rays_d; rays_o / rays_d [V][H*W][3], row-major pixels (_xy_to_ray_bundle). */
int sfb_grid_rays(const float* cams, int V, int H, int W, float min_x, float max_x, float min_y, float max_y, float* rays_o, float* rays_d,
                  void* stream);

/* ==========================================================================================
 * section 9 -- mesh extraction from a density lattice (NeRFRenderer.export_mesh, external/nerf/renderer_df.py:121-153)
 *    Volumes are fp32 [X][Y][Z] row-major (i slowest, k fastest); axis order (i, j, k) = (x, y, z).
 * ========================================================================================== */
/* scipy.ndimage.gaussian_filter(v, sigma) with its defaults: three separable passes of exp(-x^2 / 2 sigma^2) taps normalised to sum 1,
 * radius int(4 sigma + 0.5), mode 'reflect' (half-sample symmetric, folded as often as an axis shorter than the radius needs); fp32 with
 * fp32 accumulation.  in, out, tmp: X*Y*Z floats, three distinct buffers.  0 < sigma, radius <= 32. */
int sfb_gaussian_filter3d(const float* in, float* out, float* tmp, int X, int Y, int Z, float sigma, void* stream);
/* population mean and standard deviation (ddof = 0) of n floats, accumulated in fp64 in a fixed order: out2 [2] doubles = (mean, std).
 * work: SFB_VOLUME_STATS_WORK doubles of scratch (the per-CTA partial sums). */
#define SFB_VOLUME_STATS_WORK 1024
int sfb_volume_mean_std(const float* v, int64_t n, double* out2, double* work, void* stream);
/* Marching cubes at isovalue iso, in two phases around one host read of the counts.  A corner is below when v <= iso; an edge crosses when
 * one end is below.  Vertices: one per crossing lattice edge, at p0 + t (p1 - p0), t = (iso - v0) / (v1 - v0), p0 the lower-index end, in
 * index units; ordered by lattice point (i slowest, k fastest), then owned edge (+i, +j, +k).  Triangles: int32 vertex indices, ordered by
 * cell (same order) and then the triangle table (sparsefusion_b200/csrc/mc_tables.cuh); each face's normal points toward decreasing value.
 * Output is a pure function of the volume (no atomics).  Lattices of 1..SFB_MC_MAX_AXIS points per axis.
 *   scratch: sfb_marching_cubes_scratch_bytes(X, Y, Z) bytes (0 = lattice out of range), shared by the two phases.
 *   count:   counts [2] int64 (device) <- (V, F).
 *   emit:    verts [V,3] fp32, tris [F,3] int32 (either may be NULL when its count is 0; V must be below 2^31). */
#define SFB_MC_MAX_AXIS 1024
uint64_t sfb_marching_cubes_scratch_bytes(int X, int Y, int Z);
int sfb_marching_cubes_count(const float* v, int X, int Y, int Z, float iso, void* scratch, int64_t* counts, void* stream);
int sfb_marching_cubes_emit(const float* v, int X, int Y, int Z, float iso, const void* scratch, float* verts, int32_t* tris, void* stream);

/* ==========================================================================================
 * section 10 -- image metrics of a scored scene (sparsefusion/distillation.py:391-443 via utils/common_utils.py:48-64: scikit-image SSIM / PSNR)
 *    Images are fp32 [B][H][W][3] (a render's image [H*W,3] in row-major pixel order, so no transposes).
 * ========================================================================================== */
/* SSIM and mean squared error of B image pairs (a[b], b[b]) -> out [2B] doubles:
 *   out[2b]     skimage.metrics.structural_similarity(a, b, channel_axis=-1, data_range=1) as scikit-image >= 0.19 computes it for float32
 *               input: per channel, 7x7 uniform window (scipy.ndimage.uniform_filter, mode 'reflect': half-sample symmetric), sample
 *               covariance (49/48), C1 = 0.01^2, C2 = 0.03^2, the SSIM map in fp32 and its mean in fp64 over the interior (3 pixels cropped
 *               from every side); the three channel values are stored as fp32 and averaged in fp32, so the value is an fp32 number.
 *               Window sums are taken in fp64 and rounded to fp32 after each 1D pass, as scipy's line buffers do.
 *   out[2b+1]   mean of (a - b)^2 over every pixel and channel: fp32 differences and squares, fp64 sum (PSNR = 10 log10(1 / mse)).
 * Two launches: one CTA per (image, 32x32 output tile) writes four fp64 partial sums to work, then one CTA per image adds them in a fixed
 * order; no atomics, so repeated calls are bit-identical.  B >= 1, H >= 7, W >= 7 (scikit-image rejects a window larger than the image).
 *   work: sfb_image_ssim_psnr_work(B, H, W) doubles (0 = sizes rejected). */
uint64_t sfb_image_ssim_psnr_work(int B, int H, int W);
int sfb_image_ssim_psnr(const float* a, const float* b, int B, int H, int W, double* out, double* work, void* stream);

/* ==========================================================================================
 * section 11 -- GIF palettes of the sequence and circle-path gifs (sparsefusion/distillation.py:444-493, which leaves the quantisation to
 *    imageio / Pillow on the host).  Frames are uint8 [B][H][W][3]; each frame gets its own palette.
 * ========================================================================================== */
/* palette [B][256][3] (entries at or beyond ncolors[b] are zero), ncolors [B], indices [B][H][W] of B frames with 2 <= colors <= 256,
 * a pure function of the input, all integer arithmetic:
 *   1. histogram: a pixel's cell is (r>>3, g>>3, b>>3) of 32^3; per cell the pixel count n and the sums of the 8-bit r, g, b (uint32).
 *   2. median cut: a box is an inclusive cell range per axis, always shrunk to the bounding box of its non-empty cells; the first box holds
 *      every non-empty cell.  While there are fewer than `colors` boxes, the splittable box (some axis with hi > lo) with the largest pixel
 *      count, lowest index on ties, is split along its axis of largest hi - lo (ties in the order r, g, b) at the smallest t in [lo, hi-1]
 *      with 2 * (pixels in slices lo..t) >= n (t = hi-1 if there is none).  The lower part keeps the index, the upper part is appended,
 *      both shrunk.  It stops early when no box is splittable.
 *   3. palette: entry k = (2 S + N) / (2 N) per channel (box k's channel sum S over its pixel count N, rounded half up); ncolors = boxes.
 *   4. map: each pixel takes the entry of smallest squared RGB distance, the lowest index on ties.
 * Three launches (histogram, one CTA per frame for the cut, map).  B in 1..65535, H, W >= 1, H*W <= 16843009 (so that a channel sum fits
 * 32 bits).  work: sfb_palette_work_bytes(B, H, W) bytes (0 = sizes rejected), zeroed by the call itself. */
uint64_t sfb_palette_work_bytes(int B, int H, int W);
int sfb_palette_quantize(const uint8_t* rgb, int B, int H, int W, int colors, uint8_t* palette, int32_t* ncolors, uint8_t* indices, void* work,
                         void* stream);

/* ==========================================================================================
 * section 12 -- albedo texture of an extracted mesh (NeRFRenderer.export_mesh(texture_size=T); the reference's textured export,
 *    external/nerf/renderer_df.py:166-306, is never called there and needs xatlas and nvdiffrast).  A T x T texture, texel (x, y) = column x,
 *    row y counted from the top; texel coordinates run over [0, T] with texel (x, y) covering [x, x+1) x [y, y+1).
 * ========================================================================================== */
/* Atlas of F triangles: n = ceil(sqrt(ceil(F / 2))) cells per row (1 when F = 0), cell size c = floor(T / n) texels.  Triangle t takes cell
 * k = t / 2 at texel (x0, y0) = ((k % n) c, (k / n) c), half h = t % 2.  Its UV corners in tris[t, 0..2] order, in texels from (x0, y0),
 * with m = 1/2 and d = 2:  h = 0: (m, m), (c-m-d, m), (m, c-m-d);  h = 1: (c-m, c-m), (m+d, c-m), (c-m, m+d).
 * Ownership: texel (x0 + i, y0 + j), 0 <= i, j < c, belongs to triangle 2k when (2i+1) + (2j+1) < 2c and to 2k+1 otherwise, if that
 * triangle exists; texels of unused cells and outside the n c square belong to none.  Every texel that a bilinear lookup at any point
 * of a triangle's UV region weights nonzero belongs to that triangle.
 * sfb_mesh_atlas_cell returns c, or 0 when c < SFB_TEXTURE_MIN_CELL or T is outside SFB_TEXTURE_MIN..SFB_TEXTURE_MAX (or F < 0). */
#define SFB_TEXTURE_MIN 16
#define SFB_TEXTURE_MAX 8192
#define SFB_TEXTURE_MIN_CELL 4
int sfb_mesh_atlas_cell(int F, int T);
/* uv [F][3][2] fp32 <- the UV corners above in texel units, (x0 + u, y0 + v); exact (half-integers below 2^13). */
int sfb_mesh_uv_atlas(int F, int T, float* uv, void* stream);
/* Texels of rows [row0, row0 + rows), row-major: owner [rows*T] int32 (-1 = none) and xyz [rows*T][3] fp32 (0 where there is no owner).
 * For an owned texel, p is the point of the owner's UV triangle closest to the texel centre (x + 1/2, y + 1/2) (the centre itself when
 * inside), lambda its barycentrics, and xyz = sum_i lambda_i verts[tris[t, i]].  verts [V][3] fp32 (world units), tris [F][3] int32 with
 * every index in 0..V-1 (not checked here); both may be NULL when F = 0. */
int sfb_mesh_texel_points(const float* verts, const int32_t* tris, int F, int T, int row0, int rows, int32_t* owner, float* xyz, void* stream);
/* out [n][3] uint8 <- trunc(255 rgb) where owner >= 0 (the reference's (feats * 255).astype(np.uint8)), 0 elsewhere.  rgb [n][3] fp32 in
 * [0, 1], as sfb_ngp_field_forward writes it. */
int sfb_mesh_texture_pack(const int32_t* owner, const float* rgb, int64_t n, uint8_t* out, void* stream);

/* ==========================================================================================
 * section 13 -- digest of a device buffer (the scene-cache check of a resumed distillation: sparsefusion_b200/distillation.py
 *    cache_digest; the reference has no checkpoint of its distillation loop)
 * ========================================================================================== */
/* out [1] uint64 <- sum over i < n_words of mix(w[i] ^ mix(i + 0x9E3779B97F4A7C15)) modulo 2^64, w = data as uint32 words, mix = splitmix64's
 * finaliser (x ^= x >> 30; x *= 0xBF58476D1CE4E5B9; x ^= x >> 27; x *= 0x94D049BB133111EB; x ^= x >> 31).  Independent of launch geometry
 * and atomic order.  out is zeroed on `stream` first; data may be NULL when n_words = 0. */
int sfb_digest_u32(const void* data, int64_t n_words, uint64_t* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SPARSEFUSION_B200_H */
