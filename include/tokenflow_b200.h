/* tokenflow_b200 — C ABI of the H100-native TokenFlow hot path.
 *
 * The reference (omerbt/TokenFlow @ 5dd6a69) is pure Python and has no FFI layer; its boundary for
 * this path is the hook surface of tokenflow_utils.py.  This library is what a replacement for those
 * hooks binds (ctypes stub shown in INTEGRATION.md; `tokenflow_b200/ops.py` is that stub in
 * product form).  Every entry point cites the reference lines whose arithmetic it replaces.
 *
 * Conventions
 *   - plain C: raw device pointers, explicit shapes/strides, an opaque CUDA stream handle
 *     (`cudaStream_t`; pass `torch.cuda.current_stream().cuda_stream`).  No torch types.
 *   - every function returns an int status: 0 = ok, nonzero = error (tf_last_error() explains).
 *     Nothing throws, nothing allocates device memory, nothing synchronises the device: work is
 *     enqueued on `stream` and the caller owns every buffer.
 *   - "host" pointers are read synchronously during the call (small per-frame tables passed to the
 *     kernels by value); "device" pointers must be valid on the current device.
 *   - fp16 activations, int32 indices.  dim and head_dim must be multiples of 8; device pointers to
 *     activations, outputs and workspaces 16-byte aligned (a misaligned one is refused with
 *     TF_ERR_INVALID_ARGUMENT before anything is enqueued); coefficient rows, index tables and the
 *     buffers documented "any alignment" need only their element's alignment; tensors contiguous
 *     unless a stride argument says otherwise.
 *   - compiled for sm_90a only; the kernels use wgmma / TMA / mbarrier.
 */
#ifndef TOKENFLOW_B200_H_
#define TOKENFLOW_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* tf_stream_t; /* cudaStream_t */

#define TF_MAX_FRAMES 64        /* frames per kernel launch; tf_nn_field / tf_propagate take any F and chunk */
#define TF_MAX_ATTN_SAMPLES 160 /* output samples (stream, keyframe) per kernel launch; calls take any number */

/* Library ABI version (major*1000 + minor). */
int tf_version(void);
/* Thread-local description of the last error returned on this thread ("" if none). */
const char* tf_last_error(void);
/* Number of kernel launches enqueued by this library since load (all threads); bench.py reports
 * the per-step difference as `gpu_launches`. */
int64_t tf_launch_count(void);

/* Row L2-normalisation feeding the NN field:  out[r,:] = fp16(x[r,:] / ||x[r,:]||_2).
 * Replaces util.py:66-67 (`x / x.norm(dim=-1, keepdim=True)`, fp32 under autocast) plus the fp16
 * operand cast autocast applies to the following matmul (util.py:68).
 *   x            device, [rows, dim] fp32 (x_is_f32 != 0) or fp16, row pitch `x_row_stride` elements
 *   out_f16      device, [rows, dim] fp16, contiguous */
int tf_unit_rows(const void* x, int x_is_f32, int64_t rows, int dim, int64_t x_row_stride, void* out_f16,
                 tf_stream_t stream);

/* norm1 fused with the row normalisation, for the frame pass: out = fp16(LN(x) / ||LN(x)||_2) with the
 * LayerNorm evaluated in fp32 like autocast does (tokenflow_utils.py:323 norm1 + util.py:66-67).  Only
 * the source stream's rows are needed there (reference :335), so callers pass that third only.
 *   x_f16        device [rows, dim] fp16, row pitch `x_row_stride` elements (multiple of 8)
 *   gamma, beta  device [dim] fp32 (norm1.weight / norm1.bias), eps = norm1.eps
 *   out_f16      device [rows, dim] fp16 contiguous;  dim <= 1280 */
int tf_layernorm_unit_rows(const void* x_f16, int64_t rows, int dim, int64_t x_row_stride, const float* gamma,
                           const float* beta, float eps, void* out_f16, tf_stream_t stream);

/* norm1 of the PIVOTAL pass fused with both of its consumers (tokenflow_utils.py:323 -> :120-122 and
 * :326-327 + util.py:66-67): one read of hidden_states produces
 *   y_out     fp16(LN(x)) for every row — the operand autocast would cast for the to_q/to_k/to_v GEMMs
 *   unit_out  fp16(LN(x) / ||LN(x)||_2) for the first `unit_rows` rows (the source-stream samples: the
 *             pivot features the NN field correlates), from the unrounded fp32 LN like the reference
 * Either output may be NULL.  Outputs may be strided (packed all-gather buffers): row pitch in elements,
 * multiple of 8.  dim <= 1280. */
int tf_layernorm_rows(const void* x_f16, int64_t rows, int dim, int64_t x_row_stride, const float* gamma,
                      const float* beta, float eps, void* y_out_f16, int64_t y_row_stride, void* unit_out_f16,
                      int64_t unit_row_stride, int64_t unit_rows, tf_stream_t stream);

/* Token nearest-neighbour field.  Replaces tokenflow_utils.py:329-348 (+ util.py:68 `x @ y.T`,
 * fp16 output under autocast, and the two argmax reductions :340-343):
 *   idx_a[f,p] = argmax_c fp16( x_unit[f,p,:] . piv_unit[kf_a[f],c,:] )     first index on ties
 *   idx_b[f,p] = same against keyframe kf_b[f]            (skipped for frames with kf_b[f] < 0)
 *   ordered as torch.argmax orders them: a NaN similarity (the unit row of a zero token is NaN) ranks above
 *   every number and the first NaN wins, so a zero pivot token c gives c, a zero frame token 0
 *   x_unit    device [F, S, dim] fp16 unit rows (tf_unit_rows of the source-stream norm1 output)
 *   piv_unit  device [K, S, dim] fp16 unit rows of the cached source-stream pivot features
 *   kf_a,kf_b host   [F] keyframe ids in [0,K); reference batch i: kf_a = i, kf_b = i-1 (or -1)
 *   idx_a,idx_b device [F, S] int32 (idx_b may be NULL when no frame has a second keyframe) */
int tf_nn_field(const void* x_unit, const void* piv_unit, const int32_t* kf_a, const int32_t* kf_b, int F, int S,
                int dim, int K, int32_t* idx_a, int32_t* idx_b, tf_stream_t stream);

/* NN-indexed feature propagation.  Replaces tokenflow_utils.py:361-397 (keyframe slice, two
 * gathers, blend weights, blend, residual add):
 *   out[s,f,p,:] = w[f]*A[s,kf_a[f],idx_a[f,p],:] + (1-w[f])*A[s,kf_b[f],idx_b[f,p],:] (+ residual[s,f,p,:])
 *   (kf_b[f] < 0:  out = A[s,kf_a[f],idx_a[f,p],:] (+ residual))
 *   A         device [3, K, S, dim] fp16   (cached attn1 output of the pivotal pass, `kf_attn_output`)
 *   w         host   [F] fp32 blend weights (reference: sigmoid(d2/(d1+d2)), :375-383)
 *   residual  device [3, F, S, dim] fp16 or NULL  (the block's `hidden_states`, :396-397)
 *   out       device [3, F, S, dim] fp16 (out_is_f32 == 0) or fp32 (the reference's promoted dtype) */
int tf_propagate(const void* A, const int32_t* idx_a, const int32_t* idx_b, const int32_t* kf_a,
                 const int32_t* kf_b, const float* w, int F, int S, int dim, int K, const void* residual,
                 void* out, int out_is_f32, tf_stream_t stream);

/* Extended attention of one pivotal pass.  Replaces the body of the attn1 closure between the
 * q/k/v projections and `to_out` (tokenflow_utils.py:124-197 PnP flavour, :234-279 SDEdit flavour).
 *   q,k,v   device [3n, S, heads, d] fp16; consecutive tokens `tok_stride` elements apart (heads*d
 *           when contiguous, 3*heads*d for a fused qkv buffer); samples S*tok_stride apart
 *   out     device [3n, S, heads*d] fp16 contiguous
 *   inject  != 0: PnP q/k injection — uncond and cond samples read the source stream's q and k
 *           (reference :124-130) by aliasing, nothing is copied
 * Batch axis is [source | uncond | cond] thirds like the reference (:117).  Source samples attend
 * to their own frame, uncond/cond samples to all n frames of their stream. */
int tf_ext_attn_fwd(const void* q, const void* k, const void* v, int64_t tok_stride, int n_frames, int S,
                    int heads, int d, float scale, int inject, void* out, tf_stream_t stream);

/* General form: `n_out` output samples, each described by host arrays (all length n_out): which slab
 * of `out` it writes, which slab of q it reads, the first k / v slab it attends to and how many
 * consecutive slabs (1 = own frame, n = all keyframes).  q has q_slabs slabs of [S, heads, d]; k and
 * v have kv_slabs.  Only queries [q_row0, q_row0 + q_nrows) of every sample are computed (against all
 * keys), and `out` is [slabs, q_nrows, heads*d] with row = token - q_row0; q_row0 = 0, q_nrows = S is
 * the whole pass.  q_row0 must be a multiple of 128.  The multi-GPU pivotal pass splits the query
 * rows of ALL samples evenly over the ranks this way (every rank holds all K/V after the
 * all-gather), which balances the attention work exactly and keeps paired (q/k-injected) samples
 * together. */
int tf_ext_attn_fwd_rows(const void* q, int q_slabs, int64_t q_tok_stride, const void* k, const void* v,
                         int kv_slabs, int64_t kv_tok_stride, int n_out, const int32_t* out_slab,
                         const int32_t* q_slab, const int32_t* k_slab0, const int32_t* v_slab0,
                         const int32_t* n_kv, int S, int heads, int d, float scale, int q_row0, int q_nrows,
                         void* out, tf_stream_t stream);

/* Classifier-free guidance + DDIM update (eta = 0) of one denoising step, one pass over the latents.
 * Replaces run_tokenflow_pnp.py:213-217 (`u + g*(c - u)`, `scheduler.step(...)['prev_sample']`), with the
 * fp16 rounding sequence of the eager expression (bit-identical results).
 *   eps_uncond, eps_cond, x, out   device [n] fp16 contiguous (x = the latents being denoised)
 *   coef   device [4] fp32: sqrt(1-alpha_t), 1/sqrt(alpha_t), sqrt(alpha_prev), sqrt(1-alpha_prev) — in
 *          device memory so a captured CUDA graph of the step replays for every timestep */
int tf_cfg_ddim(const void* eps_uncond, const void* eps_cond, const void* x, const float* coef, float guidance,
                int64_t n, void* out, tf_stream_t stream);

/* Guidance-free DDIM update of the inversion stage (preprocess.py:217-225 inversion, :251-260 reconstruction),
 * the DDIM half of tf_cfg_ddim with the same fp16 rounding sequence:
 *     out = h( h(s3 * h( h(x - h(s1 * eps)) * inv_s2 )) + h(s4 * eps) )
 *   eps, x, out   device [n] fp16 contiguous; out == x (in place) is allowed
 *   coef   device [4] fp32 (s1, inv_s2, s3, s4): inversion (sigma_prev, 1/mu_prev, mu, sigma), reconstruction
 *          (sigma, 1/mu, mu_prev, sigma_prev) — in device memory so one captured graph serves every timestep and
 *          both directions */
int tf_ddim(const void* eps, const void* x, const float* coef, int64_t n, void* out, tf_stream_t stream);

/* The same two latent updates for v-prediction models (Stable Diffusion 2.x at 768 x 768, whose
 * scheduler_config.json says "prediction_type": "v_prediction").
 *
 * Such a UNet predicts the velocity v = sqrt(alpha) * eps - sqrt(1 - alpha) * x0 instead of the noise eps.  These
 * entry points are tf_cfg_ddim and tf_ddim with diffusers' v-branch of the DDIM step (DDIMScheduler.step /
 * DDIMInverseScheduler.step, eta = 0) in place of the eps formula.  Each operation is fp32 on fp16 operands and its
 * result is rounded to fp16 (h), as the eager fp16 expression rounds:
 *     p   = h( h(a * x) - h(b * v) )          (pred_x0)
 *     e   = h( h(a * v) + h(b * x) )          (pred_eps)
 *     out = h( h(c * p) + h(d * e) )
 * The coefficient row (a, b, c, d) is read from device memory, so one captured CUDA graph serves every timestep:
 *     edit step             sqrt(alpha_t), sqrt(1 - alpha_t), sqrt(alpha_prev), sqrt(1 - alpha_prev)
 *     inversion step        mu_prev, sigma_prev, mu, sigma
 *     reconstruction step   mu, sigma, mu_prev, sigma_prev
 * (mu = sqrt(alpha), sigma = sqrt(1 - alpha); the inversion's sample is at the level of `prev`, as in the reference's
 * eps loop, preprocess.py:211-225). */

/* Classifier-free guidance + v-parameterised DDIM update of one denoising step: v = h(u + h(g * h(c - u))), then the
 * update above.
 *   v_uncond, v_cond, x, out   device [n] fp16 contiguous (x = the latents being denoised)
 *   coef                       device [4] fp32: the edit step's row */
int tf_cfg_ddim_v(const void* v_uncond, const void* v_cond, const void* x, const float* coef, float guidance,
                  int64_t n, void* out, tf_stream_t stream);

/* Guidance-free v-parameterised DDIM update of the inversion stage, v = the model output.
 *   v, x, out   device [n] fp16 contiguous; out == x (in place) is allowed
 *   coef        device [4] fp32: the inversion or the reconstruction row */
int tf_ddim_v(const void* v, const void* x, const float* coef, int64_t n, void* out, tf_stream_t stream);

/* ---- UNet body (not part of the reference's hook surface: the Stable-Diffusion UNet it runs) ---- */

/* Channels-last GroupNorm fused with the time-embedding add before it and the SiLU after it:
 *   out[n,p,c] = [SiLU]( GroupNorm_groups( x[n,p,c] [+ bias[n,c]] ) * gamma[c] + beta[c] )
 * with the eager fp16 rounding sequence: x + bias rounded to fp16; mean, rstd = rsqrtf(var + fp16(eps)) rounded to
 * fp16 as ATen stores them; y = fp16(fmaf(rstd*gamma, x, beta - mean*rstd*gamma)) in fp32; SiLU of the fp16 y as
 * y / (1 + expf(-y)).  Statistics in fp64 over fp32 partials of shifted values;
 * deterministic (no atomics, fixed reduction order).  Two kernel launches.
 *   x, out       device [n, hw, c] fp16 dense NHWC (a channels_last [n, c, h, w] tensor), hw = h*w
 *   bias         device [n, c] fp16 or NULL; row pitch `bias_stride` elements (0 = one row for every sample)
 *   gamma, beta  device [c] fp16 (the GroupNorm's weight / bias)
 *   silu         != 0: apply SiLU
 *   workspace    device, >= tf_group_norm_nhwc_workspace(n, hw, c, groups) bytes, 16-byte aligned, uninitialised
 * c % 8 == 0 and groups | c (else TF_ERR_INVALID_ARGUMENT); c / groups == 4 or >= 8, and c <= 4096 (else unsupported).
 * Exactly 4 channels per group is the VAE's 128-channel levels with 32 groups (every 16-byte vector of 8 channels spans
 * two groups): the same rounding sequence and workspace format, but no bias add, so bias must be NULL there (else
 * unsupported). */
int64_t tf_group_norm_nhwc_workspace(int64_t n, int64_t hw, int c, int groups); /* bytes, or -1 for a bad shape */
int tf_group_norm_nhwc(const void* x, const void* bias, int64_t bias_stride, const void* gamma, const void* beta,
                       int64_t n, int64_t hw, int c, int groups, float eps, int silu, void* workspace,
                       int64_t workspace_bytes, void* out, tf_stream_t stream);

/* GEGLU gate of the transformer blocks' feed-forward: out = fp16(xh * fp16(gelu(gate))), gelu in ATen's erf form
 * (x/2 * (1 + erff(x / sqrt(2)))), so the result equals the eager `F.linear(x, w_x, b_x) * F.gelu(F.linear(x, w_g,
 * b_g))` bit for bit given the same GEMM outputs.
 *   xh, gate, out  device [n] fp16 contiguous */
int tf_geglu(const void* xh, const void* gate, int64_t n, void* out, tf_stream_t stream);

/* ---- pixels in and out of the VAE (the reference's frame loading and saving around encode / decode) ---- */

/* Encoder input from uint8 RGB frames: out = fp16(fp16(2 * fp16(v / 255)) - 1), the value of `2 * imgs - 1` on
 * `T.ToTensor()(frame).to(torch.float16)` (fp32 true quotient, rounded to fp16, then the fp16 multiply and subtract)
 * bit for bit.
 *   frames_u8   device [n_px, 3] uint8 ([N, H, W, 3] frames, n_px = N*H*W), 16-byte aligned
 *   out_f16     device [n_px, 3] fp16: a channels_last [N, 3, H, W] tensor, 16-byte aligned */
int tf_frames_to_nhwc(const void* frames_u8, int64_t n_px, void* out_f16, tf_stream_t stream);

/* uint8 frames from the decoder output: ((x / 2 + 0.5).clamp(0, 1) * 255).to(uint8) with every op rounded to fp16 and
 * truncation at the end, bit for bit; a NaN gives 0, +-Inf give 255 / 0.
 *   x_f16       device [n_px, 3] fp16 (a channels_last [N, 3, H, W] tensor), 16-byte aligned
 *   frames_u8   device [n_px, 3] uint8 ([N, H, W, 3]), 16-byte aligned */
int tf_nhwc_to_frames(const void* x_f16, int64_t n_px, void* frames_u8, tf_stream_t stream);

/* Pillow's `Image.resize((w, h), Image.LANCZOS)` of RGB uint8 frames, bit for bit (libImaging/Resample.c): the
 * reference's frame resize (util.py:28 to (W, H); run_tokenflow_pnp.py:174-175, run_tokenflow_sdedit.py:136-137,
 * preprocess.py:191-192 square frames to 512x512).  Per axis, Lanczos-3 weights in double, normalised and rounded to
 * int32 with 22 fractional bits; a horizontal pass into a uint8 intermediate, then a vertical pass, each value
 * clamp((2^21 + sum v * k) >> 22, 0, 255).  A frame more than 100 times taller than wide (h_in > 100 * w_in) whose
 * height shrinks goes through the vertical pass first, as Pillow 12 takes it.  A pass whose axis keeps its size is
 * skipped; equal sizes are a copy.
 * Sizes are in [1, 65536].
 *
 * tf_resize_taps      taps per output pixel of the table for one axis `in` -> `out` (-1 for bad sizes)
 * tf_resize_coeffs    fills that axis's tables on the host:
 *                       bounds  host [out, 2] int32: first input pixel, number of taps used (<= taps)
 *                       coeffs  host [out, taps] int32 fixed-point weights, zero past the used taps
 * tf_resize_u8        in [n, h_in, w_in, 3] -> out [n, h, w, 3], both device uint8, any alignment
 *   h_bounds, h_coeffs, h_taps   device copies of the tables for w_in -> w (unused, may be NULL, when w == w_in)
 *   v_bounds, v_coeffs, v_taps   the same for h_in -> h (unused when h == h_in)
 *   tmp                          device [n, h_in, w, 3] uint8 intermediate, used only when both axes change
 *                                ([n, h, w_in, 3] when the vertical pass goes first)
 * The device tables are trusted: they must be what tf_resize_coeffs wrote for the same sizes.  Each pass is one launch
 * of at most 2^31 - 1 blocks: the horizontal pass takes n*h_in / rows blocks (n*h / rows when it goes second; rows = 4
 * up to w_in = 4090, 3, 2, then 1 from w_in = 8187), the vertical one n*h*ceil(3w / 2048) (w_in for w when it goes
 * first; ceil(3w / 512) unless w % 16 == 0 and its input and output are 16-byte aligned); a call past either is
 * refused (TF_ERR_UNSUPPORTED) before anything is enqueued. */
int tf_resize_taps(int in, int out);
int tf_resize_coeffs(int in, int out, int32_t* bounds, int32_t* coeffs);
int tf_resize_u8(const void* in, int64_t n, int h_in, int w_in, int h, int w, const int32_t* h_bounds,
                 const int32_t* h_coeffs, int h_taps, const int32_t* v_bounds, const int32_t* v_coeffs, int v_taps,
                 void* tmp, void* out, tf_stream_t stream);

/* OpenCV's `cv2.Canny(frame, low, high)` (aperture 3, L2gradient = false) of RGB uint8 frames, bit for bit: the edge
 * maps the reference's ControlNet path conditions on (preprocess.py:113-127 get_canny_cond).  Per-channel 3x3 Sobel
 * with replicated borders, the channel of largest |dx| + |dy| (first on a tie), OpenCV's integer non-maximum
 * suppression, thresholds floor(low) < floor(high) (swapped when low > high; a magnitude must exceed them), and
 * hysteresis over 8-connected candidates.  Five launches (classify, then union-find merge, compress, flag, write),
 * nothing synchronised: capturable in a CUDA graph.  n <= 65535, 1 <= h, w <= 65536, n*h*w < 2^31.
 * tf_canny_workspace  bytes of workspace for n frames of h x w (-1 for bad sizes)
 * tf_canny_u8
 *   frames      device [n, h, w, 3] uint8, any alignment
 *   workspace   device, >= tf_canny_workspace(n, h, w) bytes, 16-byte aligned, uninitialised
 *   edges_u8    device [n, h, w] uint8, 0 / 255 (cv2.Canny's output), or NULL
 *   cond_f16    device [n, h, w, 3] fp16, 0 / 1 in every channel: get_canny_cond's [n, 3, h, w] tensor in the
 *               channels_last layout, or NULL (not both NULL) */
int64_t tf_canny_workspace(int64_t n, int h, int w);
int tf_canny_u8(const void* frames, int64_t n, int h, int w, double low, double high, void* workspace,
                int64_t workspace_bytes, void* edges_u8, void* cond_f16, tf_stream_t stream);

/* ---- multi-GPU: all-gather of keyframe tensors along the pivotal-sample axis (SURVEY.md §8e) ----
 * NCCL (all-gather over NVLink 5 / NVSwitch) bound at run time; one communicator per process/GPU.
 * Rendezvous: rank 0 calls tf_comm_unique_id and ships the TF_COMM_ID_BYTES to the other ranks by any
 * channel (the Python host uses a torch.distributed broadcast); every rank then calls tf_comm_init.
 * tf_allgather enqueues on `stream` (CUDA-graph capturable): recv = [nranks][bytes_per_rank]. */
#define TF_COMM_ID_BYTES 128
typedef void* tf_comm_t;
int tf_comm_nccl_version(void);                 /* NCCL version code, 0 if NCCL cannot be loaded */
int tf_comm_unique_id(void* id_out);
int tf_comm_init(const void* id, int nranks, int rank, tf_comm_t* comm_out);
int tf_allgather(tf_comm_t comm, const void* send, void* recv, int64_t bytes_per_rank, tf_stream_t stream);
int tf_comm_destroy(tf_comm_t comm);

#ifdef __cplusplus
}
#endif
#endif /* TOKENFLOW_B200_H_ */
