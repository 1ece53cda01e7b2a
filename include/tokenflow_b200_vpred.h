/* tokenflow_b200 — the latent updates for v-prediction models (Stable Diffusion 2.x at 768 x 768, whose
 * scheduler_config.json says "prediction_type": "v_prediction").
 *
 * Such a UNet predicts the velocity v = sqrt(alpha) * eps - sqrt(1 - alpha) * x0 instead of the noise eps.  These
 * entry points are tf_cfg_ddim and tf_ddim (include/tokenflow_b200.h) with diffusers' v-branch of the DDIM step
 * (DDIMScheduler.step / DDIMInverseScheduler.step, eta = 0) in place of the eps formula.  They are exported by the
 * same library and follow its conventions (int status, tf_last_error, nothing allocated or synchronised, device
 * pointers 16-byte aligned: a NULL or misaligned one is refused with TF_ERR_INVALID_ARGUMENT before anything is
 * enqueued).  Each operation is fp32 on fp16 operands and its result is rounded to fp16 (h), as the eager fp16
 * expression rounds:
 *     p   = h( h(a * x) - h(b * v) )          (pred_x0)
 *     e   = h( h(a * v) + h(b * x) )          (pred_eps)
 *     out = h( h(c * p) + h(d * e) )
 * The coefficient row (a, b, c, d) is read from device memory, so one captured CUDA graph serves every timestep:
 *     edit step             sqrt(alpha_t), sqrt(1 - alpha_t), sqrt(alpha_prev), sqrt(1 - alpha_prev)
 *     inversion step        mu_prev, sigma_prev, mu, sigma
 *     reconstruction step   mu, sigma, mu_prev, sigma_prev
 * (mu = sqrt(alpha), sigma = sqrt(1 - alpha); the inversion's sample is at the level of `prev`, as in the reference's
 * eps loop, preprocess.py:211-225).
 */
#ifndef TOKENFLOW_B200_VPRED_H_
#define TOKENFLOW_B200_VPRED_H_

#include <stdint.h>

#include "tokenflow_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

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

#ifdef __cplusplus
}
#endif
#endif /* TOKENFLOW_B200_VPRED_H_ */
