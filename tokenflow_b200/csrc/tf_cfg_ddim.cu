// tf_cfg_ddim — classifier-free guidance + DDIM update of one denoising step in ONE pass
// (reference run_tokenflow_pnp.py:213-217: `noise_pred_uncond + g * (noise_pred_cond - noise_pred_uncond)`
// followed by `scheduler.step(noise_pred, t, x)['prev_sample']`, eta = 0).
//
// The reference runs these as ~8 fp16 elementwise launches; each rounds its result to fp16.  This kernel
// keeps that rounding sequence (every intermediate is rounded to fp16 exactly where the eager expression
// rounds), so the fused step is bit-identical to the eager one:
//     d  = h(c - u)            m  = h(g * d)            e  = h(u + m)                 (CFG)
//     a  = h(s1 * e)           b  = h(x - a)            p  = h(b * inv_s2)            (pred_x0; ATen divides by a
//     c1 = h(s3 * p)           c2 = h(s4 * e)           out = h(c1 + c2)               host scalar as x * (1/s))
// with s1 = sqrt(1 - alpha_t), inv_s2 = 1 / sqrt(alpha_t), s3 = sqrt(alpha_prev), s4 = sqrt(1 - alpha_prev)
// as fp32 values.  The four step coefficients are read from DEVICE memory so that a CUDA graph of the step
// can be replayed for every timestep (the caller copies the step's row of its coefficient table into the
// 4-float buffer before the replay).
//
// HBM-bound and tiny (3 reads + 1 write of the latents, 0.65 MB each at C2): 8 halves per thread.
//
// tf_ddim is the same DDIM update without the guidance (the inversion stage's two directions), with the
// coefficients of the direction it runs: inversion s1 = sigma_prev, inv_s2 = 1/mu_prev, s3 = mu, s4 = sigma;
// reconstruction s1 = sigma, inv_s2 = 1/mu, s3 = mu_prev, s4 = sigma_prev.
//
// tf_cfg_ddim_v / tf_ddim_v are the same two kernels for a model that predicts the velocity
// v = sqrt(alpha) * eps - sqrt(1 - alpha) * x0 (Stable Diffusion 2.x at 768^2), with diffusers' v-branch of
// DDIMScheduler.step (eta = 0) as the DDIM half.  The coefficient row (a, b, c, d) is
// (sqrt(alpha_t), sqrt(1 - alpha_t), sqrt(alpha_prev), sqrt(1 - alpha_prev)) for the edit, (mu_prev, sigma_prev,
// mu, sigma) for the inversion and (mu, sigma, mu_prev, sigma_prev) for the reconstruction:
//     p = h(h(a * x) - h(b * v))     e = h(h(a * v) + h(b * x))     out = h(h(c * p) + h(d * e))
#include "tf_common.cuh"
#include "tf_kernels.h"

namespace tf {
namespace {

__device__ __forceinline__ float rh(float x) { return __half2float(__float2half_rn(x)); }

// What the model predicts: the parameterisation selects the DDIM half of the step, nothing else.
enum class Pred { kEps, kV };

// The DDIM half of the step, shared by both kernels so each rounding sequence lives in one place.  `m` is the model
// output (after guidance, for tf_cfg_ddim[_v]), `xv` the latent, (k0, k1, k2, k3) the coefficient row.
template <Pred P>
__device__ __forceinline__ float ddim_one(float m, float xv, float k0, float k1, float k2, float k3);

// eps: out = h(h(s3 * h(h(x - h(s1 * e)) * inv_s2)) + h(s4 * e)).
template <>
__device__ __forceinline__ float ddim_one<Pred::kEps>(float e, float xv, float s1, float inv_s2, float s3, float s4) {
  const float p = rh(rh(xv - rh(s1 * e)) * inv_s2);
  return rh(rh(s3 * p) + rh(s4 * e));
}

// v: pred_x0 = h(h(a * x) - h(b * v)), pred_eps = h(h(a * v) + h(b * x)), out = h(h(c * pred_x0) + h(d * pred_eps)).
template <>
__device__ __forceinline__ float ddim_one<Pred::kV>(float v, float xv, float a, float b, float c, float d) {
  const float p = rh(rh(a * xv) - rh(b * v));
  const float e = rh(rh(a * v) + rh(b * xv));
  return rh(rh(c * p) + rh(d * e));
}

template <Pred P>
__global__ void __launch_bounds__(256)
cfg_ddim_kernel(const __half* __restrict__ eu, const __half* __restrict__ ec, const __half* __restrict__ x,
                const float* __restrict__ coef, float g, long long n_vec, long long n, __half* __restrict__ out) {
  const float k0 = coef[0], k1 = coef[1], k2 = coef[2], k3 = coef[3];
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  auto one = [&](float u, float c, float xv) -> float {
    return ddim_one<P>(rh(u + rh(g * rh(c - u))), xv, k0, k1, k2, k3);
  };
  if (i < n_vec) {
    const uint4 ru = reinterpret_cast<const uint4*>(eu)[i];
    const uint4 rc = reinterpret_cast<const uint4*>(ec)[i];
    const uint4 rx = reinterpret_cast<const uint4*>(x)[i];
    const __half2* hu = reinterpret_cast<const __half2*>(&ru);
    const __half2* hc = reinterpret_cast<const __half2*>(&rc);
    const __half2* hx = reinterpret_cast<const __half2*>(&rx);
    uint4 w;
    __half2* ho = reinterpret_cast<__half2*>(&w);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 u = __half22float2(hu[e]), c = __half22float2(hc[e]), xv = __half22float2(hx[e]);
      ho[e] = __floats2half2_rn(one(u.x, c.x, xv.x), one(u.y, c.y, xv.y));
    }
    reinterpret_cast<uint4*>(out)[i] = w;
  }
  if (i == 0) {                                   // tail (n not a multiple of 8)
    for (long long j = n_vec * 8; j < n; ++j)
      out[j] = __float2half_rn(one(__half2float(eu[j]), __half2float(ec[j]), __half2float(x[j])));
  }
}

// Guidance-free DDIM update (both directions of the inversion stage, reference preprocess.py:217-225 and
// :251-260): one read of the model output and x, one write.  `out` may alias `x`: every element is read before it
// is written by the same thread.
template <Pred P>
__global__ void __launch_bounds__(256)
ddim_kernel(const __half* __restrict__ eps, const __half* x, const float* __restrict__ coef, long long n_vec,
            long long n, __half* out) {
  const float k0 = coef[0], k1 = coef[1], k2 = coef[2], k3 = coef[3];
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_vec) {
    const uint4 re = reinterpret_cast<const uint4*>(eps)[i];
    const uint4 rx = reinterpret_cast<const uint4*>(x)[i];
    const __half2* he = reinterpret_cast<const __half2*>(&re);
    const __half2* hx = reinterpret_cast<const __half2*>(&rx);
    uint4 w;
    __half2* ho = reinterpret_cast<__half2*>(&w);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 ev = __half22float2(he[e]), xv = __half22float2(hx[e]);
      ho[e] = __floats2half2_rn(ddim_one<P>(ev.x, xv.x, k0, k1, k2, k3), ddim_one<P>(ev.y, xv.y, k0, k1, k2, k3));
    }
    reinterpret_cast<uint4*>(out)[i] = w;
  }
  if (i == 0) {                                   // tail (n not a multiple of 8)
    for (long long j = n_vec * 8; j < n; ++j)
      out[j] = __float2half_rn(ddim_one<P>(__half2float(eps[j]), __half2float(x[j]), k0, k1, k2, k3));
  }
}

unsigned blocks_for(long long n_vec) {
  const long long threads = n_vec > 0 ? n_vec : 1;
  return (unsigned)((threads + 255) / 256);
}

template <Pred P>
int launch_ddim_as(const void* eps, const void* x, const float* coef_dev, long long n, void* out, cudaStream_t stream,
                   const char* what) {
  if (n == 0) return TF_OK;
  const long long n_vec = n / 8;
  ddim_kernel<P><<<blocks_for(n_vec), 256, 0, stream>>>(static_cast<const __half*>(eps), static_cast<const __half*>(x),
                                                        coef_dev, n_vec, n, static_cast<__half*>(out));
  return check_cuda(cudaGetLastError(), what);
}

template <Pred P>
int launch_cfg_ddim_as(const void* eps_uncond, const void* eps_cond, const void* x, const float* coef_dev,
                       float guidance, long long n, void* out, cudaStream_t stream, const char* what) {
  if (n == 0) return TF_OK;
  const long long n_vec = n / 8;
  cfg_ddim_kernel<P><<<blocks_for(n_vec), 256, 0, stream>>>(
      static_cast<const __half*>(eps_uncond), static_cast<const __half*>(eps_cond), static_cast<const __half*>(x),
      coef_dev, guidance, n_vec, n, static_cast<__half*>(out));
  return check_cuda(cudaGetLastError(), what);
}

}  // namespace

int launch_ddim(const void* eps, const void* x, const float* coef_dev, long long n, void* out, cudaStream_t stream) {
  return launch_ddim_as<Pred::kEps>(eps, x, coef_dev, n, out, stream, "tf_ddim launch");
}

int launch_ddim_v(const void* v, const void* x, const float* coef_dev, long long n, void* out, cudaStream_t stream) {
  return launch_ddim_as<Pred::kV>(v, x, coef_dev, n, out, stream, "tf_ddim_v launch");
}

int launch_cfg_ddim(const void* eps_uncond, const void* eps_cond, const void* x, const float* coef_dev, float guidance,
                    long long n, void* out, cudaStream_t stream) {
  return launch_cfg_ddim_as<Pred::kEps>(eps_uncond, eps_cond, x, coef_dev, guidance, n, out, stream,
                                        "tf_cfg_ddim launch");
}

int launch_cfg_ddim_v(const void* v_uncond, const void* v_cond, const void* x, const float* coef_dev, float guidance,
                      long long n, void* out, cudaStream_t stream) {
  return launch_cfg_ddim_as<Pred::kV>(v_uncond, v_cond, x, coef_dev, guidance, n, out, stream,
                                      "tf_cfg_ddim_v launch");
}

}  // namespace tf
