// tf_unit_rows — row L2-normalisation feeding the NN field (reference util.py:66-67).
//
//   out[r,:] = fp16_rne( x[r,:] / ||x[r,:]||_2 )        x fp32 (the autocast dtype of norm1's output)
//                                                        or fp16; no epsilon, like the reference.
// The reference normalises in fp32 and lets autocast round the GEMM operands to fp16 (SURVEY.md
// Appendix A "GPU dtype flow"); this kernel produces exactly those fp16 operands once, so the
// similarity GEMM reads 2 bytes/element and the keyframe side is normalised once per pivotal pass
// instead of once per frame batch.  The squared norm is accumulated in fp64 (the correctly rounded
// value a 1-ulp-accurate fp32 reduction approximates), the quotient is an IEEE fp32 division.
//
// One warp per row, 16-byte loads, HBM-bound: rows*dim*(esz_in + 2) bytes.
#include "tf_common.cuh"
#include "tf_kernels.h"

namespace tf {
namespace {

constexpr int kWarpsPerBlock = 8;

// x / y with one reciprocal per row: q = x*r, then one Newton correction q + (x - y*q)*r (Markstein).
// With r the correctly rounded 1/y, and the remainder x - y*q exact, this is the correctly rounded
// quotient — the IEEE division the reference's `x / norm` performs — at 3 FMA-pipe instructions per
// element instead of a MUFU.RCP + fix-up sequence per element (the kernel was XU-bound on divisions).
// Both conditions fail at extreme norms: 1/y is subnormal above 2^126 and infinite below 2^-128, and the
// remainder of an element below about 2^-103 underflows.  Every element that can reach a non-zero fp16
// output is at least 2^-26 * y, so for y in [2^-64, 2^64] both hold; rows outside that range (a zero
// or non-finite norm included) take the IEEE division.  The choice is made once per row (the norm is the
// same on every lane), so the element loop of ordinary rows is unchanged.
__device__ __forceinline__ bool div_by_needs_ieee(float y) { return !(y >= 0x1p-64f && y <= 0x1p64f); }

template <bool kIeee>
__device__ __forceinline__ float div_by(float x, float y, float r) {
  if (kIeee) return __fdiv_rn(x, y);
  const float q = x * r;
  return fmaf(fmaf(-y, q, x), r, q);
}

template <bool kInF32, bool kIeee>
__device__ __forceinline__ void write_unit_row(const void* __restrict__ x, long long r, int dim, long long row_stride,
                                               int lane, float nrm, float rcp, __half* __restrict__ orow) {
  if (kInF32) {
    const float* xr = static_cast<const float*>(x) + r * row_stride;
    for (int c = lane * 4; c < dim; c += 128) {
      float4 v = *reinterpret_cast<const float4*>(xr + c);
      __half2 lo = __floats2half2_rn(div_by<kIeee>(v.x, nrm, rcp), div_by<kIeee>(v.y, nrm, rcp));
      __half2 hi = __floats2half2_rn(div_by<kIeee>(v.z, nrm, rcp), div_by<kIeee>(v.w, nrm, rcp));
      uint2 o2;
      o2.x = *reinterpret_cast<uint32_t*>(&lo);
      o2.y = *reinterpret_cast<uint32_t*>(&hi);
      *reinterpret_cast<uint2*>(orow + c) = o2;
    }
  } else {
    const __half* xr = static_cast<const __half*>(x) + r * row_stride;
    for (int c = lane * 4; c < dim; c += 128) {
      uint2 raw = *reinterpret_cast<const uint2*>(xr + c);
      float2 a = __half22float2(*reinterpret_cast<__half2*>(&raw.x));
      float2 b = __half22float2(*reinterpret_cast<__half2*>(&raw.y));
      __half2 lo = __floats2half2_rn(div_by<kIeee>(a.x, nrm, rcp), div_by<kIeee>(a.y, nrm, rcp));
      __half2 hi = __floats2half2_rn(div_by<kIeee>(b.x, nrm, rcp), div_by<kIeee>(b.y, nrm, rcp));
      uint2 o2;
      o2.x = *reinterpret_cast<uint32_t*>(&lo);
      o2.y = *reinterpret_cast<uint32_t*>(&hi);
      *reinterpret_cast<uint2*>(orow + c) = o2;
    }
  }
}

template <bool kInF32>
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
unit_rows_kernel(const void* __restrict__ x, long long rows, int dim, long long row_stride,
                 __half* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long warp0 = (long long)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  const long long nwarps = (long long)gridDim.x * kWarpsPerBlock;
  for (long long r = warp0; r < rows; r += nwarps) {
    double ss = 0.0;
    if (kInF32) {
      const float* xr = static_cast<const float*>(x) + r * row_stride;
      for (int c = lane * 4; c < dim; c += 128) {
        float4 v = *reinterpret_cast<const float4*>(xr + c);
        ss += (double)v.x * v.x + (double)v.y * v.y + (double)v.z * v.z + (double)v.w * v.w;
      }
    } else {
      const __half* xr = static_cast<const __half*>(x) + r * row_stride;
      for (int c = lane * 4; c < dim; c += 128) {
        uint2 raw = *reinterpret_cast<const uint2*>(xr + c);
        float2 a = __half22float2(*reinterpret_cast<__half2*>(&raw.x));
        float2 b = __half22float2(*reinterpret_cast<__half2*>(&raw.y));
        ss += (double)a.x * a.x + (double)a.y * a.y + (double)b.x * b.x + (double)b.y * b.y;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    const float nrm = (float)sqrt(ss);
    const float rcp = __frcp_rn(nrm);
    __half* orow = out + r * dim;
    if (div_by_needs_ieee(nrm))
      write_unit_row<kInF32, true>(x, r, dim, row_stride, lane, nrm, rcp, orow);
    else
      write_unit_row<kInF32, false>(x, r, dim, row_stride, lane, nrm, rcp, orow);
  }
}

}  // namespace

int launch_unit_rows(const void* x, int x_is_f32, long long rows, int dim, long long row_stride, void* out_f16,
                     cudaStream_t stream) {
  if (rows == 0) return TF_OK;
  long long blocks = (rows + kWarpsPerBlock - 1) / kWarpsPerBlock;
  const long long cap = (long long)sm_count() * 8;
  if (blocks > cap) blocks = cap;
  dim3 grid((unsigned)blocks), block(kWarpsPerBlock * 32);
  if (x_is_f32)
    unit_rows_kernel<true><<<grid, block, 0, stream>>>(x, rows, dim, row_stride, static_cast<__half*>(out_f16));
  else
    unit_rows_kernel<false><<<grid, block, 0, stream>>>(x, rows, dim, row_stride, static_cast<__half*>(out_f16));
  return check_cuda(cudaGetLastError(), "tf_unit_rows launch");
}

}  // namespace tf

// ------------------------------------------------------------------------------------------------
// tf_layernorm_rows / tf_layernorm_unit_rows — norm1 (LayerNorm) fused with what consumes it.
//
//   y    = LN(x) in fp32 (autocast runs layer_norm in fp32: mean / biased variance / eps inside the rsqrt /
//          affine), rounded to fp16 — exactly the operand autocast hands to the to_q/to_k/to_v GEMMs
//          (reference tokenflow_utils.py:323 -> :120-122);
//   unit = fp16(y_fp32 / ||y_fp32||_2) — the row the NN field correlates (util.py:66-67 + the fp16 operand
//          cast of util.py:68), from the UNROUNDED fp32 y like the reference's fp32 norm1 output.
//
// Frame pass: the reference evaluates norm1 on all three streams but only the source stream's output is ever
// used, and only as the NN-field query (:335; attn1 is skipped) -> unit rows of the source third only, y is
// never written.  Pivotal pass: y of every sample feeds the fused QKV projection, unit rows are wanted for the
// source-stream samples (the first `unit_rows` rows) -> both outputs from ONE read of hidden_states, instead
// of a 4-byte norm1 output that is re-read by three casts and one normalisation.
// One warp per row, whole row held in registers (dim <= 1280).  Outputs may be strided (packed buffers).
// ------------------------------------------------------------------------------------------------
namespace tf {
namespace {

constexpr int kLnMaxVecPerLane = 5;     // 5 x 8 halves x 32 lanes = 1280 channels

template <bool kIeee>
__device__ __forceinline__ void write_ln_unit_row(const float (&v)[kLnMaxVecPerLane][8], int lane, int nvec, float nrm,
                                                  float rcp, __half* __restrict__ orow) {
#pragma unroll
  for (int j = 0; j < kLnMaxVecPerLane; ++j) {
    const int vi = lane + 32 * j;
    if (vi < nvec) {
      uint4 w;
      __half2* h = reinterpret_cast<__half2*>(&w);
#pragma unroll
      for (int e = 0; e < 4; ++e)
        h[e] = __floats2half2_rn(div_by<kIeee>(v[j][2 * e], nrm, rcp), div_by<kIeee>(v[j][2 * e + 1], nrm, rcp));
      *reinterpret_cast<uint4*>(orow + vi * 8) = w;
    }
  }
}

__global__ void __launch_bounds__(kWarpsPerBlock * 32)
layernorm_rows_kernel(const __half* __restrict__ x, long long rows, int dim, long long row_stride,
                      const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                      __half* __restrict__ y_out, long long y_row_stride, __half* __restrict__ unit_out,
                      long long unit_row_stride, long long unit_rows) {
  const int lane = threadIdx.x & 31;
  const int nvec = dim >> 3;
  const long long warp0 = (long long)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  const long long nwarps = (long long)gridDim.x * kWarpsPerBlock;
  const float inv_dim = 1.0f / (float)dim;
  for (long long r = warp0; r < rows; r += nwarps) {
    const bool want_unit = unit_out != nullptr && r < unit_rows;
    if (y_out == nullptr && !want_unit) continue;
    const __half* xr = x + r * row_stride;
    float v[kLnMaxVecPerLane][8];
    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < kLnMaxVecPerLane; ++j) {
      const int vi = lane + 32 * j;
      if (vi < nvec) {
        const uint4 raw = *reinterpret_cast<const uint4*>(xr + vi * 8);
        const __half2* h = reinterpret_cast<const __half2*>(&raw);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 f = __half22float2(h[e]);
          v[j][2 * e] = f.x;
          v[j][2 * e + 1] = f.y;
          sum += f.x + f.y;
        }
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float mean = sum * inv_dim;
    float sq = 0.f;
#pragma unroll
    for (int j = 0; j < kLnMaxVecPerLane; ++j) {
      if (lane + 32 * j < nvec) {
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const float dlt = v[j][e] - mean;
          sq += dlt * dlt;
        }
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
    const float rstd = rsqrtf(sq * inv_dim + eps);
    double ss = 0.0;
#pragma unroll
    for (int j = 0; j < kLnMaxVecPerLane; ++j) {
      const int vi = lane + 32 * j;
      if (vi < nvec) {
        const float4 g0 = *reinterpret_cast<const float4*>(gamma + vi * 8);
        const float4 g1 = *reinterpret_cast<const float4*>(gamma + vi * 8 + 4);
        const float4 b0 = *reinterpret_cast<const float4*>(beta + vi * 8);
        const float4 b1 = *reinterpret_cast<const float4*>(beta + vi * 8 + 4);
        const float g[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
        const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const float y = (v[j][e] - mean) * rstd * g[e] + b[e];
          v[j][e] = y;
          ss += (double)y * y;
        }
        if (y_out != nullptr) {
          uint4 w;
          __half2* h = reinterpret_cast<__half2*>(&w);
#pragma unroll
          for (int e = 0; e < 4; ++e) h[e] = __floats2half2_rn(v[j][2 * e], v[j][2 * e + 1]);
          *reinterpret_cast<uint4*>(y_out + r * y_row_stride + vi * 8) = w;
        }
      }
    }
    if (!want_unit) continue;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    const float nrm = (float)sqrt(ss);
    const float rcp = __frcp_rn(nrm);
    __half* orow = unit_out + r * unit_row_stride;
    if (div_by_needs_ieee(nrm))
      write_ln_unit_row<true>(v, lane, nvec, nrm, rcp, orow);
    else
      write_ln_unit_row<false>(v, lane, nvec, nrm, rcp, orow);
  }
}

}  // namespace

int launch_layernorm_rows(const void* x_f16, long long rows, int dim, long long row_stride, const float* gamma,
                          const float* beta, float eps, void* y_out, long long y_row_stride, void* unit_out,
                          long long unit_row_stride, long long unit_rows, cudaStream_t stream) {
  if (rows == 0 || (y_out == nullptr && (unit_out == nullptr || unit_rows <= 0))) return TF_OK;
  if ((dim >> 3) > 32 * kLnMaxVecPerLane) {
    set_last_error("tf_layernorm_rows: dim=%d > %d is not supported", dim, 8 * 32 * kLnMaxVecPerLane);
    return TF_ERR_UNSUPPORTED;
  }
  const long long work_rows = y_out != nullptr ? rows : (unit_rows < rows ? unit_rows : rows);
  long long blocks = (work_rows + kWarpsPerBlock - 1) / kWarpsPerBlock;
  const long long cap = (long long)sm_count() * 8;
  if (blocks > cap) blocks = cap;
  layernorm_rows_kernel<<<(unsigned)blocks, kWarpsPerBlock * 32, 0, stream>>>(
      static_cast<const __half*>(x_f16), work_rows, dim, row_stride, gamma, beta, eps, static_cast<__half*>(y_out),
      y_row_stride, static_cast<__half*>(unit_out), unit_row_stride, unit_rows);
  return check_cuda(cudaGetLastError(), "tf_layernorm_rows launch");
}

int launch_layernorm_unit_rows(const void* x_f16, long long rows, int dim, long long row_stride, const float* gamma,
                               const float* beta, float eps, void* out_f16, cudaStream_t stream) {
  return launch_layernorm_rows(x_f16, rows, dim, row_stride, gamma, beta, eps, nullptr, 0, out_f16, dim, rows, stream);
}

}  // namespace tf
