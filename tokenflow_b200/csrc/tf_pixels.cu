// tf_frames_to_nhwc / tf_nhwc_to_frames — the pixel conversions on either side of the VAE.
//
// Encoder input.  The reference turns PIL frames into the encoder's input on the host and ships fp16:
//     T.ToTensor()(frame)        uint8 -> fp32 v / 255 (a true quotient, on the CPU)
//     .to(torch.float16)         rounded to fp16
//     2 * imgs - 1               two fp16 tensor ops, each computed in fp32 and rounded
// Here only the uint8 frames cross PCIe and one pass computes the same values bit for bit, in the frames' own
// [N, H, W, 3] order: that is a channels_last [N, 3, H, W] fp16 tensor, the layout the encoder's first conv reads.
//
// Decoder output.  ((img / 2 + 0.5).clamp(0, 1) * 255).to(uint8) on the fp16 [N, 3, H, W] decoder output (the
// reference's decode_latents, then save_video / ToPILImage): every op rounded to fp16, then truncated to uint8.  ATen
// divides by the scalar 2 as a multiply by 0.5, which is exact, like the true quotient.  clamp keeps a NaN, and a
// NaN has no uint8 value (the C++ conversion is undefined): here it is defined as 0.  +-Inf clamp to 255 / 0 like
// any other value.  Read and written in channels_last order, so the output is the [N, H, W, 3] uint8 that video and
// PNG writers take.
#include "tf_common.cuh"
#include "tf_kernels.h"

namespace tf {
namespace {

__device__ __forceinline__ float round_h(float x) { return __half2float(__float2half_rn(x)); }

__device__ __forceinline__ __half byte_to_input(unsigned v) {
  const float unit = round_h(__fdiv_rn((float)v, 255.0f));     // ToTensor's fp32 quotient, .to(float16)
  return __float2half_rn(round_h(2.0f * unit) - 1.0f);          // 2 * imgs, then - 1
}

__device__ __forceinline__ unsigned char output_to_byte(float x) {
  float y = round_h(round_h(x * 0.5f) + 0.5f);                  // img / 2 + 0.5
  if (isnan(y)) return 0;
  y = fminf(fmaxf(y, 0.0f), 1.0f);                              // clamp(0, 1)
  return (unsigned char)round_h(y * 255.0f);                    // * 255, .to(uint8) truncates
}

// 8 elements a thread and iteration: 8 bytes <-> 16 bytes; the scalar tail (n % 8) is block 0's
__global__ void __launch_bounds__(256) frames_to_input_kernel(const uint8_t* __restrict__ in, long long n_vec,
                                                              long long n, __half* __restrict__ out) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_vec; i += stride) {
    const uint2 raw = reinterpret_cast<const uint2*>(in)[i];
    uint4 w;
    __half* h = reinterpret_cast<__half*>(&w);
#pragma unroll
    for (int e = 0; e < 8; ++e) h[e] = byte_to_input(((e < 4 ? raw.x : raw.y) >> (8 * (e & 3))) & 0xffu);
    reinterpret_cast<uint4*>(out)[i] = w;
  }
  if (blockIdx.x == 0)
    for (long long j = n_vec * 8 + threadIdx.x; j < n; j += blockDim.x) out[j] = byte_to_input(in[j]);
}

__global__ void __launch_bounds__(256) output_to_frames_kernel(const __half* __restrict__ in, long long n_vec,
                                                               long long n, uint8_t* __restrict__ out) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_vec; i += stride) {
    const uint4 raw = reinterpret_cast<const uint4*>(in)[i];
    const __half* h = reinterpret_cast<const __half*>(&raw);
    unsigned lo = 0, hi = 0;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      lo |= (unsigned)output_to_byte(__half2float(h[e])) << (8 * e);
      hi |= (unsigned)output_to_byte(__half2float(h[e + 4])) << (8 * e);
    }
    reinterpret_cast<uint2*>(out)[i] = make_uint2(lo, hi);
  }
  if (blockIdx.x == 0)
    for (long long j = n_vec * 8 + threadIdx.x; j < n; j += blockDim.x) out[j] = output_to_byte(__half2float(in[j]));
}

long long grid_for(long long n_vec) {
  long long blocks = (n_vec + 255) / 256;
  const long long cap = (long long)sm_count() * 16;
  if (blocks > cap) blocks = cap;
  return blocks < 1 ? 1 : blocks;
}

}  // namespace

int launch_frames_to_nhwc(const void* frames, long long n, void* out, cudaStream_t stream) {
  const long long n_vec = n / 8;
  frames_to_input_kernel<<<(unsigned)grid_for(n_vec), 256, 0, stream>>>(static_cast<const uint8_t*>(frames), n_vec, n,
                                                                        static_cast<__half*>(out));
  return check_cuda(cudaGetLastError(), "tf_frames_to_nhwc launch");
}

int launch_nhwc_to_frames(const void* x, long long n, void* frames, cudaStream_t stream) {
  const long long n_vec = n / 8;
  output_to_frames_kernel<<<(unsigned)grid_for(n_vec), 256, 0, stream>>>(static_cast<const __half*>(x), n_vec, n,
                                                                         static_cast<uint8_t*>(frames));
  return check_cuda(cudaGetLastError(), "tf_nhwc_to_frames launch");
}

}  // namespace tf
