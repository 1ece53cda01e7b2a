// tf_resize_u8 — Pillow's Image.resize((W, H), Image.LANCZOS) of RGB uint8 frames, bit for bit.
//
// The reference resizes every frame with PIL before it reaches the VAE (util.py:28 save_video_frames resizes to
// (W, H); run_tokenflow_pnp.py:174-175, run_tokenflow_sdedit.py:136-137 and preprocess.py:191-192 resize square
// frames to 512x512).  Pillow's algorithm (libImaging/Resample.c) is separable and integer:
//   - per axis, double-precision Lanczos-3 weights for every output pixel over the input window
//     [xmin, xmin + count), normalised by their sum and rounded to int32 fixed point with 22 fractional bits;
//   - a horizontal pass first, into a uint8 intermediate, then a vertical pass;
//   - every output value is clamp((2^21 + sum v * k) >> 22, 0, 255), accumulated in int32;
//   - a pass whose axis keeps its size is skipped, and an unchanged size is a copy.
// The tables are computed here on the host, with libm sin and no FMA contraction (the library's host code is built
// with -ffp-contract=off), so they are Pillow's own integers; the caller uploads them once per (in, out) pair.  Both
// passes read and write each byte once from HBM, which bounds them.
#include <cmath>
#include <vector>

#include "tf_common.cuh"
#include "tf_kernels.h"

namespace tf {

constexpr int kResizePrecisionBits = 22;          // Pillow: 32 - 8 (uint8) - 2
constexpr long long kResizeMaxSmem = 227 * 1024;  // opt-in shared memory per block on sm_90

int resize_taps(int in, int out) {
  const double scale = (double)in / out;
  const double support = 3.0 * (scale < 1.0 ? 1.0 : scale);
  return (int)std::ceil(support) * 2 + 1;
}

static double sinc(double x) {
  if (x == 0.0) return 1.0;
  x = x * M_PI;
  return std::sin(x) / x;
}

static double lanczos3(double x) { return (-3.0 <= x && x < 3.0) ? sinc(x) * sinc(x / 3) : 0.0; }

void resize_coeffs(int in, int out, int32_t* bounds, int32_t* coeffs) {
  // precompute_coeffs + normalize_coeffs_8bpc of Resample.c, with the same double operations in the same order
  const int taps = resize_taps(in, out);
  const double scale = (double)(float)in / out;   // Pillow: (double)(in1 - in0) / outSize with float box edges
  const double fs = scale < 1.0 ? 1.0 : scale;
  const double support = 3.0 * fs;
  const double ss = 1.0 / fs;
  std::vector<double> w(taps);
  for (int xx = 0; xx < out; ++xx) {
    const double center = (xx + 0.5) * scale;
    int xmin = (int)(center - support + 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = (int)(center + support + 0.5);
    if (xmax > in) xmax = in;
    xmax -= xmin;
    double ww = 0.0;
    for (int x = 0; x < xmax; ++x) {
      w[x] = lanczos3((x + xmin - center + 0.5) * ss);
      ww += w[x];
    }
    int32_t* k = coeffs + (long long)xx * taps;
    for (int x = 0; x < taps; ++x) {
      double v = 0.0;
      if (x < xmax) v = ww != 0.0 ? w[x] / ww : w[x];
      k[x] = v < 0 ? (int32_t)(-0.5 + v * (1 << kResizePrecisionBits))
                   : (int32_t)(0.5 + v * (1 << kResizePrecisionBits));
    }
    bounds[2 * xx] = xmin;
    bounds[2 * xx + 1] = xmax;
  }
}

namespace {

__device__ __forceinline__ uint8_t clip8(int v) {
  v >>= kResizePrecisionBits;
  return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

constexpr int kHThreads = 256;

// Horizontal pass: `rows` consecutive input rows per block, staged in shared memory with 16-byte loads (the rows are
// contiguous, so the block reads one contiguous byte range); each thread computes whole output pixels of every staged
// row, loading each coefficient once for all rows.
__global__ void __launch_bounds__(kHThreads) resize_h_kernel(const uint8_t* __restrict__ in, long long total_rows,
                                                             int w_in, int w, int rows,
                                                             const int32_t* __restrict__ bounds,
                                                             const int32_t* __restrict__ coeffs, int taps,
                                                             uint8_t* __restrict__ out) {
  extern __shared__ __align__(16) uint8_t srow[];
  const long long r0 = (long long)blockIdx.x * rows;
  const int nr = (int)(total_rows - r0 < rows ? total_rows - r0 : rows);
  const long long in_pitch = 3LL * w_in;
  const uint8_t* src = in + r0 * in_pitch;
  const long long len = nr * in_pitch;
  // smem[pad + i] = src[i]: src - pad is 16-byte aligned, so every whole chunk is one uint4 load and store
  const int pad = (int)(reinterpret_cast<uintptr_t>(src) & 15u);
  const uint8_t* base = src - pad;
  const long long chunks = (pad + len + 15) / 16;
  for (long long c = threadIdx.x; c < chunks; c += kHThreads) {
    const long long b0 = c * 16;
    if (b0 >= pad && b0 + 16 <= pad + len) {
      reinterpret_cast<uint4*>(srow)[c] = reinterpret_cast<const uint4*>(base)[c];
    } else {
      for (int j = 0; j < 16; ++j)
        if (b0 + j >= pad && b0 + j < pad + len) srow[b0 + j] = base[b0 + j];
    }
  }
  __syncthreads();
  const uint8_t* s = srow + pad;
  for (int xx = threadIdx.x; xx < w; xx += kHThreads) {
    const int xmin = bounds[2 * xx], cnt = bounds[2 * xx + 1];
    const int32_t* k = coeffs + (long long)xx * taps;
    for (int r = 0; r < nr; r += 4) {
      int acc[4][3];
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[i][0] = acc[i][1] = acc[i][2] = 1 << (kResizePrecisionBits - 1);
      const int rr = nr - r < 4 ? nr - r : 4;
      for (int x = 0; x < cnt; ++x) {
        const int kv = __ldg(k + x);
        const uint8_t* p = s + (long long)r * in_pitch + 3 * (xmin + x);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          if (i < rr) {
            acc[i][0] += (int)p[i * in_pitch + 0] * kv;
            acc[i][1] += (int)p[i * in_pitch + 1] * kv;
            acc[i][2] += (int)p[i * in_pitch + 2] * kv;
          }
        }
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (i < rr) {
          uint8_t* o = out + (r0 + r + i) * 3LL * w + 3LL * xx;
          o[0] = clip8(acc[i][0]);
          o[1] = clip8(acc[i][1]);
          o[2] = clip8(acc[i][2]);
        }
      }
    }
  }
}

constexpr int kVThreads = 128;

// Vertical pass: blockIdx.x / col_blocks is the output row (frame * h + yy); each thread owns VEC consecutive bytes of
// it (16 when the row pitch and both base pointers allow uint4 accesses) and walks the row's input window.  Rows of
// the window are shared by neighbouring output rows through L2.
template <int VEC>
__global__ void __launch_bounds__(kVThreads) resize_v_kernel(const uint8_t* __restrict__ in, int h_in, int h,
                                                             long long pitch, int col_blocks,
                                                             const int32_t* __restrict__ bounds,
                                                             const int32_t* __restrict__ coeffs, int taps,
                                                             uint8_t* __restrict__ out) {
  const long long row = blockIdx.x / col_blocks;
  const long long col = ((long long)(blockIdx.x % col_blocks) * kVThreads + threadIdx.x) * VEC;
  if (col >= pitch) return;
  const int yy = (int)(row % h);
  const long long frame = row / h;
  const int ymin = bounds[2 * yy], cnt = bounds[2 * yy + 1];
  const int32_t* k = coeffs + (long long)yy * taps;
  const uint8_t* src = in + (frame * h_in + ymin) * pitch + col;
  uint8_t* dst = out + (frame * h + yy) * pitch + col;
  int acc[VEC];
#pragma unroll
  for (int j = 0; j < VEC; ++j) acc[j] = 1 << (kResizePrecisionBits - 1);
  if (VEC == 16) {
    for (int y = 0; y < cnt; ++y) {
      const int kv = __ldg(k + y);
      const uint4 raw = *reinterpret_cast<const uint4*>(src + y * pitch);
      const uint32_t wv[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
      for (int j = 0; j < 16; ++j) acc[j] += (int)((wv[j >> 2] >> (8 * (j & 3))) & 0xffu) * kv;
    }
    uint32_t o[4] = {0, 0, 0, 0};
#pragma unroll
    for (int j = 0; j < 16; ++j) o[j >> 2] |= (uint32_t)clip8(acc[j]) << (8 * (j & 3));
    *reinterpret_cast<uint4*>(dst) = make_uint4(o[0], o[1], o[2], o[3]);
  } else {
    const int nb = (int)(pitch - col < VEC ? pitch - col : VEC);
    for (int y = 0; y < cnt; ++y) {
      const int kv = __ldg(k + y);
#pragma unroll
      for (int j = 0; j < VEC; ++j)
        if (j < nb) acc[j] += (int)src[y * pitch + j] * kv;
    }
#pragma unroll
    for (int j = 0; j < VEC; ++j)
      if (j < nb) dst[j] = clip8(acc[j]);
  }
}

}  // namespace

int launch_resize_h(const void* in, long long n_rows, int w_in, int w, const int32_t* bounds, const int32_t* coeffs,
                    int taps, void* out, cudaStream_t stream) {
  // up to 4 rows per block within the default 48 KB of shared memory; one wider row opts into more
  const long long pitch = 3LL * w_in;
  int rows = (int)(48 * 1024 / (pitch + 16));
  rows = rows < 1 ? 1 : (rows > 4 ? 4 : rows);
  const long long smem = rows * pitch + 16;
  if (smem > kResizeMaxSmem) {
    set_last_error("tf_resize_u8: input rows of %d pixels do not fit in shared memory", w_in);
    return TF_ERR_UNSUPPORTED;
  }
  if (smem > 48 * 1024) {
    if (int e = check_cuda(cudaFuncSetAttribute(resize_h_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                (int)smem), "tf_resize_u8 smem"))
      return e;
  }
  const long long blocks = (n_rows + rows - 1) / rows;
  resize_h_kernel<<<(unsigned)blocks, kHThreads, (size_t)smem, stream>>>(static_cast<const uint8_t*>(in), n_rows, w_in,
                                                                          w, rows, bounds, coeffs, taps,
                                                                          static_cast<uint8_t*>(out));
  return check_cuda(cudaGetLastError(), "tf_resize_u8 horizontal launch");
}

int launch_resize_v(const void* in, long long n, int h_in, int h, int w, const int32_t* bounds, const int32_t* coeffs,
                    int taps, void* out, cudaStream_t stream) {
  const long long pitch = 3LL * w;
  const bool vec = pitch % 16 == 0 && (reinterpret_cast<uintptr_t>(in) & 15u) == 0 &&
                   (reinterpret_cast<uintptr_t>(out) & 15u) == 0;
  const int per = vec ? 16 : 4;
  const int col_blocks = (int)((pitch + (long long)kVThreads * per - 1) / ((long long)kVThreads * per));
  const long long blocks = n * h * col_blocks;
  if (blocks > 0x7fffffffLL) {
    set_last_error("tf_resize_u8: %lld output rows of %d pixels are too many for one launch", n * h, w);
    return TF_ERR_UNSUPPORTED;
  }
  if (vec)
    resize_v_kernel<16><<<(unsigned)blocks, kVThreads, 0, stream>>>(static_cast<const uint8_t*>(in), h_in, h, pitch,
                                                                     col_blocks, bounds, coeffs, taps,
                                                                     static_cast<uint8_t*>(out));
  else
    resize_v_kernel<4><<<(unsigned)blocks, kVThreads, 0, stream>>>(static_cast<const uint8_t*>(in), h_in, h, pitch,
                                                                    col_blocks, bounds, coeffs, taps,
                                                                    static_cast<uint8_t*>(out));
  return check_cuda(cudaGetLastError(), "tf_resize_u8 vertical launch");
}

}  // namespace tf
