// tf_group_norm_nhwc / tf_geglu — the UNet body's GroupNorm sites and GEGLU gate as native kernels.
//
// GroupNorm.  The body runs channels_last, and ATen's CUDA GroupNorm has no channels_last kernel: it copies the
// input to NCHW, computes the moments, writes an NCHW output, SiLU reads and writes it again, and the next conv
// copies it back to NHWC — about 9 passes over the tensor.  Here
//
//     out = [SiLU]( GroupNorm( x [+ bias[n, c]] ) )        x, out dense NHWC fp16 [N, HW, C]
//
// takes two launches and three passes (read, read, write):
//   1. gn_stats_kernel  over (pixel chunk, sample): every thread owns one 8-channel column (16-byte loads) and
//      accumulates per channel; the CTA folds its channels into per-group partial sums and writes them to the
//      caller's workspace [N, G, chunks] (double2).  No atomics: every sum has a fixed order, so two launches are
//      bit-identical (the CUDA-graphed step must equal the eager one bit for bit).
//   2. gn_apply_kernel  over (pixel chunk, sample): each CTA reduces its sample's partials (fixed order), builds
//      the per-channel a = rstd * gamma, b = beta - mean * a in shared memory and streams x once.
//
// Rounding follows the eager ATen sequence:  x + bias is rounded to fp16 (the eager add is an fp16 tensor op);
// mean and rstd = rsqrtf(var_f32 + fp16(eps)) are rounded to fp16 (ATen's RowwiseMomentsCUDAKernel<Half> stores them
// in the input dtype), a = rstd * gamma, b = -a * mean + beta (ComputeFusedParamsCUDAKernel), y = fp16(fmaf(a, x, b));
// SiLU of the fp16 y as y / (1 + expf(-y)), rounded.  Each value is taken relative to a per-(sample, group) shift
// (the group's first element, so the sums do not cancel when |mean| >> std), summed in fp32 over the (<= 4) pixels
// x 8 channels of one load batch of a thread, then in fp64.  That matches or beats ATen's fp32 Welford while the
// shift is a typical element of its group.  When the shift is far from the group mean (an outlier of ~1000 in a
// group of unit spread), var = E[d^2] - mean(d)^2 cancels, the fp32 inner sums of d^2 carry that error, and rstd
// rounds to the other fp16 neighbour more often than ATen's does (tests/test_gpu_body_kernels.py, outlier_shift).
//
// At exactly 4 channels per group (the VAE's 128-channel levels with 32 groups) tf_group_norm_nhwc runs the same two
// kernels without the bias: a thread's 8-channel column then always spans two groups, the (lo, hi) pair of sums the
// kernels already carry for columns that straddle a group boundary.  They are compiled for that constant and get a
// larger apply chunk (gn_layout_g4).
//
// GEGLU.  out = fp16(float(xh) * float(fp16(gelu_erf(float(g))))) — the eager `F.linear(..) * F.gelu(F.linear(..))`
// with ATen's erf form of gelu, one read of each GEMM output and one write instead of writing and re-reading gelu(g).
#include "tf_common.cuh"
#include "tf_kernels.h"

namespace tf {
namespace {

constexpr int kGnMaxThreads = 512;                 // threads = (C / 8 columns) x rows, rows = 512 / columns
static_assert(kGnMaxChannels / 8 <= kGnMaxThreads, "one row of 8-channel columns must fit in a CTA");
constexpr int kGnStatsChunkBytes = 64 << 10;       // input bytes per statistics CTA
constexpr int kGnApplyChunkBytes = 128 << 10;      // input bytes per apply CTA
constexpr int kGnUnroll = 4;                       // 16-byte loads in flight per thread

struct GnLayout {
  int cols, rows, threads;
  long long stats_px, apply_px;
  int stats_chunks, apply_chunks;
};

GnLayout gn_layout(long long hw, int c) {
  GnLayout L;
  L.cols = c / 8;
  L.rows = kGnMaxThreads / L.cols > 0 ? kGnMaxThreads / L.cols : 1;
  L.threads = (L.cols * L.rows + 31) / 32 * 32;
  auto chunk = [&](int bytes) {
    long long px = bytes / (2LL * c);
    px = (px + L.rows - 1) / L.rows * L.rows;
    return px < L.rows ? (long long)L.rows : px;
  };
  L.stats_px = chunk(kGnStatsChunkBytes);
  L.apply_px = chunk(kGnApplyChunkBytes);
  L.stats_chunks = (int)((hw + L.stats_px - 1) / L.stats_px);
  L.apply_chunks = (int)((hw + L.apply_px - 1) / L.apply_px);
  return L;
}

// The 4-channel-group sites are the VAE's full-resolution levels (512^2 x 128 channels: 64 MB a sample).  Their
// statistics chunks are gn_layout's, so the workspace has the same [N, G, stats_chunks] format, but every apply CTA
// reduces all G x stats_chunks partials of its sample first: 512 KB at 512^2, four times a 128 KB apply chunk.  So
// an apply CTA takes at least 1/64 of the sample (1 MB there): the partials it reads, L2 hits, stay at half its input.
constexpr int kGnG4ApplyChunksPerSample = 64;

GnLayout gn_layout_g4(long long hw, int c) {
  GnLayout L = gn_layout(hw, c);
  long long px = (hw + kGnG4ApplyChunksPerSample - 1) / kGnG4ApplyChunksPerSample;
  px = (px + L.rows - 1) / L.rows * L.rows;
  if (px > L.apply_px) {
    L.apply_px = px;
    L.apply_chunks = (int)((hw + px - 1) / px);
  }
  return L;
}

__device__ __forceinline__ void unpack8(const uint4& raw, float (&v)[8]) {
  const __half2* h = reinterpret_cast<const __half2*>(&raw);
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float2 f = __half22float2(h[e]);
    v[2 * e] = f.x;
    v[2 * e + 1] = f.y;
  }
}

__device__ __forceinline__ float round_h(float x) { return __half2float(__float2half_rn(x)); }

// The group's shift: its first element (pixel 0, first channel), bias added and rounded like every other element.
template <bool kBias>
__device__ __forceinline__ float group_shift(const __half* xn, const __half* bias_n, int g, int cpg) {
  const int c = g * cpg;
  const float v = __half2float(xn[c]);
  return kBias ? round_h(v + __half2float(bias_n[c])) : v;
}

// kCpg: channels per group when known at compile time (4: the VAE's full-resolution sites), 0 = the runtime `cpg_rt`.
template <bool kBias, int kCpg>
__global__ void __launch_bounds__(kGnMaxThreads, 2)
gn_stats_kernel(const __half* __restrict__ x, const __half* __restrict__ bias, long long bias_stride, long long hw,
                int C, int cpg_rt, int G, int rows, long long chunk_px, int chunks, double2* __restrict__ ws) {
  const int cpg = kCpg ? kCpg : cpg_rt;
  extern __shared__ double2 part[];                 // [threads][2]: the (<= 2) groups a thread's 8 channels touch
  const int cols = C >> 3;
  const int tid = threadIdx.x;
  const int row = tid / cols, col = tid - row * cols;
  const int n = blockIdx.y, chunk = blockIdx.x;
  const __half* xn = x + (long long)n * hw * C;
  const __half* bias_n = kBias ? bias + (long long)n * bias_stride : nullptr;
  if (row < rows) {
    const int c0 = col * 8;
    float bv[8], shift[8];
    if (kBias) unpack8(*reinterpret_cast<const uint4*>(bias_n + c0), bv);
#pragma unroll
    for (int e = 0; e < 8; ++e) shift[e] = group_shift<kBias>(xn, bias_n, (c0 + e) / cpg, cpg);
    const int g_lo = c0 / cpg;
    int hi_mask = 0;                                // channels of the second group a column can straddle
#pragma unroll
    for (int e = 0; e < 8; ++e) hi_mask |= ((c0 + e) / cpg != g_lo) << e;
    double2 lo = make_double2(0.0, 0.0), hi = make_double2(0.0, 0.0);
    const long long p_begin = (long long)chunk * chunk_px;
    const long long p_end = p_begin + chunk_px < hw ? p_begin + chunk_px : hw;
    constexpr int kUnroll = kBias ? 2 : kGnUnroll;  // keeps the bias variant within 64 registers
    for (long long p = p_begin + row; p < p_end; p += (long long)rows * kUnroll) {
      uint4 raw[kUnroll];
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        const long long q = p + (long long)u * rows;
        if (q < p_end) raw[u] = *reinterpret_cast<const uint4*>(xn + q * C + c0);
      }
      float f1[8], f2[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) f1[e] = f2[e] = 0.f;
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        if (p + (long long)u * rows < p_end) {
          float v[8];
          unpack8(raw[u], v);
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            const float d = (kBias ? round_h(v[e] + bv[e]) : v[e]) - shift[e];
            f1[e] += d;
            f2[e] = fmaf(d, d, f2[e]);
          }
        }
      }
      float l1 = 0.f, l2 = 0.f, h1 = 0.f, h2 = 0.f;  // <= 32 values each in fp32, then fp64
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        if ((hi_mask >> e) & 1) { h1 += f1[e]; h2 += f2[e]; }
        else { l1 += f1[e]; l2 += f2[e]; }
      }
      lo.x += (double)l1;
      lo.y += (double)l2;
      hi.x += (double)h1;
      hi.y += (double)h2;
    }
    part[2 * tid] = lo;
    part[2 * tid + 1] = hi;
  }
  __syncthreads();
  for (int g = tid; g < G; g += blockDim.x) {       // fixed order: rows, then the group's columns
    const int cb = g * cpg / 8, ce = ((g + 1) * cpg - 1) / 8;
    double a = 0.0, b = 0.0;
    for (int r = 0; r < rows; ++r) {
      for (int cc = cb; cc <= ce; ++cc) {
        const double2 v = part[2 * (r * cols + cc) + (g - cc * 8 / cpg)];
        a += v.x;
        b += v.y;
      }
    }
    ws[((long long)n * G + g) * chunks + chunk] = make_double2(a, b);
  }
}

template <bool kBias, bool kSilu, int kCpg>
__global__ void __launch_bounds__(kGnMaxThreads, 2)
gn_apply_kernel(const __half* __restrict__ x, const __half* __restrict__ bias, long long bias_stride,
                const __half* __restrict__ gamma, const __half* __restrict__ beta, float eps, long long hw, int C,
                int cpg_rt, int G, int rows, long long chunk_px, const double2* __restrict__ ws, int stats_chunks,
                __half* __restrict__ out) {
  const int cpg = kCpg ? kCpg : cpg_rt;
  extern __shared__ float smem[];                   // a[C], b[C], mean[G], rstd[G]
  float* sa = smem;
  float* sb = sa + C;
  float* gmean = sb + C;
  float* grstd = gmean + G;
  const int cols = C >> 3;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  const int n = blockIdx.y, chunk = blockIdx.x;
  const __half* xn = x + (long long)n * hw * C;
  const __half* bias_n = kBias ? bias + (long long)n * bias_stride : nullptr;
  // group statistics: one warp per group, lane-strided sums then a fixed shuffle tree (lane 0's result is used)
  for (int g = warp; g < G; g += nwarps) {
    const double2* p = ws + ((long long)n * G + g) * stats_chunks;
    double a = 0.0, b = 0.0;
    for (int j = lane; j < stats_chunks; j += 32) {
      const double2 v = p[j];
      a += v.x;
      b += v.y;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      a += __shfl_down_sync(0xffffffffu, a, o);
      b += __shfl_down_sync(0xffffffffu, b, o);
    }
    if (lane == 0) {
      const double cnt = (double)hw * (double)cpg;
      const double m = a / cnt;
      double var = b / cnt - m * m;
      var = var > 0.0 ? var : 0.0;
      // ATen keeps mean / rstd in the input dtype (RowwiseMomentsCUDAKernel<Half>) and its eps argument too
      gmean[g] = round_h((float)((double)group_shift<kBias>(xn, bias_n, g, cpg) + m));
      grstd[g] = round_h(rsqrtf((float)var + round_h(eps)));
    }
  }
  __syncthreads();
  for (int c = tid; c < C; c += blockDim.x) {
    const int g = c / cpg;
    const float s = grstd[g] * __half2float(gamma[c]);
    sa[c] = s;
    sb[c] = -s * gmean[g] + __half2float(beta[c]);
  }
  __syncthreads();
  const int row = tid / cols, col = tid - row * cols;
  if (row >= rows) return;
  const int c0 = col * 8;
  float a[8], b[8], bv[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    a[e] = sa[c0 + e];
    b[e] = sb[c0 + e];
  }
  if (kBias) unpack8(*reinterpret_cast<const uint4*>(bias_n + c0), bv);
  __half* on = out + (long long)n * hw * C;
  const long long p_begin = (long long)chunk * chunk_px;
  const long long p_end = p_begin + chunk_px < hw ? p_begin + chunk_px : hw;
  constexpr int kUnroll = kBias && kSilu ? 2 : kGnUnroll;     // keeps the bias + SiLU variant within 64 registers
  for (long long p = p_begin + row; p < p_end; p += (long long)rows * kUnroll) {
    uint4 raw[kUnroll];
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const long long q = p + (long long)u * rows;
      if (q < p_end) raw[u] = *reinterpret_cast<const uint4*>(xn + q * C + c0);
    }
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const long long q = p + (long long)u * rows;
      if (q < p_end) {
        float v[8];
        unpack8(raw[u], v);
        uint4 w;
        __half2* h = reinterpret_cast<__half2*>(&w);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float y[2];
#pragma unroll
          for (int k = 0; k < 2; ++k) {
            const int i = 2 * e + k;
            const float xv = kBias ? round_h(v[i] + bv[i]) : v[i];
            y[k] = round_h(fmaf(a[i], xv, b[i]));
            if (kSilu) y[k] = y[k] / (1.0f + expf(-y[k]));
          }
          h[e] = __floats2half2_rn(y[0], y[1]);
        }
        *reinterpret_cast<uint4*>(on + q * C + c0) = w;
      }
    }
  }
}

__device__ __forceinline__ float gelu_erf(float v) {
  constexpr float kAlpha = 0.70710678118654752440f;  // M_SQRT1_2, as ATen's GeluCUDAKernelImpl rounds it
  return v * 0.5f * (1.0f + erff(v * kAlpha));
}

__device__ __forceinline__ float geglu1(float xv, float gv) { return xv * round_h(gelu_erf(gv)); }

__global__ void __launch_bounds__(256)
geglu_kernel(const __half* __restrict__ xh, const __half* __restrict__ gate, long long n_vec, long long n,
             __half* __restrict__ out) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_vec; i += stride) {
    float xv[8], gv[8];
    unpack8(reinterpret_cast<const uint4*>(xh)[i], xv);
    unpack8(reinterpret_cast<const uint4*>(gate)[i], gv);
    uint4 w;
    __half2* h = reinterpret_cast<__half2*>(&w);
#pragma unroll
    for (int e = 0; e < 4; ++e) h[e] = __floats2half2_rn(geglu1(xv[2 * e], gv[2 * e]), geglu1(xv[2 * e + 1], gv[2 * e + 1]));
    reinterpret_cast<uint4*>(out)[i] = w;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {        // tail (n not a multiple of 8)
    for (long long j = n_vec * 8; j < n; ++j)
      out[j] = __float2half_rn(geglu1(__half2float(xh[j]), __half2float(gate[j])));
  }
}

}  // namespace

long long group_norm_nhwc_workspace(long long n, long long hw, int c, int groups) {
  if (n <= 0 || hw <= 0 || c <= 0 || (c & 7) || groups <= 0 || c % groups) return 0;
  return n * groups * (long long)gn_layout(hw, c).stats_chunks * (long long)sizeof(double2);
}

namespace {

// Both channels-per-group cases: the same two kernels, the statistics layout of gn_layout (so the workspace has one
// format), and an apply layout of the caller's choice.  kCpg = 4 has no bias path (no 4-channel-group site adds one).
template <int kCpg>
int launch_gn(const GnLayout& L, const __half* xp, const __half* bp, long long bias_stride, const __half* gp,
              const __half* btp, long long n, long long hw, int c, int groups, float eps, int silu, double2* ws,
              __half* op, cudaStream_t stream, const char* stats_what, const char* apply_what) {
  const int cpg = c / groups;
  const size_t stats_smem = (size_t)L.threads * 2 * sizeof(double2);
  const size_t apply_smem = (2 * (size_t)c + 2 * (size_t)groups) * sizeof(float);   // <= 40 KB at C = 4096, G = 1024
  for (long long n0 = 0; n0 < n; n0 += 65535) {     // grid.y is the sample
    const unsigned ny = (unsigned)(n - n0 < 65535 ? n - n0 : 65535);
    const long long off = n0 * hw * c;
    const __half* bn = bp ? bp + n0 * bias_stride : nullptr;
    double2* wsn = ws + n0 * groups * (long long)L.stats_chunks;
    const dim3 gs((unsigned)L.stats_chunks, ny), ga((unsigned)L.apply_chunks, ny);
#define TF_GN_STATS(B)                                                                                             \
  gn_stats_kernel<B, kCpg><<<gs, L.threads, stats_smem, stream>>>(xp + off, bn, bias_stride, hw, c, cpg, groups,     \
                                                                  L.rows, L.stats_px, L.stats_chunks, wsn)
#define TF_GN_APPLY(B, S)                                                                                          \
  gn_apply_kernel<B, S, kCpg><<<ga, L.threads, apply_smem, stream>>>(xp + off, bn, bias_stride, gp, btp, eps, hw, c,  \
                                                                     cpg, groups, L.rows, L.apply_px, wsn,          \
                                                                     L.stats_chunks, op + off)
    if constexpr (kCpg == 0) {
      if (bn) TF_GN_STATS(true); else TF_GN_STATS(false);
    } else {
      TF_GN_STATS(false);
    }
    if (int e = check_cuda(cudaGetLastError(), stats_what)) return e;
    if constexpr (kCpg == 0) {
      if (bn) { if (silu) TF_GN_APPLY(true, true); else TF_GN_APPLY(true, false); }
      else { if (silu) TF_GN_APPLY(false, true); else TF_GN_APPLY(false, false); }
    } else {
      if (silu) TF_GN_APPLY(false, true); else TF_GN_APPLY(false, false);
    }
#undef TF_GN_STATS
#undef TF_GN_APPLY
    if (int e = check_cuda(cudaGetLastError(), apply_what)) return e;
  }
  return TF_OK;
}

}  // namespace

int launch_group_norm_nhwc(const void* x, const void* bias, long long bias_stride, const void* gamma, const void* beta,
                           long long n, long long hw, int c, int groups, float eps, int silu, void* workspace,
                           void* out, cudaStream_t stream) {
  const __half* xp = static_cast<const __half*>(x);
  const __half* gp = static_cast<const __half*>(gamma);
  const __half* btp = static_cast<const __half*>(beta);
  double2* ws = static_cast<double2*>(workspace);
  __half* op = static_cast<__half*>(out);
  if (c == 4 * groups)       // no bias here: tf_group_norm_nhwc refuses one at 4 channels per group
    return launch_gn<4>(gn_layout_g4(hw, c), xp, nullptr, 0, gp, btp, n, hw, c, groups, eps, silu, ws, op, stream,
                        "tf_group_norm_nhwc statistics launch", "tf_group_norm_nhwc apply launch");
  return launch_gn<0>(gn_layout(hw, c), xp, static_cast<const __half*>(bias), bias_stride, gp, btp, n, hw, c, groups,
                      eps, silu, ws, op, stream, "tf_group_norm_nhwc statistics launch",
                      "tf_group_norm_nhwc apply launch");
}

int launch_geglu(const void* xh, const void* gate, long long n, void* out, cudaStream_t stream) {
  if (n == 0) return TF_OK;
  const long long n_vec = n / 8;
  long long blocks = (n_vec + 255) / 256;
  const long long cap = (long long)sm_count() * 16;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  geglu_kernel<<<(unsigned)blocks, 256, 0, stream>>>(static_cast<const __half*>(xh), static_cast<const __half*>(gate),
                                                     n_vec, n, static_cast<__half*>(out));
  return check_cuda(cudaGetLastError(), "tf_geglu launch");
}

}  // namespace tf
