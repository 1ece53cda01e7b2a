// tf_canny_u8 — OpenCV's cv2.Canny(frame, low, high) of RGB uint8 frames (aperture 3, L1 gradient), bit for bit.
//
// The reference's ControlNet path conditions every UNet call on the Canny edges of its frame (preprocess.py:113-127
// get_canny_cond, cv2.Canny(img, 100, 200)).  OpenCV's algorithm (imgproc/src/canny.cpp), restated in oracle/canny.py:
//   - 3x3 Sobel dx, dy per channel with replicated borders; per pixel the channel of largest |dx| + |dy| (first on a
//     tie) gives the magnitude and the direction;
//   - non-maximum suppression with the 15-bit fixed-point tan(22.5 deg) sector test and OpenCV's asymmetric
//     neighbour comparisons, the magnitude being 0 outside the image;
//   - a surviving pixel is a candidate when its magnitude is > floor(low) and strong when > floor(high);
//   - hysteresis: the 8-connected components of candidates that contain a strong pixel.
// Five launches, no host loop and nothing read back, so the whole call can be captured in a CUDA graph:
//   1. classify: one block per 32 x 16 tile stages the frame with a 2-pixel halo in shared memory, computes the
//      gradients, the suppression and the thresholds, writes the class map and initialises the union-find labels and
//      root flags of the candidates (nothing reads them elsewhere);
//   2. merge: every candidate unites with its candidate neighbours to the left and in the row above (lock-free
//      union-find, the root of every tree is its smallest pixel index whatever the order of the atomics);
//   3. compress: every candidate points at its root;
//   4. flag: every strong pixel marks its root;
//   5. write: a candidate whose root is marked is an edge (255), written as the uint8 map and / or the fp16
//      conditioning tensor.
// The labels are a function of the components only, so the result is deterministic.
#include "tf_common.cuh"
#include "tf_kernels.h"

namespace tf {

namespace {

constexpr int kTileW = 32, kTileH = 16;
constexpr int kThreadsX = 32, kThreadsY = 8;
constexpr int kCannyShift = 15;
constexpr int kTg22 = 13573;                      // int(tan(22.5 deg) * 2^15 + 0.5)
constexpr int kInW = kTileW + 4, kInH = kTileH + 4;
constexpr int kMagW = kTileW + 2, kMagH = kTileH + 2;

struct Grad {
  int dx, dy, mag;
};

// Sobel of all three channels at input-tile position (ty, tx) (the centre of a 3 x 3 window), the channel with the
// largest L1 magnitude, first on a tie.
__device__ __forceinline__ Grad sobel3(const uint8_t (*in)[kInW][3], int ty, int tx) {
  Grad g = {0, 0, -1};
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int dx = (in[ty - 1][tx + 1][c] + 2 * in[ty][tx + 1][c] + in[ty + 1][tx + 1][c]) -
                   (in[ty - 1][tx - 1][c] + 2 * in[ty][tx - 1][c] + in[ty + 1][tx - 1][c]);
    const int dy = (in[ty + 1][tx - 1][c] + 2 * in[ty + 1][tx][c] + in[ty + 1][tx + 1][c]) -
                   (in[ty - 1][tx - 1][c] + 2 * in[ty - 1][tx][c] + in[ty - 1][tx + 1][c]);
    const int m = abs(dx) + abs(dy);
    if (m > g.mag) g = {dx, dy, m};
  }
  return g;
}

__global__ void __launch_bounds__(kThreadsX * kThreadsY) canny_classify_kernel(
    const uint8_t* __restrict__ frames, int h, int w, int low, int high, uint8_t* __restrict__ cls,
    int32_t* __restrict__ label, uint8_t* __restrict__ flag) {
  __shared__ uint8_t in[kInH][kInW][3];
  __shared__ int mag[kMagH][kMagW];
  const int n = blockIdx.z;
  const int x0 = blockIdx.x * kTileW, y0 = blockIdx.y * kTileH;
  const int tid = threadIdx.y * kThreadsX + threadIdx.x;
  const uint8_t* f = frames + (long long)n * h * w * 3;
  // input tile with a 2-pixel halo, coordinates clamped to the frame (BORDER_REPLICATE)
  for (int i = tid; i < kInH * kInW; i += kThreadsX * kThreadsY) {
    const int ty = i / kInW, tx = i % kInW;
    const int gy = min(max(y0 + ty - 2, 0), h - 1), gx = min(max(x0 + tx - 2, 0), w - 1);
    const uint8_t* p = f + ((long long)gy * w + gx) * 3;
    in[ty][tx][0] = p[0];
    in[ty][tx][1] = p[1];
    in[ty][tx][2] = p[2];
  }
  __syncthreads();
  // magnitude over the tile and a 1-pixel ring; 0 outside the frame
  for (int i = tid; i < kMagH * kMagW; i += kThreadsX * kThreadsY) {
    const int my = i / kMagW, mx = i % kMagW;
    const int gy = y0 + my - 1, gx = x0 + mx - 1;
    mag[my][mx] = (gy >= 0 && gy < h && gx >= 0 && gx < w) ? sobel3(in, my + 1, mx + 1).mag : 0;
  }
  __syncthreads();
  const int gx = x0 + threadIdx.x;
  if (gx >= w) return;
  for (int ly = threadIdx.y; ly < kTileH; ly += kThreadsY) {
    const int gy = y0 + ly;
    if (gy >= h) break;
    const int my = ly + 1, mx = threadIdx.x + 1;
    const Grad g = sobel3(in, ly + 2, threadIdx.x + 2);
    const int m = g.mag;
    bool keep = false;
    if (m > low) {
      const int ax = abs(g.dx);
      const int ay = abs(g.dy) << kCannyShift;
      const int tg22x = ax * kTg22;
      if (ay < tg22x) {
        keep = m > mag[my][mx - 1] && m >= mag[my][mx + 1];
      } else {
        const int tg67x = tg22x + (ax << (kCannyShift + 1));
        if (ay > tg67x) {
          keep = m > mag[my - 1][mx] && m >= mag[my + 1][mx];
        } else {
          const int s = (g.dx ^ g.dy) < 0 ? -1 : 1;
          keep = m > mag[my - 1][mx - s] && m > mag[my + 1][mx + s];
        }
      }
    }
    const long long p = ((long long)n * h + gy) * w + gx;
    const uint8_t c = keep ? (m > high ? 2 : 1) : 0;
    cls[p] = c;
    if (c) {          // labels and flags are only ever read at candidates
      label[p] = (int32_t)p;
      flag[p] = 0;
    }
  }
}

__device__ __forceinline__ int32_t find_root(const int32_t* label, int32_t x) {
  const volatile int32_t* l = label;
  int32_t nx = l[x];
  while (nx != x) {
    x = nx;
    nx = l[x];
  }
  return x;
}

// Unite the trees of a and b: the larger root is linked under the smaller one with atomicMin; when another thread
// changed that root first, retry from what it now points to.
__device__ __forceinline__ void unite(int32_t* label, int32_t a, int32_t b) {
  while (true) {
    a = find_root(label, a);
    b = find_root(label, b);
    if (a == b) return;
    if (a < b) {
      const int32_t old = atomicMin(&label[b], a);
      if (old == b) return;
      b = old;
    } else {
      const int32_t old = atomicMin(&label[a], b);
      if (old == a) return;
      a = old;
    }
  }
}

__global__ void canny_merge_kernel(const uint8_t* __restrict__ cls, int h, int w, long long total,
                                   int32_t* label) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= total || !cls[p]) return;
  const int x = (int)(p % w);
  const int y = (int)((p / w) % h);
  if (x > 0 && cls[p - 1]) unite(label, (int32_t)p, (int32_t)(p - 1));
  if (y > 0) {
    const long long up = p - w;
    if (x > 0 && cls[up - 1]) unite(label, (int32_t)p, (int32_t)(up - 1));
    if (cls[up]) unite(label, (int32_t)p, (int32_t)up);
    if (x + 1 < w && cls[up + 1]) unite(label, (int32_t)p, (int32_t)(up + 1));
  }
}

__global__ void canny_compress_kernel(const uint8_t* __restrict__ cls, long long total, int32_t* label) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= total || !cls[p]) return;
  label[p] = find_root(label, (int32_t)p);
}

__global__ void canny_flag_kernel(const uint8_t* __restrict__ cls, long long total, const int32_t* __restrict__ label,
                                  uint8_t* flag) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= total || cls[p] != 2) return;
  flag[label[p]] = 1;
}

__global__ void canny_write_kernel(const uint8_t* __restrict__ cls, long long total,
                                   const int32_t* __restrict__ label, const uint8_t* __restrict__ flag,
                                   uint8_t* __restrict__ edges, __half* __restrict__ cond) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= total) return;
  const bool e = cls[p] && flag[label[p]];      // label / flag are read only where cls is set
  if (edges) edges[p] = e ? 255 : 0;
  if (cond) {
    const __half v = __float2half(e ? 1.0f : 0.0f);
    cond[3 * p] = v;
    cond[3 * p + 1] = v;
    cond[3 * p + 2] = v;
  }
}

constexpr int kFlatThreads = 256;

}  // namespace

long long canny_workspace(long long n, int h, int w) {
  const long long px = n * h * w;
  const long long cls = (px + 15) / 16 * 16;
  return cls + 4 * cls + cls;        // class map, int32 labels, root flags
}

int launch_canny(const void* frames, long long n, int h, int w, int low, int high, void* workspace, void* edges,
                 void* cond, cudaStream_t stream) {
  const long long px = n * h * w;
  const long long cls_bytes = (px + 15) / 16 * 16;
  uint8_t* cls = static_cast<uint8_t*>(workspace);
  int32_t* label = reinterpret_cast<int32_t*>(cls + cls_bytes);
  uint8_t* flag = cls + 5 * cls_bytes;
  const dim3 tiles((w + kTileW - 1) / kTileW, (h + kTileH - 1) / kTileH, (unsigned)n);
  canny_classify_kernel<<<tiles, dim3(kThreadsX, kThreadsY), 0, stream>>>(static_cast<const uint8_t*>(frames), h, w,
                                                                          low, high, cls, label, flag);
  if (int e = check_cuda(cudaGetLastError(), "tf_canny_u8 classify launch")) return e;
  const unsigned blocks = (unsigned)((px + kFlatThreads - 1) / kFlatThreads);
  canny_merge_kernel<<<blocks, kFlatThreads, 0, stream>>>(cls, h, w, px, label);
  canny_compress_kernel<<<blocks, kFlatThreads, 0, stream>>>(cls, px, label);
  canny_flag_kernel<<<blocks, kFlatThreads, 0, stream>>>(cls, px, label, flag);
  canny_write_kernel<<<blocks, kFlatThreads, 0, stream>>>(cls, px, label, flag, static_cast<uint8_t*>(edges),
                                                          static_cast<__half*>(cond));
  return check_cuda(cudaGetLastError(), "tf_canny_u8 hysteresis launches");
}

}  // namespace tf
