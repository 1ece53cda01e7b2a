// C-ABI layer (include/tokenflow_b200.h): argument validation, per-frame tables, error plumbing.
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <initializer_list>
#include <vector>

#include "../../include/tokenflow_b200.h"
#include "tf_common.cuh"
#include "tf_kernels.h"

namespace tf {

static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int check_cuda(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return TF_OK;
  set_last_error("%s: %s (%s)", what, cudaGetErrorName(e), cudaGetErrorString(e));
  return TF_ERR_CUDA;
}

int sm_count() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cached[dev] = n;
  }
  return cached[dev];
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

CUresult encode_tiled(CUtensorMap* map, CUtensorMapDataType dtype, uint32_t rank, const void* base,
                      const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box,
                      CUtensorMapSwizzle swizzle) {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || !p)
      return CUDA_ERROR_NOT_FOUND;
    fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  cuuint64_t gdims[5];
  cuuint64_t gstrides[4];
  cuuint32_t gbox[5];
  cuuint32_t estr[5];
  for (uint32_t i = 0; i < rank; ++i) {
    gdims[i] = dims[i];
    gbox[i] = box[i];
    estr[i] = 1;
    if (i + 1 < rank) gstrides[i] = strides_bytes[i];
  }
  return fn(map, dtype, rank, const_cast<void*>(base), gdims, gstrides, gbox, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// The pointer rule of every entry point that enqueues work: each `required` pointer non-NULL and 16-byte aligned (the
// kernels move 16-byte vectors and address operands through TMA), each `optional` one NULL or 16-byte aligned, and
// `others_ok` the caller's verdict on the pointers that need less (coefficient rows, index and host tables).
static int check_pointers(const char* who, std::initializer_list<const void*> required,
                          std::initializer_list<const void*> optional = {}, bool others_ok = true) {
  bool ok = others_ok;
  for (const void* p : required) ok = ok && p && aligned16(p);
  for (const void* p : optional) ok = ok && aligned16(p);
  if (ok) return TF_OK;
  set_last_error("%s: NULL or misaligned pointer", who);
  return TF_ERR_INVALID_ARGUMENT;
}

// The status of `n_launches` kernel launches, counted for tf_launch_count when they were enqueued.
static int launched(int e, long long n_launches = 1) {
  if (!e) g_launches += n_launches;
  return e;
}

// An element-wise entry point: a length outside [0, max_n] is refused, an empty call succeeds without looking at a
// pointer, and `launch()` enqueues one kernel once the pointers pass check_pointers(who, ptrs, {}, others_ok).
template <class Launch>
static int elementwise(const char* who, int64_t n, int64_t max_n, std::initializer_list<const void*> ptrs,
                       bool others_ok, Launch launch) {
  if (n < 0 || n > max_n) { set_last_error("%s: n=%lld", who, (long long)n); return TF_ERR_INVALID_ARGUMENT; }
  if (n == 0) return TF_OK;
  if (int e = check_pointers(who, ptrs, {}, others_ok)) return e;
  return launched(launch());
}

// Frames [f0, f0 + n) of one tf_nn_field / tf_propagate launch.
struct FrameChunk {
  int f0, n;
  FrameTable tab;
};

// The launches of F frames, kMaxFrames per launch, every one validated before the caller enqueues the first.
// need_b: some frame has a second keyframe.
static int frame_chunks(std::vector<FrameChunk>& chunks, bool& need_b, const int32_t* kf_a, const int32_t* kf_b,
                        const float* w, int F, int K, const char* who) {
  if (F > 0 && !kf_a) { set_last_error("%s: kf_a is NULL", who); return TF_ERR_INVALID_ARGUMENT; }
  need_b = false;
  for (int f0 = 0; f0 < F; f0 += kMaxFrames) {
    chunks.push_back({f0, std::min(F - f0, kMaxFrames), {}});
    FrameTable& tab = chunks.back().tab;
    for (int f = 0; f < chunks.back().n; ++f) {
      const int a = kf_a[f0 + f];
      const int b = kf_b ? kf_b[f0 + f] : -1;
      if (a < 0 || a >= K || b >= K) {
        set_last_error("%s: frame %d has keyframe ids (%d,%d) outside [0,%d)", who, f, a, b, K);
        return TF_ERR_INVALID_ARGUMENT;
      }
      tab.kf_a[f] = a;
      tab.kf_b[f] = b < 0 ? -1 : b;
      tab.w[f] = w ? w[f0 + f] : 1.0f;
      need_b |= b >= 0;
    }
  }
  return TF_OK;
}

static int check_group_norm_shape(int64_t n, int64_t hw, int c, int groups) {
  if (n < 0 || hw < 0 || c <= 0 || (c & 7) || groups <= 0 || c % groups) {
    set_last_error("tf_group_norm_nhwc: bad shape n=%lld hw=%lld c=%d groups=%d (c %% 8 == 0 and groups | c required)",
                   (long long)n, (long long)hw, c, groups);
    return TF_ERR_INVALID_ARGUMENT;
  }
  if ((c / groups != 4 && c / groups < 8) || c > kGnMaxChannels) {
    set_last_error("tf_group_norm_nhwc: c=%d groups=%d not supported (c / groups == 4 or >= 8, c <= %d)", c, groups,
                   kGnMaxChannels);
    return TF_ERR_UNSUPPORTED;
  }
  return TF_OK;
}

constexpr int kResizeMaxSide = 1 << 16;

static bool resize_sizes_ok(int in, int out, const char* who) {
  if (in < 1 || out < 1 || in > kResizeMaxSide || out > kResizeMaxSide) {
    set_last_error("%s: sizes in=%d out=%d outside [1, %d]", who, in, out, kResizeMaxSide);
    return false;
  }
  return true;
}

// Canny: every pixel index of the call is an int32 label of the hysteresis pass
static bool canny_sizes_ok(int64_t n, int h, int w, const char* who) {
  if (n < 0 || n > 65535 || h < 1 || w < 1 || h > 65536 || w > 65536 ||
      (n > 0 && (int64_t)h * w > (INT32_MAX - 1) / n)) {
    set_last_error("%s: bad size n=%lld h=%d w=%d (n <= 65535, 1 <= h, w <= 65536, n*h*w < 2^31)", who, (long long)n,
                   h, w);
    return false;
  }
  return true;
}

}  // namespace tf

using namespace tf;

extern "C" {

int tf_version(void) { return 1004; }

const char* tf_last_error(void) { return g_err; }

int64_t tf_launch_count(void) { return (int64_t)g_launches.load(); }

int tf_unit_rows(const void* x, int x_is_f32, int64_t rows, int dim, int64_t x_row_stride, void* out_f16,
                 tf_stream_t stream) {
  if (rows < 0 || dim <= 0 || (dim & 7) || (x_row_stride & 3) || x_row_stride < dim) {
    set_last_error("tf_unit_rows: bad shape rows=%lld dim=%d stride=%lld (dim %% 8 == 0 required)", (long long)rows,
                   dim, (long long)x_row_stride);
    return TF_ERR_INVALID_ARGUMENT;
  }
  if (rows == 0) return TF_OK;
  if (int e = check_pointers("tf_unit_rows", {x, out_f16})) return e;
  return launched(launch_unit_rows(x, x_is_f32, rows, dim, x_row_stride, out_f16, static_cast<cudaStream_t>(stream)));
}

int tf_layernorm_unit_rows(const void* x_f16, int64_t rows, int dim, int64_t x_row_stride, const float* gamma,
                           const float* beta, float eps, void* out_f16, tf_stream_t stream) {
  if (rows < 0 || dim <= 0 || (dim & 7) || (x_row_stride & 7) || x_row_stride < dim) {
    set_last_error("tf_layernorm_unit_rows: bad shape rows=%lld dim=%d stride=%lld (dim %% 8 == 0 required)",
                   (long long)rows, dim, (long long)x_row_stride);
    return TF_ERR_INVALID_ARGUMENT;
  }
  if (rows == 0) return TF_OK;
  if (int e = check_pointers("tf_layernorm_unit_rows", {x_f16, gamma, beta, out_f16})) return e;
  return launched(launch_layernorm_unit_rows(x_f16, rows, dim, x_row_stride, gamma, beta, eps, out_f16,
                                             static_cast<cudaStream_t>(stream)));
}

int tf_layernorm_rows(const void* x_f16, int64_t rows, int dim, int64_t x_row_stride, const float* gamma,
                      const float* beta, float eps, void* y_out_f16, int64_t y_row_stride, void* unit_out_f16,
                      int64_t unit_row_stride, int64_t unit_rows, tf_stream_t stream) {
  if (rows < 0 || dim <= 0 || (dim & 7) || (x_row_stride & 7) || x_row_stride < dim ||
      (y_out_f16 && ((y_row_stride & 7) || y_row_stride < dim)) ||
      (unit_out_f16 && ((unit_row_stride & 7) || unit_row_stride < dim)) || unit_rows < 0) {
    set_last_error("tf_layernorm_rows: bad shape rows=%lld dim=%d strides=(%lld,%lld,%lld) (multiples of 8 required)",
                   (long long)rows, dim, (long long)x_row_stride, (long long)y_row_stride, (long long)unit_row_stride);
    return TF_ERR_INVALID_ARGUMENT;
  }
  if (rows == 0) return TF_OK;
  if (int e = check_pointers("tf_layernorm_rows", {x_f16, gamma, beta}, {y_out_f16, unit_out_f16})) return e;
  if (!y_out_f16 && (!unit_out_f16 || unit_rows == 0)) return TF_OK;
  return launched(launch_layernorm_rows(x_f16, rows, dim, x_row_stride, gamma, beta, eps, y_out_f16, y_row_stride,
                                        unit_out_f16, unit_row_stride, unit_rows, static_cast<cudaStream_t>(stream)));
}

int tf_cfg_ddim(const void* eps_uncond, const void* eps_cond, const void* x, const float* coef, float guidance,
                int64_t n, void* out, tf_stream_t stream) {
  return elementwise("tf_cfg_ddim", n, INT64_MAX, {eps_uncond, eps_cond, x, out}, coef != nullptr, [&] {
    return launch_cfg_ddim(eps_uncond, eps_cond, x, coef, guidance, n, out, static_cast<cudaStream_t>(stream));
  });
}

int tf_ddim(const void* eps, const void* x, const float* coef, int64_t n, void* out, tf_stream_t stream) {
  return elementwise("tf_ddim", n, INT64_MAX, {eps, x, out}, coef != nullptr, [&] {
    return launch_ddim(eps, x, coef, n, out, static_cast<cudaStream_t>(stream));
  });
}

int tf_cfg_ddim_v(const void* v_uncond, const void* v_cond, const void* x, const float* coef, float guidance,
                  int64_t n, void* out, tf_stream_t stream) {
  return elementwise("tf_cfg_ddim_v", n, INT64_MAX, {v_uncond, v_cond, x, out}, coef != nullptr, [&] {
    return launch_cfg_ddim_v(v_uncond, v_cond, x, coef, guidance, n, out, static_cast<cudaStream_t>(stream));
  });
}

int tf_ddim_v(const void* v, const void* x, const float* coef, int64_t n, void* out, tf_stream_t stream) {
  return elementwise("tf_ddim_v", n, INT64_MAX, {v, x, out}, coef != nullptr, [&] {
    return launch_ddim_v(v, x, coef, n, out, static_cast<cudaStream_t>(stream));
  });
}

int64_t tf_group_norm_nhwc_workspace(int64_t n, int64_t hw, int c, int groups) {
  if (check_group_norm_shape(n, hw, c, groups)) return -1;
  return (int64_t)group_norm_nhwc_workspace(n, hw, c, groups);
}

int tf_group_norm_nhwc(const void* x, const void* bias, int64_t bias_stride, const void* gamma, const void* beta,
                       int64_t n, int64_t hw, int c, int groups, float eps, int silu, void* workspace,
                       int64_t workspace_bytes, void* out, tf_stream_t stream) {
  if (int e = check_group_norm_shape(n, hw, c, groups)) return e;
  if (bias && c == 4 * groups) {
    set_last_error("tf_group_norm_nhwc: c=%d groups=%d: no bias add at 4 channels per group", c, groups);
    return TF_ERR_UNSUPPORTED;
  }
  if (bias && (bias_stride < 0 || (bias_stride & 7) || (bias_stride > 0 && bias_stride < c))) {
    set_last_error("tf_group_norm_nhwc: bias row stride %lld (0, or >= c and a multiple of 8)", (long long)bias_stride);
    return TF_ERR_INVALID_ARGUMENT;
  }
  if (n == 0 || hw == 0) return TF_OK;
  const long long need = group_norm_nhwc_workspace(n, hw, c, groups);
  if (workspace_bytes < need) {
    set_last_error("tf_group_norm_nhwc: workspace of %lld bytes, %lld needed", (long long)workspace_bytes, need);
    return TF_ERR_INVALID_ARGUMENT;
  }
  if (int e = check_pointers("tf_group_norm_nhwc", {x, workspace, out}, {bias}, gamma && beta)) return e;
  return launched(launch_group_norm_nhwc(x, bias, bias_stride, gamma, beta, n, hw, c, groups, eps, silu, workspace,
                                         out, static_cast<cudaStream_t>(stream)),
                  2 * ((n + 65534) / 65535));
}

int tf_frames_to_nhwc(const void* frames_u8, int64_t n_px, void* out_f16, tf_stream_t stream) {
  return elementwise("tf_frames_to_nhwc", n_px, INT64_MAX / 3, {frames_u8, out_f16}, true, [&] {
    return launch_frames_to_nhwc(frames_u8, 3 * n_px, out_f16, static_cast<cudaStream_t>(stream));
  });
}

int tf_nhwc_to_frames(const void* x_f16, int64_t n_px, void* frames_u8, tf_stream_t stream) {
  return elementwise("tf_nhwc_to_frames", n_px, INT64_MAX / 3, {x_f16, frames_u8}, true, [&] {
    return launch_nhwc_to_frames(x_f16, 3 * n_px, frames_u8, static_cast<cudaStream_t>(stream));
  });
}

int tf_resize_taps(int in, int out) {
  if (!resize_sizes_ok(in, out, "tf_resize_taps")) return -1;
  return resize_taps(in, out);
}

int tf_resize_coeffs(int in, int out, int32_t* bounds, int32_t* coeffs) {
  if (!resize_sizes_ok(in, out, "tf_resize_coeffs")) return TF_ERR_INVALID_ARGUMENT;
  if (!bounds || !coeffs) { set_last_error("tf_resize_coeffs: NULL table"); return TF_ERR_INVALID_ARGUMENT; }
  resize_coeffs(in, out, bounds, coeffs);
  return TF_OK;
}

int tf_resize_u8(const void* in, int64_t n, int h_in, int w_in, int h, int w, const int32_t* h_bounds,
                 const int32_t* h_coeffs, int h_taps, const int32_t* v_bounds, const int32_t* v_coeffs, int v_taps,
                 void* tmp, void* out, tf_stream_t stream) {
  if (n < 0 || !resize_sizes_ok(w_in, w, "tf_resize_u8") || !resize_sizes_ok(h_in, h, "tf_resize_u8")) {
    if (n < 0) set_last_error("tf_resize_u8: n=%lld", (long long)n);
    return TF_ERR_INVALID_ARGUMENT;
  }
  const bool need_h = w != w_in, need_v = h != h_in;
  if (need_h && h_taps != resize_taps(w_in, w)) {
    set_last_error("tf_resize_u8: horizontal table of %d taps, %d -> %d has %d", h_taps, w_in, w, resize_taps(w_in, w));
    return TF_ERR_INVALID_ARGUMENT;
  }
  if (need_v && v_taps != resize_taps(h_in, h)) {
    set_last_error("tf_resize_u8: vertical table of %d taps, %d -> %d has %d", v_taps, h_in, h, resize_taps(h_in, h));
    return TF_ERR_INVALID_ARGUMENT;
  }
  // Pillow's Image.resize takes a frame more than 100 times taller than wide through the vertical pass first when its
  // height shrinks (a vertical-only resize to (w_in, h), then a horizontal-only one); every other frame goes through
  // the horizontal pass first.  The two orders round the intermediate differently.
  const bool v_first = need_h && need_v && h_in > 100LL * w_in && h < h_in;
  const long long h_rows = v_first ? h : h_in;           // input rows per frame of the horizontal pass
  const int v_w = v_first ? w_in : w;                    // row width of the vertical pass
  const void* v_in = need_h && !v_first ? tmp : in;
  void* v_out = v_first ? tmp : out;
  // Both passes' grids (at most 2^31 - 1 blocks) are checked before the first launch, so that a refused call enqueues
  // nothing.  The horizontal pass runs one block per `rows` input rows, the vertical pass one per output row and
  // column block of 128 threads of 16 bytes (4 unless the row pitch and both pointers are 16-byte aligned):
  // launch_resize_h / launch_resize_v.  Written as divisions, so that no product overflows.
  constexpr long long kMaxBlocks = 0x7fffffffLL;
  if (need_h) {
    const long long rows = std::min(std::max(48LL * 1024 / (3LL * w_in + 16), 1LL), 4LL);
    if (n > kMaxBlocks * rows / h_rows) {
      set_last_error("tf_resize_u8: %lld frames of %lld rows of %d pixels are too many for one horizontal launch",
                     (long long)n, h_rows, w_in);
      return TF_ERR_UNSUPPORTED;
    }
  }
  if (need_v) {
    const uintptr_t src = reinterpret_cast<uintptr_t>(v_in), dst = reinterpret_cast<uintptr_t>(v_out);
    const long long per = (3LL * v_w) % 16 == 0 && (src & 15u) == 0 && (dst & 15u) == 0 ? 16 : 4;
    const long long col_blocks = (3LL * v_w + 128 * per - 1) / (128 * per);
    if (n > kMaxBlocks / (h * col_blocks)) {
      set_last_error("tf_resize_u8: %lld frames of %d rows of %d pixels are too many for one vertical launch",
                     (long long)n, h, v_w);
      return TF_ERR_UNSUPPORTED;
    }
  }
  if (n == 0) return TF_OK;
  if (!in || !out || (need_h && (!h_bounds || !h_coeffs)) || (need_v && (!v_bounds || !v_coeffs)) ||
      (need_h && need_v && !tmp)) {
    set_last_error("tf_resize_u8: NULL pointer");
    return TF_ERR_INVALID_ARGUMENT;
  }
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (!need_h && !need_v)          // Pillow returns a copy when the size is unchanged
    return check_cuda(cudaMemcpyAsync(out, in, (size_t)n * h * w * 3, cudaMemcpyDeviceToDevice, st), "tf_resize_u8 copy");
  if (v_first) {
    if (int e = launched(launch_resize_v(in, n, h_in, h, w_in, v_bounds, v_coeffs, v_taps, tmp, st))) return e;
    return launched(launch_resize_h(tmp, n * h, w_in, w, h_bounds, h_coeffs, h_taps, out, st));
  }
  if (need_h)
    if (int e = launched(launch_resize_h(in, n * h_in, w_in, w, h_bounds, h_coeffs, h_taps, need_v ? tmp : out, st)))
      return e;
  if (need_v) return launched(launch_resize_v(v_in, n, h_in, h, w, v_bounds, v_coeffs, v_taps, out, st));
  return TF_OK;
}

int64_t tf_canny_workspace(int64_t n, int h, int w) {
  if (!canny_sizes_ok(n, h, w, "tf_canny_workspace")) return -1;
  return (int64_t)canny_workspace(n, h, w);
}

int tf_canny_u8(const void* frames, int64_t n, int h, int w, double low, double high, void* workspace,
                int64_t workspace_bytes, void* edges_u8, void* cond_f16, tf_stream_t stream) {
  if (!canny_sizes_ok(n, h, w, "tf_canny_u8")) return TF_ERR_INVALID_ARGUMENT;
  if (!(low == low) || !(high == high)) {
    set_last_error("tf_canny_u8: NaN threshold");
    return TF_ERR_INVALID_ARGUMENT;
  }
  if (low > high) std::swap(low, high);          // cv2.Canny swaps, then floors
  const double lo = std::floor(low), hi = std::floor(high);
  // magnitudes are in [0, 2040]: thresholds past either end act like the ends
  const int ilo = (int)std::min(std::max(lo, -1.0), 2040.0), ihi = (int)std::min(std::max(hi, -1.0), 2040.0);
  if (n == 0) return TF_OK;
  const long long need = canny_workspace(n, h, w);
  if (workspace_bytes < need) {
    set_last_error("tf_canny_u8: workspace of %lld bytes, %lld needed", (long long)workspace_bytes, need);
    return TF_ERR_INVALID_ARGUMENT;
  }
  // the fp16 conditioning output is written element by element: 2-byte alignment is enough
  const bool cond_ok = !(reinterpret_cast<uintptr_t>(cond_f16) & 1u);
  if (int e = check_pointers("tf_canny_u8", {workspace}, {}, frames && (edges_u8 || cond_f16) && cond_ok)) return e;
  return launched(
      launch_canny(frames, n, h, w, ilo, ihi, workspace, edges_u8, cond_f16, static_cast<cudaStream_t>(stream)), 5);
}

int tf_geglu(const void* xh, const void* gate, int64_t n, void* out, tf_stream_t stream) {
  return elementwise("tf_geglu", n, INT64_MAX, {xh, gate, out}, true,
                     [&] { return launch_geglu(xh, gate, n, out, static_cast<cudaStream_t>(stream)); });
}

int tf_nn_field(const void* x_unit, const void* piv_unit, const int32_t* kf_a, const int32_t* kf_b, int F, int S,
                int dim, int K, int32_t* idx_a, int32_t* idx_b, tf_stream_t stream) {
  if (F < 0 || S < 0 || dim <= 0 || (dim & 7) || K <= 0) {
    set_last_error("tf_nn_field: bad shape F=%d S=%d dim=%d K=%d", F, S, dim, K);
    return TF_ERR_INVALID_ARGUMENT;
  }
  std::vector<FrameChunk> chunks;
  bool need_b;
  if (int e = frame_chunks(chunks, need_b, kf_a, kf_b, nullptr, F, K, "tf_nn_field")) return e;
  if (F == 0 || S == 0) return TF_OK;
  if (int e = check_pointers("tf_nn_field", {x_unit, piv_unit}, {}, idx_a && (!need_b || idx_b))) return e;
  const __half* xu = static_cast<const __half*>(x_unit);
  for (const FrameChunk& c : chunks) {                  // any number of frames: kMaxFrames per launch
    const long long off = (long long)c.f0 * S;
    if (int e = launched(launch_nn_field(xu + off * dim, piv_unit, c.tab, c.n, S, dim, K, idx_a + off,
                                         idx_b ? idx_b + off : nullptr, static_cast<cudaStream_t>(stream))))
      return e;
  }
  return TF_OK;
}

int tf_propagate(const void* A, const int32_t* idx_a, const int32_t* idx_b, const int32_t* kf_a,
                 const int32_t* kf_b, const float* w, int F, int S, int dim, int K, const void* residual,
                 void* out, int out_is_f32, tf_stream_t stream) {
  if (F < 0 || S < 0 || dim <= 0 || (dim & 7) || K <= 0) {
    set_last_error("tf_propagate: bad shape F=%d S=%d dim=%d K=%d", F, S, dim, K);
    return TF_ERR_INVALID_ARGUMENT;
  }
  std::vector<FrameChunk> chunks;
  bool need_b;
  if (int e = frame_chunks(chunks, need_b, kf_a, kf_b, w, F, K, "tf_propagate")) return e;
  if (F == 0 || S == 0) return TF_OK;
  if (int e = check_pointers("tf_propagate", {A, out}, {residual}, idx_a && (!need_b || (idx_b && w)))) return e;
  const size_t out_esz = out_is_f32 ? 4 : 2;
  for (const FrameChunk& c : chunks) {                  // any number of frames: kMaxFrames per launch, no copies
    const long long off = (long long)c.f0 * S;
    if (int e = launched(launch_propagate(A, idx_a + off, idx_b ? idx_b + off : nullptr, c.tab, c.n, S, dim, K,
                                          residual ? static_cast<const __half*>(residual) + off * dim : nullptr,
                                          static_cast<char*>(out) + (size_t)off * dim * out_esz, out_is_f32, F,
                                          static_cast<cudaStream_t>(stream))))
      return e;
  }
  return TF_OK;
}

int tf_ext_attn_fwd_rows(const void* q, int q_slabs, int64_t q_tok_stride, const void* k, const void* v,
                         int kv_slabs, int64_t kv_tok_stride, int n_out, const int32_t* out_slab,
                         const int32_t* q_slab, const int32_t* k_slab0, const int32_t* v_slab0,
                         const int32_t* n_kv, int S, int heads, int d, float scale, int q_row0, int q_nrows,
                         void* out, tf_stream_t stream) {
  if (q_row0 < 0 || q_nrows < 0 || (q_row0 & 127)) {
    set_last_error("tf_ext_attn: bad query row range [%d, +%d) (start must be a multiple of 128)", q_row0, q_nrows);
    return TF_ERR_INVALID_ARGUMENT;
  }
  if (n_out < 0 || S < 0 || heads <= 0 || d <= 0 || (d & 7) ||
      q_tok_stride < (int64_t)heads * d || kv_tok_stride < (int64_t)heads * d || (q_tok_stride & 7) ||
      (kv_tok_stride & 7)) {
    set_last_error("tf_ext_attn: bad shape n_out=%d S=%d heads=%d d=%d strides=(%lld,%lld)", n_out, S, heads, d,
                   (long long)q_tok_stride, (long long)kv_tok_stride);
    return TF_ERR_INVALID_ARGUMENT;
  }
  if (n_out == 0 || S == 0 || q_nrows == 0 || q_row0 >= S) return TF_OK;
  if (int e = check_pointers("tf_ext_attn", {q, k, v, out}, {}, out_slab && q_slab && k_slab0 && v_slab0 && n_kv))
    return e;
  for (int i = 0; i < n_out; ++i) {
    if (q_slab[i] < 0 || q_slab[i] >= q_slabs || n_kv[i] <= 0 || k_slab0[i] < 0 || v_slab0[i] < 0 ||
        k_slab0[i] + n_kv[i] > kv_slabs || v_slab0[i] + n_kv[i] > kv_slabs || out_slab[i] < 0) {
      set_last_error("tf_ext_attn: sample %d has an out-of-range slab (q=%d k0=%d v0=%d n_kv=%d)", i, q_slab[i],
                     k_slab0[i], v_slab0[i], n_kv[i]);
      return TF_ERR_INVALID_ARGUMENT;
    }
  }
  // Samples that share q and k (PnP q/k injection: the uncond and cond sample of a keyframe, reference :124-130) have
  // identical scores and probabilities: pair them and let one kernel compute S / P once and both P V products.
  std::vector<int> partner(n_out, -1);
  int n_pairs = 0;
  if (ext_attn_pairs_supported(d)) {
    for (int i = 0; i < n_out; ++i) {
      if (partner[i] >= 0) continue;
      for (int j = i + 1; j < n_out; ++j) {
        if (partner[j] < 0 && q_slab[j] == q_slab[i] && k_slab0[j] == k_slab0[i] && n_kv[j] == n_kv[i] &&
            v_slab0[j] != v_slab0[i] && out_slab[j] != out_slab[i]) {
          partner[i] = j;
          partner[j] = i;
          ++n_pairs;
          break;
        }
      }
    }
  }
  if (n_pairs > 0) {
    std::vector<int> lead;
    for (int i = 0; i < n_out; ++i)
      if (partner[i] > i) lead.push_back(i);
    std::stable_sort(lead.begin(), lead.end(), [&](int a, int b) { return n_kv[a] > n_kv[b]; });
    for (int p0 = 0; p0 < n_pairs; p0 += kMaxAttnPairs) {
      const int nc = n_pairs - p0 < kMaxAttnPairs ? n_pairs - p0 : kMaxAttnPairs;
      AttnPairTable ptab;
      memset(&ptab, 0, sizeof(ptab));
      for (int slot = 0; slot < nc; ++slot) {
        const int i = lead[p0 + slot], j = partner[i];
        ptab.p[slot].out_u = out_slab[i];
        ptab.p[slot].out_c = out_slab[j];
        ptab.p[slot].q_sample = q_slab[i];
        ptab.p[slot].k_sample0 = k_slab0[i];
        ptab.p[slot].v_u0 = v_slab0[i];
        ptab.p[slot].v_c0 = v_slab0[j];
        ptab.p[slot].n_kv = n_kv[i];
      }
      if (int e = launched(launch_ext_attn_pairs(q, k, v, q_tok_stride, kv_tok_stride, q_slabs, kv_slabs, ptab, nc, S,
                                                 heads, d, scale, out, q_row0, q_nrows,
                                                 static_cast<cudaStream_t>(stream))))
        return e;
    }
  }
  // heavy samples (most key slabs) first: the hardware block scheduler then fills the tail of the
  // grid with the cheap own-frame (source stream) samples
  std::vector<int> order;
  for (int i = 0; i < n_out; ++i)
    if (partner[i] < 0) order.push_back(i);
  const int n_single = (int)order.size();
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return n_kv[a] > n_kv[b]; });
  for (int s0 = 0; s0 < n_single; s0 += kMaxAttnSamples) {    // any number of samples: kMaxAttnSamples per launch
    const int nc = n_single - s0 < kMaxAttnSamples ? n_single - s0 : kMaxAttnSamples;
    AttnTable tab;
    memset(&tab, 0, sizeof(tab));
    for (int slot = 0; slot < nc; ++slot) {
      const int i = order[s0 + slot];
      tab.s[slot].out_sample = out_slab[i];
      tab.s[slot].q_sample = q_slab[i];
      tab.s[slot].k_sample0 = k_slab0[i];
      tab.s[slot].v_sample0 = v_slab0[i];
      tab.s[slot].n_kv = n_kv[i];
    }
    if (int e = launched(launch_ext_attn(q, k, v, q_tok_stride, kv_tok_stride, q_slabs, kv_slabs, tab, nc, S, heads, d,
                                         scale, out, q_row0, q_nrows, static_cast<cudaStream_t>(stream))))
      return e;
  }
  return TF_OK;
}

int tf_ext_attn_fwd(const void* q, const void* k, const void* v, int64_t tok_stride, int n_frames, int S,
                    int heads, int d, float scale, int inject, void* out, tf_stream_t stream) {
  const int n = n_frames;
  if (n < 0) {
    set_last_error("tf_ext_attn_fwd: n_frames=%d", n);
    return TF_ERR_INVALID_ARGUMENT;
  }
  std::vector<int32_t> out_slab(3 * n), q_slab(3 * n), k0(3 * n), v0(3 * n), nkv(3 * n);
  for (int s = 0; s < 3; ++s) {
    for (int f = 0; f < n; ++f) {
      const int i = s * n + f;
      out_slab[i] = i;
      if (s == 0) {                       // source stream: own frame only (reference :173,:177)
        q_slab[i] = f; k0[i] = f; v0[i] = f; nkv[i] = 1;
      } else {                            // uncond / cond: all n frames of the stream (:133-138)
        q_slab[i] = inject ? f : i;       // injection (:126,:129): q of the source stream
        k0[i] = inject ? 0 : s * n;       // injection (:127,:130): k of the source stream
        v0[i] = s * n;                    // v is never injected
        nkv[i] = n;
      }
    }
  }
  return tf_ext_attn_fwd_rows(q, 3 * n, tok_stride, k, v, 3 * n, tok_stride, 3 * n, out_slab.data(), q_slab.data(),
                              k0.data(), v0.data(), nkv.data(), S, heads, d, scale, 0, S, out, stream);
}

}  // extern "C"
