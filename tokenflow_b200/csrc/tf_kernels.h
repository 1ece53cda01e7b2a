// Internal launch interface between the C-ABI layer (tf_capi.cu) and the kernels.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace tf {

// Per-frame keyframe table, passed by value in kernel parameter space (no device allocation, no
// H2D copy).  Generalises the reference's scalar `batch_idx` (tokenflow_utils.py:331-333) to a
// per-frame (kf_a, kf_b, w) triple so frames — not only whole batches — can be sharded across GPUs.
constexpr int kMaxFrames = 64;
struct FrameTable {
  int32_t kf_a[kMaxFrames];
  int32_t kf_b[kMaxFrames];   // < 0: no second keyframe (reference batch 0)
  float w[kMaxFrames];        // blend weight of kf_a (reference :375-383)
};

int launch_unit_rows(const void* x, int x_is_f32, long long rows, int dim, long long row_stride, void* out_f16,
                     cudaStream_t stream);

int launch_layernorm_unit_rows(const void* x_f16, long long rows, int dim, long long row_stride, const float* gamma,
                               const float* beta, float eps, void* out_f16, cudaStream_t stream);

int launch_layernorm_rows(const void* x_f16, long long rows, int dim, long long row_stride, const float* gamma,
                          const float* beta, float eps, void* y_out, long long y_row_stride, void* unit_out,
                          long long unit_row_stride, long long unit_rows, cudaStream_t stream);

int launch_cfg_ddim(const void* eps_uncond, const void* eps_cond, const void* x, const float* coef_dev, float guidance,
                    long long n, void* out, cudaStream_t stream);
int launch_ddim(const void* eps, const void* x, const float* coef_dev, long long n, void* out, cudaStream_t stream);
// The same two updates for a v-prediction model (tf_cfg_ddim_v / tf_ddim_v).
int launch_cfg_ddim_v(const void* v_uncond, const void* v_cond, const void* x, const float* coef_dev, float guidance,
                      long long n, void* out, cudaStream_t stream);
int launch_ddim_v(const void* v, const void* x, const float* coef_dev, long long n, void* out, cudaStream_t stream);

// Channels-last GroupNorm (tf_body.cu): C / groups == 4 (no bias) or >= 8, C % 8 == 0, C <= kGnMaxChannels.
constexpr int kGnMaxChannels = 4096;
long long group_norm_nhwc_workspace(long long n, long long hw, int c, int groups);
int launch_group_norm_nhwc(const void* x, const void* bias, long long bias_stride, const void* gamma, const void* beta,
                           long long n, long long hw, int c, int groups, float eps, int silu, void* workspace,
                           void* out, cudaStream_t stream);
int launch_geglu(const void* xh, const void* gate, long long n, void* out, cudaStream_t stream);

// Pixel conversions around the VAE (tf_pixels.cu); n = elements (pixels x 3).
int launch_frames_to_nhwc(const void* frames, long long n, void* out, cudaStream_t stream);
int launch_nhwc_to_frames(const void* x, long long n, void* frames, cudaStream_t stream);

// Pillow's LANCZOS resize of RGB uint8 frames (tf_resize.cu): host-side tables, then one launch per pass.
int resize_taps(int in, int out);
void resize_coeffs(int in, int out, int32_t* bounds, int32_t* coeffs);
int launch_resize_h(const void* in, long long n_rows, int w_in, int w, const int32_t* bounds, const int32_t* coeffs,
                    int taps, void* out, cudaStream_t stream);
int launch_resize_v(const void* in, long long n, int h_in, int h, int w, const int32_t* bounds, const int32_t* coeffs,
                    int taps, void* out, cudaStream_t stream);

// OpenCV's Canny of RGB uint8 frames (tf_canny.cu): a classify launch and four union-find hysteresis launches.
long long canny_workspace(long long n, int h, int w);
int launch_canny(const void* frames, long long n, int h, int w, int low, int high, void* workspace, void* edges,
                 void* cond, cudaStream_t stream);

int launch_propagate(const void* A, const int32_t* idx_a, const int32_t* idx_b, const FrameTable& tab, int F,
                     int S, int dim, int K, const void* residual, void* out, int out_is_f32, long long F_total,
                     cudaStream_t stream);

int launch_nn_field(const void* x_unit, const void* piv_unit, const FrameTable& tab, int F, int S, int dim,
                    int K, int32_t* idx_a, int32_t* idx_b, cudaStream_t stream);

// One query sample of the extended-attention launch.
struct AttnSample {
  int32_t out_sample;  // which [S, dim] slab of `out` receives this sample's result
  int32_t q_sample;    // which [S, dim] slab of the q tensor holds this sample's queries
  int32_t k_sample0;   // first [S, dim] slab of the k tensor this sample attends to
  int32_t v_sample0;   // first [S, dim] slab of the v tensor
  int32_t n_kv;        // number of consecutive slabs attended to (1 = own frame, n = all keyframes)
};
constexpr int kMaxAttnSamples = 160;
struct AttnTable {
  AttnSample s[kMaxAttnSamples];
};

// One PAIR of output samples that share q and k and differ in v (PnP q/k injection: the uncond and the cond
// sample of a keyframe, reference tokenflow_utils.py:124-130).
constexpr int kMaxAttnPairs = 80;
struct AttnPair {
  int32_t out_u, out_c;      // output slabs of the two samples
  int32_t q_sample;          // shared query slab
  int32_t k_sample0;         // shared first key slab
  int32_t v_u0, v_c0;        // first value slab of each sample
  int32_t n_kv;
};
struct AttnPairTable {
  AttnPair p[kMaxAttnPairs];
};


bool ext_attn_pairs_supported(int d);
int launch_ext_attn_pairs(const void* q, const void* k, const void* v, long long q_tok_stride, long long kv_tok_stride,
                          int q_samples_total, int kv_samples_total, const AttnPairTable& tab, int n_pairs, int S,
                          int heads, int d, float scale, void* out, int q_row0, int q_nrows, cudaStream_t stream);

int launch_ext_attn(const void* q, const void* k, const void* v, long long q_tok_stride, long long kv_tok_stride,
                    int q_samples_total, int kv_samples_total, const AttnTable& tab, int n_out, int S, int heads,
                    int d, float scale, void* out, int q_row0, int q_nrows, cudaStream_t stream);

}  // namespace tf
