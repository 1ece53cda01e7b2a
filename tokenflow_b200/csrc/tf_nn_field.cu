// tf_nn_field — token nearest-neighbour field (reference tokenflow_utils.py:329-348 + util.py:61-69).
//
// For every token p of every frame f and each adjacent keyframe kf in {kf_a[f], kf_b[f]}:
//     idx[f,p] = argmax_c  fp16( x̂[f,p,:] . ŷ[kf,c,:] )          first index wins ties, NaN above every number
// with x̂, ŷ the fp16 unit rows produced by tf_unit_rows.  This is the arithmetic of the reference's
// GPU path (fp32 normalise -> fp16 operands -> fp32-accumulated GEMM -> *fp16 output* -> argmax),
// but the [B*S, 2S] similarity matrix (512 MB fp16 per block per batch at the 40-frame SD1.5
// config, written once and re-read twice by the reference) never exists: it lives 128xN tiles at
// a time in registers and is consumed by a running (max, first-argmax) epilogue.
//
// Kernel shape (one CTA per work item; kBlockN = 128):
//   work item   = (frame f, tile of 128 tokens, keyframe kf)                     -> 128 indices
//   warp 8      = TMA producer: the item's A tile (tokens x dim, resident for the whole N sweep
//                 when it fits in shared memory, else streamed with B) and a ring of B tiles
//                 (kBlockN keyframe tokens x 64 channels)
//   warpgroups  = 2, 64 token rows each: wgmma D[64 x kBlockN] (+)= A[64 x 16] . B[kBlockN x 16]^T
//                 with fp32 accumulators in registers, one 64-channel chunk in flight while the next
//                 is issued; after each N tile the epilogue rounds to fp16 and keeps a running
//                 (max, first index) per row and thread, merged across the 4 threads of a row at the end
// Operands are K-major with the 128-byte swizzle (TMA writes it, the wgmma descriptor reads it).
//
// Roofline: tensor-bound, 2*rows*S*dim flops per (frame, keyframe) pair; HBM traffic is only the
// operands (a few MB, L2 resident) and the int32 indices.
#include <cmath>

#include "tf_common.cuh"
#include "tf_kernels.h"
#include "tf_wgmma.cuh"

namespace tf {
namespace {

constexpr int kChunkK = 64;                 // channels per smem tile row: 64 x fp16 = one 128 B swizzle row
constexpr int kBlockM = 128;
constexpr int kBlockN = 128;
constexpr int kMaxStages = 8;
constexpr int kSmemBudget = 227 * 1024;

struct NNItems {
  int32_t n_a;                      // items [0, n_a): (frame, tile) against kf_a
  int32_t n_b;                      // items [n_a, n_a+n_b): frames listed in b_frames against kf_b
  int32_t tiles_per_frame;
  int32_t n_b_frames;
  int32_t b_frames[kMaxFrames];
};

struct SmemCtl {
  uint64_t full[kMaxStages];
  uint64_t empty[kMaxStages];
  uint64_t a_full;
};

template <bool kResidentA>
__global__ void __launch_bounds__(288, 1)
nn_field_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_p,
                const FrameTable tab, const NNItems items, int S, int dim, int stages,
                int32_t* __restrict__ idx_a, int32_t* __restrict__ idx_b) {
  constexpr int kAChunkBytes = kBlockM * 128;         // one 64-channel chunk of the A tile
  constexpr int kBChunkBytes = kBlockN * 128;
  constexpr int kStageBytes = kBChunkBytes + (kResidentA ? 0 : kAChunkBytes);
  constexpr int kAcc = kBlockN / 2;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int nkc = (dim + kChunkK - 1) / kChunkK;
  uint8_t* a_res = smem;                                               // resident A: nkc chunks
  uint8_t* ring = smem + (kResidentA ? nkc * kAChunkBytes : 0);        // stages x (B chunk + A chunk?)
  SmemCtl* ctl = reinterpret_cast<SmemCtl*>(ring + stages * kStageBytes);

  // work item -> (frame, first token of the tile, keyframe, output array)
  int f, m0, kf;
  int32_t* out;
  if ((int)blockIdx.x < items.n_a) {
    f = blockIdx.x / items.tiles_per_frame;
    m0 = (blockIdx.x - f * items.tiles_per_frame) * kBlockM;
    kf = tab.kf_a[f];
    out = idx_a;
  } else {
    const int j = blockIdx.x - items.n_a;
    const int fi = j / items.tiles_per_frame;
    f = items.b_frames[fi];
    m0 = (j - fi * items.tiles_per_frame) * kBlockM;
    kf = tab.kf_b[f];
    out = idx_b;
  }
  const int n_tiles = (S + kBlockN - 1) / kBlockN;
  const int J = n_tiles * nkc;                          // loads: (N tile, channel chunk), chunk fastest

  auto load = [&](int j) {
    const int st = j % stages;
    const int nt = j / nkc, kc = j - nt * nkc;
    uint8_t* dst = ring + st * kStageBytes;
    mbar_arrive_expect_tx(&ctl->full[st], (uint32_t)kStageBytes);
    tma_load_3d(dst, &map_p, &ctl->full[st], kc * kChunkK, nt * kBlockN, kf);
    if (!kResidentA) tma_load_3d(dst + kBChunkBytes, &map_x, &ctl->full[st], kc * kChunkK, m0, f);
  };

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_x);
    tma_prefetch_desc(&map_p);
    for (int i = 0; i < stages; ++i) {
      mbar_init(&ctl->full[i], 1);
      mbar_init(&ctl->empty[i], 8);                     // one arrival per warp
    }
    mbar_init(&ctl->a_full, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (threadIdx.x >= 256) {
    // ===================== TMA producer warp =====================
    if (threadIdx.x == 256) {
      if (kResidentA) {
        mbar_arrive_expect_tx(&ctl->a_full, (uint32_t)(nkc * kAChunkBytes));
        for (int kc = 0; kc < nkc; ++kc) tma_load_3d(a_res + kc * kAChunkBytes, &map_x, &ctl->a_full, kc * kChunkK, m0, f);
      }
      for (int j = 0; j < J; ++j) {
        if (j >= stages) mbar_wait(&ctl->empty[j % stages], (uint32_t)(j / stages - 1) & 1u);
        load(j);
      }
    }
    return;
  }

  const int wg = threadIdx.x >> 7;
  const int lane = threadIdx.x & 31;
  const int qcol = 2 * (lane & 3);
  const uint32_t ring_addr = smem_u32(ring);
  const uint32_t a_res_addr = smem_u32(a_res) + wg * 64 * 128;
  if (kResidentA) {
    mbar_wait(&ctl->a_full, 0);
    __syncwarp();
  }

  // the stage of load j may be refilled (every consumer warp arrives once)
  auto release = [&](int j) {
    __syncwarp();
    if (lane == 0) mbar_arrive(&ctl->empty[j % stages]);
  };

  float best[2] = {-INFINITY, -INFINITY};
  int best_idx[2] = {0, 0};
  int j = 0;
  for (int nt = 0; nt < n_tiles; ++nt) {
    float acc[kAcc];
    for (int kc = 0; kc < nkc; ++kc, ++j) {
      const int st = j % stages;
      mbar_wait(&ctl->full[st], (uint32_t)(j / stages) & 1u);
      __syncwarp();
      const uint32_t b_addr = ring_addr + st * kStageBytes;
      const uint32_t a_addr = kResidentA ? a_res_addr + kc * kAChunkBytes : b_addr + kBChunkBytes + wg * 64 * 128;
      wgmma_fence();
#pragma unroll
      for (int k4 = 0; k4 < kChunkK / 16; ++k4)
        wgmma_ss<kBlockN>(acc, wgmma_desc(a_addr + k4 * 32, 16, 1024), wgmma_desc(b_addr + k4 * 32, 16, 1024),
                          (kc > 0 || k4 > 0) ? 1u : 0u);
      wgmma_commit();
      if (kc > 0) {                                    // the previous chunk's MMAs are done: its stage is free
        wgmma_wait<1>();
        release(j - 1);
      }
    }
    wgmma_wait<0>();
    reg_fence(acc);
    release(j - 1);

    // epilogue: fp16-rounded similarities in torch.argmax's order (a NaN ranks above every number; a zero
    // token's unit row is NaN).  Each thread visits its columns in increasing order, so taking a value only
    // when it is greater or NaN, and nothing once the best is NaN, keeps the first of equal values or NaNs.
    const int n0 = nt * kBlockN;
#pragma unroll
    for (int jb = 0; jb < kBlockN / 8; ++jb) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int r = e >> 1;
        const int c = n0 + 8 * jb + qcol + (e & 1);
        const float h = __half2float(__float2half_rn(acc[4 * jb + e]));
        if (c < S && !(h <= best[r]) && best[r] == best[r]) { best[r] = h; best_idx[r] = c; }
      }
    }
  }

  // merge the four threads of each row in the same order: NaN above every number, the smaller index among
  // equal values or NaNs
#pragma unroll
  for (int r = 0; r < 2; ++r) {
#pragma unroll
    for (int off = 1; off <= 2; off <<= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best[r], off);
      const int oi = __shfl_xor_sync(0xffffffffu, best_idx[r], off);
      const bool o_nan = ob != ob, b_nan = best[r] != best[r];
      if ((!b_nan && !(ob <= best[r])) || ((ob == best[r] || (o_nan && b_nan)) && oi < best_idx[r])) {
        best[r] = ob;
        best_idx[r] = oi;
      }
    }
    const int p = m0 + wg * 64 + ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2) + 8 * r;
    if ((lane & 3) == 0 && p < S) out[(long long)f * S + p] = best_idx[r];
  }
}

template <bool kResidentA>
int launch_cfg(const void* x_unit, const void* piv_unit, const FrameTable& tab, const NNItems& items, int F, int S,
               int dim, int K, int32_t* idx_a, int32_t* idx_b, cudaStream_t stream) {
  const int nkc = (dim + kChunkK - 1) / kChunkK;
  const int a_bytes = kResidentA ? nkc * kBlockM * 128 : 0;
  const int stage_bytes = kBlockN * 128 + (kResidentA ? 0 : kBlockM * 128);
  int stages = (kSmemBudget - 2048 - a_bytes) / stage_bytes;
  if (stages > kMaxStages) stages = kMaxStages;
  if (stages < 2) {
    set_last_error("tf_nn_field: dim=%d does not fit the resident-A configuration", dim);
    return TF_ERR_UNSUPPORTED;
  }
  const size_t smem_bytes = 1024 + (size_t)a_bytes + (size_t)stages * stage_bytes + sizeof(SmemCtl);

  CUtensorMap map_x, map_p;
  {
    const uint64_t dims[3] = {(uint64_t)dim, (uint64_t)S, (uint64_t)F};
    const uint64_t strides[2] = {(uint64_t)dim * 2, (uint64_t)S * dim * 2};
    const uint32_t box[3] = {(uint32_t)kChunkK, (uint32_t)kBlockM, 1};
    CUresult r = encode_tiled(&map_x, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, x_unit, dims, strides, box,
                              CU_TENSOR_MAP_SWIZZLE_128B);
    if (r != CUDA_SUCCESS) { set_last_error("tf_nn_field: cuTensorMapEncodeTiled(x) failed: %d", (int)r); return TF_ERR_DRIVER; }
  }
  {
    const uint64_t dims[3] = {(uint64_t)dim, (uint64_t)S, (uint64_t)K};
    const uint64_t strides[2] = {(uint64_t)dim * 2, (uint64_t)S * dim * 2};
    const uint32_t box[3] = {(uint32_t)kChunkK, (uint32_t)kBlockN, 1};
    CUresult r = encode_tiled(&map_p, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, piv_unit, dims, strides, box,
                              CU_TENSOR_MAP_SWIZZLE_128B);
    if (r != CUDA_SUCCESS) { set_last_error("tf_nn_field: cuTensorMapEncodeTiled(pivots) failed: %d", (int)r); return TF_ERR_DRIVER; }
  }
  auto kern = nn_field_kernel<kResidentA>;
  if (check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes),
                 "tf_nn_field smem attribute"))
    return TF_ERR_CUDA;
  const int n_items = items.n_a + items.n_b;
  kern<<<n_items, 288, smem_bytes, stream>>>(map_x, map_p, tab, items, S, dim, stages, idx_a, idx_b);
  return check_cuda(cudaGetLastError(), "tf_nn_field launch");
}

}  // namespace

int launch_nn_field(const void* x_unit, const void* piv_unit, const FrameTable& tab, int F, int S, int dim, int K,
                    int32_t* idx_a, int32_t* idx_b, cudaStream_t stream) {
  if (F == 0 || S == 0) return TF_OK;
  NNItems items;
  items.tiles_per_frame = (S + kBlockM - 1) / kBlockM;
  items.n_a = F * items.tiles_per_frame;
  items.n_b_frames = 0;
  for (int f = 0; f < F; ++f)
    if (tab.kf_b[f] >= 0) items.b_frames[items.n_b_frames++] = f;
  items.n_b = items.n_b_frames * items.tiles_per_frame;
  if (items.n_b > 0 && idx_b == nullptr) {
    set_last_error("tf_nn_field: idx_b is NULL but some frame has a second keyframe");
    return TF_ERR_INVALID_ARGUMENT;
  }
  // The token tile stays in shared memory for the whole keyframe sweep while at least four B stages fit
  // beside it (dim <= 640: every SD level but the 1280-channel one); above that A streams with B.
  if (dim <= 640) return launch_cfg<true>(x_unit, piv_unit, tab, items, F, S, dim, K, idx_a, idx_b, stream);
  return launch_cfg<false>(x_unit, piv_unit, tab, items, F, S, dim, K, idx_a, idx_b, stream);
}

}  // namespace tf
