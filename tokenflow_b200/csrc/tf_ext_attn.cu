// tf_ext_attn — extended cross-frame self-attention over the keyframes
// (reference tokenflow_utils.py:114-199 PnP flavour, :224-281 SDEdit flavour).
//
// For every output sample (stream s, keyframe f), head j and query token p:
//     O[p,:] = softmax_c( Q[p,:] . K[c,:] * scale ) V[c,:]
// where c runs over the S tokens of the sample's own frame (source stream) or over the n*S tokens
// of ALL keyframes of its stream, frame-major (uncond / cond streams).  The reference materialises
// per head an [n, S, n*S] fp16 score tensor and an fp32 probability tensor (0.84 + 1.68 GB at the
// 40-frame SD1.5 top level), replicates K and V n times and shuffles heads through ~10 copies
// (SURVEY.md §2.1 k1-k6).  Here none of that exists: one CTA owns a 128-query tile of one
// (sample, head), streams the key/value tiles of every attended keyframe through shared memory
// with TMA, keeps scores, probabilities and the output accumulator in registers, and addresses
// heads by stride inside the [sample, S, heads, d] tensors.  PnP q/k injection (:124-130) is pure
// aliasing: the per-sample table names which q / k slab to read.
//
// CTA = 2 warpgroups, 64 query rows each (FlashAttention-2 online softmax, fp32 statistics):
//   S = Q K_t^T      wgmma, both operands from shared memory (K-major, 128-byte swizzle)
//   P = exp2(S * scale*log2e - m + 8)   in registers, rounded to fp16 into the wgmma A-fragment layout
//   O = O*corr + P V_t   wgmma, P from registers, V from shared memory (MN-major), into a fresh accumulator
//                    that is added to O with one fp32 FMA per tile
//   l += sum_t(P)    fp32: each thread sums its columns of the tile into a fresh partial, then adds it to l
//
// Rounding: P is at most 2^8, so fp16 P is relative to 2^-11 down to 2^-22 of the row maximum and below that
// absolute to 2^-33 of it (fp16 subnormals; the offset keeps that far below the relative term even over
// 204 800 keys).  Both running sums, O and l, take one rounding per tile, not one per key: a running sum near
// the row maximum would otherwise swamp every key below about 2^-24 of it.  The tensor core's fp32
// accumulation drops such products from O, and l summed key by key dropped them on its own terms, so the two
// disagreed by up to N * 2^-25 of the row mass: on an H100 (700 W), at 204 800 keys whose tail sits 2^-25
// below a maximum in the first tile, the output was 0.4 % off with both sums taken key by key and 0.5 % off
// with only l taken per tile.  The fresh accumulator costs kO registers per value tensor: the paired kernels
// at d = 40 and 64 reach 255 registers and spill 24-28 bytes, and run 2-3.5 % slower than with O += P V_t.
// Thread 0 also issues the TMA loads: the Q tile once, then a ring of {K tile, V tile} stages; a
// stage is refilled one tile after both warpgroups released it, so neither waits on the other.
// The two warpgroups' softmax and MMA phases interleave on the SM.
//
// Paired samples (PnP q/k injection: the uncond and cond sample of a keyframe share q and k, so
// their scores and probabilities are identical): one CTA computes P once and P V_u, P V_c into two
// accumulators.
//
// Head dims that are not a multiple of 64 (SD1.5: 40, 80, 160) are zero-padded by TMA out-of-bound
// fill: the tensor maps describe [d, heads, S, samples] with the true inner extent d and a 64-wide
// box, so shared-memory rows are always one full 128-byte swizzle row.
//
// Roofline: tensor-bound, 4*S_q*S_kv*d flops per (sample, head); HBM traffic is q,k,v,out once
// (K/V tiles re-read by the other query tiles hit L2).
#include <cmath>
#include <type_traits>

#include "tf_common.cuh"
#include "tf_kernels.h"
#include "tf_wgmma.cuh"

namespace tf {
namespace {

constexpr int kBlockM = 128;
constexpr int kMaxStages = 8;
constexpr int kSmemBudget = 227 * 1024;
constexpr float kPOffset = 8.f;   // log2 of the largest P: moves the fp16 subnormal range 8 octaves further down

struct AttnCtl {
  uint64_t q_full;
  uint64_t full[kMaxStages];
  uint64_t empty[kMaxStages];
};

struct AttnParams {
  int S, heads, d;
  int tiles_m;            // query tiles per (sample, head)
  int stages;
  float scale_log2;       // scale * log2(e)
  long long out_tok_stride;   // elements between consecutive tokens of `out` (= heads*d)
  int q_row0;             // first query token this launch computes (multi-GPU: query rows are split across ranks)
  int q_row_end;          // one past the last query token (<= S)
  int out_rows;           // rows per slab of `out`: out is [slabs, out_rows, heads*d], row = token - q_row0
};

// One CTA's sample, single or paired (out_c / v_c0 unused for a single sample).
struct Item {
  int out_u, out_c, q, k0, v_u0, v_c0, n_kv;
};
__device__ __forceinline__ Item item_of(const AttnTable& t, int i) {
  const AttnSample& s = t.s[i];
  return {s.out_sample, -1, s.q_sample, s.k_sample0, s.v_sample0, -1, s.n_kv};
}
__device__ __forceinline__ Item item_of(const AttnPairTable& t, int i) {
  const AttnPair& p = t.p[i];
  return {p.out_u, p.out_c, p.q_sample, p.k_sample0, p.v_u0, p.v_c0, p.n_kv};
}

// kDChunks: 64-channel chunks of the head dim; kBlockN: keys per tile; kNPV: head dim rounded up to 16
// (N of the P V MMA).
template <int kDChunks, int kBlockN, int kNPV, class Tab>
__global__ void __launch_bounds__(256, 1)
ext_attn_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
                const __grid_constant__ CUtensorMap map_v, const __grid_constant__ Tab tab, const AttnParams prm,
                __half* __restrict__ out) {
  constexpr int kNV = std::is_same<Tab, AttnPairTable>::value ? 2 : 1;   // value tensors per stage
  constexpr int kQChunkBytes = kBlockM * 128;
  constexpr int kKVChunkBytes = kBlockN * 128;
  constexpr int kQBytes = kDChunks * kQChunkBytes;
  constexpr int kTileBytes = kDChunks * kKVChunkBytes;         // one K tile or one V tile
  constexpr int kStageBytes = (1 + kNV) * kTileBytes;
  constexpr int kS = kBlockN / 2;                               // score registers per thread
  constexpr int kO = kNPV / 2;                                  // output registers per thread and value tensor
  static_assert(kNPV <= 64 * kDChunks, "P V width exceeds the loaded channels");

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* q_smem = smem;
  uint8_t* ring = smem + kQBytes;
  AttnCtl* ctl = reinterpret_cast<AttnCtl*>(ring + prm.stages * kStageBytes);

  // ---- work item: heavy (extended) samples first so the tail of the grid is made of light items ----
  const int S = prm.S, d = prm.d, stages = prm.stages;
  const int per_sample = prm.heads * prm.tiles_m;
  const int slot = blockIdx.x / per_sample;
  const int rem = blockIdx.x - slot * per_sample;
  const int head = rem / prm.tiles_m;
  const int m0 = prm.q_row0 + (rem - head * prm.tiles_m) * kBlockM;
  const Item it = item_of(tab, slot);
  const int tiles_per_slab = (S + kBlockN - 1) / kBlockN;
  const int T = it.n_kv * tiles_per_slab;
  const int ksteps = (d + 15) / 16;                             // QK^T k-steps (zero padded to 16)

  auto load_tile = [&](int t) {
    const int st = t % stages;
    const int slab = t / tiles_per_slab;
    const int n0 = (t - slab * tiles_per_slab) * kBlockN;
    uint8_t* dst = ring + st * kStageBytes;
    mbar_arrive_expect_tx(&ctl->full[st], (uint32_t)kStageBytes);
#pragma unroll
    for (int c = 0; c < kDChunks; ++c) {
      tma_load_4d(dst + c * kKVChunkBytes, &map_k, &ctl->full[st], c * 64, head, n0, it.k0 + slab);
      tma_load_4d(dst + kTileBytes + c * kKVChunkBytes, &map_v, &ctl->full[st], c * 64, head, n0, it.v_u0 + slab);
      if (kNV == 2)
        tma_load_4d(dst + 2 * kTileBytes + c * kKVChunkBytes, &map_v, &ctl->full[st], c * 64, head, n0,
                    it.v_c0 + slab);
    }
  };

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_q);
    tma_prefetch_desc(&map_k);
    tma_prefetch_desc(&map_v);
    mbar_init(&ctl->q_full, 1);
    for (int i = 0; i < stages; ++i) {
      mbar_init(&ctl->full[i], 1);
      mbar_init(&ctl->empty[i], 8);                             // one arrival per warp
    }
    fence_mbar_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_arrive_expect_tx(&ctl->q_full, (uint32_t)kQBytes);
#pragma unroll
    for (int c = 0; c < kDChunks; ++c) tma_load_4d(q_smem + c * kQChunkBytes, &map_q, &ctl->q_full, c * 64, head, m0, it.q);
    for (int t = 0; t < stages && t < T; ++t) load_tile(t);
  }
  __syncwarp();

  const int wg = threadIdx.x >> 7;
  const int lane = threadIdx.x & 31;
  const int wrow = ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2);   // first of the thread's two rows in the warpgroup
  const int qcol = 2 * (lane & 3);                                // first of the thread's two columns in an n8 block

  float o[kNV][kO];
#pragma unroll
  for (int v = 0; v < kNV; ++v)
#pragma unroll
    for (int i = 0; i < kO; ++i) o[v][i] = 0.f;
  float m_r[2] = {-INFINITY, -INFINITY}, l_r[2] = {0.f, 0.f};
  const float sl2 = prm.scale_log2;

  const uint32_t q_addr = smem_u32(q_smem) + wg * 64 * 128;
  const uint32_t ring_addr = smem_u32(ring);
  mbar_wait(&ctl->q_full, 0);
  __syncwarp();

  for (int t = 0; t < T; ++t) {
    const int st = t % stages;
    mbar_wait(&ctl->full[st], (uint32_t)(t / stages) & 1u);
    __syncwarp();
    const uint32_t k_addr = ring_addr + st * kStageBytes;

    // ---- S = Q K^T ----
    float s[kS];
    wgmma_fence();
    for (int kk = 0; kk < ksteps; ++kk) {
      const uint32_t off = (kk & 3) * 32;
      wgmma_ss<kBlockN>(s, wgmma_desc(q_addr + (kk >> 2) * kQChunkBytes + off, 16, 1024),
                        wgmma_desc(k_addr + (kk >> 2) * kKVChunkBytes + off, 16, 1024), kk > 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(s);

    // ---- keys past the end of the keyframe (ragged last tile of a slab) ----
    const int n0 = (t % tiles_per_slab) * kBlockN;
    if (n0 + kBlockN > S) {
      const int valid = S - n0;
#pragma unroll
      for (int j = 0; j < kBlockN / 8; ++j) {
        const int c = 8 * j + qcol;
        if (c >= valid) { s[4 * j] = -INFINITY; s[4 * j + 2] = -INFINITY; }
        if (c + 1 >= valid) { s[4 * j + 1] = -INFINITY; s[4 * j + 3] = -INFINITY; }
      }
    }

    // ---- online softmax (log2 domain) ----
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int j = 0; j < kBlockN / 8; ++j) {
      mx[0] = fmaxf(mx[0], fmaxf(s[4 * j], s[4 * j + 1]));
      mx[1] = fmaxf(mx[1], fmaxf(s[4 * j + 2], s[4 * j + 3]));
    }
    float corr[2], mneg[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      const float m_new = fmaxf(m_r[r], mx[r] * sl2);
      corr[r] = fast_exp2(m_r[r] - m_new);
      m_r[r] = m_new;
      mneg[r] = kPOffset - m_new;
      l_r[r] *= corr[r];
    }
    uint32_t pa[kBlockN / 16][4];
    float lt[2] = {0.f, 0.f};                                     // this tile's share of l
#pragma unroll
    for (int j = 0; j < kBlockN / 8; ++j) {
      const float p0 = fast_exp2(fmaf(s[4 * j], sl2, mneg[0]));
      const float p1 = fast_exp2(fmaf(s[4 * j + 1], sl2, mneg[0]));
      const float p2 = fast_exp2(fmaf(s[4 * j + 2], sl2, mneg[1]));
      const float p3 = fast_exp2(fmaf(s[4 * j + 3], sl2, mneg[1]));
      lt[0] += p0 + p1;
      lt[1] += p2 + p3;
      pa[j >> 1][(j & 1) * 2 + 0] = pack_f16x2_rn(p0, p1);
      pa[j >> 1][(j & 1) * 2 + 1] = pack_f16x2_rn(p2, p3);
    }
    l_r[0] += lt[0];
    l_r[1] += lt[1];

    // ---- O = O * corr + P V_t (the tile's product in a fresh accumulator, added with one rounding) ----
    float ot[kNV][kO];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kBlockN / 16; ++kk)
#pragma unroll
      for (int v = 0; v < kNV; ++v)
        wgmma_rs<kNPV>(ot[v], pa[kk], wgmma_desc(k_addr + (1 + v) * kTileBytes + kk * 16 * 128, kKVChunkBytes, 1024),
                       kk > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int v = 0; v < kNV; ++v) {
      reg_fence(ot[v]);
#pragma unroll
      for (int j = 0; j < kO / 4; ++j) {
        o[v][4 * j] = fmaf(o[v][4 * j], corr[0], ot[v][4 * j]);
        o[v][4 * j + 1] = fmaf(o[v][4 * j + 1], corr[0], ot[v][4 * j + 1]);
        o[v][4 * j + 2] = fmaf(o[v][4 * j + 2], corr[1], ot[v][4 * j + 2]);
        o[v][4 * j + 3] = fmaf(o[v][4 * j + 3], corr[1], ot[v][4 * j + 3]);
      }
    }

    __syncwarp();
    if (lane == 0) mbar_arrive(&ctl->empty[st]);
    // refill the stage of the previous tile (both warpgroups are past it by now, typically)
    if (threadIdx.x == 0 && t >= 1 && t - 1 + stages < T) {
      const int pt = t - 1;
      mbar_wait(&ctl->empty[pt % stages], (uint32_t)(pt / stages) & 1u);
      load_tile(pt + stages);
    }
    __syncwarp();
  }

  // ---- O / l, fp16, rows inside [q_row0, q_row_end) ----
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_r[r] += __shfl_xor_sync(0xffffffffu, l_r[r], 1);
    l_r[r] += __shfl_xor_sync(0xffffffffu, l_r[r], 2);
    l_r[r] = 1.f / l_r[r];
  }
#pragma unroll
  for (int v = 0; v < kNV; ++v) {
    const int out_slab = v == 0 ? it.out_u : it.out_c;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int tok = m0 + wg * 64 + wrow + 8 * r;
      if (tok >= prm.q_row_end) continue;
      __half* dst = out + ((long long)out_slab * prm.out_rows + (tok - prm.q_row0)) * prm.out_tok_stride + head * d;
#pragma unroll
      for (int j = 0; j < kO / 4; ++j) {
        const int c = 8 * j + qcol;
        if (c < d)
          *reinterpret_cast<uint32_t*>(dst + c) = pack_f16x2_rn(o[v][4 * j + 2 * r] * l_r[r], o[v][4 * j + 2 * r + 1] * l_r[r]);
      }
    }
  }
}

template <int kDChunks, int kBlockN, int kNPV, class Tab>
int launch_cfg(const void* q, const void* k, const void* v, long long q_tok_stride, long long kv_tok_stride,
               int q_samples_total, int kv_samples_total, const Tab& tab, int n_items, int S, int heads, int d,
               float scale, void* out, int q_row0, int q_nrows, cudaStream_t stream) {
  constexpr int kNV = std::is_same<Tab, AttnPairTable>::value ? 2 : 1;
  constexpr int kQBytes = kDChunks * kBlockM * 128;
  constexpr int kStageBytes = (1 + kNV) * kDChunks * kBlockN * 128;
  int stages = (kSmemBudget - 2048 - kQBytes) / kStageBytes;
  if (stages > kMaxStages) stages = kMaxStages;
  if (stages < 2) { set_last_error("tf_ext_attn: configuration does not fit shared memory"); return TF_ERR_UNSUPPORTED; }
  const size_t smem_bytes = 1024 + kQBytes + (size_t)stages * kStageBytes + sizeof(AttnCtl);

  CUtensorMap map_q, map_k, map_v;
  auto make = [&](CUtensorMap* m, const void* base, long long tok_stride, int samples, int box_rows) -> int {
    const uint64_t dims[4] = {(uint64_t)d, (uint64_t)heads, (uint64_t)S, (uint64_t)samples};
    const uint64_t strides[3] = {(uint64_t)d * 2, (uint64_t)tok_stride * 2, (uint64_t)S * tok_stride * 2};
    const uint32_t box[4] = {64, 1, (uint32_t)box_rows, 1};
    CUresult r = encode_tiled(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, base, dims, strides, box,
                              CU_TENSOR_MAP_SWIZZLE_128B);
    if (r != CUDA_SUCCESS) { set_last_error("tf_ext_attn: cuTensorMapEncodeTiled failed: %d", (int)r); return TF_ERR_DRIVER; }
    return TF_OK;
  };
  if (int e = make(&map_q, q, q_tok_stride, q_samples_total, kBlockM)) return e;
  if (int e = make(&map_k, k, kv_tok_stride, kv_samples_total, kBlockN)) return e;
  if (int e = make(&map_v, v, kv_tok_stride, kv_samples_total, kBlockN)) return e;

  AttnParams prm;
  prm.S = S; prm.heads = heads; prm.d = d;
  prm.q_row0 = q_row0; prm.q_row_end = (q_row0 + q_nrows < S) ? q_row0 + q_nrows : S; prm.out_rows = q_nrows;
  prm.tiles_m = (prm.q_row_end - q_row0 + kBlockM - 1) / kBlockM;
  prm.stages = stages;
  prm.scale_log2 = scale * 1.4426950408889634f;
  prm.out_tok_stride = (long long)heads * d;

  auto kern = ext_attn_kernel<kDChunks, kBlockN, kNPV, Tab>;
  if (check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes),
                 "tf_ext_attn smem attribute"))
    return TF_ERR_CUDA;
  const long long grid = (long long)n_items * heads * prm.tiles_m;
  kern<<<(unsigned)grid, 256, smem_bytes, stream>>>(map_q, map_k, map_v, tab, prm, static_cast<__half*>(out));
  return check_cuda(cudaGetLastError(), "tf_ext_attn launch");
}

// Head dim -> kernel shape: 64-channel chunks, 128 keys per tile up to d = 128 (64 above, for shared memory),
// P V width = d rounded up to 16.
template <class Tab>
int dispatch(const void* q, const void* k, const void* v, long long q_tok_stride, long long kv_tok_stride,
             int q_samples_total, int kv_samples_total, const Tab& tab, int n_items, int S, int heads, int d,
             float scale, void* out, int q_row0, int q_nrows, cudaStream_t stream) {
  constexpr bool kPair = std::is_same<Tab, AttnPairTable>::value;
#define TF_CFG(C, N, P)                                                                                          \
  case P:                                                                                                       \
    if constexpr (!kPair || P <= 64)                                                                            \
      return launch_cfg<C, N, P, Tab>(q, k, v, q_tok_stride, kv_tok_stride, q_samples_total, kv_samples_total,  \
                                      tab, n_items, S, heads, d, scale, out, q_row0, q_nrows, stream);          \
    break
  switch ((d + 15) / 16 * 16) {
    TF_CFG(1, 128, 16); TF_CFG(1, 128, 32); TF_CFG(1, 128, 48); TF_CFG(1, 128, 64);
    TF_CFG(2, 128, 80); TF_CFG(2, 128, 96); TF_CFG(2, 128, 112); TF_CFG(2, 128, 128);
    TF_CFG(3, 64, 144); TF_CFG(3, 64, 160); TF_CFG(3, 64, 176); TF_CFG(3, 64, 192);
    default: break;
  }
#undef TF_CFG
  set_last_error("tf_ext_attn: head dim %d > 192 is not supported", d);
  return TF_ERR_UNSUPPORTED;
}

}  // namespace

int launch_ext_attn(const void* q, const void* k, const void* v, long long q_tok_stride, long long kv_tok_stride,
                    int q_samples_total, int kv_samples_total, const AttnTable& tab, int n_out, int S, int heads,
                    int d, float scale, void* out, int q_row0, int q_nrows, cudaStream_t stream) {
  if (n_out == 0 || S == 0 || q_nrows <= 0 || q_row0 >= S) return TF_OK;
  return dispatch(q, k, v, q_tok_stride, kv_tok_stride, q_samples_total, kv_samples_total, tab, n_out, S, heads, d,
                  scale, out, q_row0, q_nrows, stream);
}

// The paired kernel holds two output accumulators; above d = 64 a pair would cost more registers than the
// shared score computation saves, so such samples run singly.
bool ext_attn_pairs_supported(int d) {
  return d <= 64;
}

int launch_ext_attn_pairs(const void* q, const void* k, const void* v, long long q_tok_stride, long long kv_tok_stride,
                          int q_samples_total, int kv_samples_total, const AttnPairTable& tab, int n_pairs, int S,
                          int heads, int d, float scale, void* out, int q_row0, int q_nrows, cudaStream_t stream) {
  if (n_pairs == 0 || S == 0 || q_nrows <= 0 || q_row0 >= S) return TF_OK;
  if (!ext_attn_pairs_supported(d)) {
    set_last_error("tf_ext_attn: paired kernel does not cover d=%d", d);
    return TF_ERR_UNSUPPORTED;
  }
  return dispatch(q, k, v, q_tok_stride, kv_tok_stride, q_samples_total, kv_samples_total, tab, n_pairs, S, heads, d,
                  scale, out, q_row0, q_nrows, stream);
}

}  // namespace tf
