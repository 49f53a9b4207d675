// Tensor-core path (sm_90a): 16-bit operands (bf16, or fp16 in the fp16 mode) staged by TMA into 128B-swizzled shared memory, fp32 accumulators in registers of
// two consumer warpgroups (wgmma.mma_async), an mbarrier ring between one TMA producer warp and the consumers.
//
//   tc_conv_kernel   1x1 conv == GEMM  D[pixels, Cout] = A[pixels, Cin] * W[Cout, Cin]^T          (mode 0, 2D TMA)
//                    RxS conv (stride 1/2, dilation) as implicit GEMM: per tap (r,s) the A tile is a shifted [8 x 16] pixel box
//                    of the NHWC input fetched by a 4D TMA (out-of-bounds = the reference's explicit zero padding,
//                    backbones/efficientnet.py:1127-1161)                                             (mode 1)
//                    epilogue: registers -> + folded-BN bias, activation, + residual, 16-bit NHWC store.
//   tc_conv3x3s1_kernel  3x3 stride-1 conv with Cin, Cout <= 64 (EfficientNetV2 stage 1, ResNet conv2_x): the input of a
//                    tile as three column-shifted boxes instead of one box per tap, the weights resident; same MMA order
//                    and the same epilogue as tc_conv_kernel.
//   tc_head_kernel   MetrabsHeads (models/metrabs.py:75-85): swapped operands, D[channel, pixel] = W[N, C] * F^T, so every
//                    epilogue thread owns one (d,j) channel and reduces its pixels in registers: the J x D x H x W logits
//                    never leave the SM.
//
// tc_conv_kernel is persistent (one CTA per SM walking output tiles of 128 rows x BN columns, two consumer warpgroups
// taking alternate tiles, so one tile's epilogue overlaps the next tile's main loop); tc_head_kernel runs one CTA per tile.
// Descriptor encodings: the sm_90 GMMA shared-memory descriptor (PTX ISA, "Matrix Descriptor Format" of wgmma).
#pragma once
#include <cuda.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "common.cuh"
#include "conv_simt.cuh"
#include "decode.cuh"
#include "wgmma.cuh"

namespace mtb {

// ------------------------------------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n"
      "selp.u32 %0, 1, 0, P1;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a pipeline bug (wrong expect_tx bytes, missing arrive) traps after ~seconds instead of hanging the GPU.  Kept
// inline and free of calls: a call between wgmma instructions makes ptxas serialise the whole wgmma pipeline.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity))
    if (clock64() - t0 > 8000000000LL) __trap();  // ~4 s at 2 GHz
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ uint4 ld_shared_u4(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ void st_shared_u4(uint32_t addr, const uint4& v) {
  asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
// 4-byte shared-memory store and load with no "memory" clobber: global loads may be scheduled across them (a .shared access
// cannot alias global memory), while volatile keeps them in order with the fences and barriers, which do clobber memory
__device__ __forceinline__ void st_shared_b32(uint32_t addr, uint32_t v) { asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v)); }
__device__ __forceinline__ uint32_t ld_shared_b32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// named barrier of one consumer warpgroup (ids 1, 2; id 0 is __syncthreads)
__device__ __forceinline__ void wg_sync(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory"); }

__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, const void* src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(map), "r"(smem_u32(src)), "r"(c0),
               "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* map, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(map), "r"(smem_u32(src)),
               "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// the shared-memory source of every committed bulk store has been read (it may be overwritten)
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void prefetch_l1(const void* p) { asm volatile("prefetch.global.L1 [%0];" ::"l"(p)); }
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}

// K-major operand tile with rows of RB bytes (128: SWIZZLE_128B, 64: SWIZZLE_64B), 8-row groups 8 * RB bytes apart (SBO);
// LBO is unused for swizzled K-major layouts.  Advancing along K inside the swizzle atom = advancing the start address.
template <int RB>
__device__ __forceinline__ uint64_t gmma_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);    // start address, bits [0,14)
  d |= (uint64_t)1 << 16;                         // leading byte offset (ignored)
  d |= (uint64_t)((8 * RB) >> 4) << 32;           // stride byte offset, bits [32,46)
  d |= (uint64_t)(RB == 128 ? 1 : 2) << 62;       // layout type: 1 = SWIZZLE_128B, 2 = SWIZZLE_64B
  return d;
}

// ------------------------------------------------------------------------------------------- conv/GEMM kernel
constexpr int TC_BM = 128, TC_BK = 64;
constexpr int TC_A_BYTES = TC_BM * TC_BK * 2;       // 16 KB
constexpr int TC_THREADS = 288;                     // warps 0-7: two consumer warpgroups; warp 8: TMA producer
constexpr int TC_CONSUMER_WARPS = 8;
constexpr int TC_TILE_W = 16, TC_TILE_H = 8;        // spatial M tile of mode 1 (16 x 8 = 128 output pixels)
constexpr int TCP_THREADS = 384;                    // tc_conv_kernel: warpgroup 0 TMA producer, warpgroups 1, 2 consumers

// tc_conv_kernel's shared memory (one CTA per SM): the ring, shared by the CTA's whole tile sequence, then one output staging
// tile per consumer warpgroup, [BN / SW slabs][128 rows][SW columns] 16-bit in the TMA's swizzled layout (SW = 64: 128-byte
// rows, SWIZZLE_128B; SW = 32: 64-byte rows, SWIZZLE_64B).  BN = 128: 5 x 32 KB + 2 x 32 KB; BN = 64: 8 x 24 KB + 2 x 16 KB;
// BN = 32: 8 x 20 KB + 2 x 8 KB.
template <int BN>
struct TcRing {
  static constexpr int stages = BN >= 128 ? 5 : 8;
  static constexpr int stage_bytes = TC_A_BYTES + BN * TC_BK * 2;
  static constexpr int slab_cols = BN < 64 ? BN : 64;
  static constexpr int out_bytes = TC_BM * BN * 2;
  static constexpr int out_off = stages * stage_bytes;
  static constexpr int bar_off = out_off + 2 * out_bytes;
  static constexpr int smem_bytes = bar_off + 256 /*barriers*/ + 1024 /*align slack*/;
};

struct TcConvParams {
  const void* res;
  const float* bias;
  void* out;
  int mode;     // 0: flat 1x1 stride 1 (rows = B*H*W, 2D maps); 1: spatial 16x8 tiles, A tile per tap by 4D TMA
  int Hin, Win;
  int M;        // mode 0: number of rows
  int Cout, Cin;
  int kchunks, taps;
  int Hout, Wout, tiles_w, tiles_h, pad_t, pad_l, S, stride, dil;
  int m_tiles, n_tiles;  // tc_conv_kernel's tile grid (tile t = m_blk * n_tiles + n_blk)
};

// warpgroup register budgets of tc_conv_kernel: 128 x 40 + 256 x 232 = 64512 of the SM's 65536 registers; the SE instances,
// whose warpgroup 0 also scales the A tiles: 128 x 56 + 256 x 224 = 64512
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
// named barrier between the two consumer warpgroups (256 threads): one side arrives, the other waits
__device__ __forceinline__ void named_bar_sync(int id) { asm volatile("bar.sync %0, 256;" ::"r"(id) : "memory"); }
__device__ __forceinline__ void named_bar_arrive(int id) { asm volatile("bar.arrive %0, 256;" ::"r"(id) : "memory"); }

__device__ __forceinline__ float tanh_approx(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// Epilogue activation, COMPILE-TIME selected (a runtime switch inside the per-element code gets if-converted into all
// branches: ncu showed ~110 executed instructions per output element).  bf16 outputs: SiLU(x) = h + h*tanh(h), h = x/2: one
// MUFU op, error ~2^-11, below bf16 resolution.  fp16 outputs (T = __half): silu_f16out, one more MUFU op per element,
// because 2^-11 is a whole fp16 ulp.
template <int ACT, typename T = __nv_bfloat16>
__device__ __forceinline__ float tc_act(float x) {
  if constexpr (ACT == ACT_SILU && is_f16<T>) {
    return silu_f16out(x);
  } else if constexpr (ACT == ACT_SILU) {
    float h = 0.5f * x;
    return fmaf(h, tanh_approx(h), h);
  } else if constexpr (ACT == ACT_RELU) {
    return fmaxf(x, 0.0f);
  } else if constexpr (ACT == ACT_HSWISH) {
    return x * __saturatef(fmaf(x, 1.0f / 6.0f, 0.5f));
  } else {
    return x;
  }
}
// Output row r (0..127) of a tile -> (valid, element offset of channel 0) in the NHWC output
__device__ __forceinline__ bool tile_row_offset(int mode, int m_blk, int r, int M, int Cout, int tiles_w, int tiles_h, int Hout, int Wout,
                                                size_t& off) {
  if (mode == 0) {
    const int m = m_blk * TC_BM + r;
    off = (size_t)m * Cout;
    return m < M;
  }
  const int tw = m_blk % tiles_w, th = (m_blk / tiles_w) % tiles_h, b = m_blk / (tiles_w * tiles_h);
  const int oh = th * TC_TILE_H + (r >> 4), ow = tw * TC_TILE_W + (r & 15);
  off = ((size_t)(b * Hout + oh) * Wout + ow) * Cout;
  return oh < Hout && ow < Wout;
}

// The A tile of k-block kb (tap = kb / kchunks, channel chunk kc = kb % kchunks) for output tile m_blk: 2D box of 128 rows
// (mode 0) or the shifted 16 x 8 pixel box of tap (r, s) (mode 1).  BKE: channels per k-block.
template <int BKE, typename P>
__device__ __forceinline__ void tma_load_a_tile(void* dst, const CUtensorMap* map, uint64_t* bar, const P& p, int m_blk, int kb) {
  const int tap = kb / p.kchunks, kc = kb - tap * p.kchunks;
  if (p.mode == 0) {
    tma_load_2d(dst, map, bar, kc * BKE, m_blk * TC_BM);
  } else {
    const int tw = m_blk % p.tiles_w, th = (m_blk / p.tiles_w) % p.tiles_h, b = m_blk / (p.tiles_w * p.tiles_h);
    const int r = tap / p.S, s = tap - r * p.S;
    tma_load_4d(dst, map, bar, kc * BKE, tw * TC_TILE_W * p.stride - p.pad_l + s * p.dil, th * TC_TILE_H * p.stride - p.pad_t + r * p.dil, b);
  }
}

// The p.S column-shifted input boxes of a stride-1, dilation-1 RxS conv for output tile m_blk and channel chunk kc: box s
// (at dst + s * box_bytes) holds TC_TILE_W x (TC_TILE_H + R - 1) pixels from input row th * TC_TILE_H - pad_t and column
// tw * TC_TILE_W - pad_l + s (map: make_tmap_nhwc with box_h = TC_TILE_H + R - 1).  The A tile of tap (r, s) is then box s
// from pixel row r on, r * TC_TILE_W * 128 bytes in: a multiple of 1024, so it keeps the SWIZZLE_128B phase and the
// descriptors of a 1024-byte-aligned tile, and holds what tma_load_a_tile loads for that tap.  One load per column offset
// instead of one per tap: R x fewer boxes and (TC_TILE_H + R - 1) / (R x TC_TILE_H) of the bytes.
template <typename P>
__device__ __forceinline__ void tma_load_tap_boxes(uint8_t* dst, int box_bytes, const CUtensorMap* map, uint64_t* bar, const P& p, int m_blk,
                                                   int kc) {
  const int tw = m_blk % p.tiles_w, th = (m_blk / p.tiles_w) % p.tiles_h, b = m_blk / (p.tiles_w * p.tiles_h);
  for (int s = 0; s < p.S; ++s)
    tma_load_4d(dst + s * box_bytes, map, bar, kc * TC_BK, tw * TC_TILE_W - p.pad_l + s, th * TC_TILE_H - p.pad_t, b);
}

// Epilogue of one 128-row x BN-column output tile held by consumer warpgroup c (rows [0, 64) in acc, [64, 128) in
// acc + BN/2, as two m64nBNk16 wgmma accumulators): + folded-BN bias, activation, + residual read from global, rounded to
// 16 bits into the warpgroup's staging tile stg in the TMA's swizzled layout ([BN / SW slabs][128 rows][SW columns], SW =
// min(BN, 64)), then one thread stores the slabs with the TMA (2D box for mode 0, 4D 16 x 8-pixel box for mode 1).  The
// TMA clips what lies outside the tensor: the M tail, the parts of a 16 x 8 box beyond the map, the Cout tail.  Uses the
// named barrier 3 + c; the staging tile is rewritten only after the warpgroup's previous stores have read it.
//
// PRE (ResNet V2, mode 0): the tile is also the input of the next block's pre-activation, a 1x1 depthwise op
// z = relu(x * pre.w[c] + pre.b[c]) (its BatchNorm folded).  Once the TMA has read the stored tile out of the staging tile,
// every thread rewrites the elements it wrote with z, computed from the stored 16-bit value exactly as dwconv_kernel
// computes it (fmaf(x, w, b), then fmaxf(., 0), rounded to nearest even), and the leader stores the tile again through
// tmZ.  The two outputs are bit-identical to the GEMM and dwconv_kernel launched one after the other.
struct TcPreact {
  const float* w;  // [Cout] folded BN scale of the absorbed op
  const float* b;  // [Cout] folded BN shift
};
// a 16-bit pair as the 32 bits st_shared_b32 stores, and back
template <typename T>
__device__ __forceinline__ uint32_t pair16_bits(typename Pair16<T>::type v) {
  uint32_t u;
  memcpy(&u, &v, 4);
  return u;
}
template <typename T>
__device__ __forceinline__ typename Pair16<T>::type pair16_from_bits(uint32_t u) {
  typename Pair16<T>::type v;
  memcpy(&v, &u, 4);
  return v;
}
template <int BN>
__device__ __forceinline__ void tc_store_staging(const uint8_t* stg, const CUtensorMap* map, const TcConvParams& p, int m_blk, int n_blk) {
  constexpr int SW = BN < 64 ? BN : 64, RB = SW * 2;
#pragma unroll
  for (int sl = 0; sl < BN / SW; ++sl) {
    const int col0 = n_blk * BN + sl * SW;
    if (col0 >= p.Cout) break;
    if (p.mode == 0) {
      tma_store_2d(map, stg + sl * TC_BM * RB, col0, m_blk * TC_BM);
    } else {
      const int tw = m_blk % p.tiles_w, th = (m_blk / p.tiles_w) % p.tiles_h, b = m_blk / (p.tiles_w * p.tiles_h);
      tma_store_4d(map, stg + sl * TC_BM * RB, col0, tw * TC_TILE_W, th * TC_TILE_H, b);
    }
  }
  bulk_commit();
}
template <typename T, int ACT, int RES, int BN, bool PRE = false>
__device__ __forceinline__ void tc_tile_epilogue(const float* acc, uint8_t* stg, const CUtensorMap* tmO, const TcConvParams& p, int m_blk,
                                                 int n_blk, int c, const CUtensorMap* tmZ = nullptr, TcPreact pre = {}) {
  constexpr int SW = BN < 64 ? BN : 64, RB = SW * 2;  // staging slab: columns, bytes per row
  typedef typename Pair16<T>::type T2;
  const T* __restrict__ res = (const T*)p.res;
  const int warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  // rows 64 mh + 16 warp + lane / 4 (+ 8 h), columns 8 j + 2 (lane % 4) + {0, 1} -> staging tile
  const bool leader = (threadIdx.x & 127) == 0;  // issues and waits for this warpgroup's bulk stores
  if (leader) bulk_wait_read();  // the previous tile's stores have read the staging tile
  wg_sync(2 + c);                // named barriers 3, 4 (1 and 2 order tc_conv_kernel's main loops)
  const int c0 = n_blk * BN + 2 * (lane & 3);
  const uint32_t stg_s = smem_u32(stg);
  // Column blocks of JB 8-column groups outside, the thread's four rows inside: the block's bias pairs are loaded once per
  // tile, in one batch ahead of its arithmetic, and each row's residual pairs in one batch too.  The staging writes are
  // .shared stores, which no global load has to wait behind: with generic stores to `stg`, which might have aliased global
  // memory, every load stayed behind the previous column's store and each column pair ran as one dependent chain.  Blocks
  // are up to 8 groups wide.  At BN = 128 with a residual, the bias batch does not fit next to the 128 accumulators and the
  // residual batch within the 168 registers of __launch_bounds__, and narrower blocks, whose residual batches are smaller,
  // made the ResNet projections slower; so there the bias pairs are loaded at their use, free of the stores.
  constexpr int JB = BN / 8 < 8 ? BN / 8 : 8;
  constexpr bool BIAS_BATCH = RES == 0 || BN < 128;
#pragma unroll
  for (int j0 = 0; j0 < BN / 8; j0 += JB) {
    float2 bv[BIAS_BATCH ? JB : 1];
    if constexpr (BIAS_BATCH) {
#pragma unroll
      for (int jj = 0; jj < JB; ++jj)
        if (c0 + 8 * (j0 + jj) < p.Cout) bv[jj] = __ldg(reinterpret_cast<const float2*>(p.bias + c0 + 8 * (j0 + jj)));
    }
#pragma unroll
    for (int g = 0; g < 4; ++g) {  // rows 64 mh + 16 warp + lane / 4 + 8 h, g = 2 mh + h
      const int mh = g >> 1, h = g & 1;
      const float* accm = acc + mh * (BN / 2);
      const int r = mh * 64 + warp * 16 + (lane >> 2) + 8 * h;
      T2 rv2[RES != 0 ? JB : 1];
      if constexpr (RES != 0) {
        size_t off = 0;
        if (!tile_row_offset(p.mode, m_blk, r, p.M, p.Cout, p.tiles_w, p.tiles_h, p.Hout, p.Wout, off)) continue;
#pragma unroll
        for (int jj = 0; jj < JB; ++jj)
          if (c0 + 8 * (j0 + jj) < p.Cout) rv2[jj] = *reinterpret_cast<const T2*>(res + off + c0 + 8 * (j0 + jj));
      }
      const uint32_t swz = RB == 128 ? (uint32_t)(r & 7) : (uint32_t)((r >> 1) & 3);
#pragma unroll
      for (int jj = 0; jj < JB; ++jj) {
        const int j = j0 + jj, cc = c0 + 8 * j;
        if (cc >= p.Cout) break;  // Cout % 8 == 0: column cc + 1 is valid with cc
        const float2 b = BIAS_BATCH ? bv[BIAS_BATCH ? jj : 0] : __ldg(reinterpret_cast<const float2*>(p.bias + cc));
        float o0 = accm[4 * j + 2 * h] + b.x, o1 = accm[4 * j + 2 * h + 1] + b.y;
        if constexpr (RES != 0) {
          const float2 rv = Pair16<T>::unpack(rv2[jj]);
          if constexpr (RES == 2) {
            o0 = tc_act<ACT, T>(o0 + rv.x);
            o1 = tc_act<ACT, T>(o1 + rv.y);
          } else {
            o0 = tc_act<ACT, T>(o0) + rv.x;
            o1 = tc_act<ACT, T>(o1) + rv.y;
          }
        } else {
          o0 = tc_act<ACT, T>(o0);
          o1 = tc_act<ACT, T>(o1);
        }
        const int col = 8 * j + 2 * (lane & 3), cs = col % SW;  // column within the tile, within its slab
        const uint32_t o = (uint32_t)(col / SW) * (TC_BM * RB) + (uint32_t)r * RB + ((((uint32_t)cs >> 3) ^ swz) << 4) + (cs & 7) * 2;
        st_shared_b32(stg_s + o, pair16_bits<T>(Pair16<T>::pack(o0, o1)));
      }
    }
  }
  fence_proxy_async();  // generic-proxy writes -> visible to the TMA (async proxy)
  wg_sync(2 + c);
  if (leader) tc_store_staging<BN>(stg, tmO, p, m_blk, n_blk);
  if constexpr (PRE) {
    if (leader) bulk_wait_read();  // the block output has left the staging tile
    wg_sync(2 + c);
    // Column blocks outside, the four rows inside, as above: each pre.w / pre.b pair is loaded once per tile, not once per
    // row.  The blocks are one 8-column group wide: wider batches spill at BN = 128.
    constexpr int JP = 1;
    for (int j0 = 0; j0 < BN / 8; j0 += JP) {
      float2 wv[JP], bv[JP];
#pragma unroll
      for (int jj = 0; jj < JP; ++jj) {
        const int cc = c0 + 8 * (j0 + jj);
        if (cc < p.Cout) {
          wv[jj] = __ldg(reinterpret_cast<const float2*>(pre.w + cc));
          bv[jj] = __ldg(reinterpret_cast<const float2*>(pre.b + cc));
        }
      }
#pragma unroll
      for (int g = 0; g < 4; ++g) {
        const int r = (g >> 1) * 64 + warp * 16 + (lane >> 2) + 8 * (g & 1);  // rows past M hold what the TMA clips
        const uint32_t swz = RB == 128 ? (uint32_t)(r & 7) : (uint32_t)((r >> 1) & 3);
#pragma unroll
        for (int jj = 0; jj < JP; ++jj) {
          const int j = j0 + jj;
          if (c0 + 8 * j >= p.Cout) break;
          const int col = 8 * j + 2 * (lane & 3), cs = col % SW;
          const uint32_t q = stg_s + (uint32_t)(col / SW) * (TC_BM * RB) + (uint32_t)r * RB + ((((uint32_t)cs >> 3) ^ swz) << 4) + (cs & 7) * 2;
          const float2 x = Pair16<T>::unpack(pair16_from_bits<T>(ld_shared_b32(q)));
          st_shared_b32(q, pair16_bits<T>(Pair16<T>::pack(act_t<ACT_RELU>(fmaf(x.x, wv[jj].x, bv[jj].x)),
                                                          act_t<ACT_RELU>(fmaf(x.y, wv[jj].y, bv[jj].y)))));
        }
      }
    }
    fence_proxy_async();
    wg_sync(2 + c);
    if (leader) tc_store_staging<BN>(stg, tmZ, p, m_blk, n_blk);
  }
}

// Squeeze-excitation scale of the landed mode-0 A tiles (128 rows of the flat [M][Cin] input from row m0, 64 channels per
// k-block), in place: x[m][k] = round16(x[m][k] * s[m / P][k]), the fp32 product rounded to nearest even, so the wgmma reads
// the bits a separate in-place pass over the tensor would have stored.  Transform thread u (0..95) owns logical 16-byte chunk
// L = u % 8 (8 channels) of the contiguous rows [r0, r1) of row block u / 8 (12 blocks of 11 or 10 rows); SWIZZLE_128B puts
// that chunk at physical chunk L ^ (r & 7) of row r.  A warp's 32 accesses then cover four whole 128-byte rows (no bank
// conflicts), and a block of 11 rows spans at most two crops, ca and cb, when P >= 10: the thread loads both crops' 8
// scales before it waits for the stage, and prefetches those of its next k-block into L1.  Crops strictly between them
// (maps below 10 pixels) load their scales row by row.  Rows m >= M and channels k >= Cin are the TMA's zero fill and are
// left alone (Cin % 8 == 0: a chunk lies wholly inside or outside Cin).
struct SeRows {
  int r0, r1;  // the thread's rows of the tile, r1 clipped to the M tail (r1 <= r0: none)
  int ca, cb;  // crops of rows r0 and r1 - 1
};
__device__ __forceinline__ SeRows se_rows(int u, int m0, int M, int P) {
  const int g = u >> 3;
  SeRows w;
  w.r0 = 10 * g + min(g, 8);
  w.r1 = min(w.r0 + (g < 8 ? 11 : 10), M - m0);
  w.ca = (m0 + w.r0) / P;
  w.cb = (m0 + max(w.r1, w.r0 + 1) - 1) / P;
  return w;
}
template <typename T>
__device__ __forceinline__ void se_scale_chunk(uint32_t addr, const float4& s0, const float4& s1) {
  typedef typename Pair16<T>::type T2;
  uint4 v = ld_shared_u4(addr);
  T2* v2 = reinterpret_cast<T2*>(&v);
  float2 f = Pair16<T>::unpack(v2[0]);
  v2[0] = Pair16<T>::pack(f.x * s0.x, f.y * s0.y);
  f = Pair16<T>::unpack(v2[1]);
  v2[1] = Pair16<T>::pack(f.x * s0.z, f.y * s0.w);
  f = Pair16<T>::unpack(v2[2]);
  v2[2] = Pair16<T>::pack(f.x * s1.x, f.y * s1.y);
  f = Pair16<T>::unpack(v2[3]);
  v2[3] = Pair16<T>::pack(f.x * s1.z, f.y * s1.w);
  st_shared_u4(addr, v);
}
// rows [rb, re) of chunk L with one crop's scales, two rows per step so that their shared-memory loads overlap
template <typename T>
__device__ __forceinline__ void se_scale_rows(uint32_t a, int L, int rb, int re, const float4& s0, const float4& s1) {
  typedef typename Pair16<T>::type T2;
  int r = rb;
#pragma unroll 1
  for (; r + 1 < re; r += 2) {
    const uint32_t p0 = a + r * 128 + ((L ^ (r & 7)) << 4), p1 = a + (r + 1) * 128 + ((L ^ ((r + 1) & 7)) << 4);
    uint4 v = ld_shared_u4(p0), w = ld_shared_u4(p1);
    T2* v2 = reinterpret_cast<T2*>(&v);
    T2* w2 = reinterpret_cast<T2*>(&w);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float sx = j < 2 ? (j == 0 ? s0.x : s0.z) : (j == 2 ? s1.x : s1.z);
      const float sy = j < 2 ? (j == 0 ? s0.y : s0.w) : (j == 2 ? s1.y : s1.w);
      const float2 f = Pair16<T>::unpack(v2[j]), g = Pair16<T>::unpack(w2[j]);
      v2[j] = Pair16<T>::pack(f.x * sx, f.y * sy);
      w2[j] = Pair16<T>::pack(g.x * sx, g.y * sy);
    }
    st_shared_u4(p0, v);
    st_shared_u4(p1, w);
  }
  if (r < re) se_scale_chunk<T>(a + r * 128 + ((L ^ (r & 7)) << 4), s0, s1);
}
// One stage: k-block kb's A tile at shared address a, landing on `full` with parity `ph`; waits for it in every case.
template <typename T>
__device__ __forceinline__ void se_scale_a_tile(uint32_t a, uint64_t* full, uint32_t ph, const SeRows& w, const float* __restrict__ s, int m0,
                                                int P, int Cin, int kb, int u) {
  const int L = u & 7, k = kb * TC_BK + 8 * L;
  if (k >= Cin || w.r1 <= w.r0) {
    mbar_wait(full, ph);
    return;
  }
  const float4* sa = reinterpret_cast<const float4*>(s + (size_t)w.ca * Cin + k);
  const float4* sb = reinterpret_cast<const float4*>(s + (size_t)w.cb * Cin + k);
  const float4 a0 = __ldg(sa), a1 = __ldg(sa + 1), b0 = __ldg(sb), b1 = __ldg(sb + 1);
  if (k + TC_BK < Cin) {  // the next k-block's scales, into L1 a whole stage ahead of their loads
    prefetch_l1(sa + TC_BK / 4);
    prefetch_l1(sb + TC_BK / 4);
  }
  mbar_wait(full, ph);
  const int ra = min((w.ca + 1) * P - m0, w.r1);        // first row past crop ca
  const int rb = max(min(w.cb * P - m0, w.r1), ra);     // first row of crop cb (when cb > ca)
  se_scale_rows<T>(a, L, w.r0, ra, a0, a1);
#pragma unroll 1
  for (int r = ra; r < rb; ++r) {                       // crops between ca and cb: maps of fewer than 10 pixels
    const float4* sr = reinterpret_cast<const float4*>(s + (size_t)((m0 + r) / P) * Cin + k);
    se_scale_chunk<T>(a + r * 128 + ((L ^ (r & 7)) << 4), __ldg(sr), __ldg(sr + 1));
  }
  se_scale_rows<T>(a, L, rb, w.r1, b0, b1);
}

// Persistent conv / GEMM kernel.  ACT: epilogue activation; RES: 0 no residual, 1 residual added AFTER the activation
// (EfficientNet), 2 BEFORE (ResNet); BN: output channels per tile (wgmma N); T: operand and activation element type
// (__nv_bfloat16 or __half); SE (mode 0 only): scale the A rows by the squeeze-excitation vector of their crop,
// a_scale [B][Cin] (crop of row m: m / (Hin * Win)), in shared memory before the consumers read them.
//
// CTA b walks tiles t = b, b + gridDim.x, ...; tile t is (m_blk, n_blk) = (t / n_tiles, t % n_tiles): N fastest, so the CTAs
// running at the same time cover every N tile of a few M blocks and each A tile comes from HBM once, the re-reads from L2.
// Warpgroup 0 (one thread) streams the k-blocks of the CTA's whole tile sequence through one ring; consumer warpgroups 1
// and 2 take alternate tiles (ping-pong), each owning a whole 128-row tile (two m64nBNk16 wgmmas per K step).  A named
// barrier orders their main loops: a consumer starts waiting on its tile's stages only after the other finished the previous
// tile's, which keeps every mbarrier wait within one phase of the barrier, and lets one warpgroup's epilogue run under the
// other's MMAs.  Every output element sees the wgmma sequence and the roundings of a one-CTA-per-tile kernel.
//
// With SE, warps 1-3 of warpgroup 0 walk the producer's (tile, k-block) sequence too: wait for full[s], scale the stage's A
// tile in place (se_scale_a_tile), fence the generic-proxy writes for the wgmma's async proxy, and arrive on ready[s] (one
// arrive per warp); the consumers wait on ready[s] instead of full[s].  The parities stay in phase: full[s] completes phase
// k + 1 only after the producer saw empty[s] complete phase k, which needs the consumers to have taken ready[s] phase k,
// which needs every transform warp to have finished phase k; so no barrier runs more than one phase ahead of its waiters.
//
// PRE: the epilogue also writes the next op's pre-activation through tmZ (tc_tile_epilogue); tc_conv_preact_kernel.
template <typename T, int ACT, int RES, int BN, bool SE, bool PRE>
__device__ __forceinline__ void tc_conv_body(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmO, const CUtensorMap* tmZ,
                                             const TcConvParams& p, const float* __restrict__ a_scale, TcPreact pre) {
  using Ring = TcRing<BN>;
  constexpr int STAGES = Ring::stages;
  extern __shared__ uint8_t tc_smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)tc_smem_raw + 1023) & ~(uintptr_t)1023);  // SWIZZLE_128B needs 1024 B alignment
  uint64_t* full = (uint64_t*)(smem + Ring::bar_off);
  uint64_t* empty = full + STAGES;
  uint64_t* ready = empty + STAGES;  // SE only: the stage's A tile is scaled
  uint64_t* landed = SE ? ready : full;  // what the consumers wait for

  const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    tma_prefetch_desc(&tmO);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full[i], 1);  // the producer's arrive.expect_tx
      mbar_init(&empty[i], 4); // one arrive per warp of the consuming warpgroup
      if constexpr (SE) mbar_init(&ready[i], 3);  // one arrive per transform warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  const int tiles = p.m_tiles * p.n_tiles;
  const int num_kb = SE ? p.kchunks : p.taps * p.kchunks;  // SE: mode 0, one tap; read as is, warpgroup 0 would spill the product
  if (wg == 0) {
    // ===== TMA producer =====
    setmaxnreg_dec<SE ? 56 : 40>();
    if (threadIdx.x == 0) {
      int it = 0;
      for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
        const int m_blk = t / p.n_tiles, n_blk = t - m_blk * p.n_tiles;
        for (int kb = 0; kb < num_kb; ++kb, ++it) {
          const int s = it % STAGES;
          mbar_wait(&empty[s], ((it / STAGES) & 1) ^ 1);
          uint8_t* sa = smem + s * Ring::stage_bytes;
          const int tap = kb / p.kchunks, kc = kb - tap * p.kchunks;
          mbar_expect_tx(&full[s], Ring::stage_bytes);
          tma_load_a_tile<TC_BK>(sa, &tmA, &full[s], p, m_blk, kb);
          tma_load_2d(sa + TC_A_BYTES, &tmB, &full[s], tap * p.Cin + kc * TC_BK, n_blk * BN);
        }
      }
    } else if constexpr (SE) {
      if (threadIdx.x >= 32) {
        // ===== warps 1-3: squeeze-excitation scale of each landed A tile (mode 0: k-block kb = channel chunk kb) =====
        const int u = threadIdx.x - 32, P = p.Hin * p.Win;
        int it = 0;
        for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
          const int m0 = (t / p.n_tiles) * TC_BM;
          const SeRows w = se_rows(u, m0, p.M, P);
          for (int kb = 0; kb < num_kb; ++kb, ++it) {
            const int s = it % STAGES;
            se_scale_a_tile<T>(smem_u32(smem + s * Ring::stage_bytes), &full[s], (it / STAGES) & 1, w, a_scale, m0, P, p.Cin, kb, u);
            fence_proxy_async();  // generic-proxy writes -> visible to the wgmma (async proxy)
            __syncwarp();
            if (lane == 0) mbar_arrive(&ready[s]);
          }
        }
      }
    }
    return;
  }
  // ===== consumers: warpgroup 1 + c computes the CTA's tiles c, c + 2, ... (rows [0, 64) in acc, [64, 128) in acc + BN/2) =====
  setmaxnreg_inc<SE ? 224 : 232>();
  const int c = wg - 1;
  for (int i = c, t = blockIdx.x + c * gridDim.x; t < tiles; i += 2, t += 2 * gridDim.x) {
    const int m_blk = t / p.n_tiles, n_blk = t - m_blk * p.n_tiles;
    float acc[BN];
#pragma unroll
    for (int q = 0; q < BN; ++q) acc[q] = 0.f;
    if (t != (int)blockIdx.x) named_bar_sync(1 + c);  // the other consumer finished the previous tile's main loop
    int it = i * num_kb, prev = -1;
    for (int kb = 0; kb < num_kb; ++kb, ++it) {
      const int s = it % STAGES;
      mbar_wait(&landed[s], (it / STAGES) & 1);
      const uint32_t a = smem_u32(smem + s * Ring::stage_bytes);
      const uint32_t b = smem_u32(smem + s * Ring::stage_bytes + TC_A_BYTES);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < TC_BK / 16; ++k) {
        const uint64_t db = gmma_desc<128>(b + 32 * k);
        wgmma_16b<T, BN>(acc, gmma_desc<128>(a + 32 * k), db, (uint32_t)(kb | k));
        wgmma_16b<T, BN>(acc + BN / 2, gmma_desc<128>(a + 64 * 128 + 32 * k), db, (uint32_t)(kb | k));
      }
      wgmma_commit();
      wgmma_wait<1>();  // the previous k-block's MMAs are done: its stage goes back to the producer
      if (prev >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[prev]);
      }
      prev = s;
    }
    wgmma_wait<0>();
    wgmma_fence_regs<BN>(acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[prev]);
    if (t + (int)gridDim.x < tiles) named_bar_arrive(2 - c);  // the other consumer may start the next tile
    tc_tile_epilogue<T, ACT, RES, BN, PRE>(acc, smem + Ring::out_off + c * Ring::out_bytes, &tmO, p, m_blk, n_blk, c, tmZ, pre);
  }
  if ((threadIdx.x & 127) == 0) bulk_wait();
}

template <typename T, int ACT, int RES, int BN, bool SE = false>
__global__ void __launch_bounds__(TCP_THREADS, 1)
tc_conv_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmO,
               const TcConvParams p, const float* __restrict__ a_scale) {
  tc_conv_body<T, ACT, RES, BN, SE, false>(tmA, tmB, tmO, nullptr, p, a_scale, TcPreact{});
}

// tc_conv_kernel whose epilogue also stores the next op's pre-activation (ResNet V2: a block's _3_conv and the next block's
// _preact_bn + _preact_relu, or the last block's and post_bn + post_relu) through tmZ
template <typename T, int ACT, int RES, int BN>
__global__ void __launch_bounds__(TCP_THREADS, 1)
tc_conv_preact_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmO,
                      const __grid_constant__ CUtensorMap tmZ, const TcConvParams p, const TcPreact pre) {
  tc_conv_body<T, ACT, RES, BN, false, true>(tmA, tmB, tmO, &tmZ, p, nullptr, pre);
}

// ------------------------------------------------------------------- 3x3 stride-1 conv with Cin, Cout <= 64
// tc_conv3x3s1_kernel's shared memory for K per tap = N tile = CK (32: 64-byte rows, SWIZZLE_64B; 64: 128-byte rows,
// SWIZZLE_128B): the 9 taps' [CK][CK] weight blocks, resident for the CTA's whole tile sequence; per consumer warpgroup
// `sets` sets of the three 16 x 10-pixel input boxes of a tile; one output staging tile per consumer warpgroup.
// CK = 32: 18 KB + 4 x 30 KB + 2 x 8 KB = 154 KB; CK = 64: 72 KB + 2 x 60 KB + 2 x 16 KB = 224 KB.
template <int CK>
struct Tc3x3Smem {
  static constexpr int RB = CK * 2;                              // bytes per pixel of a box, per output channel of a weight block
  static constexpr int w_tap_bytes = CK * RB;
  static constexpr int box_bytes = TC_TILE_W * (TC_TILE_H + 2) * RB;  // 10 / 20 KB, a multiple of 1024
  static constexpr int sets = CK == 32 ? 2 : 1;
  static constexpr int box_off = 9 * w_tap_bytes;
  static constexpr int out_bytes = TC_BM * CK * 2;
  static constexpr int out_off = box_off + 2 * sets * 3 * box_bytes;
  static constexpr int bar_off = out_off + 2 * out_bytes;
  static constexpr int smem_bytes = bar_off + 256 /*barriers*/ + 1024 /*align slack*/;
};

// Shapes tc_conv3x3s1_kernel takes: 3x3, stride 1, dilation 1, Cin and Cout multiples of 8 up to 64, SiLU or ReLU (the
// stage-1 convs of EfficientNetV2, the conv2_x 3x3 convs of the ResNets); its K per tap and N tile is 32 when Cin and Cout
// fit in 32, else 64.
inline bool tc3x3s1_eligible(int R, int S, int stride, int dil, int cin, int cout, int act) {
  return R == 3 && S == 3 && stride == 1 && dil == 1 && cin <= 64 && cout <= 64 && cin % 8 == 0 && cout % 8 == 0 &&
         (act == ACT_SILU || act == ACT_RELU);
}
inline int tc3x3s1_width(int cin, int cout) { return std::max(cin, cout) <= 32 ? 32 : 64; }

// Persistent 3x3 stride-1 conv, one N tile (BN = CK >= Cout), mode-1 16 x 8-pixel output tiles.  The input of a tile is
// loaded once, as the three column-shifted 16 x 10-pixel boxes of tma_load_tap_boxes with CK channels (those beyond Cin
// are zeros from the TMA); the A tile of tap (r, s) is box s from pixel row r on, r x 16 x RB bytes in, a multiple of
// the swizzle atom, so its descriptors are those of an aligned per-tap tile.  The weights are loaded once per CTA.  At
// Cin < CK the 32-column weight block of tap t also holds the first weights of tap t + 1 (of the last tap: the map's
// out-of-bounds zeros); they meet zero A channels.
//
// Warpgroup 0 (one thread) loads the weights, then the boxes of the CTA's tiles; consumer warpgroups 1 and 2 take
// alternate tiles, each into box sets of its own, so both may be in their MMAs at once.  A box set goes back to the producer
// once its tile's last wgmma has retired, before the epilogue.  The MMA sequence of every output element is that of
// tc_conv_kernel (taps in order, channels ascending, K = 16 per wgmma, fp32 accumulators) without the k16 steps whose A
// columns are all zeros (channels >= 32 at Cin <= 32), and the epilogue is tc_conv_kernel's.
template <typename T, int ACT, int RES, int CK>
__global__ void __launch_bounds__(TCP_THREADS, 1)
tc_conv3x3s1_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                    const __grid_constant__ CUtensorMap tmO, const TcConvParams p) {
  using L = Tc3x3Smem<CK>;
  constexpr int BN = CK, SETS = L::sets, RB = L::RB;
  extern __shared__ uint8_t tc_smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)tc_smem_raw + 1023) & ~(uintptr_t)1023);
  uint64_t* w_full = (uint64_t*)(smem + L::bar_off);
  uint64_t* box_full = w_full + 1;           // [consumer][set]
  uint64_t* box_empty = box_full + 2 * SETS;

  const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    tma_prefetch_desc(&tmO);
    mbar_init(w_full, 1);
    for (int i = 0; i < 2 * SETS; ++i) {
      mbar_init(&box_full[i], 1);   // the producer's arrive.expect_tx
      mbar_init(&box_empty[i], 4);  // one arrive per warp of the consuming warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();

  const int tiles = p.m_tiles;
  if (wg == 0) {
    // ===== TMA producer: the weights, then tile n's boxes into set (n / 2) % SETS of consumer n % 2 =====
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      mbar_expect_tx(w_full, 9 * L::w_tap_bytes);
      for (int tap = 0; tap < 9; ++tap) tma_load_2d(smem + tap * L::w_tap_bytes, &tmB, w_full, tap * p.Cin, 0);
      int n = 0;
      for (int t = blockIdx.x; t < tiles; t += gridDim.x, ++n) {
        const int j = n >> 1, b = (n & 1) * SETS + j % SETS;
        mbar_wait(&box_empty[b], ((j / SETS) & 1) ^ 1);
        mbar_expect_tx(&box_full[b], 3 * L::box_bytes);
        tma_load_tap_boxes(smem + L::box_off + b * 3 * L::box_bytes, L::box_bytes, &tmA, &box_full[b], p, t, 0);
      }
    }
    return;
  }
  // ===== consumers: warpgroup 1 + c computes the CTA's tiles c, c + 2, ... =====
  setmaxnreg_inc<232>();
  const int c = wg - 1;
  const uint32_t wts = smem_u32(smem);
  mbar_wait(w_full, 0);
  for (int j = 0, t = blockIdx.x + c * gridDim.x; t < tiles; ++j, t += 2 * gridDim.x) {
    const int b = c * SETS + j % SETS;
    float acc[BN];
#pragma unroll
    for (int q = 0; q < BN; ++q) acc[q] = 0.f;
    mbar_wait(&box_full[b], (j / SETS) & 1);
    const uint32_t box = smem_u32(smem + L::box_off + b * 3 * L::box_bytes);
    wgmma_fence();
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      const int r = tap / 3, s = tap - 3 * r;
      const uint32_t a = box + s * L::box_bytes + r * TC_TILE_W * RB, w = wts + tap * L::w_tap_bytes;
#pragma unroll
      for (int k = 0; k < CK / 16; ++k) {
        const uint64_t db = gmma_desc<RB>(w + 32 * k);
        wgmma_16b<T, BN>(acc, gmma_desc<RB>(a + 32 * k), db, (uint32_t)(tap | k));
        wgmma_16b<T, BN>(acc + BN / 2, gmma_desc<RB>(a + 64 * RB + 32 * k), db, (uint32_t)(tap | k));
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs<BN>(acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(&box_empty[b]);  // the boxes go back to the producer under the epilogue
    tc_tile_epilogue<T, ACT, RES, BN>(acc, smem + L::out_off + c * L::out_bytes, &tmO, p, t, 0, c);
  }
  if ((threadIdx.x & 127) == 0) bulk_wait();
}

// in-place squeeze-excitation scaling  x[b,p,c] *= s[b,c]  ahead of a tensor-core projection GEMM (T: bf16 or fp16)
template <typename T>
__global__ void __launch_bounds__(256) se_scale_kernel(T* __restrict__ x, const float* __restrict__ s, int P, int C,
                                                       size_t total8) {
  typedef typename Pair16<T>::type T2;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total8; i += (size_t)gridDim.x * blockDim.x) {
    size_t e = i * 8;
    int c = (int)(e % C);
    int b = (int)(e / ((size_t)P * C));
    uint4 v = *reinterpret_cast<uint4*>(x + e);
    T2* v2 = reinterpret_cast<T2*>(&v);
    const float4 s0 = *reinterpret_cast<const float4*>(s + (size_t)b * C + c);
    const float4 s1 = *reinterpret_cast<const float4*>(s + (size_t)b * C + c + 4);
    const float sc[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float2 f = Pair16<T>::unpack(v2[k]);
      v2[k] = Pair16<T>::pack(f.x * sc[2 * k], f.y * sc[2 * k + 1]);
    }
    *reinterpret_cast<uint4*>(x + e) = v;
  }
}

// ------------------------------------------------------------------------------------------------ host side
typedef CUresult (*tmap_encode_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline tmap_encode_fn get_tmap_encode() {
  static tmap_encode_fn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = (tmap_encode_fn)p;
  }
  return fn;
}

template <typename T>
constexpr CUtensorMapDataType tmap_dtype() {
  return std::is_same<T, float>::value    ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
         : std::is_same<T, __half>::value ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16
                                          : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
}

// Encodes the tensor map of a dense T tensor (float, bf16 or fp16) with `rank` dims, innermost first, and a box of
// box[i] elements taken every estr[i] elements along dim i (to load N elements with traversal stride s, box = N * s).
// Out-of-bounds elements read as 0.  The swizzle is the caller's: it must match how the kernel addresses the box in shared
// memory, and cannot be derived from the box's row bytes (dw3x3s1_tma_kernel reads 128-byte rows unswizzled).
template <typename T>
inline const char* make_tmap(CUtensorMap* m, const void* ptr, int rank, const uint64_t* dims, const uint32_t* box, const uint32_t* estr,
                             CUtensorMapSwizzle swizzle) {
  tmap_encode_fn enc = get_tmap_encode();
  if (!enc) return "cuTensorMapEncodeTiled unavailable";
  cuuint64_t strides[3];
  for (int i = 1; i < rank; ++i) strides[i - 1] = (i == 1 ? sizeof(T) : strides[i - 2]) * dims[i - 1];
  CUresult r = enc(m, tmap_dtype<T>(), rank, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? nullptr : "cuTensorMapEncodeTiled failed";
}
// row-major matrix [rows][cols], box [box_rows][box_cols]
template <typename T>
inline const char* make_tmap_2d(CUtensorMap* m, const void* ptr, uint64_t rows, uint64_t cols, uint32_t box_rows, uint32_t box_cols,
                             CUtensorMapSwizzle swizzle) {
  const uint64_t dims[2] = {cols, rows};
  const uint32_t box[2] = {box_cols, box_rows}, estr[2] = {1, 1};
  return make_tmap<T>(m, ptr, 2, dims, box, estr, swizzle);
}
// NHWC tensor [B][H][W][C], box box_c channels x box_w x box_h pixels sampled every `stride` pixels x box_b images
template <typename T>
inline const char* make_tmap_nhwc(CUtensorMap* m, const void* ptr, uint64_t B, uint64_t H, uint64_t W, uint64_t C, uint32_t box_c,
                             uint32_t box_w, uint32_t box_h, uint32_t box_b, uint32_t stride, CUtensorMapSwizzle swizzle) {
  const uint64_t dims[4] = {C, W, H, B};
  const uint32_t box[4] = {box_c, box_w * stride, box_h * stride, box_b}, estr[4] = {1, stride, stride, 1};
  return make_tmap<T>(m, ptr, 4, dims, box, estr, swizzle);
}

// The tensor maps one kernel's launches take, for one weight set.  An entry's key holds every device pointer and size its
// maps encode, plus the kernel variant, so an entry is only ever reused for the buffers and shapes it was encoded for: a
// copied Op that runs on other buffers encodes its own.  Encoding on every launch would sit on the host's launch path; a
// handle alternates between a few (workspace, batch) pairs, and past kEntries the oldest entry is replaced.
struct TmapCache {
  static constexpr int kEntries = 16, kKeyWords = 15;
  struct Entry {
    uint64_t key[kKeyWords];
    CUtensorMap map[4];
  };
  std::vector<Entry> entries;
  size_t replaced = 0;

  // *maps = the maps of `key` (device pointers and integers); on a miss encode(CUtensorMap*) makes them (nullptr on success)
  template <typename Encode, typename... K>
  const char* get(const CUtensorMap** maps, Encode&& encode, K... key) {
    static_assert(sizeof...(K) <= kKeyWords, "TmapCache key too long");
    Entry n = {};
    int i = 0;
    ((n.key[i++] = key_word(key)), ...);
    for (const Entry& e : entries)
      if (std::equal(e.key, e.key + kKeyWords, n.key)) {
        *maps = e.map;
        return nullptr;
      }
    if (const char* err = encode(n.map)) return err;
    Entry& slot = entries.size() < kEntries ? entries.emplace_back(n) : (entries[replaced++ % kEntries] = n);
    *maps = slot.map;
    return nullptr;
  }
  template <typename X>
  static uint64_t key_word(X x) {
    if constexpr (std::is_pointer<X>::value) return (uint64_t)(uintptr_t)x;
    else return (uint64_t)x;
  }
};

// cudaMalloc, record the allocation in `allocs` (freed with the handle) and copy `bytes` from the host; nullptr on success
inline const char* upload_dev(std::vector<void*>& allocs, void** dev, const void* host, size_t bytes) {
  cudaError_t e = cudaMalloc(dev, bytes);
  if (e == cudaSuccess) {
    allocs.push_back(*dev);
    e = cudaMemcpy(*dev, host, bytes, cudaMemcpyHostToDevice);
  }
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

struct TcWeights {
  bool ready = false;
  void* d_w = nullptr;           // [Cout][taps*Cin] K-major, bf16 or fp16 (the mode's storage type)
  float* d_bias = nullptr;       // [Cout]
  int Cout = 0, Cin = 0, taps = 1, S = 1;
  int n_real = 0;                // head
  mutable TmapCache maps;        // conv: (input, weights, output); head: (weights, features)
};

inline bool tc_eligible(bool is_conv, bool depthwise, bool small_io, int k, int stride, int cin, int cout) {
  if (!is_conv || depthwise || small_io) return false;
  if (cin % 8 != 0 || cout % 8 != 0) return false;
  return (stride == 1 || stride == 2) && (k == 1 || k == 3);
}

inline __nv_bfloat16 host_bf16(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  uint32_t lsb = (u >> 16) & 1u;
  u += 0x7FFFu + lsb;  // round to nearest even
  uint16_t h = (uint16_t)(u >> 16);
  __nv_bfloat16 out;
  memcpy(&out, &h, 2);
  return out;
}

// fp16 twin of host_bf16: round to nearest even, overflow to inf
inline __half host_f16(float f) { return __float2half_rn(f); }
template <typename T>
inline T host_16b(float f) {
  if constexpr (std::is_same<T, __half>::value) return host_f16(f);
  else return host_bf16(f);
}

// wk: fp32 [K = taps*Cin][Cout] (BN folded) -> T (bf16 or fp16) [Cout][K]
template <typename T>
inline const char* tc_prepare_weights(TcWeights& w, const float* wk, const float* bias, int K, int cout, int R, int S, int cin,
                                      std::vector<void*>& allocs) {
  std::vector<T> t((size_t)K * cout);
  for (int k = 0; k < K; ++k)
    for (int n = 0; n < cout; ++n) t[(size_t)n * K + k] = host_16b<T>(wk[(size_t)k * cout + n]);
  const char* e = upload_dev(allocs, &w.d_w, t.data(), t.size() * sizeof(T));
  if (!e) e = upload_dev(allocs, (void**)&w.d_bias, bias, (size_t)cout * 4);
  if (e) return e;
  w.Cout = cout; w.Cin = cin; w.taps = R * S; w.S = S;
  w.ready = true;
  return nullptr;
}

// N-tile width: the narrowest wgmma N in {32, 64, 128} that covers Cout, else 128 (Cout > 128 runs several N tiles)
inline int tc_pick_bn(int cout) { return cout <= 32 ? 32 : cout <= 64 ? 64 : 128; }
// The GEMMs tc_conv_preact_kernel runs: 1x1 stride 1, no activation, a residual added, one or more 128-wide N tiles
// (every ResNet V2 _3_conv: Cout 256 to 2048)
inline bool tc_preact_eligible(int R, int stride, int cout, int act, bool res) {
  return R == 1 && stride == 1 && act == ACT_NONE && res && tc_pick_bn(cout) == 128 && cout % 8 == 0;
}
// Where a 1x1 projection's squeeze-excitation scale is applied: inside tc_conv_kernel (SE instances) when the GEMM has at
// most two N tiles (Cout <= 256), else by se_scale_kernel in place ahead of it.  The GEMM scales its A tile once per N tile,
// in warps whose throughput bounds the projection: at 2 N tiles that costs less than the separate pass's read and write of
// the tensor, at 3 and 5 (EfficientNetV2-L stages 6 and 7, Cout 384 and 640) more (DESIGN.md section 2).
inline bool tc_se_in_gemm(int cout) { return cout <= 256; }

// T: the storage type the weights were prepared in (tc_prepare_weights<T>).  s1: run tc_conv3x3s1_kernel, for a shape
// that tc3x3s1_eligible takes; else tc_conv_kernel.  z (tc_preact_eligible shapes): run tc_conv_preact_kernel, which also
// stores relu(out * pre.w + pre.b) to z.
template <typename T>
inline const char* tc_conv_launch(const TcWeights& w, const ConvParams& p, bool res_first, bool s1, cudaStream_t st, void* z = nullptr,
                                  TcPreact pre = {}) {
  TcConvParams q;
  q.res = p.res; q.bias = w.d_bias; q.out = p.out;
  q.mode = (p.R == 1 && p.stride == 1) ? 0 : 1;
  q.Hin = p.Hin; q.Win = p.Win;
  q.Cout = p.Cout; q.Cin = p.Cin;
  q.taps = w.taps; q.S = w.S; q.stride = p.stride; q.dil = p.dil;
  q.kchunks = (p.Cin + TC_BK - 1) / TC_BK;
  q.Hout = p.Hout; q.Wout = p.Wout; q.pad_t = p.pad_t; q.pad_l = p.pad_l;
  q.tiles_w = (p.Wout + TC_TILE_W - 1) / TC_TILE_W;
  q.tiles_h = (p.Hout + TC_TILE_H - 1) / TC_TILE_H;
  q.M = p.B * p.Hout * p.Wout;
  if (p.a_scale && (q.mode != 0 || !tc_se_in_gemm(p.Cout)))
    return "squeeze-excitation scale outside the 1x1 projections tc_conv_kernel scales (tc_se_in_gemm)";
  if (z && (q.mode != 0 || s1 || p.a_scale || tc_pick_bn(p.Cout) != 128))
    return "pre-activation output outside the 1x1 GEMMs tc_conv_preact_kernel runs (tc_preact_eligible)";
  // tc_conv3x3s1_kernel: bn is its K per tap and N tile
  const int bn = s1 ? tc3x3s1_width(p.Cin, p.Cout) : tc_pick_bn(p.Cout);
  q.m_tiles = q.mode == 0 ? (q.M + TC_BM - 1) / TC_BM : p.B * q.tiles_w * q.tiles_h;
  q.n_tiles = (p.Cout + bn - 1) / bn;
  const CUtensorMap* m = nullptr;  // input, weights, output
  const char* e = w.maps.get(&m, [&](CUtensorMap* c) {
    const CUtensorMapSwizzle sw = CU_TENSOR_MAP_SWIZZLE_128B;
    const uint32_t slab = (uint32_t)std::min(bn, 64);  // output box: 64 (SWIZZLE_128B) or 32 (SWIZZLE_64B) channels
    const CUtensorMapSwizzle out_sw = slab == 64 ? sw : CU_TENSOR_MAP_SWIZZLE_64B;
    const char* r;
    if (s1) {  // 16 x 10-pixel input boxes and [bn][bn] weight blocks, both with rows of bn channels like the output box
      r = make_tmap_nhwc<T>(&c[0], p.in, p.B, p.Hin, p.Win, p.Cin, bn, TC_TILE_W, TC_TILE_H + 2, 1, 1, out_sw);
      if (!r) r = make_tmap_2d<T>(&c[1], w.d_w, p.Cout, (uint64_t)w.taps * p.Cin, bn, bn, out_sw);
    } else {
      r = q.mode == 0 ? make_tmap_2d<T>(&c[0], p.in, q.M, p.Cin, TC_BM, TC_BK, sw)
                      : make_tmap_nhwc<T>(&c[0], p.in, p.B, p.Hin, p.Win, p.Cin, TC_BK, TC_TILE_W, TC_TILE_H, 1, p.stride, sw);
      if (!r) r = make_tmap_2d<T>(&c[1], w.d_w, p.Cout, (uint64_t)w.taps * p.Cin, bn, TC_BK, sw);
    }
    if (!r)
      r = q.mode == 0 ? make_tmap_2d<T>(&c[2], p.out, q.M, p.Cout, TC_BM, slab, out_sw)
                      : make_tmap_nhwc<T>(&c[2], p.out, p.B, p.Hout, p.Wout, p.Cout, slab, TC_TILE_W, TC_TILE_H, 1, 1, out_sw);
    if (!r && z) r = make_tmap_2d<T>(&c[3], z, q.M, p.Cout, TC_BM, slab, out_sw);
    return r;
  }, p.in, p.out, w.d_w, p.B, p.Hin, p.Win, p.Cin, p.Hout, p.Wout, p.Cout, w.taps, p.stride, bn, s1, z);
  if (e) return e;
  const dim3 grid(std::min(q.m_tiles * q.n_tiles, num_sms()));  // persistent: one CTA per SM
  const int res_mode = p.res ? (res_first ? 2 : 1) : 0;
  if (z)  // ResNet V2 _3_conv: no activation, the shortcut added, Cout >= 256
    return with_const<ACT_NONE>(p.act, "unsupported activation in tc_conv_preact_kernel", [&](auto act) {
      return with_const<1>(res_mode, "tc_conv_preact_kernel adds a residual after the (identity) activation", [&](auto res) {
        return launch_smem(tc_conv_preact_kernel<T, act, res, 128>, grid, dim3(TCP_THREADS), TcRing<128>::smem_bytes, st, m[0], m[1], m[2],
                           m[3], q, pre);
      });
    });
  if (s1)
    return with_const<ACT_SILU, ACT_RELU>(p.act, "unsupported activation in tc_conv3x3s1_kernel", [&](auto act) {
      return with_const<0, 1, 2>(res_mode, "unsupported residual mode", [&](auto res) {
        return with_const<32, 64>(bn, "unsupported width of tc_conv3x3s1_kernel", [&](auto ck) {
          return launch_smem(tc_conv3x3s1_kernel<T, act, res, ck>, grid, dim3(TCP_THREADS), Tc3x3Smem<ck>::smem_bytes, st, m[0], m[1], m[2],
                             q);
        });
      });
    });
  if (p.a_scale)  // the MBConv / MobileNetV3 projections: no activation, residual after it or none
    return with_const<ACT_NONE>(p.act, "unsupported activation with a squeeze-excitation scale", [&](auto act) {
      return with_const<0, 1>(res_mode, "unsupported residual mode with a squeeze-excitation scale", [&](auto res) {
        return with_const<32, 64, 128>(bn, "unsupported N tile", [&](auto bn_) {
          return launch_smem(tc_conv_kernel<T, act, res, bn_, true>, grid, dim3(TCP_THREADS), TcRing<bn_>::smem_bytes, st, m[0], m[1], m[2],
                             q, p.a_scale);
        });
      });
    });
  return with_const<ACT_NONE, ACT_SILU, ACT_RELU, ACT_HSWISH>(p.act, "unsupported activation in the tensor-core epilogue", [&](auto act) {
    return with_const<0, 1, 2>(res_mode, "unsupported residual mode", [&](auto res) {
      return with_const<32, 64, 128>(bn, "unsupported N tile", [&](auto bn_) {
        return launch_smem(tc_conv_kernel<T, act, res, bn_>, grid, dim3(TCP_THREADS), TcRing<bn_>::smem_bytes, st, m[0], m[1], m[2], q,
                           (const float*)nullptr);
      });
    });
  });
}

template <typename T>
inline const char* tc_se_scale_launch(void* x, const float* s, int B, int P, int C, cudaStream_t st) {
  size_t total8 = (size_t)B * P * C / 8;
  launch_k(se_scale_kernel<T>, dim3(grid_for(total8, 256)), dim3(256), 0, st, (T*)x, s, P, C, total8);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? nullptr : cudaGetErrorString(e);
}

// ----------------------------------------------------------------------------------------- fused head kernel
// MetrabsHeads.forward (models/metrabs.py:75-85) with ptu.soft_argmax (ptu.py:47-75) fused behind the 1x1 conv:
//   D[n, pixel] = sum_c W[n, c] * F[pixel, c]        A = head weights [N_out][C] (M = channels, 128 per tile)
//                                                     B = features     [B*P][C]  (N = pixels, <= 256 per tile)
// Each consumer warpgroup computes 64 channels x 256 pixels in registers and parks them in its half of a shared-memory
// staging tile; then one thread per channel n = J + d*J + j (or n = j < J for the 2D head) adds the bias and keeps the
// online-softmax state (max, sum e, sum e*x, sum e*y) of ITS pixels in registers, across the pixel tiles of a crop;
// one float4 per (crop, channel) goes to a scratch, and head_finalize_kernel merges the D depth slices of every
// joint (sum e*z = d * sum e), applies linspace(0,1,n) and heatmap_to_image / heatmap_to_metric.
struct TcHeadParams {
  float4* states;     // [B][n_out] (m, s, sx, sy)
  const float* bias;  // [n_out]
  int B, P, W, n_out, C;
  int bnp;            // pixels per tile (N)
  int cpt;            // crops per tile when P <= 256, else 0
  int npt;            // pixel tiles per crop when P > 256, else 1
  int m_tiles;        // ceil(n_out / 128)
  int kblocks;        // ceil(C / 64)
};
constexpr int TCH_STAGES = 2;
constexpr int TCH_STAGE_BYTES = TC_A_BYTES + 256 * TC_BK * 2;      // 48 KB
constexpr int TCH_STG_OFF = TCH_STAGES * TCH_STAGE_BYTES;           // staging: [128 channels][256 pixels] fp32 = 128 KB
constexpr int TCH_BAR_OFF = TCH_STG_OFF + 128 * 256 * 4;
constexpr int TCH_SMEM_BYTES = TCH_BAR_OFF + 64 + 1024 /*align slack*/;

// staging element (row, col): 16-byte chunks of a row XOR-rotated by row & 7 (the row owners read along their rows)
__device__ __forceinline__ uint32_t tch_stg(int row, int col) {
  return (uint32_t)(row * 256 + ((((col >> 2) ^ (row & 7))) << 2) + (col & 3)) * 4u;
}

template <typename T>
__global__ void __launch_bounds__(TC_THREADS, 1)
tc_head_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmF, const TcHeadParams p) {
  extern __shared__ uint8_t tc_smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)tc_smem_raw + 1023) & ~(uintptr_t)1023);
  uint64_t* full = (uint64_t*)(smem + TCH_BAR_OFF);
  uint64_t* empty = full + TCH_STAGES;
  float* stg = (float*)(smem + TCH_STG_OFF);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == TC_CONSUMER_WARPS * 32) {
    tma_prefetch_desc(&tmW);
    tma_prefetch_desc(&tmF);
    for (int i = 0; i < TCH_STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], TC_CONSUMER_WARPS);
    }
    fence_barrier_init();
  }
  __syncthreads();

  const int g = blockIdx.x / p.m_tiles, m_blk = blockIdx.x - g * p.m_tiles;
  const int n_kb = p.npt * p.kblocks;
  if (warp == TC_CONSUMER_WARPS) {
    if (lane == 0) {
      const uint32_t stage_tx = TC_A_BYTES + (uint32_t)p.bnp * TC_BK * 2;
      for (int i = 0; i < n_kb; ++i) {
        const int s = i % TCH_STAGES, pt = i / p.kblocks, kb = i - pt * p.kblocks;
        mbar_wait(&empty[s], ((i / TCH_STAGES) & 1) ^ 1);
        uint8_t* sa = smem + s * TCH_STAGE_BYTES;
        const int row0 = p.cpt > 0 ? g * p.bnp : g * p.P + pt * p.bnp;
        mbar_expect_tx(&full[s], stage_tx);
        tma_load_2d(sa, &tmW, &full[s], kb * TC_BK, m_blk * TC_BM);
        tma_load_2d(sa + TC_A_BYTES, &tmF, &full[s], kb * TC_BK, row0);
      }
    }
    return;
  }
  const int wg = warp >> 2, tid = threadIdx.x & 127;
  // row owners: threads 0-63 of each warpgroup, one channel each
  const int row = wg * 64 + tid;
  const int n = m_blk * TC_BM + row;
  const bool owner = tid < 64;
  const bool nvalid = owner && n < p.n_out;
  const float bias_n = nvalid ? p.bias[n] : 0.f;
  constexpr float L2E = 1.4426950408889634f;
  int crop = p.cpt > 0 ? g * p.cpt : g;
  int pix = 0, x = 0, y = 0;
  float m = -INFINITY, mL = -INFINITY, s_ = 0.f, sx = 0.f, sy = 0.f;
  int i = 0;
  for (int pt = 0; pt < p.npt; ++pt) {
    float acc[128];
#pragma unroll
    for (int k = 0; k < 128; ++k) acc[k] = 0.f;
    int prev = -1;
    for (int kb = 0; kb < p.kblocks; ++kb, ++i) {
      const int s = i % TCH_STAGES;
      mbar_wait(&full[s], (i / TCH_STAGES) & 1);
      const uint32_t a = smem_u32(smem + s * TCH_STAGE_BYTES) + wg * 64 * 128;
      const uint32_t b = smem_u32(smem + s * TCH_STAGE_BYTES + TC_A_BYTES);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < TC_BK / 16; ++k) wgmma_16b<T, 256>(acc, gmma_desc<128>(a + 32 * k), gmma_desc<128>(b + 32 * k), (uint32_t)(kb | k));
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[prev]);
      }
      prev = s;
    }
    wgmma_wait<0>();
    wgmma_fence_regs<128>(acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[prev]);
    // fragment -> staging (this warpgroup's 64 rows)
    {
      const int fr = wg * 64 + (warp & 3) * 16 + (lane >> 2), fc = 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        *reinterpret_cast<float2*>((uint8_t*)stg + tch_stg(fr, fc + 8 * j)) = make_float2(acc[4 * j], acc[4 * j + 1]);
        *reinterpret_cast<float2*>((uint8_t*)stg + tch_stg(fr + 8, fc + 8 * j)) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
      }
    }
    wg_sync(wg);
    if (owner) {
      for (int c0 = 0; c0 < p.bnp; c0 += 16) {
        float v[16];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float4 f = *reinterpret_cast<const float4*>((const uint8_t*)stg + tch_stg(row, c0 + 4 * q));
          v[4 * q] = f.x; v[4 * q + 1] = f.y; v[4 * q + 2] = f.z; v[4 * q + 3] = f.w;
        }
        if (pix + 16 <= p.P) {
          // whole chunk inside one crop: one rescale, then 16 exps
          float vm = v[0];
#pragma unroll
          for (int q = 1; q < 16; ++q) vm = fmaxf(vm, v[q]);
          vm += bias_n;
          if (vm > m) {
            const float mL_new = vm * L2E;
            float f = ex2_fast(mL - mL_new);  // same rounded offsets as the elements use
            s_ *= f; sx *= f; sy *= f;
            m = vm;
            mL = mL_new;
          }
          const float cL = fmaf(bias_n, L2E, -mL);
#pragma unroll
          for (int q = 0; q < 16; ++q) {
            float e = ex2_fast(fmaf(v[q], L2E, cL));
            s_ += e;
            sx = fmaf(e, (float)x, sx);
            sy = fmaf(e, (float)y, sy);
            if (++x == p.W) { x = 0; ++y; }
          }
          pix += 16;
          if (pix == p.P) {
            if (nvalid && crop < p.B) p.states[(size_t)crop * p.n_out + n] = make_float4(m, s_, sx, sy);
            ++crop; pix = 0; x = 0; y = 0;
            m = -INFINITY; mL = -INFINITY; s_ = 0.f; sx = 0.f; sy = 0.f;
          }
        } else {
          // chunk straddles a crop boundary (P % 16 != 0): element-wise
#pragma unroll
          for (int q = 0; q < 16; ++q) {
            float vv = v[q] + bias_n;
            if (vv > m) {
              const float mL_new = vv * L2E;
              float f = ex2_fast(mL - mL_new);
              s_ *= f; sx *= f; sy *= f;
              m = vv;
              mL = mL_new;
            }
            float e = ex2_fast(fmaf(vv, L2E, -mL));
            s_ += e;
            sx = fmaf(e, (float)x, sx);
            sy = fmaf(e, (float)y, sy);
            if (++x == p.W) { x = 0; ++y; }
            if (++pix == p.P) {
              if (nvalid && crop < p.B) p.states[(size_t)crop * p.n_out + n] = make_float4(m, s_, sx, sy);
              ++crop; pix = 0; x = 0; y = 0;
              m = -INFINITY; mL = -INFINITY; s_ = 0.f; sx = 0.f; sy = 0.f;
            }
          }
        }
      }
    }
    wg_sync(wg);  // the staging tile is rewritten by the next pixel tile
  }
}

// merges the per-channel states of one crop into coords2d [J,2] (px) and coords3d_rel [J,3] (mm)
__global__ void __launch_bounds__(128) head_finalize_kernel(const float4* __restrict__ states, float* __restrict__ out2d,
                                                            float* __restrict__ out3d, int J, int D, int H, int W,
                                                            DecodeScale sc) {
  const int b = blockIdx.x;
  const int n_out = J * (1 + D);
  for (int j = threadIdx.x; j < J; j += blockDim.x) {
    const float4* st = states + (size_t)b * n_out;
    {
      float4 c = st[j];
      float x = soft_coord(c.z, c.y, W), y = soft_coord(c.w, c.y, H);
      if (sc.apply) {
        x = fmaf(x, sc.img_mul, sc.img_add);
        y = fmaf(y, sc.img_mul, sc.img_add);
      }
      out2d[((size_t)b * J + j) * 2 + 0] = x;
      out2d[((size_t)b * J + j) * 2 + 1] = y;
    }
    SoftState a;
    soft_init(a);
    for (int d = 0; d < D; ++d) {
      float4 c = st[J + d * J + j];
      SoftState bb;
      bb.m = c.x; bb.s = c.y; bb.sx = c.z; bb.sy = c.w; bb.sz = c.y * (float)d;
      soft_merge(a, bb);
    }
    float x = soft_coord(a.sx, a.s, W), y = soft_coord(a.sy, a.s, H), z = soft_coord(a.sz, a.s, D);
    if (sc.apply) {
      x = fmaf(x, sc.met_mul, sc.met_add);
      y = fmaf(y, sc.met_mul, sc.met_add);
      z = z * sc.z_mul;
    }
    out3d[((size_t)b * J + j) * 3 + 0] = x;
    out3d[((size_t)b * J + j) * 3 + 1] = y;
    out3d[((size_t)b * J + j) * 3 + 2] = z;
  }
}

// w: fp32 [n_out][C] (torch conv weight [N,C,1,1]) -> T (bf16 or fp16); returns nullptr on success.  Not eligible -> ready
// stays false.
template <typename T>
inline const char* tc_prepare_head(TcWeights& w, const float* wt, const float* bias, int C, int n_out, std::vector<void*>& allocs) {
  if (C % 8 != 0) return nullptr;
  std::vector<T> t((size_t)n_out * C);
  for (size_t i = 0; i < t.size(); ++i) t[i] = host_16b<T>(wt[i]);
  const char* e = upload_dev(allocs, &w.d_w, t.data(), t.size() * sizeof(T));
  if (!e) e = upload_dev(allocs, (void**)&w.d_bias, bias, (size_t)n_out * 4);
  if (e) return e;
  w.Cout = n_out; w.Cin = C; w.n_real = n_out;
  w.ready = true;
  return nullptr;
}

inline bool tc_head_plan(int P, int* bnp, int* cpt, int* npt) {
  if (P <= 256) {
    for (int c = 256 / P; c >= 1; --c)
      if ((c * P) % 16 == 0) {
        *bnp = c * P; *cpt = c; *npt = 1;
        return true;
      }
    return false;
  }
  if (P % 256 != 0) return false;
  *bnp = 256; *cpt = 0; *npt = P / 256;
  return true;
}

template <typename T>
inline const char* tc_head_launch(const TcWeights& w, const void* features, int B, int H, int W, int J, int D, DecodeScale sc,
                                  float* c2d, float* c3d, void* scratch, cudaStream_t st) {
  TcHeadParams q;
  q.states = (float4*)scratch;
  q.bias = w.d_bias;
  q.B = B; q.P = H * W; q.W = W; q.n_out = w.n_real; q.C = w.Cin;
  if (!tc_head_plan(q.P, &q.bnp, &q.cpt, &q.npt)) return "unsupported feature map shape for the fused head";
  const int n_groups = q.cpt > 0 ? (B + q.cpt - 1) / q.cpt : B;
  q.m_tiles = (q.n_out + TC_BM - 1) / TC_BM;
  q.kblocks = (q.C + TC_BK - 1) / TC_BK;
  const CUtensorMap* m = nullptr;  // weights, features
  const char* e = w.maps.get(&m, [&](CUtensorMap* c) {
    const char* r = make_tmap_2d<T>(&c[0], w.d_w, q.n_out, q.C, TC_BM, TC_BK, CU_TENSOR_MAP_SWIZZLE_128B);
    return r ? r : make_tmap_2d<T>(&c[1], features, (uint64_t)B * q.P, q.C, q.bnp, TC_BK, CU_TENSOR_MAP_SWIZZLE_128B);
  }, w.d_w, features, B, H, W, q.C, q.n_out);
  if (!e) e = launch_smem(tc_head_kernel<T>, dim3(n_groups * q.m_tiles), dim3(TC_THREADS), TCH_SMEM_BYTES, st, m[0], m[1], q);
  if (e) return e;
  launch_k(head_finalize_kernel, dim3(B), dim3(128), 0, st, q.states, c2d, c3d, J, D, H, W, sc);
  const cudaError_t ce = cudaGetLastError();
  return ce == cudaSuccess ? nullptr : cudaGetErrorString(ce);
}

}  // namespace mtb
