// Depthwise 3x3 stride-1 conv + bias + activation + squeeze-excitation pooling for bf16 or fp16 NHWC tensors (the MBConv middle
// op, backbones/efficientnet.py:110-173), staged through shared memory by TMA.
//
// Why: the strip kernel (dwconv3x3_pool_16b_kernel) ran at ~2 TB/s whatever the batch (so not HBM-bound): every thread
// lived for ONE strip - one global-load round trip, then compute, then a block reduction - and nothing overlapped the
// load latency.  Here a persistent CTA walks (crop group, 64-channel group, row band) items; the (rows+2) x (W+2) x 64ch
// input patch of the NEXT item is in flight (one 4D TMA box, out-of-image halo = TMA zero fill = the reference's explicit
// zero padding, efficientnet.py:1127-1161) while the current one is computed from shared memory, each input row is read
// and unpacked once per 4-row run (input-stationary: a row updates the three output rows it feeds), and the SE means are
// reduced in a fixed order inside the CTA.
//
// Dilation d (2 or 4, the dilated EfficientNetV2 stages): the outputs (py + d i, px + d j) of one phase (py, px) are an
// undilated 3x3 SAME conv of the input sub-grid X[py::d, px::d].  An item then walks the d^2 phases in order, each staged as the
// undilated item's patch of that sub-grid (one TMA box with element stride d), computed by the same loop with the output
// addressing scaled by d, and summed into the same pooling slice: the patch is as small as an undilated one and the pooling
// order stays fixed.
#pragma once
#include "tc_gemm.cuh"

namespace mtb {

constexpr int DWT_THREADS = 128;   // 8 channel vectors (8 ch each) x 16 strips per pass
constexpr int DWT_CG = 64;         // channels per item (128-byte pixel rows in shared memory)
constexpr int DWT_RUN = 4;         // output rows per thread run (RUN + 2 input rows)
constexpr int DWT_OW = 4;          // output columns per thread (OW + 2 input columns)
constexpr int DWT_STAGES = 2;
constexpr int DWT_MAX_STAGE = 52 * 1024;
constexpr int DWT_MAX_G = 8;

struct DwTmaParams {
  void* out;           // bf16 / fp16 NHWC
  const float* w;      // [9][C] fp32 (BN folded)
  const float* bias;   // [C]
  float* pooled;       // [n_rb][B][C] partial means (nullptr: no squeeze-excitation behind this op)
  int B, H, W, C;
  int pad_t, pad_l;
  int G, BH;           // crops per item, output rows per item
  int n_cg, n_rb, items;
  int strips_w, bands, nstrips;  // per item: column strips, row runs per crop, G * bands * strips_w
  int stage_bytes;
  float inv_hw;
};

struct DwTmaPlan {
  bool ok = false;
  int G = 1, BH = 0, n_rb = 1;
};

// (crops per item, rows per item): maximise (busy strip slots) x (useful rows / staged rows) within the stage budget.  H x W:
// the map, or with dilation `dil` the largest phase sub-grid; a TMA box spans at most 256 pixels per axis
inline DwTmaPlan dw_tma_plan(int H, int W, int dil = 1) {
  DwTmaPlan best;
  double best_score = -1.0;
  const int PW = W + 2;
  const int strips_w = (W + DWT_OW - 1) / DWT_OW;
  if (PW * dil > 256) return best;
  for (int BH = DWT_RUN; BH <= H + DWT_RUN - 1; BH += DWT_RUN) {
    const int bh = BH > H ? H : BH;
    if ((bh + 2) * dil > 256) break;
    const long patch = 128L * PW * (bh + 2);
    if (patch > DWT_MAX_STAGE) break;
    const int gmax = (int)std::min<long>(DWT_MAX_G, DWT_MAX_STAGE / patch);
    const int bands = (bh + DWT_RUN - 1) / DWT_RUN;
    const int n_rb = (H + bh - 1) / bh;
    for (int G = 1; G <= (n_rb == 1 ? gmax : 1); ++G) {
      const int nstrips = G * bands * strips_w;
      const double eff = (double)nstrips / (16.0 * ((nstrips + 15) / 16));
      const double score = eff * bh / (bh + 2.0) - 1e-3 * G;
      if (score > best_score) {
        best_score = score;
        best.ok = true; best.G = G; best.BH = bh; best.n_rb = n_rb;
      }
    }
  }
  return best;
}

// activation of a pair; SiLU(x) = h + h * tanh(h), h = x / 2 for bf16 outputs, silu_f16out for fp16 ones (same arithmetic as
// fast_act<ACT_SILU, T>)
template <int ACT, typename T>
__device__ __forceinline__ f32x2 f2_act(f32x2 x) {
  if constexpr (ACT == ACT_SILU && is_f16<T>) {
    float x0, x1;
    f2_unpack(x, x0, x1);
    return f2_pack(silu_f16out(x0), silu_f16out(x1));
  } else if constexpr (ACT == ACT_SILU) {
    const f32x2 h = f2_mul(x, f2_pack(0.5f, 0.5f));
    float h0, h1;
    f2_unpack(h, h0, h1);
    return f2_fma(h, f2_pack(fast_tanh(h0), fast_tanh(h1)), h);
  } else {
    float x0, x1;
    f2_unpack(x, x0, x1);
    return f2_pack(fast_act<ACT, T>(x0), fast_act<ACT, T>(x1));
  }
}

// 64 channels per item, 8 per thread (4 fp32 pairs); T: element type (__nv_bfloat16 or __half)
template <typename T, int ACT>
__global__ void __launch_bounds__(DWT_THREADS, 2)
dw3x3s1_tma_kernel(const __grid_constant__ CUtensorMap tmIn, const DwTmaParams p) {
  constexpr int NV = 4;                    // fp32 pairs per thread
  constexpr int CPT = 2 * NV;              // channels per thread
  extern __shared__ uint8_t dwt_smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)dwt_smem_raw + 127) & ~(uintptr_t)127);
  __shared__ uint64_t full[DWT_STAGES];
  __shared__ float red[16][DWT_CG];            // per pass: activated-output sums of each strip slot
  __shared__ float blocksum[DWT_MAX_G][DWT_CG];  // per item: sums per (crop of the group, channel), owner thread = channel

  const int tid = threadIdx.x;
  const int j = tid & 7;        // channel vector inside the 64-channel group
  const int sidx = tid >> 3;    // strip slot 0..15
  if (tid == 0) {
    tma_prefetch_desc(&tmIn);
    for (int i = 0; i < DWT_STAGES; ++i) mbar_init(&full[i], 1);
    fence_barrier_init();
  }
  __syncthreads();

  const int PW = p.W + 2, PHB = p.BH + 2;
  const uint32_t stage_tx = (uint32_t)(128 * PW * PHB * p.G);
  const int strips_per_crop = p.bands * p.strips_w;
  constexpr int GSTEP = DWT_THREADS / DWT_CG;
  const int own_ch = tid & (DWT_CG - 1), own_g0 = tid / DWT_CG;  // blocksum owner: channel own_ch, crops own_g0, own_g0 + GSTEP, ...

  // Items are walked last-to-first: the expand GEMM before this op wrote its output first-crop-to-last, all channels of a
  // pixel block together (tc_conv_kernel's tile order is N fastest), so the END of the whole tensor is what the L2 still
  // holds, and the BEGINNING of this op's output stays in L2 for the projection GEMM that follows.
  auto issue = [&](int it_, int stage) {
    const int it = p.items - 1 - it_;
    const int cg = it % p.n_cg;
    const int t2 = it / p.n_cg;
    const int rb = t2 % p.n_rb, bg = t2 / p.n_rb;
    mbar_expect_tx(&full[stage], stage_tx);
    tma_load_4d(smem + (size_t)stage * p.stage_bytes, &tmIn, &full[stage], cg * DWT_CG, -p.pad_l, rb * p.BH - p.pad_t, bg * p.G);
  };

  if (tid == 0 && (int)blockIdx.x < p.items) issue(blockIdx.x, 0);
  int li = 0;
  for (int it_ = blockIdx.x; it_ < p.items; it_ += gridDim.x, ++li) {
    const int stage = li & 1;
    if (tid == 0 && it_ + (int)gridDim.x < p.items) issue(it_ + gridDim.x, stage ^ 1);
    const int it = p.items - 1 - it_;
    const int cg = it % p.n_cg;
    const int t2 = it / p.n_cg;
    const int rb = t2 % p.n_rb, bg = t2 / p.n_rb;
    const int c = cg * DWT_CG + j * CPT;
    const bool c_ok = c < p.C;
    const int b0 = bg * p.G, row0 = rb * p.BH;
    const int rows_item = min(p.BH, p.H - row0);  // output rows of this item

    // this thread's 8 channels: 9 taps + bias, fp32 pairs (channels 2k, 2k+1), in registers for the whole item
    f32x2 w[9][NV], bias[NV];
#pragma unroll
    for (int t = 0; t < 9; ++t) {
#pragma unroll
      for (int q = 0; q < NV / 2; ++q) {
        float4 w0 = make_float4(0.f, 0.f, 0.f, 0.f);
        if (c_ok) w0 = __ldg(reinterpret_cast<const float4*>(p.w + (size_t)t * p.C + c + 4 * q));
        w[t][2 * q] = f2_pack(w0.x, w0.y); w[t][2 * q + 1] = f2_pack(w0.z, w0.w);
      }
    }
#pragma unroll
    for (int q = 0; q < NV / 2; ++q) {
      float4 b0v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (c_ok) b0v = __ldg(reinterpret_cast<const float4*>(p.bias + c + 4 * q));
      bias[2 * q] = f2_pack(b0v.x, b0v.y); bias[2 * q + 1] = f2_pack(b0v.z, b0v.w);
    }
    if (p.pooled) {
      for (int g = own_g0; g < p.G; g += GSTEP) blocksum[g][own_ch] = 0.f;
    }
    mbar_wait(&full[stage], (uint32_t)((li >> 1) & 1));
    const uint8_t* patch = smem + (size_t)stage * p.stage_bytes + j * 16;

    for (int s0 = 0; s0 < p.nstrips; s0 += 16) {
      const int s = s0 + sidx;
      f32x2 psum[NV];
#pragma unroll
      for (int k = 0; k < NV; ++k) psum[k] = f2_pack(0.f, 0.f);
      if (s < p.nstrips && c_ok) {
        const int g = s / strips_per_crop;
        const int rem = s - g * strips_per_crop;
        const int band = rem / p.strips_w;
        const int ow0 = (rem - band * p.strips_w) * DWT_OW;
        const int b = b0 + g;
        const int orow0 = band * DWT_RUN;                       // first output row of the run, relative to the item
        const int rows_run = min(DWT_RUN, rows_item - orow0);   // >= 1 by construction of `bands`
        if (b < p.B && rows_run > 0) {
          const uint8_t* prow = patch + (size_t)((g * PHB + orow0) * PW + ow0) * 128;
          T* obase = reinterpret_cast<T*>(p.out) + ((size_t)(b * p.H + row0 + orow0) * p.W + ow0) * p.C + c;
          f32x2 acc[3][DWT_OW][NV];
#pragma unroll
          for (int pr = 0; pr < DWT_RUN + 2; ++pr) {
            if (pr < rows_run + 2) {
              // one input row of the run (OW + 2 pixels x 8 channels, each read and unpacked once); it is tap row r of output
              // row pr - r (slot (pr - r) % 3); the first tap of an output row (r = 0, s = 0) starts from the bias
#pragma unroll
              for (int x = 0; x < DWT_OW + 2; ++x) {
                const uint4 raw = *reinterpret_cast<const uint4*>(prow + (size_t)(pr * PW + x) * 128);
                const unsigned wd[4] = {raw.x, raw.y, raw.z, raw.w};
                f32x2 v[NV];
#pragma unroll
                for (int k = 0; k < NV; ++k) v[k] = unpack2_16b<T>(wd[k]);
#pragma unroll
                for (int r = 0; r < 3; ++r) {
                  const int o = pr - r;  // compile-time
                  if (o < 0 || o >= DWT_RUN) continue;
#pragma unroll
                  for (int i = 0; i < DWT_OW; ++i) {
                    const int s_ = x - i;  // compile-time
                    if (s_ >= 0 && s_ < 3) {
#pragma unroll
                      for (int k = 0; k < NV; ++k)
                        acc[o % 3][i][k] = f2_fma(v[k], w[r * 3 + s_][k], (r == 0 && s_ == 0) ? bias[k] : acc[o % 3][i][k]);
                    }
                  }
                }
              }
              // output row pr - 2 is complete
              if (pr >= 2 && pr - 2 < rows_run) {
                const int o = pr - 2, slot = o % 3;
                T* orow = obase + (size_t)o * p.W * p.C;
#pragma unroll
                for (int i = 0; i < DWT_OW; ++i) {
                  if (ow0 + i < p.W) {
                    uint4 ov;
                    typename Pair16<T>::type* o2 = reinterpret_cast<typename Pair16<T>::type*>(&ov);
#pragma unroll
                    for (int k = 0; k < NV; ++k) {
                      const f32x2 a = f2_act<ACT, T>(acc[slot][i][k]);
                      float a0, a1;
                      f2_unpack(a, a0, a1);
                      o2[k] = Pair16<T>::pack(a0, a1);
                      psum[k] = f2_add(psum[k], a);
                    }
                    *reinterpret_cast<uint4*>(orow + (size_t)i * p.C) = ov;
                  }
                }
              }
            }
          }
        }
      }
      if (p.pooled) {
        // fixed-order reduction of this pass: strip slots -> (crop, channel) owner threads
        *reinterpret_cast<float4*>(&red[sidx][j * CPT]) = make_float4(psum[0].x, psum[0].y, psum[1].x, psum[1].y);
        *reinterpret_cast<float4*>(&red[sidx][j * CPT + 4]) = make_float4(psum[2].x, psum[2].y, psum[3].x, psum[3].y);
        __syncthreads();
        for (int g = own_g0; g < p.G; g += GSTEP) {
          // strip slots of crop g in this pass: [g * strips_per_crop, (g + 1) * strips_per_crop) - s0, clipped
          const int qlo = max(g * strips_per_crop - s0, 0);
          const int qhi = min(min((g + 1) * strips_per_crop, p.nstrips) - s0, 16);
          float t = blocksum[g][own_ch];
          for (int q = qlo; q < qhi; ++q) t += red[q][own_ch];
          blocksum[g][own_ch] = t;
        }
        __syncthreads();
      }
    }
    if (p.pooled) {
      const int ch = cg * DWT_CG + own_ch;
      if (ch < p.C) {
        for (int g = own_g0; g < p.G; g += GSTEP) {
          if (b0 + g < p.B) p.pooled[((size_t)rb * p.B + b0 + g) * p.C + ch] = blocksum[g][own_ch] * p.inv_hw;
        }
      }
    }
    __syncthreads();  // every thread is done with `stage` (the next iteration's TMA may overwrite it) and with blocksum
  }
}

// dw3x3s1_tma_kernel for dilation DIL (2 or 4) and SiLU: the same item, strip loop and arithmetic per output, run once per phase
// of the dilation on that phase's sub-grid (header comment); the SE sums of all phases go to the item's pooling slice
template <typename T, int DIL>
__global__ void __launch_bounds__(DWT_THREADS, 2)
dw3x3s1_dil_tma_kernel(const __grid_constant__ CUtensorMap tmIn, const DwTmaParams p) {
  constexpr int NV = 4;                    // fp32 pairs per thread
  constexpr int CPT = 2 * NV;              // channels per thread
  constexpr int NPH = DIL * DIL;           // phases per item
  extern __shared__ uint8_t dwt_smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)dwt_smem_raw + 127) & ~(uintptr_t)127);
  __shared__ uint64_t full[DWT_STAGES];
  __shared__ float red[16][DWT_CG];            // per pass: activated-output sums of each strip slot
  __shared__ float blocksum[DWT_MAX_G][DWT_CG];  // per item: sums per (crop of the group, channel), owner thread = channel

  const int tid = threadIdx.x;
  const int j = tid & 7;        // channel vector inside the 64-channel group
  const int sidx = tid >> 3;    // strip slot 0..15
  if (tid == 0) {
    tma_prefetch_desc(&tmIn);
    for (int i = 0; i < DWT_STAGES; ++i) mbar_init(&full[i], 1);
    fence_barrier_init();
  }
  __syncthreads();

  const int PW = (p.W + DIL - 1) / DIL + 2, PHB = p.BH + 2;
  const uint32_t stage_tx = (uint32_t)(128 * PW * PHB * p.G);
  const int strips_per_crop = p.bands * p.strips_w;
  constexpr int GSTEP = DWT_THREADS / DWT_CG;
  const int own_ch = tid & (DWT_CG - 1), own_g0 = tid / DWT_CG;  // blocksum owner: channel own_ch, crops own_g0, own_g0 + GSTEP, ...

  // Items are walked last-to-first: the expand GEMM before this op wrote its output first-crop-to-last, all channels of a
  // pixel block together (tc_conv_kernel's tile order is N fastest), so the END of the whole tensor is what the L2 still
  // holds, and the BEGINNING of this op's output stays in L2 for the projection GEMM that follows.
  // phase (py, px) = (ph / DIL, ph % DIL) of the item: its sub-grid rows from rb * BH on, with one halo row / column
  auto issue = [&](int it_, int ph, int stage) {
    const int it = p.items - 1 - it_;
    const int cg = it % p.n_cg;
    const int t2 = it / p.n_cg;
    const int rb = t2 % p.n_rb, bg = t2 / p.n_rb;
    mbar_expect_tx(&full[stage], stage_tx);
    tma_load_4d(smem + (size_t)stage * p.stage_bytes, &tmIn, &full[stage], cg * DWT_CG, ph % DIL - p.pad_l,
                ph / DIL + rb * p.BH * DIL - p.pad_t, bg * p.G);
  };
  // the unit after phase ph of item it_: the next phase, or the first phase of this CTA's next item
  auto issue_next = [&](int it_, int ph, int stage) {
    if (ph + 1 < NPH) issue(it_, ph + 1, stage);
    else if (it_ + (int)gridDim.x < p.items) issue(it_ + gridDim.x, 0, stage);
  };

  if (tid == 0 && (int)blockIdx.x < p.items) issue(blockIdx.x, 0, 0);
  int li = 0;
  for (int it_ = blockIdx.x; it_ < p.items; it_ += gridDim.x) {
    if (tid == 0) issue_next(it_, 0, (li & 1) ^ 1);
    const int it = p.items - 1 - it_;
    const int cg = it % p.n_cg;
    const int t2 = it / p.n_cg;
    const int rb = t2 % p.n_rb, bg = t2 / p.n_rb;
    const int c = cg * DWT_CG + j * CPT;
    const bool c_ok = c < p.C;
    const int b0 = bg * p.G, row0 = rb * p.BH;

    // this thread's 8 channels: 9 taps + bias, fp32 pairs (channels 2k, 2k+1), in registers for the whole item
    f32x2 w[9][NV], bias[NV];
#pragma unroll
    for (int t = 0; t < 9; ++t) {
#pragma unroll
      for (int q = 0; q < NV / 2; ++q) {
        float4 w0 = make_float4(0.f, 0.f, 0.f, 0.f);
        if (c_ok) w0 = __ldg(reinterpret_cast<const float4*>(p.w + (size_t)t * p.C + c + 4 * q));
        w[t][2 * q] = f2_pack(w0.x, w0.y); w[t][2 * q + 1] = f2_pack(w0.z, w0.w);
      }
    }
#pragma unroll
    for (int q = 0; q < NV / 2; ++q) {
      float4 b0v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (c_ok) b0v = __ldg(reinterpret_cast<const float4*>(p.bias + c + 4 * q));
      bias[2 * q] = f2_pack(b0v.x, b0v.y); bias[2 * q + 1] = f2_pack(b0v.z, b0v.w);
    }
    if (p.pooled) {
      for (int g = own_g0; g < p.G; g += GSTEP) blocksum[g][own_ch] = 0.f;
    }
    for (int ph = 0; ph < NPH; ++ph, ++li) {
      const int stage = li & 1;
      if (ph > 0 && tid == 0) issue_next(it_, ph, stage ^ 1);
      // this phase's sub-grid: Hq x Wq pixels from (py, px) in steps of DIL
      const int py = ph / DIL, px = ph % DIL;
      const int Hq = (p.H - py + DIL - 1) / DIL, Wq = (p.W - px + DIL - 1) / DIL;
      const int rows_item = min(p.BH, Hq - row0);  // output rows of this item
      mbar_wait(&full[stage], (uint32_t)((li >> 1) & 1));
      const uint8_t* patch = smem + (size_t)stage * p.stage_bytes + j * 16;

      for (int s0 = 0; s0 < p.nstrips; s0 += 16) {
        const int s = s0 + sidx;
        f32x2 psum[NV];
#pragma unroll
        for (int k = 0; k < NV; ++k) psum[k] = f2_pack(0.f, 0.f);
        if (s < p.nstrips && c_ok) {
          const int g = s / strips_per_crop;
          const int rem = s - g * strips_per_crop;
          const int band = rem / p.strips_w;
          const int ow0 = (rem - band * p.strips_w) * DWT_OW;
          const int b = b0 + g;
          const int orow0 = band * DWT_RUN;                       // first output row of the run, relative to the item
          const int rows_run = min(DWT_RUN, rows_item - orow0);   // < 1 in a phase that ends above the run
          if (b < p.B && rows_run > 0) {
            const uint8_t* prow = patch + (size_t)((g * PHB + orow0) * PW + ow0) * 128;
            T* obase = reinterpret_cast<T*>(p.out) + ((size_t)(b * p.H + py + (row0 + orow0) * DIL) * p.W + px + ow0 * DIL) * p.C + c;
            f32x2 acc[3][DWT_OW][NV];
#pragma unroll
            for (int pr = 0; pr < DWT_RUN + 2; ++pr) {
              if (pr < rows_run + 2) {
                // one input row of the run (OW + 2 pixels x 8 channels, each read and unpacked once); it is tap row r of output
                // row pr - r (slot (pr - r) % 3); the first tap of an output row (r = 0, s = 0) starts from the bias
#pragma unroll
                for (int x = 0; x < DWT_OW + 2; ++x) {
                  const uint4 raw = *reinterpret_cast<const uint4*>(prow + (size_t)(pr * PW + x) * 128);
                  const unsigned wd[4] = {raw.x, raw.y, raw.z, raw.w};
                  f32x2 v[NV];
#pragma unroll
                  for (int k = 0; k < NV; ++k) v[k] = unpack2_16b<T>(wd[k]);
#pragma unroll
                  for (int r = 0; r < 3; ++r) {
                    const int o = pr - r;  // compile-time
                    if (o < 0 || o >= DWT_RUN) continue;
#pragma unroll
                    for (int i = 0; i < DWT_OW; ++i) {
                      const int s_ = x - i;  // compile-time
                      if (s_ >= 0 && s_ < 3) {
#pragma unroll
                        for (int k = 0; k < NV; ++k)
                          acc[o % 3][i][k] = f2_fma(v[k], w[r * 3 + s_][k], (r == 0 && s_ == 0) ? bias[k] : acc[o % 3][i][k]);
                      }
                    }
                  }
                }
                // output row pr - 2 is complete
                if (pr >= 2 && pr - 2 < rows_run) {
                  const int o = pr - 2, slot = o % 3;
                  T* orow = obase + (size_t)o * DIL * p.W * p.C;
#pragma unroll
                  for (int i = 0; i < DWT_OW; ++i) {
                    if (ow0 + i < Wq) {
                      uint4 ov;
                      typename Pair16<T>::type* o2 = reinterpret_cast<typename Pair16<T>::type*>(&ov);
#pragma unroll
                      for (int k = 0; k < NV; ++k) {
                        const f32x2 a = f2_act<ACT_SILU, T>(acc[slot][i][k]);
                        float a0, a1;
                        f2_unpack(a, a0, a1);
                        o2[k] = Pair16<T>::pack(a0, a1);
                        psum[k] = f2_add(psum[k], a);
                      }
                      *reinterpret_cast<uint4*>(orow + (size_t)i * DIL * p.C) = ov;
                    }
                  }
                }
              }
            }
          }
        }
        if (p.pooled) {
          // fixed-order reduction of this pass: strip slots -> (crop, channel) owner threads
          *reinterpret_cast<float4*>(&red[sidx][j * CPT]) = make_float4(psum[0].x, psum[0].y, psum[1].x, psum[1].y);
          *reinterpret_cast<float4*>(&red[sidx][j * CPT + 4]) = make_float4(psum[2].x, psum[2].y, psum[3].x, psum[3].y);
          __syncthreads();
          for (int g = own_g0; g < p.G; g += GSTEP) {
            // strip slots of crop g in this pass: [g * strips_per_crop, (g + 1) * strips_per_crop) - s0, clipped
            const int qlo = max(g * strips_per_crop - s0, 0);
            const int qhi = min(min((g + 1) * strips_per_crop, p.nstrips) - s0, 16);
            float t = blocksum[g][own_ch];
            for (int q = qlo; q < qhi; ++q) t += red[q][own_ch];
            blocksum[g][own_ch] = t;
          }
          __syncthreads();
        }
      }
      if (ph + 1 < NPH) __syncthreads();  // every thread is done with `stage` before the phase after next refills it
    }
    if (p.pooled) {
      const int ch = cg * DWT_CG + own_ch;
      if (ch < p.C) {
        for (int g = own_g0; g < p.G; g += GSTEP) {
          if (b0 + g < p.B) p.pooled[((size_t)rb * p.B + b0 + g) * p.C + ch] = blocksum[g][own_ch] * p.inv_hw;
        }
      }
    }
    __syncthreads();  // every thread is done with `stage` (the next iteration's TMA may overwrite it) and with blocksum
  }
}

template <typename T>
inline const char* dw_tma_launch(TmapCache& cache, const DwTmaPlan& plan, const void* in, void* out, const float* w, const float* bias,
                                 float* pooled, int B, int H, int W, int C, int pad_t, int pad_l, int act, int dil, cudaStream_t st) {
  const int Wq = (W + dil - 1) / dil;  // columns of the widest phase sub-grid (W when dil = 1)
  DwTmaParams p;
  p.out = out; p.w = w; p.bias = bias; p.pooled = pooled;
  p.B = B; p.H = H; p.W = W; p.C = C; p.pad_t = pad_t; p.pad_l = pad_l;
  p.G = plan.G; p.BH = plan.BH; p.n_rb = plan.n_rb;
  p.n_cg = (C + DWT_CG - 1) / DWT_CG;
  const int n_bg = (B + plan.G - 1) / plan.G;
  p.items = n_bg * p.n_rb * p.n_cg;
  p.strips_w = (Wq + DWT_OW - 1) / DWT_OW;
  p.bands = (plan.BH + DWT_RUN - 1) / DWT_RUN;
  p.nstrips = plan.G * p.bands * p.strips_w;
  p.stage_bytes = 128 * (Wq + 2) * (plan.BH + 2) * plan.G;
  p.inv_hw = 1.0f / (float)(H * W);
  // input box: 64 channels (128 bytes) x (Wq+2) x (BH+2) pixels (every dil-th of the map) x G crops, unswizzled (quarter-warps
  // read whole 128-byte pixel rows: conflict-free as is)
  const CUtensorMap* m = nullptr;
  const char* e = cache.get(&m, [&](CUtensorMap* c) {
    return make_tmap_nhwc<T>(c, in, B, H, W, C, DWT_CG, Wq + 2, plan.BH + 2, plan.G, dil, CU_TENSOR_MAP_SWIZZLE_NONE);
  }, in, B, H, W, C, plan.BH, plan.G, dil);
  if (e) return e;
  // + one pixel row of slack: the last strip of a ragged row may read (never use) a few pixels past the patch
  const int smem = DWT_STAGES * p.stage_bytes + 128 + 8 * 128;
  const int grid = std::min(p.items, 2 * num_sms());
  if (dil != 1) {  // the dilated stages of EfficientNetV2: SiLU only
    if (act != ACT_SILU) return "unsupported activation in dw3x3s1_dil_tma_kernel";
    return with_const<2, 4>(dil, "unsupported dilation in dw3x3s1_dil_tma_kernel", [&](auto d) {
      return launch_smem(dw3x3s1_dil_tma_kernel<T, d>, dim3(grid), dim3(DWT_THREADS), smem, st, m[0], p);
    });
  }
  return with_const<ACT_SILU, ACT_RELU, ACT_HSWISH>(act, "unsupported activation in dw3x3s1_tma_kernel", [&](auto a) {
    return launch_smem(dw3x3s1_tma_kernel<T, a>, dim3(grid), dim3(DWT_THREADS), smem, st, m[0], p);
  });
}

}  // namespace mtb
