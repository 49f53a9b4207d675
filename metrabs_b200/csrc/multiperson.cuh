// The callers either side of the crop model (SURVEY.md 8f), device-resident so that frames -> joints never leaves the GPU:
//
//   pyramid_kernel        gamma decoding + the 3-level box-filter pyramid   (multiperson_model.py:200, warping.py:9-13)
//   crop_setup_kernel     per box: undistorted box points, look-at rotation, box scale; per (aug, box): new intrinsics,
//                         R = rotflip[aug] @ R_noaug, inverse projection, pyramid level
//                                                                           (multiperson_model.py:264-293, 321-355; warping.py:20-21)
//   warp_crops_kernel     ALL num_aug x n_boxes crops in one launch: homography, 12-coefficient lens distortion, pyramid
//                         level select, bilinear gather with zero padding, antialias 1 / 2 / 4 supersampling, gamma
//                                                                           (warping.py:6-107, multiperson_model.py:295-319)
//   warp_crops_aa_kernel  the same render at antialias 5..16, shrunk by the antialiased bilinear resize per output tile
//                         without the render reaching global memory      (multiperson_model.py:311-314)
//   tta_merge_kernel      mirror joint swap, poses @ R, joint_transform_matrix, 2D projection with distortion and the
//                         image intrinsics, inverse extrinsics, skeleton gather, mean over augmentations
//                                                                           (multiperson_model.py:143-178, 246-259)
//   pose_filter_kernel    plausibility checks + pose-similarity NMS         (plausibility_check.py:8-119; the call site is
//                                                                            commented out in the PyTorch reference, :158-163)
//
// Crop order everywhere: flat index = aug * n_box + box  (reshape of [num_aug, n_box, ...], multiperson_model.py:236-239).
#pragma once
#include "common.cuh"
#include "decode.cuh"  // inv3x3 (fp64 closed form)

namespace mtb {

constexpr int MP_MAX_AUG = 16;
constexpr int MP_NDIST = 12;  // (k1, k2, p1, p2, k3, k4, k5, k6, s1, s2, s3, s4), warping.py:81-83

struct Dist12 {
  float d[MP_NDIST];
};

__device__ __forceinline__ Dist12 load_dist(const float* __restrict__ p, int ncoef) {
  Dist12 r;
#pragma unroll
  for (int i = 0; i < MP_NDIST; ++i) r.d[i] = i < ncoef ? p[i] : 0.f;  // pad_axis_to_size(..., 12)
  return r;
}
// distortion_formula_parts (warping.py:80-99)
__device__ __forceinline__ void dist_parts(float x, float y, const Dist12& k, float& a, float& b, float& cx, float& cy) {
  const float* d = k.d;
  const float r2 = x * x + y * y;
  a = (((d[4] * r2 + d[1]) * r2 + d[0]) * r2 + 1.f) / (((d[7] * r2 + d[6]) * r2 + d[5]) * r2 + 1.f);
  b = 2.f * (x * d[3] + y * d[2]);
  cx = (d[9] * r2 + d[3] + d[8]) * r2;
  cy = (d[11] * r2 + d[2] + d[10]) * r2;
}
// distort_points (warping.py:50-55); with all-zero coefficients a = 1, b = c = 0 and the point comes back bit-identical
__device__ __forceinline__ void distort_point(float& x, float& y, const Dist12& k) {
  float a, b, cx, cy;
  dist_parts(x, y, k, a, b, cx, cy);
  const float s = a + b;
  x = x * s + cx;
  y = y * s + cy;
}
// undistort_points (warping.py:58-66): five fixed-point iterations
__device__ __forceinline__ void undistort_point(float& x, float& y, const Dist12& k) {
  const float dx = x, dy = y;
  float ux = x, uy = y;
#pragma unroll 1
  for (int i = 0; i < 5; ++i) {
    float a, b, cx, cy;
    dist_parts(ux, uy, k, a, b, cx, cy);
    ux = (dx - cx - ux * b) / a;
    uy = (dy - cy - uy * b) / a;
  }
  x = ux;
  y = uy;
}
__device__ __forceinline__ void mat3_mul(const float* a, const float* b, float* o) {
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) o[r * 3 + c] = a[r * 3 + 0] * b[0 * 3 + c] + a[r * 3 + 1] * b[1 * 3 + c] + a[r * 3 + 2] * b[2 * 3 + c];
}

// ---------------------------------------------------------------------------------------------------- pyramid
// images u8 NCHW [N,3,H,W].  level 0 is never materialised (the warp kernel decodes u8 through the same 256-entry table);
// level 1 / 2 = avg_pool2d(2, 2) of the gamma-decoded image, floor sizes (odd last row / column dropped).
__global__ void __launch_bounds__(256) pyramid_level1_kernel(const uint8_t* __restrict__ img, float* __restrict__ l1, int planes, int H,
                                                             int W) {
  __shared__ float lut[256];
  lut[threadIdx.x] = powf((float)threadIdx.x / 255.f, 2.2f);  // (images.float() / 255) ** 2.2, multiperson_model.py:200
  __syncthreads();
  const int H1 = H >> 1, W1 = W >> 1;
  const size_t total = (size_t)planes * H1 * W1;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % W1), y = (int)((i / W1) % H1);
    const size_t pl = i / ((size_t)W1 * H1);
    const uint8_t* s = img + (pl * H + 2 * y) * (size_t)W + 2 * x;
    l1[i] = (lut[s[0]] + lut[s[1]] + lut[s[W]] + lut[s[W + 1]]) * 0.25f;
  }
}
__global__ void __launch_bounds__(256) pyramid_down_kernel(const float* __restrict__ src, float* __restrict__ dst, int planes, int H, int W) {
  const int H1 = H >> 1, W1 = W >> 1;
  const size_t total = (size_t)planes * H1 * W1;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % W1), y = (int)((i / W1) % H1);
    const size_t pl = i / ((size_t)W1 * H1);
    const float* s = src + (pl * H + 2 * y) * (size_t)W + 2 * x;
    dst[i] = (s[0] + s[1] + s[W] + s[W + 1]) * 0.25f;
  }
}

// ------------------------------------------------------------------------------------------------- crop setup
struct CropSetupParams {
  const float* boxes;       // [n, box_stride] (x, y, w, h, ...)
  int box_stride;
  const float* K;           // [n,3,3] intrinsics of the box's image
  const float* dist;        // [n, ncoef]
  int ncoef;
  const float* up;          // [n,3] world-up in camera space
  const float* rotflip;     // [A,3,3] aug_rotflipmat
  const float* aug_scales;  // [A]
  int n_box, num_aug, res, antialias;
  float* new_K;             // [A*n,3,3]
  float* R;                 // [A*n,3,3]
  float* invproj;           // [A*n,3,3]
  int* level;               // [A*n]
};

__global__ void __launch_bounds__(128) crop_setup_kernel(const CropSetupParams p) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= p.n_box) return;
  const float* bx = p.boxes + (size_t)b * p.box_stride;
  const float x = bx[0], y = bx[1], w = bx[2], h = bx[3];
  float K[9], Kinv[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) K[i] = p.K[(size_t)b * 9 + i];
  inv3x3(K, Kinv);
  const Dist12 dk = load_dist(p.dist + (size_t)b * p.ncoef, p.ncoef);
  // five box points: centre and the midpoints of the four sides (multiperson_model.py:323-330)
  const float px[5] = {x + w / 2, x + w / 2, x + w, x + w / 2, x};
  const float py[5] = {y + h / 2, y, y + h / 2, y + h, y + h / 2};
  float cam[5][3];
#pragma unroll
  for (int i = 0; i < 5; ++i) {
    // einsum('bpc,bCc->bpC', homog, inv(K)), then undistort the first two components and re-homogenise (:332-335)
    float cx = Kinv[0] * px[i] + Kinv[1] * py[i] + Kinv[2];
    float cy = Kinv[3] * px[i] + Kinv[4] * py[i] + Kinv[5];
    undistort_point(cx, cy, dk);
    cam[i][0] = cx; cam[i][1] = cy; cam[i][2] = 1.f;
  }
  // lookat_matrix(forward = box centre, up = camspace_up)  (ptu3d.py lookat_matrix)
  float R0[9];
  {
    const float* f = cam[0];
    const float fn = sqrtf(f[0] * f[0] + f[1] * f[1] + f[2] * f[2]);
    const float z0 = f[0] / fn, z1 = f[1] / fn, z2 = f[2] / fn;
    const float u0 = p.up[(size_t)b * 3 + 0], u1 = p.up[(size_t)b * 3 + 1], u2 = p.up[(size_t)b * 3 + 2];
    float x0 = z1 * u2 - z2 * u1, x1 = z2 * u0 - z0 * u2, x2 = z0 * u1 - z1 * u0;
    float xn = sqrtf(x0 * x0 + x1 * x1 + x2 * x2);
    if (xn == 0.f) {  // look direction parallel to up: rotate the new Z around the old Y by 90 degrees
      x0 = z2; x1 = 0.f; x2 = -z0;
      xn = sqrtf(x0 * x0 + x1 * x1 + x2 * x2);
    }
    x0 /= xn; x1 /= xn; x2 /= xn;
    const float y0 = z1 * x2 - z2 * x1, y1 = z2 * x0 - z0 * x2, y2 = z0 * x1 - z1 * x0;
    R0[0] = x0; R0[1] = x1; R0[2] = x2; R0[3] = y0; R0[4] = y1; R0[5] = y2; R0[6] = z0; R0[7] = z1; R0[8] = z2;
  }
  // side midpoints in the new frame: project((K @ R_noaug) p)  (:342-345), box size = larger extent (:349-351)
  float M[9];
  mat3_mul(K, R0, M);
  float sx[4], sy[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float* q = cam[i + 1];
    const float a = M[0] * q[0] + M[1] * q[1] + M[2] * q[2];
    const float bq = M[3] * q[0] + M[4] * q[1] + M[5] * q[2];
    const float c = M[6] * q[0] + M[7] * q[1] + M[8] * q[2];
    sx[i] = a / c;
    sy[i] = bq / c;
  }
  const float vert = sqrtf((sx[0] - sx[2]) * (sx[0] - sx[2]) + (sy[0] - sy[2]) * (sy[0] - sy[2]));
  const float horiz = sqrtf((sx[1] - sx[3]) * (sx[1] - sx[3]) + (sy[1] - sy[3]) * (sy[1] - sy[3]));
  const float box_scale = (float)p.res / fmaxf(vert, horiz);
  for (int a = 0; a < p.num_aug; ++a) {
    const float cs = p.aug_scales[a] * box_scale;  // crop_scales (:271)
    const size_t o = ((size_t)a * p.n_box + b) * 9;
    float nK[9] = {K[0] * cs, K[1] * cs, (float)p.res / 2, K[3] * cs, K[4] * cs, (float)p.res / 2, 0.f, 0.f, 1.f};  // (:276-286)
    float R[9], PM[9], inv[9];
    mat3_mul(p.rotflip + (size_t)a * 9, R0, R);  // R = aug_rotflipmat[:, None] @ R_noaug (:287)
    mat3_mul(nK, R, PM);
    inv3x3(PM, inv);                              // new_invprojmat (:288)
    if (p.antialias > 1) {                        // @ corner_aligned_scale_mat(1 / antialias_factor) (:292-295, warping.py:121-127)
      const float fct = 1.f / (float)p.antialias, sh = (fct - 1.f) / 2.f;
      const float S[9] = {fct, 0.f, sh, 0.f, fct, sh, 0.f, 0.f, 1.f};
      float t[9];
      mat3_mul(inv, S, t);
#pragma unroll
      for (int i = 0; i < 9; ++i) inv[i] = t[i];
    }
#pragma unroll
    for (int i = 0; i < 9; ++i) {
      p.new_K[o + i] = nK[i];
      p.R[o + i] = R[i];
      p.invproj[o + i] = inv[i];
    }
    // pyramid level: clip(floor(-log2(crop_scale * antialias)), 0, 2)  (warping.py:20-21, multiperson_model.py:303)
    float lv = floorf(-log2f(cs * (float)p.antialias));
    lv = fminf(fmaxf(lv, 0.f), 2.f);
    p.level[(size_t)a * p.n_box + b] = (int)lv;
  }
}

// ------------------------------------------------------------------------------------------------------- warp
struct WarpParams {
  const uint8_t* img;   // [N,3,H,W] u8
  const float* l1;      // [N,3,H/2,W/2] gamma-decoded
  const float* l2;      // [N,3,H/4,W/4]
  int N, H, W;
  const float* K;       // [n,3,3] per box
  const float* dist;    // [n,ncoef]
  int ncoef;
  const int* image_ids; // [n]
  const float* invproj; // [A*n,3,3]
  const int* level;     // [A*n]
  const float* gamma_exp;  // [A] = aug_gammas / 2.2
  int n_box, num_aug, res, antialias;
  float* crops;         // [A*n,3,res,res]
};

template <typename T, bool LUT>
__device__ __forceinline__ float tap(const T* __restrict__ plane, int W, int xi, int yi, int Wl, int Hl, const float* lut) {
  if (xi < 0 || yi < 0 || xi >= Wl || yi >= Hl) return 0.f;  // padding_mode='zeros'
  if constexpr (LUT) return lut[plane[(size_t)yi * W + xi]];
  else return (float)plane[(size_t)yi * W + xi];
}

// Block-wide (256 threads): the decode table into `lut`; into `sp` the inverse projection (9), the level intrinsics (6)
// and the distortion (12) of crop `crop` (box b); then a barrier.  -> the crop's pyramid level.  The kernels derive the
// level image themselves: returning it from here as well changes the code ptxas generates for warp_crops_kernel.
__device__ __forceinline__ int warp_load_crop(const WarpParams& p, int crop, int b, float* lut, float* sp) {
  lut[threadIdx.x] = powf((float)threadIdx.x / 255.f, 2.2f);
  const int lv = p.level[crop];
  if (threadIdx.x < 9) sp[threadIdx.x] = p.invproj[(size_t)crop * 9 + threadIdx.x];
  if (threadIdx.x >= 32 && threadIdx.x < 38) {
    // intrinsic_matrix_levels = corner_aligned_scale_mat(1 / 2**level) @ K (warping.py:15-17): rows 0/1 scaled, shift added
    const int i = threadIdx.x - 32, r = i / 3, c = i - r * 3;
    const float f = 1.f / (float)(1 << lv), sh = (f - 1.f) / 2.f;
    sp[9 + i] = f * p.K[(size_t)b * 9 + r * 3 + c] + sh * p.K[(size_t)b * 9 + 6 + c];
  }
  if (threadIdx.x >= 64 && threadIdx.x < 64 + MP_NDIST) {
    const int i = threadIdx.x - 64;
    sp[15 + i] = i < p.ncoef ? p.dist[(size_t)b * p.ncoef + i] : 0.f;
  }
  __syncthreads();
  return lv;
}

// Sample (nx, ny) of the crop's render grid: adds the bilinear blend of each channel to acc, nothing when all four taps
// are outside the level image.
__device__ __forceinline__ void warp_sample(const float* sp, const Dist12& dk, int lv, int Wl, int Hl, size_t plane_sz,
                                            const uint8_t* im0, const float* imf, const float* lut, float nx, float ny, float acc[3]) {
  // old = invproj @ (x, y, 1); project; distort; K_level @ (q, 1)   (warping.py:41-47)
  const float hx = sp[0] * nx + sp[1] * ny + sp[2];
  const float hy = sp[3] * nx + sp[4] * ny + sp[5];
  const float hz = sp[6] * nx + sp[7] * ny + sp[8];
  float qx = hx / hz, qy = hy / hz;
  distort_point(qx, qy, dk);
  const float u = sp[9] * qx + sp[10] * qy + sp[11];
  const float v = sp[12] * qx + sp[13] * qy + sp[14];
  // grid_sample(align_corners=True, bilinear, zeros) on coordinates normalised by (size - 1) (warping.py:48-52)
  const float gx = ((u / (float)(Wl - 1) * 2.f - 1.f) + 1.f) * 0.5f * (float)(Wl - 1);
  const float gy = ((v / (float)(Hl - 1) * 2.f - 1.f) + 1.f) * 0.5f * (float)(Hl - 1);
  if (!(gx > -1.f && gx < (float)Wl && gy > -1.f && gy < (float)Hl)) return;  // all four taps outside (also NaN)
  const float fx0 = floorf(gx), fy0 = floorf(gy);
  const int x0 = (int)fx0, y0 = (int)fy0;
  const float wx1 = gx - fx0, wx0 = (fx0 + 1.f) - gx, wy1 = gy - fy0, wy0 = (fy0 + 1.f) - gy;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float v00, v01, v10, v11;
    if (lv == 0) {
      const uint8_t* pl = im0 + (size_t)c * plane_sz;
      v00 = tap<uint8_t, true>(pl, Wl, x0, y0, Wl, Hl, lut);
      v01 = tap<uint8_t, true>(pl, Wl, x0 + 1, y0, Wl, Hl, lut);
      v10 = tap<uint8_t, true>(pl, Wl, x0, y0 + 1, Wl, Hl, lut);
      v11 = tap<uint8_t, true>(pl, Wl, x0 + 1, y0 + 1, Wl, Hl, lut);
    } else {
      const float* pl = imf + (size_t)c * plane_sz;
      v00 = tap<float, false>(pl, Wl, x0, y0, Wl, Hl, nullptr);
      v01 = tap<float, false>(pl, Wl, x0 + 1, y0, Wl, Hl, nullptr);
      v10 = tap<float, false>(pl, Wl, x0, y0 + 1, Wl, Hl, nullptr);
      v11 = tap<float, false>(pl, Wl, x0 + 1, y0 + 1, Wl, Hl, nullptr);
    }
    acc[c] += v00 * (wx0 * wy0) + v01 * (wx1 * wy0) + v10 * (wx0 * wy1) + v11 * (wx1 * wy1);
  }
}

// antialias 1, 2 and 4: the af x af supersamples of each output pixel, averaged (the reference's avg_pool2d(af))
__global__ void __launch_bounds__(256) warp_crops_kernel(const WarpParams p) {
  __shared__ float lut[256];
  __shared__ float sp[9 + 6 + MP_NDIST];
  const int crop = blockIdx.y;
  const int a = crop / p.n_box, b = crop - a * p.n_box;
  const int lv = warp_load_crop(p, crop, b, lut, sp);
  Dist12 dk;
#pragma unroll
  for (int i = 0; i < MP_NDIST; ++i) dk.d[i] = sp[15 + i];
  const int Hl = p.H >> lv, Wl = p.W >> lv;
  const int img_id = p.image_ids[b];
  const size_t plane_sz = (size_t)Hl * Wl;
  const uint8_t* im0 = p.img + (size_t)img_id * 3 * plane_sz;
  const float* imf = (lv == 1 ? p.l1 : p.l2) + (size_t)img_id * 3 * plane_sz;
  const float gexp = p.gamma_exp[a];
  const int af = p.antialias;
  const float inv_n = 1.f / (float)(af * af);
  const int npix = p.res * p.res;
  for (int pix = blockIdx.x * blockDim.x + threadIdx.x; pix < npix; pix += gridDim.x * blockDim.x) {
    const int oy = pix / p.res, ox = pix - oy * p.res;
    float acc[3] = {0.f, 0.f, 0.f};
    for (int sy = 0; sy < af; ++sy)
      for (int sx = 0; sx < af; ++sx)
        warp_sample(sp, dk, lv, Wl, Hl, plane_sz, im0, imf, lut, (float)(ox * af + sx), (float)(oy * af + sy), acc);
    float* o = p.crops + (size_t)crop * 3 * npix + pix;
#pragma unroll
    for (int c = 0; c < 3; ++c) o[(size_t)c * npix] = powf(acc[c] * inv_n, gexp);  // crops **= aug_gammas / 2.2 (:318)
  }
}

// ------------------------------------------------------------------------------------------ warp, antialias 5..16
// The reference renders res*f and shrinks it with torchvision's resize(BILINEAR, antialias=True) (multiperson_model.py:
// 311-314), i.e. F.interpolate(bilinear, align_corners=False, antialias=True): per axis, output i takes the render taps
// j in [lo, lo + n) around center f (i + 0.5) with weight max(0, 1 - |j - center + 0.5| / f), clipped to the render and
// renormalised over the taps that remain; the width pass runs first, then the height pass (ATen's separable CPU kernel).
// One CTA per (crop, AA_TILE x AA_TILE output tile): it computes each supersample of the tile's footprint once, in chunks
// of rows held in shared memory, reduces every chunk row by the width pass into a strip of [rows][AA_TILE][3], then runs
// the height pass and the gamma.  Sums run in ascending tap order without atomics: a crop's output does not depend on
// the launch it is part of.
constexpr int AA_TILE = 8;
constexpr int AA_MAX_F = 16;
constexpr int AA_SPAN = (AA_TILE + 1) * AA_MAX_F;  // footprint of a tile, supersamples per axis, at most
constexpr int AA_TAPS = 2 * AA_MAX_F;               // taps per output and axis, at most
constexpr int AA_RAW = 2304;                        // supersamples per row chunk: 16 rows of the widest footprint

// Taps [lo, lo + n) of output i (ATen's _compute_weights_aa, scale and support f, no align-corners shift)
__device__ __forceinline__ void aa_range(int i, int f, int n_in, int& lo, int& n) {
  const float center = (float)f * ((float)i + 0.5f);
  lo = max((int)(center - (float)f + 0.5f), 0);
  n = min((int)(center + (float)f + 0.5f), n_in) - lo;
}

// The renormalised fp32 weights of output i, in ATen's operations: |t| * fl(1 / f), 1 - x, the running total, w / total
__device__ __forceinline__ void aa_weights(int i, int f, int n_in, float* w, int* range) {
  int lo, n;
  aa_range(i, f, n_in, lo, n);
  const float center = (float)f * ((float)i + 0.5f), invscale = 1.f / (float)f;
  float total = 0.f;
  for (int j = 0; j < n; ++j) {
    const float x = fabsf(((float)(j + lo) - center + 0.5f) * invscale);
    w[j] = x < 1.f ? 1.f - x : 0.f;
    total += w[j];
  }
  for (int j = 0; j < n; ++j) w[j] /= total;  // the tap nearest the center has weight >= 1/2
  range[0] = lo;
  range[1] = n;
}

__global__ void __launch_bounds__(256) warp_crops_aa_kernel(const WarpParams p) {
  __shared__ float lut[256];
  __shared__ float sp[9 + 6 + MP_NDIST];
  __shared__ float raw[3][AA_RAW];                 // one chunk of footprint rows, per channel
  __shared__ float strip[AA_SPAN][AA_TILE][3];     // width-pass output of every footprint row
  __shared__ float wx[AA_TILE][AA_TAPS + 1], wy[AA_TILE][AA_TAPS + 1];
  __shared__ int rx[AA_TILE][2], ry[AA_TILE][2];
  const int crop = blockIdx.y;
  const int a = crop / p.n_box, b = crop - a * p.n_box;
  const int f = p.antialias, n_in = p.res * f;
  const int tiles_x = (p.res + AA_TILE - 1) / AA_TILE;
  const int ty = blockIdx.x / tiles_x, tx = blockIdx.x - ty * tiles_x;
  const int ox0 = tx * AA_TILE, oy0 = ty * AA_TILE;
  const int nox = min(AA_TILE, p.res - ox0), noy = min(AA_TILE, p.res - oy0);
  const int t = threadIdx.x;
  if (t >= 128 && t < 128 + nox) aa_weights(ox0 + t - 128, f, n_in, wx[t - 128], rx[t - 128]);
  if (t >= 160 && t < 160 + noy) aa_weights(oy0 + t - 160, f, n_in, wy[t - 160], ry[t - 160]);
  const int lv = warp_load_crop(p, crop, b, lut, sp);  // its barrier also publishes the weights
  Dist12 dk;
#pragma unroll
  for (int i = 0; i < MP_NDIST; ++i) dk.d[i] = sp[15 + i];
  const int Hl = p.H >> lv, Wl = p.W >> lv;
  const int img_id = p.image_ids[b];
  const size_t plane_sz = (size_t)Hl * Wl;
  const uint8_t* im0 = p.img + (size_t)img_id * 3 * plane_sz;
  const float* imf = (lv == 1 ? p.l1 : p.l2) + (size_t)img_id * 3 * plane_sz;
  const int x_lo = rx[0][0], nx = rx[nox - 1][0] + rx[nox - 1][1] - x_lo;  // the tile's footprint
  const int y_lo = ry[0][0], ny = ry[noy - 1][0] + ry[noy - 1][1] - y_lo;
  const int chunk = AA_RAW / nx;
  for (int r0 = 0; r0 < ny; r0 += chunk) {
    const int nr = min(chunk, ny - r0);
    for (int k = t; k < nr * nx; k += blockDim.x) {
      const int r = k / nx, x = k - r * nx;
      float acc[3] = {0.f, 0.f, 0.f};
      warp_sample(sp, dk, lv, Wl, Hl, plane_sz, im0, imf, lut, (float)(x_lo + x), (float)(y_lo + r0 + r), acc);
      raw[0][k] = acc[0];
      raw[1][k] = acc[1];
      raw[2][k] = acc[2];
    }
    __syncthreads();
    for (int k = t; k < nr * AA_TILE * 3; k += blockDim.x) {  // width pass: (row, channel, output column)
      const int ox = k % AA_TILE, c = (k / AA_TILE) % 3, r = k / (AA_TILE * 3);
      if (ox >= nox) continue;
      const float* row = raw[c] + r * nx + (rx[ox][0] - x_lo);
      const float* w = wx[ox];
      float s = 0.f;
      for (int j = 0; j < rx[ox][1]; ++j) s += row[j] * w[j];
      strip[r0 + r][ox][c] = s;
    }
    __syncthreads();
  }
  const float gexp = p.gamma_exp[a];
  const int npix = p.res * p.res;
  for (int k = t; k < AA_TILE * AA_TILE * 3; k += blockDim.x) {  // height pass and gamma: (channel, row, column)
    const int ox = k % AA_TILE, oy = (k / AA_TILE) % AA_TILE, c = k / (AA_TILE * AA_TILE);
    if (ox >= nox || oy >= noy) continue;
    const int lo = ry[oy][0] - y_lo;
    const float* w = wy[oy];
    float s = 0.f;
    for (int j = 0; j < ry[oy][1]; ++j) s += strip[lo + j][ox][c] * w[j];
    p.crops[(size_t)crop * 3 * npix + (size_t)c * npix + (size_t)(oy0 + oy) * p.res + ox0 + ox] = powf(s, gexp);  // (:318)
  }
}

// -------------------------------------------------------------------------------------------------- TTA merge
struct TtaParams {
  const float* poses;       // [A*n, J, 3] crop-model output (camera space of each crop)
  const float* R;           // [A*n,3,3]
  const uint8_t* flip;      // [A] aug_should_flip
  const int* mirror;        // [J] joint_info.mirror_mapping
  const float* jt;          // [J, J2] joint_transform_matrix or nullptr (J2 = J)
  const int* skel;          // [Js] skeleton joint indices into J2 (nullptr: identity, Js = J2)
  const float* K;           // [n,3,3]
  const float* dist;        // [n,ncoef]
  int ncoef;
  const float* ext_inv;     // [n,4,4] inverse extrinsics of the box's image (row-major)
  int n_box, num_aug, J, J2, Js, average;
  float* poses3d;           // [n, (A,) Js, 3] world space
  float* poses2d;           // [n, (A,) Js, 2] image pixels
};

// one thread per (box, output joint): loops over the augmentations in index order (deterministic mean)
__global__ void __launch_bounds__(128) tta_merge_kernel(const TtaParams p) {
  const int b = blockIdx.x;
  const Dist12 dk = load_dist(p.dist + (size_t)b * p.ncoef, p.ncoef);
  const float* K = p.K + (size_t)b * 9;
  const float* E = p.ext_inv + (size_t)b * 16;
  for (int js = threadIdx.x; js < p.Js; js += blockDim.x) {
    const int N = p.skel ? p.skel[js] : js;
    float s3[3] = {0.f, 0.f, 0.f}, s2[2] = {0.f, 0.f};
    for (int a = 0; a < p.num_aug; ++a) {
      const size_t crop = (size_t)a * p.n_box + b;
      const float* R = p.R + crop * 9;
      const float* P = p.poses + crop * p.J * 3;
      const bool fl = p.flip[a] != 0;
      // poses (mirror-swapped) @ R, then einsum('bank,nN->baNk') with the joint transform  (:246-256, :146-148)
      float c0 = 0.f, c1 = 0.f, c2 = 0.f;
      if (p.jt) {
        for (int n = 0; n < p.J; ++n) {
          const float t = p.jt[(size_t)n * p.J2 + N];
          if (t == 0.f) continue;
          const float* q = P + (size_t)(fl ? p.mirror[n] : n) * 3;
          c0 += (q[0] * R[0] + q[1] * R[3] + q[2] * R[6]) * t;
          c1 += (q[0] * R[1] + q[1] * R[4] + q[2] * R[7]) * t;
          c2 += (q[0] * R[2] + q[1] * R[5] + q[2] * R[8]) * t;
        }
      } else {
        const float* q = P + (size_t)(fl ? p.mirror[N] : N) * 3;
        c0 = q[0] * R[0] + q[1] * R[3] + q[2] * R[6];
        c1 = q[0] * R[1] + q[1] * R[4] + q[2] * R[7];
        c2 = q[0] * R[2] + q[1] * R[5] + q[2] * R[8];
      }
      // poses2d = [distort(project(pose)), 1] @ K[:2,:]^T  (:151-155)
      float qx = c0 / c2, qy = c1 / c2;
      distort_point(qx, qy, dk);
      const float u = qx * K[0] + qy * K[1] + K[2];
      const float v = qx * K[3] + qy * K[4] + K[5];
      // world = [pose, 1] @ inv(extrinsic)[:3,:]^T  (:170-174)
      const float w0 = c0 * E[0] + c1 * E[1] + c2 * E[2] + E[3];
      const float w1 = c0 * E[4] + c1 * E[5] + c2 * E[6] + E[7];
      const float w2 = c0 * E[8] + c1 * E[9] + c2 * E[10] + E[11];
      if (p.average) {
        s3[0] += w0; s3[1] += w1; s3[2] += w2; s2[0] += u; s2[1] += v;
      } else {
        float* o3 = p.poses3d + (((size_t)b * p.num_aug + a) * p.Js + js) * 3;
        float* o2 = p.poses2d + (((size_t)b * p.num_aug + a) * p.Js + js) * 2;
        o3[0] = w0; o3[1] = w1; o3[2] = w2; o2[0] = u; o2[1] = v;
      }
    }
    if (p.average) {
      const float inv = 1.f / (float)p.num_aug;  // torch.mean over the augmentation axis (:180-182)
      float* o3 = p.poses3d + ((size_t)b * p.Js + js) * 3;
      float* o2 = p.poses2d + ((size_t)b * p.Js + js) * 2;
      o3[0] = s3[0] * inv; o3[1] = s3[1] * inv; o3[2] = s3[2] * inv;
      o2[0] = s2[0] * inv; o2[1] = s2[1] * inv;
    }
  }
}

// ------------------------------------------------------------------------------------------ plausibility + NMS
struct FilterParams {
  const float* poses3d;     // [n, A, J, 3] camera-space poses of every augmentation
  const float* poses2d;     // [n, A, J, 2]
  const float* boxes;       // [n, box_stride] (x, y, w, h, score)
  int box_stride;
  const int* bones;         // [nb, 2] joint index pairs (joint2bone_mat rows)
  const float* mean_bones;  // [nb]
  int n_bones;
  const int* image_start;   // [n_images + 1] box ranges per image
  int num_aug, J;
  uint8_t* plausible;       // [n] out: the three plausibility checks
  uint8_t* keep;            // [n] out: plausible AND surviving the pose NMS
  float* scratch;           // [n, J, 3] mean-over-aug poses
  int max_boxes;            // bound on every image's box count: sizes the dynamic shared memory
};
// dynamic shared memory of pose_filter_kernel per box of the largest image: score, sqscale, order, valid, supp
constexpr int MP_FILTER_SMEM_PER_BOX = 4 + 4 + 4 + 1 + 1;
constexpr int FILTER_THREADS = 128;

// one CTA per image.  Phase 1 (thread per box): the three checks.  Phase 2: pose similarity on demand + greedy NMS.
__global__ void __launch_bounds__(FILTER_THREADS) pose_filter_kernel(const FilterParams p) {
  __shared__ float sq_all[MP_MAX_AUG * FILTER_THREADS];
  extern __shared__ __align__(16) unsigned char filter_smem[];
  float* score = reinterpret_cast<float*>(filter_smem);
  float* sqscale = score + p.max_boxes;
  int* order = reinterpret_cast<int*>(sqscale + p.max_boxes);
  uint8_t* valid = reinterpret_cast<uint8_t*>(order + p.max_boxes);
  uint8_t* supp = valid + p.max_boxes;
  const int b0 = p.image_start[blockIdx.x], b1 = p.image_start[blockIdx.x + 1];
  const int n = b1 - b0;  // <= max_boxes
  const int J = p.J, A = p.num_aug;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int b = b0 + i;
    const float* P3 = p.poses3d + (size_t)b * A * J * 3;
    const float* P2 = p.poses2d + (size_t)b * A * J * 2;
    float* mean3 = p.scratch + (size_t)b * J * 3;
    // mean over augmentations
    float bx0 = INFINITY, by0 = INFINITY, bx1 = -INFINITY, by1 = -INFINITY;
    float ss = 0.f;
    for (int j = 0; j < J; ++j) {
      float m0 = 0.f, m1 = 0.f, m2 = 0.f, u = 0.f, v = 0.f;
      for (int a = 0; a < A; ++a) {
        const float* q = P3 + ((size_t)a * J + j) * 3;
        m0 += q[0]; m1 += q[1]; m2 += q[2];
        u += P2[((size_t)a * J + j) * 2];
        v += P2[((size_t)a * J + j) * 2 + 1];
      }
      m0 /= A; m1 /= A; m2 /= A; u /= A; v /= A;
      mean3[j * 3] = m0; mean3[j * 3 + 1] = m1; mean3[j * 3 + 2] = m2;
      ss += m0 * m0 + m1 * m1 + m2 * m2;
      bx0 = fminf(bx0, u); by0 = fminf(by0, v); bx1 = fmaxf(bx1, u); by1 = fmaxf(by1, v);
    }
    sqscale[i] = ss / (float)(J * 3);
    // is_pose_plausible (plausibility_check.py:8-28): any bone both relatively (<0.1x or >3x) and absolutely (>300 mm) off
    bool implausible = false;
    for (int k = 0; k < p.n_bones; ++k) {
      const float* q0 = mean3 + p.bones[2 * k] * 3;
      const float* q1 = mean3 + p.bones[2 * k + 1] * 3;
      const float len = sqrtf((q0[0] - q1[0]) * (q0[0] - q1[0]) + (q0[1] - q1[1]) * (q0[1] - q1[1]) + (q0[2] - q1[2]) * (q0[2] - q1[2]));
      const float rel = len / p.mean_bones[k], ad = fabsf(len - p.mean_bones[k]);
      implausible |= (rel > 3.f || rel < 0.1f) && ad > 300.f;
    }
    // are_augmentation_results_consistent (:63-67): scale-align the A poses, per-joint stdev over augmentations (unbiased
    // variance, summed over xyz), more than J//4 joints under 200 mm
    // per-augmentation square scales in shared memory, not a local array: a stack frame makes ptxas spill around the
    // IEEE division / square-root calls
    float* sq = sq_all + threadIdx.x;  // sq[a * FILTER_THREADS]
    float msq = 0.f;
    for (int a = 0; a < A; ++a) {
      float s = 0.f;
      for (int j = 0; j < J * 3; ++j) s += P3[(size_t)a * J * 3 + j] * P3[(size_t)a * J * 3 + j];
      sq[a * FILTER_THREADS] = s / (float)(J * 3);
      msq += sq[a * FILTER_THREADS];
    }
    msq /= A;
    int n_stable = 0;
    for (int j = 0; j < J; ++j) {
      float var = 0.f;
      for (int c = 0; c < 3; ++c) {
        float m = 0.f;
        for (int a = 0; a < A; ++a) m += P3[((size_t)a * J + j) * 3 + c] * sqrtf(msq / sq[a * FILTER_THREADS]);
        m /= A;
        float vs = 0.f;
        for (int a = 0; a < A; ++a) {
          const float d = P3[((size_t)a * J + j) * 3 + c] * sqrtf(msq / sq[a * FILTER_THREADS]) - m;
          vs += d * d;
        }
        var += vs / (float)(A - 1);  // torch.var default: unbiased
      }
      n_stable += sqrtf(var) < 200.f ? 1 : 0;
    }
    const bool consistent = n_stable > J / 4;
    // is_pose_consistent_with_box (:88-106): intersection(pose box, detection) > half the detection area
    const float* bx = p.boxes + (size_t)b * p.box_stride;
    const float ix0 = fmaxf(bx[0], bx0), iy0 = fmaxf(bx[1], by0);
    const float ix1 = fminf(bx[0] + bx[2], bx1), iy1 = fminf(bx[1] + bx[3], by1);
    const float inter = fmaxf(ix1 - ix0, 0.f) * fmaxf(iy1 - iy0, 0.f);
    const bool in_box = inter > 0.5f * (bx[2] * bx[3]);
    const bool ok = !implausible && consistent && in_box;
    valid[i] = ok ? 1 : 0;
    supp[i] = 0;
    score[i] = bx[4];
    p.plausible[b] = ok ? 1 : 0;
  }
  __syncthreads();
  // stable descending order by score among the valid poses (rank by counting)
  __shared__ int n_valid_s;
  if (threadIdx.x == 0) n_valid_s = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    if (!valid[i]) continue;
    int rank = 0;
    for (int k = 0; k < n; ++k)
      if (valid[k] && (score[k] > score[i] || (score[k] == score[i] && k < i))) ++rank;
    order[rank] = i;
    atomicAdd(&n_valid_s, 1);
  }
  __syncthreads();
  const int nv = n_valid_s;
  const int kq = J / 4;  // topk(dists, k = J // 4): the k LARGEST per-joint distances (torch.topk default)
  // greedy NMS (non_max_suppression_overlaps :31-53): for each unsuppressed i in order, suppress later j with sim > 0.4.
  for (int oi = 0; oi < nv; ++oi) {
    const int i = order[oi];
    if (supp[i]) { __syncthreads(); continue; }  // block-uniform: supp[] is only written between barriers
    const float* Pi = p.scratch + (size_t)(b0 + i) * J * 3;
    for (int oj = oi + 1 + (int)threadIdx.x; oj < nv; oj += blockDim.x) {
      const int j = order[oj];
      if (supp[j]) continue;
      const float* Pj = p.scratch + (size_t)(b0 + j) * J * 3;
      // compute_pose_similarity (:70-85): pairwise scale alignment, per-joint distances, mean of relu(1 - d/300) over the
      // k largest distances
      const float ms = (sqscale[i] + sqscale[j]) * 0.5f;
      const float fi = sqrtf(ms / sqscale[i]), fj = sqrtf(ms / sqscale[j]);
      // k largest of J values without a buffer: repeated selection (J <= 122, k <= 30)
      float acc = 0.f, last = INFINITY;
      int last_idx = -1;
      for (int t = 0; t < kq; ++t) {
        float best = -1.f;
        int best_idx = -1;
        for (int jj = 0; jj < J; ++jj) {
          const float d0 = fi * Pi[jj * 3] - fj * Pj[jj * 3], d1 = fi * Pi[jj * 3 + 1] - fj * Pj[jj * 3 + 1],
                      d2 = fi * Pi[jj * 3 + 2] - fj * Pj[jj * 3 + 2];
          const float d = sqrtf(d0 * d0 + d1 * d1 + d2 * d2);
          // strictly after (last, last_idx) in the (value desc, index asc) order
          const bool after = d < last || (d == last && jj > last_idx);
          if (after && (d > best || best_idx < 0)) { best = d; best_idx = jj; }
        }
        acc += fmaxf(1.f - best / 300.f, 0.f);
        last = best;
        last_idx = best_idx;
      }
      if (kq > 0 && acc / (float)kq > 0.4f) supp[j] = 1;
    }
    __syncthreads();
  }
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) p.keep[b0 + i] = (valid[i] && !supp[i]) ? 1 : 0;
}

}  // namespace mtb
