/*
 * metrabs_b200.h - C ABI of libmetrabs_b200.so: the H100 (sm_90a) implementation of the MeTRAbs per-crop
 * inference hot path   crops -> CNN backbone -> 1x1-conv head -> 2D + volumetric soft-argmax -> metric scaling
 * -> reconstruct_absolute -> joints [B,J,3].
 *
 * The reference (isarandi/metrabs) is pure Python and has no FFI; its boundary for this path is the nn.Module
 * contract consumed at metrabs_pytorch/multiperson/multiperson_model.py:240-242.  Each entry point below names
 * the reference function it replaces (file:line relative to /root/reference/metrabs_pytorch/).  INTEGRATION.md
 * shows the ctypes binding a maintainer would add on the reference side.
 *
 * Conventions: plain C, raw pointers + sizes, no torch types.  Unless a function says "host", pointers are
 * DEVICE pointers on the handle's device and work is enqueued on `stream` (a cudaStream_t passed as void*;
 * NULL = legacy default stream) without synchronising the host and without allocating: the caller owns inputs,
 * outputs and the workspace; the library owns only its weight arena.  Every function returns 0 (MTB_OK) or a
 * negative mtb_status; mtb_last_error() gives the message of the last failure on that handle (or the global
 * one when the handle is NULL).  A handle is bound to one device and is not re-entrant; distinct handles are
 * independent (one process per GPU drives one handle).
 */
#ifndef METRABS_B200_H_
#define METRABS_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MTB_ABI_VERSION 2

typedef enum {
  MTB_OK = 0,
  MTB_ERR_INVALID_ARG = -1,
  MTB_ERR_CUDA = -2,
  MTB_ERR_NOT_FINALIZED = -3,
  MTB_ERR_MISSING_WEIGHT = -4,
  MTB_ERR_WORKSPACE = -5,
  MTB_ERR_UNSUPPORTED = -6,
  MTB_ERR_NCCL = -7
} mtb_status;

typedef enum { MTB_DTYPE_F32 = 0, MTB_DTYPE_BF16 = 1, MTB_DTYPE_F16 = 2, MTB_DTYPE_I64 = 3 } mtb_dtype;

/* Backbone families.  EFFNET covers EfficientNetV2-S/M/L, EfficientNet-B5/B6/B7 and any table in the same block grammar
 * (backbones/efficientnet.py:379-433) with BatchNorm epsilon 1e-3; EFFNET_EPS1E5 is the same grammar with torchvision's
 * default epsilon 1e-5, for EfficientNet-B0..B4 (:753-960), and takes MBConv rows only (kernel 3 or 5, stride 1 or 2;
 * anything else fails with MTB_ERR_UNSUPPORTED); the RESNET* values (V1, metrabs_tf/backbones/resnet.py: ResNet-18/34 with the
 * basic block :322-388, ResNet-50/101/152 with the bottleneck :239-319), the RESNET*V2 values (the pre-activation
 * ResNet-50/101/152, ResNetUnifiedV2 :710-745 with block2_dense :391-456, output strides 8, 16 and 32), the RESNET*V1_5 values
 * (ResNetUnified(v1_5=True) :621-666: the V1 bottleneck nets with block 1's stride on the 3x3 _2_conv, dilated by dil_in of
 * its stack, and torch_preproc (x - mean) / std, builder.py:99-103; output strides 8, 16 and 32) and MOBILENETV3_SMALL /
 * _LARGE (metrabs_tf/backbones/mobilenet_v3.py:348-384 / :387-428, alpha 1; the _MINI values are the minimalistic=True
 * form, :250-257: 3x3 depthwise kernels, ReLU everywhere, no squeeze-excitation) follow the TF-only
 * metrabs_tf/backbones/{resnet,mobilenet_v3}.py. */
typedef enum { MTB_ARCH_EFFNET = 0, MTB_ARCH_RESNET50 = 1, MTB_ARCH_MOBILENETV3_SMALL = 2,
               MTB_ARCH_HEAD_ONLY = 3, MTB_ARCH_RESNET18 = 4, MTB_ARCH_RESNET34 = 5, MTB_ARCH_RESNET101 = 6,
               MTB_ARCH_RESNET152 = 7, MTB_ARCH_MOBILENETV3_LARGE = 8, MTB_ARCH_EFFNET_EPS1E5 = 9,
               MTB_ARCH_RESNET50V2 = 10, MTB_ARCH_RESNET101V2 = 11, MTB_ARCH_RESNET152V2 = 12,
               MTB_ARCH_RESNET50V1_5 = 13, MTB_ARCH_RESNET101V1_5 = 14, MTB_ARCH_RESNET152V1_5 = 15,
               MTB_ARCH_MOBILENETV3_SMALL_MINI = 16, MTB_ARCH_MOBILENETV3_LARGE_MINI = 17 } mtb_arch;

/* Arithmetic of the conv/GEMM kernels.  FP32: CUDA-core fp32 FMA everywhere (the 1e-3 parity mode).
 * BF16_TC: bf16 operands on wgmma tensor cores with fp32 accumulation in registers, bf16 activations in HBM
 * (the throughput mode; the reference itself deploys under fp16 autocast, multiperson_model.py:241). */
typedef enum { MTB_PRECISION_FP32 = 0, MTB_PRECISION_BF16_TC = 1,
               /* verification mode: same bf16 storage and bf16-rounded weights as BF16_TC, but every conv on CUDA
                * cores (fp32 FMA) - lets tests separate tensor-core kernel bugs from bf16 rounding effects */
               MTB_PRECISION_BF16_SIMT = 2,
               /* the 1e-3 parity mode ON TENSOR CORES: fp32 storage, every conv/GEMM as three wgmma tf32
                * products of hi/lo-split operands (a_hi*b_hi + a_lo*b_hi + a_hi*b_lo) with fp32 accumulation in registers;
                * conv outputs agree with the fp32 FMA chain to ~1e-6 */
               MTB_PRECISION_TF32X3 = 3,
               /* the reference's deployment arithmetic (fp16 autocast, multiperson_model.py:240-242) on tensor cores: fp16
                * activations in HBM, fp16-rounded GEMM weights, wgmma .f32.f16.f16 with fp32 accumulation in registers;
                * outputs round to nearest even and overflow to inf (no saturation), as under autocast */
               MTB_PRECISION_F16_TC = 4,
               /* verification mode: same fp16 storage and fp16-rounded weights as F16_TC, but every conv on CUDA cores
                * (fp32 FMA) - what BF16_SIMT is for BF16_TC */
               MTB_PRECISION_F16_SIMT = 5 } mtb_precision;

/* Layout of a logits tensor handed to the standalone soft-argmax. */
typedef enum {
  MTB_LAYOUT_BDJHW = 0, /* reference layout after rearrange 'b (d j) h w -> b d j h w' (models/metrabs.py:79) */
  MTB_LAYOUT_BHWN = 1   /* library-internal NHWC, channel n = J + d*J + j (2D logits in n < J) */
} mtb_layout;

#define MTB_MAX_STAGES 16

/* One row of EfficientNet's inverted_residual_setting (backbones/efficientnet.py:47-107). */
typedef struct {
  int32_t block;       /* 0 = FusedMBConv (:176-234), 1 = MBConv (:110-173) */
  int32_t expand;      /* expand_ratio */
  int32_t kernel;      /* 3 or 5 */
  int32_t stride;      /* stride of the first block of the stage */
  int32_t cin, cout;
  int32_t layers;
  int32_t bottomright; /* bottomright_stride: pad (pb-1, pe+1) on the first block (:140-141, :195-196) */
  int32_t dilation_in;  /* dilation of the first block's depthwise conv (`din` of metrabs_tf effnetv2_configs.py), 1..8 */
  int32_t dilation_out; /* dilation of the later blocks (`dout`); both 1 in the stride-32 tables.  A table whose output
                         * stride (2 x the product of the stage strides) is below 32 must equal stride_test, and dilates
                         * MBConv rows only (the reference's efficientnetv2-{s,l}-stride{16,8}, :163-228) */
} mtb_stage;

/* Frozen copy of the get_config() keys the path reads (util.py:41-57; config/config_l.yaml:1-21). */
typedef struct {
  int32_t abi_version;                /* MTB_ABI_VERSION */
  int32_t arch;                       /* mtb_arch */
  int32_t precision;                  /* mtb_precision */
  int32_t device;                     /* CUDA device ordinal */
  int32_t proc_side;                  /* S */
  int32_t stride_train, stride_test;
  int32_t centered_stride;
  int32_t legacy_centered_stride_bug; /* models/util.py:17-18 */
  int32_t depth;                      /* D */
  int32_t n_joints;                   /* J (n_raw_points) */
  int32_t feature_channels;           /* C: channels entering the head (needed for MTB_ARCH_HEAD_ONLY) */
  float box_size_mm;
  float mix_3d_inside_fov;            /* < 0 means None (ptu3d.py:28) */
  int32_t weak_perspective;           /* must be 0: the reference's weak-perspective solve crashes (ptu.py:30) */
  int32_t n_stages;                   /* EFFNET / EFFNET_EPS1E5 only */
  int32_t last_channel;               /* EFFNET / EFFNET_EPS1E5 only: 1280 (V2), 4 * last cout (B0-B7) */
  mtb_stage stages[MTB_MAX_STAGES];
} mtb_config;

typedef struct mtb_handle mtb_handle;

/* Metrabs.__init__ (models/metrabs.py:12-45) + backbone construction (backbones/efficientnet.py:237-357). */
int mtb_create(const mtb_config* cfg, mtb_handle** out);
int mtb_destroy(mtb_handle* h);
const char* mtb_last_error(const mtb_handle* h);
const char* mtb_version(void);

/* load_state_dict (scripts/demo_image.py:73): one call per entry, `name` in the reference key schema
 * ("backbone.1.<stage>.<block>.block.<i>.0.weight", "heatmap_heads.conv_final.bias", ...).  `data` is a HOST
 * pointer to a contiguous tensor in torch layout; it is copied.  Unknown names are ignored
 * (num_batches_tracked).  mtb_finalize_weights folds BN, repacks to NHWC / K-major, uploads, and fails with
 * MTB_ERR_MISSING_WEIGHT naming the first absent key. */
int mtb_load_weight(mtb_handle* h, const char* name, const void* data, int dtype, const int64_t* shape, int ndim);
int mtb_finalize_weights(mtb_handle* h);

/* Latent-point models (Metrabs.__init__ with affine_weights, models/metrabs.py:23-45 and :53-62; the recombination itself
 * is metrabs_tf/models/metrabs.py:80-81).  `weights` is a HOST fp32 array [n_latents][n_out] (the autoencoder's w2; it is
 * copied).  From then on the forward reconstructs head points [0, n_latents) and maps them to n_out joints per crop:
 * joints[b,J',c] = sum_l abs[b,l,c] * w2[l,J'].  transform_coords: n_latents = cfg.n_joints; predict_all_and_latents:
 * cfg.n_joints = n_latents + J, and mtb_finalize_weights keeps only the head channels of the first n_latents points (the
 * checkpoint still holds the full [(n_latents+J)(1+D),C,1,1] weight).  mtb_head_decode, mtb_reconstruct_absolute and the
 * all-gather of mtb_forward_sharded then work on n_latents points; mtb_forward* write n_out joints per crop.  Must be called
 * before mtb_finalize_weights; a second call replaces the first.  MTB_ERR_INVALID_ARG for n_latents outside
 * [1, cfg.n_joints], n_out outside [1, 4096], a null pointer, a non-finite weight, a finalized or a head-only handle. */
int mtb_set_latent_recombination(mtb_handle* h, const float* weights, int n_latents, int n_out);
/* Joints per crop that mtb_forward / mtb_forward_host* / mtb_forward_sharded write: n_out after
 * mtb_set_latent_recombination, cfg.n_joints otherwise (0 for a null handle). */
int mtb_output_joints(const mtb_handle* h);
/* tfu3d.linear_combine_points (metrabs_tf/tfu3d.py:48-49), handle-free: points [batch,n_in,3] and weights [n_in,n_out]
 * (device, fp32) -> out [batch,n_out,3] = einsum('bjc,jJ->bJc').  fp32 FMA over the n_in points in ascending order, the
 * kernel the forward of a latent-point model runs.  n_in <= 4096, n_out <= 4096. */
int mtb_linear_combine_points(const float* points, int batch, int n_in, const float* weights, int n_out, float* out,
                              void* stream);

/* Model classes of metrabs_tf/main.py:172-185 (--model-class, metrabs_tf/init.py:218).  METRABS (the default) is the path
 * above.  METRO (metrabs_tf/models/metro.py:13-45) and MODEL_25D (metrabs_tf/models/twofive.py:14-57) share a head without
 * the 2D block: conv_final has D*J channels (key "heatmap_head.conv_final.*", weight [D*J,C,1,1]), channel d*J + j, soft-argmax
 * jointly over (W, H, D) with tf.linspace (a one-long axis decodes to 0, not 0.5).  METRO outputs heatmap_to_metric of it:
 * root-relative joints in mm, crop-box frame; it takes no intrinsics.  MODEL_25D decodes heatmap_to_25d (x, y in crop pixels,
 * z in mm) and reconstructs absolute camera-space joints with reconstruct_absolute_by_bone_lengths (metrabs_tf/tfu3d.py:
 * 219-269): a 10-step Levenberg-Marquardt fit of each crop's depth to the ideal bone lengths, whose accept decision is taken
 * on the objective of the whole batch, so a crop's absolute joints depend on the batch it runs in (its decoded coords25d do
 * not). */
typedef enum { MTB_MODEL_METRABS = 0, MTB_MODEL_METRO = 1, MTB_MODEL_25D = 2 } mtb_model_class;
/* Sets the handle's model class; must be called before mtb_finalize_weights.  MODEL_25D takes `edges` [n_bones][2] (joint
 * indices in [0, cfg.n_joints)) and `bone_lengths` [n_bones] (mm, finite and positive), HOST arrays that are copied; the other
 * classes ignore them.  mean_relative != 0: depths relative to the mean joint (the reference default, init.py:228), else to the
 * last joint.  On a METRO or MODEL_25D handle:
 *   - mtb_head_decode writes the decoded [B,J,3] (Metro: mm; 2.5D: x px, y px, z mm) into coords3d_rel and its x, y into
 *     coords2d when coords2d is non-null;
 *   - mtb_forward, mtb_forward_host*, and mtb_forward_sharded run the whole class (METRO ignores intrinsics, which may be null);
 *     MODEL_25D's sharded forward all-gathers coords25d (3 floats per joint) and solves the full batch on every rank;
 *   - mtb_reconstruct_absolute fails with MTB_ERR_UNSUPPORTED.
 * MTB_ERR_INVALID_ARG for an unknown class, a bone index out of range, a bad length, n_bones outside [1, 4096] (MODEL_25D), a
 * METRO / MODEL_25D class with cfg.legacy_centered_stride_bug (the TF decode has no such term), a finalized or head-only
 * handle, or one with a latent recombination (mtb_set_latent_recombination in turn refuses a METRO / MODEL_25D handle). */
int mtb_set_model_class(mtb_handle* h, int model_class, const int32_t* edges, const float* bone_lengths, int n_bones,
                        int mean_relative);
/* The MODEL_25D absolute step on its own: coords25d [batch,J,3] (as mtb_head_decode writes them) + intrinsics [batch,3,3] ->
 * coords3d_abs [batch,J,3], one bone_solve_kernel launch, no host synchronisation.  Bit-identical from run to run.
 * scratch >= mtb_bone_lengths_scratch_bytes(h, batch) bytes (0 for a handle of another class). */
size_t mtb_bone_lengths_scratch_bytes(const mtb_handle* h, int batch);
int mtb_reconstruct_by_bone_lengths(mtb_handle* h, const float* coords25d, const float* intrinsics, int batch, float* coords3d_abs,
                                    void* scratch, void* stream);

size_t mtb_workspace_bytes(const mtb_handle* h, int batch);
/* Elements per crop of the feature map [H*W*C] and its spatial side, after finalize. */
int mtb_feature_shape(const mtb_handle* h, int* hw_side, int* channels);

/* self.backbone(image) (models/metrabs.py:50): crops fp32 NCHW [B,3,S,S] in [0,1] -> features NHWC
 * [B,S/s,S/s,C]: fp32 in FP32 / TF32X3 mode, bf16 in BF16_TC / BF16_SIMT, fp16 in F16_TC / F16_SIMT. */
int mtb_backbone_forward(mtb_handle* h, const float* crops, int batch, void* features, void* workspace,
                         size_t workspace_bytes, void* stream);

/* MetrabsHeads.forward (models/metrabs.py:75-85) incl. heatmap_to_image / heatmap_to_metric
 * (models/util.py:6-33): features NHWC -> coords2d [B,J,2] px, coords3d_rel [B,J,3] mm (fp32). */
int mtb_head_decode(mtb_handle* h, const void* features, int batch, float* coords2d, float* coords3d_rel,
                    void* workspace, size_t workspace_bytes, void* stream);

/* ptu.soft_argmax (ptu.py:54-75), standalone over materialised logits (config c5 / roofline sweep); dtype f32, bf16 or
 * f16 (f16: what the reference's head emits under autocast, multiperson_model.py:241; reference layout only).
 * BDJHW: logits [B,D,J,H,W] -> out [B,J,3] = (x,y,z) in [0,1];  with depth == 0: logits [B,J,H,W] -> out
 * [B,J,2].  BHWN: logits [B,H,W,J*(1+D)] -> out2d [B,J,2] and out3d [B,J,3] (either may be NULL). */
int mtb_softargmax(const void* logits, int dtype, int layout, int batch, int n_joints, int depth, int height,
                   int width, float* out2d, float* out3d, void* stream);

/* ptu3d.reconstruct_absolute (ptu3d.py:9-33) with reconstruct_ref_fullpersp (:56-105), is_within_fov
 * (:113-121), back_project (:108-110).  scratch: >= mtb_reconstruct_scratch_bytes(batch) bytes. */
size_t mtb_reconstruct_scratch_bytes(int batch);
int mtb_reconstruct_absolute(mtb_handle* h, const float* coords2d, const float* coords3d_rel,
                             const float* intrinsics, int batch, float* coords3d_abs, void* scratch,
                             void* stream);

/* Metrabs.forward (models/metrabs.py:47-64): crops [B,3,S,S] fp32 + intrinsics [B,3,3] fp32 -> [B,J,3] fp32
 * (J = mtb_output_joints(h)). */
int mtb_forward(mtb_handle* h, const float* crops, const float* intrinsics, int batch, float* coords3d_abs,
                void* workspace, size_t workspace_bytes, void* stream);

/* Same call for HOST buffers (the reference-facing end-to-end path): pinned or pageable host crops/intrinsics
 * in, host joints out; H2D/D2H copies and the forward are enqueued on `stream`, then the stream is
 * synchronised.  The library keeps a device staging area sized by the largest batch seen. */
int mtb_forward_host(mtb_handle* h, const float* host_crops, const float* host_intrinsics, int batch,
                     float* host_coords3d_abs, void* stream);

/* Pipelined form of the same call for back-to-back batches (the reference's caller feeds chunk after chunk,
 * multiperson_model.py:190-207): `submit` enqueues the H2D copies of this batch on an internal copy stream and the forward +
 * joints read-back on `stream` behind them, and returns without synchronising; `wait` blocks until that slot's joints are
 * in `host_coords3d_abs`.  Two slots (0/1): submit batch i+1 on the other slot before waiting for batch i, and its
 * host->device copy overlaps batch i's forward.  Host buffers must be pinned for the copies to be asynchronous and must
 * stay valid until the matching wait. */
int mtb_forward_host_submit(mtb_handle* h, const float* host_crops, const float* host_intrinsics, int batch,
                            float* host_coords3d_abs, int slot, void* stream);
int mtb_forward_host_wait(mtb_handle* h, int slot);

/* Multi-GPU (SURVEY.md 8e): crops shard across ranks; one all-gather of the decoded joints over NVLink.
 * mtb_comm_* wrap a NCCL communicator owned by the handle (libnccl is dlopen'ed). */
int mtb_comm_unique_id(void* id128 /* host, 128 bytes */);
int mtb_comm_init(mtb_handle* h, const void* id128, int rank, int world_size);
int mtb_allgather_joints(mtb_handle* h, const float* local, int floats_per_rank, float* all, void* stream);
/* The sharded forward in one call, no allocation: this rank's `batch_local` crops (the same count on every rank) ->
 * backbone -> head decode -> ONE ncclAllGather of [coords2d | coords3d_rel] (5 floats per joint) -> absolute reconstruction
 * of the full batch on every rank (reconstruct_ref_fullpersp uses batch-global RMS scalars, ptu3d.py:71-74, so the result
 * equals the unsharded Metrabs.forward on the concatenated batch).  intrinsics_all [world*batch_local,3,3] and
 * coords3d_abs_all [world*batch_local,J,3] are in rank order; scratch >= mtb_sharded_scratch_bytes(h, batch_local). */
size_t mtb_sharded_scratch_bytes(const mtb_handle* h, int batch_local);
int mtb_forward_sharded(mtb_handle* h, const float* crops_local, int batch_local, const float* intrinsics_all,
                        float* coords3d_abs_all, void* scratch, void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * The callers either side of the crop model (SURVEY.md 8f; /root/reference/metrabs_pytorch/multiperson/).  Handle-free
 * device functions: every pointer is a DEVICE pointer, work is enqueued on `stream`, nothing is allocated or synchronised.
 * Crop order: flat index = aug * n_boxes + box (multiperson_model.py:236-239).
 * ------------------------------------------------------------------------------------------------------------------ */

/* Gamma decoding `(images / 255) ** 2.2` (multiperson_model.py:200) + the box-filter pyramid of warp_images_with_pyramid
 * (warping.py:9-13).  images: u8 NCHW [n,3,H,W].  level1 [n,3,H/2,W/2] and level2 [n,3,H/4,W/4] are fp32 (floor sizes);
 * level 0 is decoded on the fly by mtb_warp_crops. */
int mtb_image_pyramid(const uint8_t* images, int n_images, int height, int width, float* level1, float* level2,
                      void* stream);

/* _get_new_rotation_and_scale (multiperson_model.py:321-355) + the per-crop matrices of _get_crops (:264-293) + the
 * pyramid level choice (warping.py:20-21). */
typedef struct {
  const float* boxes;            /* [n_boxes, box_stride]: x, y, w, h(, score) in image pixels */
  int32_t box_stride;
  const float* intrinsics;       /* [n_boxes,3,3] of the image each box lives in */
  const float* distortion;       /* [n_boxes, n_dist] OpenCV order (k1,k2,p1,p2,k3,k4,k5,k6,s1..s4), zero padded */
  int32_t n_dist;                /* 0..12 */
  const float* camspace_up;      /* [n_boxes,3] */
  const float* aug_rotflipmat;   /* [num_aug,3,3] */
  const float* aug_scales;       /* [num_aug] */
  int32_t n_boxes, num_aug, resolution, antialias_factor;
  float* new_intrinsics;         /* out [num_aug*n_boxes,3,3] (the intrinsics mtb_forward takes) */
  float* rotations;              /* out [num_aug*n_boxes,3,3] R = aug_rotflipmat @ R_noaug */
  float* inv_projections;        /* out [num_aug*n_boxes,3,3] inv(new_intrinsics @ R) (@ antialias scaling) */
  int32_t* pyramid_levels;       /* out [num_aug*n_boxes] */
} mtb_crop_setup_args;
int mtb_crop_setup(const mtb_crop_setup_args* args, void* stream);

/* warp_images_with_pyramid + the gamma of _get_crops (warping.py:6-52, multiperson_model.py:295-319): every crop of the
 * batch in ONE launch, written as the fp32 NCHW [num_aug*n_boxes,3,res,res] tensor mtb_forward reads.  antialias_factor
 * 1, 2 or 4 (rendered by supersampling = the reference's larger render followed by avg_pool2d) or 5..16 (the larger
 * render shrunk by the antialiased bilinear resize, per output tile in on-chip memory); mtb_crop_setup takes the same
 * factors.  Others, 3 included, return MTB_ERR_UNSUPPORTED. */
typedef struct {
  const uint8_t* images;         /* [n_images,3,H,W] u8 */
  const float* level1;           /* from mtb_image_pyramid */
  const float* level2;
  int32_t n_images, height, width;
  const float* intrinsics;       /* [n_boxes,3,3] */
  const float* distortion;       /* [n_boxes, n_dist] */
  int32_t n_dist;
  const int32_t* image_ids;      /* [n_boxes] */
  const float* inv_projections;  /* [num_aug*n_boxes,3,3] */
  const int32_t* pyramid_levels; /* [num_aug*n_boxes] */
  const float* gamma_exponents;  /* [num_aug] = aug_gammas / 2.2 */
  int32_t n_boxes, num_aug, resolution, antialias_factor;
  float* crops;                  /* out [num_aug*n_boxes,3,res,res] */
} mtb_warp_args;
int mtb_warp_crops(const mtb_warp_args* args, void* stream);

/* The epilogue of _predict_single_batch (mirror swap, poses @ R; multiperson_model.py:246-259) and of
 * _estimate_poses_batched (joint transform, 2D projection with distortion + intrinsics, inverse extrinsics, skeleton
 * gather, mean over augmentations; :143-182). */
typedef struct {
  const float* poses;            /* [num_aug*n_boxes, J, 3] crop-model output */
  const float* rotations;        /* [num_aug*n_boxes,3,3] */
  const uint8_t* aug_should_flip;/* [num_aug] */
  const int32_t* mirror_mapping; /* [J] */
  const float* joint_transform;  /* [J, J2] or NULL (J2 = J) */
  const int32_t* skeleton;       /* [Js] indices into J2, or NULL (Js = J2) */
  const float* intrinsics;       /* [n_boxes,3,3] */
  const float* distortion;       /* [n_boxes, n_dist] */
  int32_t n_dist;
  const float* extrinsics_inv;   /* [n_boxes,4,4] inverse extrinsic matrix of the box's image */
  int32_t n_boxes, num_aug, n_joints, n_joints_transformed, n_skeleton, average_aug;
  float* poses3d;                /* out [n_boxes,(num_aug,)Js,3] */
  float* poses2d;                /* out [n_boxes,(num_aug,)Js,2] */
} mtb_tta_args;
int mtb_tta_merge(const mtb_tta_args* args, void* stream);

/* plausibility_check.py:8-119: is_pose_plausible, are_augmentation_results_consistent, is_pose_consistent_with_box and
 * pose_non_max_suppression (similarity threshold 0.4) per image.  num_aug <= 16.  The per-box state of one image lives in
 * shared memory, 14 B per box sized for n_boxes: at most about 16,000 boxes per call on an H100 (227 KB per block);
 * above what the device holds the call fails with MTB_ERR_UNSUPPORTED and filters nothing. */
typedef struct {
  const float* poses3d;          /* [n_boxes, num_aug, J, 3] camera space */
  const float* poses2d;          /* [n_boxes, num_aug, J, 2] */
  const float* boxes;            /* [n_boxes, box_stride] x, y, w, h, score */
  int32_t box_stride;
  const int32_t* bones;          /* [n_bones,2] joint pairs (rows of joint2bone_mat) */
  const float* mean_bones;       /* [n_bones] mm */
  int32_t n_bones;
  const int32_t* image_start;    /* [n_images+1] box range of each image */
  int32_t n_images, n_boxes, num_aug, n_joints;
  uint8_t* plausible;            /* out [n_boxes] */
  uint8_t* keep;                 /* out [n_boxes]: plausible and not suppressed */
  float* scratch;                /* [n_boxes, J, 3] */
} mtb_filter_args;
int mtb_filter_poses(const mtb_filter_args* args, void* stream);

/* Introspection for tests / profiling. */
int mtb_num_ops(const mtb_handle* h);
const char* mtb_op_name(const mtb_handle* h, int op);
/* Runs the first `n_ops` backbone ops and copies that op's NHWC output (as fp32) to `out` (device). */
int mtb_debug_run_ops(mtb_handle* h, const float* crops, int batch, int n_ops, float* out, size_t out_floats,
                      void* workspace, size_t workspace_bytes, void* stream);
int mtb_op_output_shape(const mtb_handle* h, int op, int* height, int* width, int* channels);
int mtb_op_input_shape(const mtb_handle* h, int op, int* height, int* width, int* channels, int* has_residual,
                       int* has_scale);
/* The workspace buffers the forward's planner gave backbone op `op`: its input, its output, its residual and its
 * squeeze-excitation scale.  Ids: -2 the feature output, -1 none (the stem's input: it reads the crops), 0-3 the large
 * activation buffers, 4-6 the small [B,C] ones.  An operand of op k is the output of the latest op j < k whose out_buf is that id (not always k - 1: a projection
 * reads the depthwise output before the SE ops, its residual is the block input), so a test can take an op's operands
 * from mtb_debug_run_ops prefixes.  Any output pointer may be null.  MTB_ERR_INVALID_ARG for an index out of range. */
int mtb_debug_op_buffers(const mtb_handle* h, int op, int* in_buf, int* out_buf, int* res_buf, int* scale_buf);
/* Runs ONE backbone op in isolation on caller-provided fp32 NHWC device tensors (converted to the handle's
 * storage type - fp32, or bf16 / fp16 rounded to nearest even): in [B,Hin,Win,Cin] (the stem takes NCHW crops), optional residual [B,Hout,Wout,Cout] and
 * squeeze-excitation scale [B,Cin]; out receives [B,Hout,Wout,Cout] as fp32.  Lets tests compare the tensor-core
 * kernels with the CUDA-core kernels on identical inputs. */
int mtb_debug_run_op(mtb_handle* h, int op_index, const float* in, const float* res, const float* scale, int batch,
                     float* out, size_t out_floats, void* workspace, size_t workspace_bytes, void* stream);
/* FusedMBConv block fusion (BF16_TC and F16_TC modes): 1 when backbone op `op_index` (a 3x3 stride-1 expand conv) and the op
 * after it (the 1x1 projection, + residual) run as ONE fmb_kernel launch (reference block:
 * metrabs_pytorch/backbones/efficientnet.py:176-234).  mtb_debug_run_fused_block runs that pair in isolation on a
 * caller-provided fp32 NHWC device tensor `in` [B,H,W,Cin] (also the residual when the block has one); `out` receives the
 * block output [B,H,W,Cout] as fp32. */
int mtb_op_is_fused_block(const mtb_handle* h, int op_index);
int mtb_debug_run_fused_block(mtb_handle* h, int op_index, const float* in, int batch, float* out, size_t out_floats,
                              void* workspace, size_t workspace_bytes, void* stream);
/* ResNet V2 pre-activation fusion (BF16_TC and F16_TC modes): 1 when backbone op `op_index` (a block's 1x1 _3_conv, + shortcut)
 * and the op after it (the next block's _preact_bn + ReLU, or post_bn + ReLU: a 1x1 depthwise op) run as ONE
 * tc_conv_preact_kernel launch [tc_conv_preact_kernel] that stores both outputs, bit-identical to the two launches.
 * mtb_debug_run_preact_pair runs that pair in isolation on caller-provided fp32 NHWC device tensors `in` [B,H,W,Cin] and
 * `res` [B,H,W,Cout]; `out` receives the GEMM's output and `out_preact` the pre-activation, both [B,H,W,Cout] as fp32. */
int mtb_op_is_preact_pair(const mtb_handle* h, int op_index);
int mtb_debug_run_preact_pair(mtb_handle* h, int op_index, const float* in, const float* res, int batch, float* out, float* out_preact,
                              size_t out_floats, void* workspace, size_t workspace_bytes, void* stream);
/* CUDA-event profiler (bench.py's live roofline measurement): between begin and end, every kernel launch of the
 * classes selected by `class_mask` (bit i = class i) is bracketed by cudaEventRecord on the launching stream.
 * mtb_profile_end synchronises those events and returns, per class, the summed device time (ms), algorithmic
 * FLOPs, algorithmic bytes and launch count; arrays must hold mtb_num_kernel_classes() entries. */
int mtb_profile_begin(mtb_handle* h, unsigned class_mask);
int mtb_profile_end(mtb_handle* h, double* ms, double* flops, double* bytes, int64_t* launches);
/* Per-op view of the last profiling window: device ms per backbone op, its algorithmic FLOPs and bytes per crop and
 * its kernel class; arrays hold mtb_num_ops() entries. */
int mtb_profile_op_times(const mtb_handle* h, double* ms, double* flops_per_crop, double* bytes_per_crop, int* cls, int n);
/* Weight bytes the op reads once per launch (bf16 / fp16 on the tensor-core path, fp32 otherwise); `bytes_per_crop` above counts
 * activations (input + output + residual) only, so a launch on B crops moves B * bytes_per_crop + weight bytes. */
double mtb_op_weight_bytes(const mtb_handle* h, int op);
int mtb_num_kernel_classes(void);
const char* mtb_kernel_class_name(int cls);
/* Number of kernels the last mtb_forward / mtb_backbone_forward / ... call on this handle launched. */
int64_t mtb_last_launch_count(const mtb_handle* h);
double mtb_backbone_flops_per_crop(const mtb_handle* h);
/* Host-side tiling plan of the TMA-staged depthwise 3x3 kernel for an HxW map (no device needed): crops per item, output
 * rows per item, row bands per crop (= SE pooling slices) and bytes of one shared-memory stage; all 0 when the shape falls
 * back to the strip kernel. */
int mtb_debug_dw_plan(int height, int width, int* crops_per_item, int* rows_per_item, int* row_bands, int* stage_bytes);
/* The kernel mtb_finalize_weights chose for each op; the profiler class its launches count under is in brackets.
 * Stem [stem_conv_kernel]: STEM_3X3S2 is stem3x3s2_kernel, EfficientNet's 3x3 stride-2 stem with 24 or 32 output channels
 * (bit-identical to the generic kernels; the environment variable MTB_STEM_FAST=0, read once per process, turns it off for
 * tests); STEM_WIDE is stem_conv_wide_kernel, for a multiple of 32, 24 or 16 output channels; STEM_GENERIC is
 * stem_conv_kernel for any other width.
 * MAXPOOL is maxpool_kernel [other].  POOL_MEAN is pool_mean_kernel [pool_mean_kernel], the squeeze-excitation (SE) mean;
 * POOL_FUSED launches nothing, because the depthwise kernel before it wrote the SE pooling slices (fc1 sums them).
 * SE_FC is conv_igemm_kernel on the SE fully-connected layers, plus se_reduce_kernel when fc1 splits K [se_fc(...)].
 * IGEMM is conv_igemm_kernel [conv_igemm_kernel], every conv of the FP32 and _SIMT modes and what no other kernel takes.
 * Tensor cores, BF16_TC / F16_TC [tc_conv_kernel]: TC_CONV is tc_conv_kernel; TC_CONV_SE is tc_conv_kernel scaling its A
 * tiles by the SE scale (the 1x1 projections to at most 256 channels); SE_SCALE_TC_CONV is se_scale_kernel
 * [se_scale_kernel] applying the scale in place, then tc_conv_kernel (the wider projections); TC_CONV3X3S1 is
 * tc_conv3x3s1_kernel, which takes the 3x3 stride-1 undilated convs with Cin and Cout <= 64 and SiLU or ReLU from input
 * boxes and weights resident in shared memory.  TC32 is tc32_conv_kernel [tc32_conv_kernel], the TF32X3 mode's GEMMs.
 * Depthwise [dwconv_kernel]: DW_GENERIC is dwconv_kernel (one thread per pixel and 4 channels; every fp32 / 3xTF32 / _SIMT
 * mode op that no other kernel covers), DW_TMA the TMA-staged 3x3 stride-1 kernel and DW_STRIP_16B / DW_STRIP_F32 the 3x3
 * strip kernels (these three also write the SE pooling slices), DW_5X5_16B the 16-bit 5x5 kernel of the BF16_TC / F16_TC
 * modes for ReLU / hard-swish (bit-identical to dwconv_kernel, no pooling), DW_5X5_POOL_16B the same kernel for SiLU
 * (bit-identical outputs, and it also writes the SE pooling slices of the stored outputs), DW_TMA_DIL the TMA-staged kernel
 * for the 3x3 stride-1 SiLU ops with dilation 2 or 4 of the BF16_TC / F16_TC modes (one undilated pass per phase of the
 * dilation, same arithmetic per output as DW_TMA, also writes the SE pooling slices).
 * Head (mtb_head_decode and the forward): HEAD_FUSED is tc_head_kernel + head_finalize_kernel
 * [tc_head_softargmax_kernel], the BF16_TC / F16_TC modes when a fused tile fits the feature map; HEAD_TC32 is
 * tc32_conv_kernel [tc32_conv_kernel] and HEAD_IGEMM conv_igemm_kernel [head_conv(...)], both followed by
 * softargmax_bhwn_kernel [softargmax_bhwn_kernel].
 * The two ops of a fused FusedMBConv block (mtb_op_is_fused_block) run as one fmb_kernel launch [fmb_kernel] on the forward;
 * each reports the kernel that runs it alone, as on a mtb_debug_run_ops prefix that ends after the first.  In isolation
 * (mtb_debug_run_op) a depthwise op writes no pooling slices and a POOL_FUSED op runs pool_mean_kernel. */
typedef enum {
  /* depthwise values first: their numbers (0-6) are stable for existing callers */
  MTB_DW_GENERIC = 0, MTB_DW_TMA = 1, MTB_DW_STRIP_16B = 2, MTB_DW_STRIP_F32 = 3, MTB_DW_5X5_16B = 4,
  MTB_DW_5X5_POOL_16B = MTB_DW_5X5_16B + 1 /* 5 */,
  MTB_DW_TMA_DIL = MTB_DW_5X5_POOL_16B + 1 /* 6 */,
  MTB_STEM_3X3S2 = 7, MTB_STEM_WIDE = 8, MTB_STEM_GENERIC = 9,
  MTB_MAXPOOL = 10, MTB_POOL_MEAN = 11, MTB_POOL_FUSED = 12,
  MTB_SE_FC = 13, MTB_IGEMM = 14,
  MTB_TC_CONV = 15, MTB_TC_CONV_SE = 16, MTB_SE_SCALE_TC_CONV = 17, MTB_TC_CONV3X3S1 = 18,
  MTB_TC32 = 19,
  MTB_HEAD_FUSED = 20, MTB_HEAD_TC32 = 21, MTB_HEAD_IGEMM = 22
} mtb_kernel;
/* The mtb_kernel value of backbone op `op` (the head's is not reported here).  MTB_ERR_NOT_FINALIZED before
 * mtb_finalize_weights, MTB_ERR_INVALID_ARG for an index out of range. */
int mtb_op_kernel(const mtb_handle* h, int op);

#ifdef __cplusplus
}
#endif
#endif /* METRABS_B200_H_ */
