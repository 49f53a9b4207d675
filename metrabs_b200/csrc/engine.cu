// libmetrabs_b200.so - engine: handle, weight arena (BN folding + repack), op plan, forward executor, C ABI.
// See include/metrabs_b200.h for the contract and the reference file:line each entry point replaces.
#include "../../include/metrabs_b200.h"

#include <dlfcn.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <iterator>
#include <map>
#include <string>
#include <vector>

#include "common.cuh"
#include "conv_simt.cuh"
#include "decode.cuh"
#include "tc_gemm.cuh"
#include "tc_fmb.cuh"
#include "tc_tf32.cuh"
#include "dw_tma.cuh"
#include "multiperson.cuh"

using namespace mtb;

namespace {

std::string g_error;

enum OpType { OP_STEM = 0, OP_CONV = 1, OP_DW = 2, OP_POOL = 3, OP_MAXPOOL = 4 };
// kernel classes for the CUDA-event profiler (mtb_profile_begin / mtb_profile_end)
enum KClass { KC_STEM = 0, KC_IGEMM_SIMT = 1, KC_DWCONV = 2, KC_POOL = 3, KC_SE_FC = 4, KC_TC_GEMM = 5, KC_FMB = 6,
              KC_HEAD_FUSED = 7, KC_HEAD_CONV_SIMT = 8, KC_SOFTARGMAX = 9, KC_RECON = 10, KC_OTHER = 11, KC_SE_SCALE = 12, KC_TC32 = 13,
              KC_COMBINE = 14, KC_TC_PREACT = 15, KC_BONE_SOLVE = 16, KC_COUNT = 17 };
const char* kKClassNames[KC_COUNT] = {"stem_conv_kernel", "conv_igemm_kernel", "dwconv_kernel", "pool_mean_kernel",
                                      "se_fc(conv_igemm_kernel)", "tc_conv_kernel", "fmb_kernel",
                                      "tc_head_softargmax_kernel", "head_conv(conv_igemm_kernel)",
                                      "softargmax_bhwn_kernel", "recon_pass1+2_kernel", "other", "se_scale_kernel", "tc32_conv_kernel",
                                      "combine_points_kernel", "tc_conv_preact_kernel", "bone_solve_kernel"};
// One row per mtb_kernel value: the profiler class of its launches, whether it exists for 16-bit storage only (bf16 /
// fp16), and whether it also writes the SE pooling slices of its output (depthwise)
struct KernelTraits { mtb_kernel kernel; KClass cls; bool only16, pools; };
constexpr KernelTraits kKernels[] = {
    {MTB_DW_GENERIC, KC_DWCONV, false, false},        {MTB_DW_TMA, KC_DWCONV, true, true},
    {MTB_DW_STRIP_16B, KC_DWCONV, true, true},        {MTB_DW_STRIP_F32, KC_DWCONV, false, true},
    {MTB_DW_5X5_16B, KC_DWCONV, true, false},         {MTB_DW_5X5_POOL_16B, KC_DWCONV, true, true},
    {MTB_DW_TMA_DIL, KC_DWCONV, true, true},          {MTB_STEM_3X3S2, KC_STEM, false, false},
    {MTB_STEM_WIDE, KC_STEM, false, false},           {MTB_STEM_GENERIC, KC_STEM, false, false},
    {MTB_MAXPOOL, KC_OTHER, false, false},            {MTB_POOL_MEAN, KC_POOL, false, false},
    {MTB_POOL_FUSED, KC_POOL, false, false},          {MTB_SE_FC, KC_SE_FC, false, false},
    {MTB_IGEMM, KC_IGEMM_SIMT, false, false},         {MTB_TC_CONV, KC_TC_GEMM, true, false},
    {MTB_TC_CONV_SE, KC_TC_GEMM, true, false},        {MTB_SE_SCALE_TC_CONV, KC_TC_GEMM, true, false},
    {MTB_TC_CONV3X3S1, KC_TC_GEMM, true, false},      {MTB_TC32, KC_TC32, false, false},
    {MTB_HEAD_FUSED, KC_HEAD_FUSED, true, false},     {MTB_HEAD_TC32, KC_TC32, false, false},
    {MTB_HEAD_IGEMM, KC_HEAD_CONV_SIMT, false, false}};
constexpr bool kernel_rows_in_order() {
  for (int i = 0; i < (int)std::size(kKernels); ++i)
    if (kKernels[i].kernel != i) return false;
  return std::size(kKernels) == MTB_HEAD_IGEMM + 1;
}
static_assert(kernel_rows_in_order(), "kKernels: one row per mtb_kernel value, in order");
constexpr int kMaxCombinePoints = 4096;  // n_in and n_out of combine_points_kernel (its shared memory holds n_in * 3 floats)
enum { BUF_FEATURES = -2, BUF_NONE = -1, BUF_SMALL0 = 4 };  // 0..3 big activation buffers, 4..6 small [B,C]
constexpr int kNumBig = 4, kNumSmall = 3;
constexpr int kPoolSlices = 8;  // the fused depthwise+pool kernel leaves up to 8 partial slices [slice][B][C]

struct HostTensor {
  std::vector<float> data;
  std::vector<int64_t> shape;
};

struct Op {
  OpType type;
  std::string name;     // reference key prefix of the layer
  std::string wkey;     // conv weight key
  std::string bnkey;    // BN key prefix ("" = none)
  std::string biaskey;  // conv bias key ("" = none)
  int in_buf = 0, out_buf = 0, res_buf = BUF_NONE, scale_buf = BUF_NONE;
  int Hin = 1, Win = 1, Cin = 0, Hout = 1, Wout = 1, Cout = 0;
  int R = 1, S = 1, stride = 1, dil = 1, pad_t = 0, pad_l = 0, act = ACT_NONE;
  bool depthwise = false;
  bool small_io = false;  // squeeze-excitation FCs on [B,1,1,C] fp32 tensors
  float pre_scale[3] = {2.f, 2.f, 2.f}, pre_shift[3] = {-1.f, -1.f, -1.f};  // stem input affine (PreprocLayer: x*2-1)
  mtb_kernel kernel = MTB_IGEMM;  // the kernel that runs it (choose_kernels, at mtb_finalize_weights)
  bool fused_pool = false;  // depthwise: also writes the SE pooling slices of the pool op behind it (MTB_POOL_FUSED)
  DwTmaPlan dw_plan;                // DW_TMA / DW_TMA_DIL: its tiling plan (DW_TMA_DIL: of one phase of the dilation)
  int pool_slices = 1;              // DW_TMA* / DW_STRIP_* / DW_5X5_POOL_16B: partial pooling slices it leaves (= its gridDim.y / dw_plan.n_rb)
  bool res_first = false;  // residual added BEFORE the activation (ResNet); EfficientNet adds it after
  int pool_src = -1;       // fc1: index of the OP_POOL op that produces its input (fused pooling leaves partial slices)
  int ksplit = 1;          // split-K (squeeze-excitation fc1): raw sums, bias/act deferred to the consumer
  bool pad_ok = false;    // weight tensor may be smaller than [Cout,Cin]: channels zero-padded to a multiple of 4
  float bn_eps = 1e-3f;
  float* d_w = nullptr;     // fp32 [R*S*Cin][Cout]  (dw: [R*S][C])
  float* d_bias = nullptr;  // fp32 [Cout]
  TcWeights tc;             // 16-bit (bf16 / fp16) K-major copy + TMA descriptor state for the wgmma path
  Tc32Weights tc32;         // fp32 K-major copy + TMA descriptor state for the 3xTF32 wgmma path (MTB_PRECISION_TF32X3)
  FmbWeights fmb;           // 16-bit tensor-core modes: this 3x3 expand conv and the NEXT op (1x1 projection) run as one fmb_kernel launch
  bool preact_next = false;  // 16-bit tensor-core modes: this 1x1 GEMM also writes the NEXT op's output (ResNet V2 pre-activation,
                             // a 1x1 depthwise BN + ReLU) in one tc_conv_preact_kernel launch
  mutable TmapCache dw_maps;    // DW_TMA / DW_TMA_DIL: its input tensor maps
  double flops = 0;         // 2*MACs per crop
};

}  // namespace

struct mtb_handle {
  mtb_config cfg;
  std::map<std::string, HostTensor> raw;
  std::vector<Op> ops;
  Op head;
  // latent-point model (mtb_set_latent_recombination): the forward reconstructs head points [0, n_latents) and maps them to
  // n_out joints with recomb [n_latents][n_out]; n_latents == 0 for a plain model
  int n_latents = 0, n_out = 0;
  std::vector<float> recomb;
  float* d_recomb = nullptr;  // device copy in the weight arena (uploaded by mtb_finalize_weights)
  // model class (mtb_set_model_class): MeTRAbs, Metro (root-relative metric output) or Model25D (2.5D head + bone-length
  // depth solve over bone_edges / bone_len); the device copies live in the weight arena
  int model_class = MTB_MODEL_METRABS;
  std::vector<int32_t> bone_edges;  // [n_bones][2]
  std::vector<float> bone_len;      // [n_bones] mm
  int mean_relative = 1;
  int2* d_edges = nullptr;
  float* d_len = nullptr;
  bool finalized = false;
  mutable std::string err;
  std::vector<void*> dev_allocs;
  // geometry
  int feat_side = 0, feat_c = 0;
  size_t big_elems_per_crop = 0;   // capacity of one big buffer, elements per crop
  int small_c = 0;                 // capacity of one small buffer, floats per crop
  int64_t launches = 0;
  double flops_per_crop = 0;
  // host-path staging
  void* stage = nullptr;
  size_t stage_bytes = 0, stage_ws_bytes = 0;
  int stage_batch = 0;
  // pipelined host path (mtb_forward_host_submit / _wait): two input/output slots, one shared workspace, a copy stream
  struct HostSlot {
    void* buf = nullptr;       // [crops | intrinsics | joints] device staging of this slot
    size_t bytes = 0;
    cudaEvent_t h2d_done = nullptr, done = nullptr;
    bool used = false;         // `done` has been recorded at least once
  };
  HostSlot slots[2];
  // mtb_forward's captured forwards keyed by (buffers, batch, stream)
  struct GraphEntry {
    const void *crops = nullptr, *k = nullptr, *out = nullptr, *ws = nullptr;
    int batch = 0;
    cudaStream_t st = nullptr;
    cudaGraphExec_t exec = nullptr;
    int64_t launches = 0;
    bool failed = false;
  };
  std::vector<GraphEntry> graphs;
  void* pipe_ws = nullptr;
  size_t pipe_ws_bytes = 0;
  cudaStream_t copy_stream = nullptr;
  cudaStream_t graph_stream = nullptr;  // mtb_forward on the legacy default stream: captured forwards run here
  cudaEvent_t graph_in = nullptr, graph_out = nullptr;
  // profiler
  unsigned prof_mask = 0;
  std::vector<cudaEvent_t> prof_events;  // pairs
  std::vector<int> prof_cls;
  std::vector<int> prof_op;      // backbone op index of each timed launch (-1: head / decode / reconstruction)
  int prof_cur_op = -1;
  std::vector<double> prof_flops, prof_bytes;
  size_t prof_used = 0;
  std::vector<double> prof_op_ms;
  // NCCL (dlopen'ed)
  void* nccl_lib = nullptr;
  void* nccl_comm = nullptr;
  int nccl_world = 0;
};

namespace {

int fail(const mtb_handle* h, int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  if (h) h->err = buf;
  g_error = buf;
  return code;
}

#define CUDA_TRY(h, expr)                                                                               \
  do {                                                                                                  \
    cudaError_t e__ = (expr);                                                                           \
    if (e__ != cudaSuccess)                                                                             \
      return fail(h, MTB_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
  } while (0)

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }
// element type of the activations in HBM: bf16 (BF16_TC / BF16_SIMT), fp16 (F16_TC / F16_SIMT) or fp32 (FP32 / TF32X3)
enum Storage { ST_F32 = 0, ST_BF16 = 1, ST_F16 = 2 };
inline Storage storage(const mtb_handle* h) {
  switch (h->cfg.precision) {
    case MTB_PRECISION_BF16_TC:
    case MTB_PRECISION_BF16_SIMT: return ST_BF16;
    case MTB_PRECISION_F16_TC:
    case MTB_PRECISION_F16_SIMT: return ST_F16;
    default: return ST_F32;
  }
}
inline bool is_16b(const mtb_handle* h) { return storage(h) != ST_F32; }
inline size_t elem_size(const mtb_handle* h) { return is_16b(h) ? 2 : 4; }
// the wgmma modes with 16-bit operands (bf16 or fp16): tc_conv_kernel, fmb_kernel, tc_head_kernel, the TMA depthwise kernel
inline bool is_tc16(const mtb_handle* h) {
  return h->cfg.precision == MTB_PRECISION_BF16_TC || h->cfg.precision == MTB_PRECISION_F16_TC;
}
// calls f((T*)nullptr) with T the storage element type of the handle's mode
template <typename F>
auto with_storage(const mtb_handle* h, F&& f) {
  switch (storage(h)) {
    case ST_BF16: return f((__nv_bfloat16*)nullptr);
    case ST_F16: return f((__half*)nullptr);
    default: return f((float*)nullptr);
  }
}
// with_storage for the code that only exists for 16-bit storage (the tensor-core kernels): T is __half in the fp16 modes,
// __nv_bfloat16 otherwise
template <typename F>
auto with_storage16(const mtb_handle* h, F&& f) {
  return storage(h) == ST_F16 ? f((__half*)nullptr) : f((__nv_bfloat16*)nullptr);
}
// points the head decodes and the reconstruction solves for: the latents of a latent-point model, cfg.n_joints otherwise
inline int head_points(const mtb_handle* h) { return h->n_latents > 0 ? h->n_latents : h->cfg.n_joints; }
inline int output_joints(const mtb_handle* h) { return h->n_latents > 0 ? h->n_out : h->cfg.n_joints; }
// the TF-only Metro / Model25D head: D*J channels (channel d*J + j), no 2D block
inline bool head3d(const mtb_handle* h) { return h->model_class != MTB_MODEL_METRABS; }
// head channels before padding: 1 + D per point (MeTRAbs), D per point (Metro / Model25D)
inline int head_channels(const mtb_handle* h) { return head_points(h) * (h->cfg.depth + (head3d(h) ? 0 : 1)); }
// head channel count padded to a multiple of 4 with zero weights (J=122: 1098 -> 1100), and its FLOPs
inline void size_head(mtb_handle* h) {
  Op& hd = h->head;
  hd.Cout = (head_channels(h) + 3) / 4 * 4;
  hd.flops = 2.0 * hd.Hout * hd.Wout * hd.Cin * hd.Cout;
}

// ------------------------------------------------------------------------------------------- plan building
struct Planner {
  mtb_handle* h;
  int H, W, C;       // current activation
  int cur = BUF_NONE;
  size_t max_elems = 0;
  int max_small = 0;

  int pick(std::initializer_list<int> busy) {
    for (int i = 0; i < kNumBig; ++i)
      if (std::find(busy.begin(), busy.end(), i) == busy.end()) return i;
    return 0;
  }
  void track(int h_, int w_, int c_) { max_elems = std::max(max_elems, (size_t)h_ * w_ * c_); }

  // Keras-named conv (TF-only backbones): explicit weight / bias / BN keys
  Op& conv_k(const std::string& name, const std::string& wkey, const std::string& biaskey, const std::string& bnkey, int cout,
             int k, int stride, int pad_beg, int pad_total, int act, int in_buf, int out_buf, bool depthwise = false,
             int dil = 1, float eps = 1e-3f) {
    Op& op = conv(name, cout, k, stride, pad_beg, pad_total, act, in_buf, out_buf, depthwise, dil);
    op.wkey = wkey; op.biaskey = biaskey; op.bnkey = bnkey; op.bn_eps = eps;
    return op;
  }

  // squeeze-excitation on the tensor in `buf` (H x W x C): pool + fc1 + fc2 -> scale in BUF_SMALL0+2
  void squeeze_excite(const std::string& name, const std::string& fc1, const std::string& fc2, int csq_real, int buf,
                      int act1, int act2) {
    const int cexp = C;
    const int csq = (csq_real + 3) / 4 * 4;  // hidden channels zero-padded to a multiple of 4 (128-bit accesses)
    Op op;
    op.type = OP_POOL; op.name = name + ".avgpool";
    op.Hin = H; op.Win = W; op.Cin = op.Cout = cexp;
    op.in_buf = buf; op.out_buf = BUF_SMALL0;
    h->ops.push_back(op);
    const int pool_index = (int)h->ops.size() - 1;
    Op f1;
    f1.type = OP_CONV; f1.name = name + ".fc1"; f1.wkey = fc1 + ".weight"; f1.biaskey = fc1 + ".bias";
    f1.Cin = cexp; f1.Cout = csq; f1.act = act1; f1.small_io = true; f1.pad_ok = true;
    f1.in_buf = BUF_SMALL0; f1.out_buf = BUF_SMALL0 + 1;
    f1.pool_src = pool_index;
    f1.flops = 2.0 * cexp * csq_real;
    // K = cexp is long and M = batch is short: split K over CTAs; the ksplit partial slices [ksplit][B][csq] must fit
    // the small buffer (capacity >= cexp floats per crop)
    f1.ksplit = std::max(1, std::min({32, cexp / 64, cexp / csq}));
    h->ops.push_back(f1);
    Op f2;
    f2.type = OP_CONV; f2.name = name + ".fc2"; f2.wkey = fc2 + ".weight"; f2.biaskey = fc2 + ".bias";
    f2.Cin = csq; f2.Cout = cexp; f2.act = act2; f2.small_io = true; f2.pad_ok = true;
    f2.in_buf = BUF_SMALL0 + 1; f2.out_buf = BUF_SMALL0 + 2;
    f2.flops = 2.0 * cexp * csq_real;
    // (fc2 summing fc1's split-K slices on its A load was measured slower than the tiny reduce kernel)
    h->ops.push_back(f2);
    max_small = std::max(max_small, cexp);
  }

  // conv with explicit begin pad; output size = floor((in + pad_total - eff_k)/stride) + 1
  Op& conv(const std::string& name, int cout, int k, int stride, int pad_beg, int pad_total, int act, int in_buf,
           int out_buf, bool depthwise = false, int dil = 1) {
    Op op;
    op.type = depthwise ? OP_DW : OP_CONV;
    op.name = name;
    op.wkey = name + ".0.weight";
    op.bnkey = name + ".1";
    op.Hin = H; op.Win = W; op.Cin = C; op.Cout = cout;
    op.R = op.S = k; op.stride = stride; op.dil = dil; op.pad_t = op.pad_l = pad_beg; op.act = act;
    int eff = k + (k - 1) * (dil - 1);
    op.Hout = (H + pad_total - eff) / stride + 1;
    op.Wout = (W + pad_total - eff) / stride + 1;
    op.depthwise = depthwise;
    op.in_buf = in_buf; op.out_buf = out_buf;
    op.flops = 2.0 * op.Hout * op.Wout * cout * k * k * (depthwise ? 1 : C);
    H = op.Hout; W = op.Wout; C = cout;
    track(H, W, C);
    h->ops.push_back(op);
    return h->ops.back();
  }
};

// EfficientNet.features (backbones/efficientnet.py:286-324) with PreprocLayer (:1181-1186) folded in the stem, every BatchNorm
// with epsilon `bn_eps`: 1e-3 for EfficientNetV2 (:1051) and B5-B7 (:973, :1011), torchvision's default 1e-5 for B0-B4
void plan_effnet(mtb_handle* h, float bn_eps) {
  const mtb_config& c = h->cfg;
  Planner P{h, c.proc_side, c.proc_side, 3};
  const std::string pre = "backbone.1";
  {
    Op op;
    op.type = OP_STEM;
    op.name = pre + ".0";
    op.wkey = op.name + ".0.weight";
    op.bnkey = op.name + ".1";
    op.Hin = op.Win = c.proc_side; op.Cin = 3; op.Cout = c.stages[0].cin;
    op.R = op.S = 3; op.stride = 2; op.pad_t = op.pad_l = 1; op.act = ACT_SILU;
    op.Hout = op.Wout = (c.proc_side + 2 - 3) / 2 + 1;
    op.in_buf = BUF_NONE; op.out_buf = 0;
    op.flops = 2.0 * op.Hout * op.Wout * op.Cout * 27;
    P.H = op.Hout; P.W = op.Wout; P.C = op.Cout; P.cur = 0;
    P.track(P.H, P.W, P.C);
    h->ops.push_back(op);
  }
  for (int si = 0; si < c.n_stages; ++si) {
    const mtb_stage& st = c.stages[si];
    for (int bi = 0; bi < st.layers; ++bi) {
      const bool first = bi == 0;
      const int cin = first ? st.cin : st.cout;
      const int stride = first ? st.stride : 1;
      const int shift = (first && st.bottomright) ? 1 : 0;
      const bool residual = stride == 1 && cin == st.cout;
      const int cexp = cin * st.expand;
      const int k = st.kernel;
      // dilation of the depthwise conv: din on the first block, dout on the rest (metrabs_tf effnetv2_model.py:574-600);
      // mtb_create admits dilation > 1 on MBConv rows only
      const int dil = first ? st.dilation_in : st.dilation_out;
      const int pad_total = (k - 1) * dil, pad_beg = pad_total / 2 - shift;  // fixed_padding_layer (:1127-1161)
      char key[64];
      snprintf(key, sizeof(key), "%s.%d.%d.block", pre.c_str(), si + 1, bi);
      const std::string kb = key;
      const int x_in = P.cur;
      if (st.block == 0) {  // FusedMBConv (:176-234)
        if (st.expand != 1) {
          int t1 = P.pick({x_in});
          P.conv(kb + ".0", cexp, k, stride, pad_beg, pad_total, ACT_SILU, x_in, t1);
          int t2 = P.pick({x_in, t1});
          Op& pr = P.conv(kb + ".1", st.cout, 1, 1, 0, 0, ACT_NONE, t1, t2);
          if (residual) pr.res_buf = x_in;
          P.cur = t2;
        } else {
          int t1 = P.pick({x_in});
          Op& cv = P.conv(kb + ".0", st.cout, k, stride, pad_beg, pad_total, ACT_SILU, x_in, t1);
          if (residual) cv.res_buf = x_in;
          P.cur = t1;
        }
      } else {  // MBConv (:110-173)
        int i = 0;
        int t1 = x_in;
        if (st.expand != 1) {
          t1 = P.pick({x_in});
          P.conv(kb + "." + std::to_string(i), cexp, 1, 1, 0, 0, ACT_SILU, x_in, t1);
          ++i;
        }
        int t2 = P.pick({x_in, t1});
        P.conv(kb + "." + std::to_string(i), cexp, k, stride, pad_beg, pad_total, ACT_SILU, t1, t2, true, dil);
        ++i;
        // squeeze-excitation: avgpool -> fc1 + SiLU -> fc2 + sigmoid -> scale (folded into the projection's A load)
        const std::string se = kb + "." + std::to_string(i);
        P.squeeze_excite(se, se + ".fc1", se + ".fc2", std::max(1, cin / 4), t2, ACT_SILU, ACT_SIGMOID);
        ++i;
        int t3 = P.pick({x_in, t2});
        Op& pr = P.conv(kb + "." + std::to_string(i), st.cout, 1, 1, 0, 0, ACT_NONE, t2, t3);
        pr.scale_buf = BUF_SMALL0 + 2;
        if (residual) pr.res_buf = x_in;
        P.cur = t3;
      }
    }
  }
  {
    char key[64];
    snprintf(key, sizeof(key), "%s.%d", pre.c_str(), c.n_stages + 1);
    P.conv(key, c.last_channel, 1, 1, 0, 0, ACT_SILU, P.cur, BUF_FEATURES);  // :319-324
  }
  for (Op& op : h->ops) op.bn_eps = bn_eps;
  h->feat_side = P.H;
  h->feat_c = P.C;
  h->big_elems_per_crop = P.max_elems;
  h->small_c = std::max(P.max_small, 4);
}

// get_strides_and_dilations(output_stride) (metrabs_tf/backbones/resnet.py:601-618), output_stride in {8, 16, 32}
void resnet_stride_plan(int output_stride, bool centered, int strides[3], int dil_in[3], int dil_out[3], bool brs[3]) {
  for (int i = 0; i < 3; ++i) { strides[i] = 2; dil_in[i] = dil_out[i] = 1; brs[i] = false; }
  int i_last = 0;
  for (int s_ = output_stride; s_ > 8; s_ >>= 1) ++i_last;  // log2(stride) - 3
  if (centered) brs[i_last] = true;
  for (int i = i_last + 1; i < 3; ++i) {
    strides[i] = 1;
    dil_in[i] = 1 << (i - (i_last + 1));
    dil_out[i] = dil_in[i] * 2;
  }
}

// The ResNet V1 family at output stride `stride_test` (metrabs_tf/backbones/resnet.py:75-236 stem/pool, :601-666
// stride/dilation plan; BN eps 1e-5 :71), `counts` blocks in conv2..conv5:
// * bottleneck (ResNet-50/101/152, ResNetUnified :621-666): block1_dense :239-319, every conv has a bias (:270);
// * basic (ResNet-18/34, ResNetUnifiedBasic :669-707): block1_basic_dense :322-388, no conv has a bias (stem included,
//   :704-707), conv2_block1 has an identity shortcut (conv1_shortcut=False, :689-692).
// * V1.5 (bottleneck only, ResNetUnified(v1_5=True)): _1_conv is a plain 1x1 at stride 1 (:282-283); the stack's stride and
//   the bottom-right shift move to the 3x3 _2_conv (:295-303), which takes dil_in of its stack in block1 (striding_infos_in,
//   :629-634) and dil_out in the other blocks; preprocessing torch_preproc (builder.py:99-103).
// Key schema: Keras layer names, "backbone.<layer>.{weight,bias}" / "backbone.<layer>.{weight,bias,running_mean,running_var}"
// in torch layout (the same for V1 and V1.5).
int plan_resnet(mtb_handle* h, const int counts[4], bool basic, bool v1_5) {
  const mtb_config& c = h->cfg;
  auto valid_stride = [](int s) { return s == 8 || s == 16 || s == 32; };
  if (!valid_stride(c.stride_test))
    return fail(h, MTB_ERR_UNSUPPORTED, "ResNet: stride_test must be 8, 16 or 32 (got %d)", c.stride_test);
  int strides[3], dil_in[3], dil_out[3];
  bool brs[3];
  resnet_stride_plan(c.stride_test, c.centered_stride, strides, dil_in, dil_out, brs);
  // the basic block's second 3x3 has dilation dilation_rate_test * strides / strides_test (:377-383), with `strides`
  // from the training stride plan
  int strides_train[3] = {1, 1, 1};
  if (basic) {
    if (!valid_stride(c.stride_train))
      return fail(h, MTB_ERR_UNSUPPORTED, "ResNet-18/34: stride_train must be 8, 16 or 32 (got %d)", c.stride_train);
    int di[3], dout[3];
    bool b_[3];
    resnet_stride_plan(c.stride_train, c.centered_stride, strides_train, di, dout, b_);
    for (int i = 0; i < 3; ++i)
      if (dil_out[i] * strides_train[i] / strides[i] < 1)  // the reference truncates 1 * 1 / 2 to a dilation of 0
        return fail(h, MTB_ERR_UNSUPPORTED, "ResNet-18/34: stride_train %d below stride_test %d gives a dilation of 0",
                    c.stride_train, c.stride_test);
  }
  Planner P{h, c.proc_side, c.proc_side, 3};
  const std::string pre = "backbone.";
  const float eps = 1e-5f;
  {
    Op op;
    op.type = OP_STEM;
    op.name = pre + "conv1_conv";
    op.wkey = op.name + ".weight"; op.biaskey = basic ? "" : op.name + ".bias"; op.bnkey = pre + "conv1_bn"; op.bn_eps = eps;
    op.Hin = op.Win = c.proc_side; op.Cin = 3; op.Cout = 64;
    op.R = op.S = 7; op.stride = 2; op.pad_t = op.pad_l = 3; op.act = ACT_RELU;
    op.Hout = op.Wout = (c.proc_side + 6 - 7) / 2 + 1;
    if (v1_5) {
      // torch_preproc (builder.py:99-103): (x - mean) / std, applied as x * (1/std) + (-mean/std) with both constants
      // rounded once to fp32
      const float mean[3] = {0.485f, 0.456f, 0.406f}, stdev[3] = {0.229f, 0.224f, 0.225f};
      for (int i = 0; i < 3; ++i) { op.pre_scale[i] = 1.f / stdev[i]; op.pre_shift[i] = -mean[i] / stdev[i]; }
    } else {
      const float mean[3] = {103.939f, 116.779f, 123.68f};  // caffe_preproc (builder.py:106-108): 255*x - mean, no channel swap
      for (int i = 0; i < 3; ++i) { op.pre_scale[i] = 255.f; op.pre_shift[i] = -mean[i]; }
    }
    op.in_buf = BUF_NONE; op.out_buf = 0;
    op.flops = 2.0 * op.Hout * op.Wout * 64 * 147;
    P.H = op.Hout; P.W = op.Wout; P.C = 64; P.cur = 0;
    P.track(P.H, P.W, P.C);
    h->ops.push_back(op);
    Op mp;  // ZeroPadding2D((1,1)) + MaxPooling2D(3, 2) (:187-193): the zero pad value takes part in the max
    mp.type = OP_MAXPOOL; mp.name = pre + "pool1_pool";
    mp.Hin = P.H; mp.Win = P.W; mp.Cin = mp.Cout = 64; mp.R = mp.S = 3; mp.stride = 2; mp.pad_t = mp.pad_l = 1;
    mp.Hout = (P.H + 2 - 3) / 2 + 1; mp.Wout = (P.W + 2 - 3) / 2 + 1;
    mp.in_buf = 0; mp.out_buf = 1;
    P.H = mp.Hout; P.W = mp.Wout; P.cur = 1;
    h->ops.push_back(mp);
  }
  const int filters[4] = {64, 128, 256, 512};
  for (int st = 0; st < 4; ++st) {
    for (int bi = 0; bi < counts[st]; ++bi) {
      const bool first = bi == 0;
      // V1: stride on the first conv and on the shortcut of block1; the 3x3 uses dil_out of its stack in EVERY block
      const int stride = (st > 0 && first) ? strides[st - 1] : 1;
      const int shift = (st > 0 && first && brs[st - 1]) ? 1 : 0;
      const int dil = st == 0 ? dil_in[0] : dil_out[st - 1];
      const int f = filters[st];
      char nm[64];
      snprintf(nm, sizeof(nm), "conv%d_block%d", st + 2, bi + 1);
      const std::string b = pre + nm;
      auto bias = [&](int j) { return basic ? std::string() : b + "_" + std::to_string(j) + "_conv.bias"; };
      const int x_in = P.cur;
      const int Hin = P.H, Win = P.W, Cin = P.C;
      const bool last = st == 3 && bi == counts[3] - 1;
      int sc = x_in;
      if (first && !(basic && st == 0)) {  // conv shortcut: strided 1x1 sampled at pixels shift::stride (Conv2DDenseSame)
        sc = P.pick({x_in});
        P.conv_k(b + "_0_conv", b + "_0_conv.weight", bias(0), b + "_0_bn", basic ? f : 4 * f, 1, stride, -shift, 0, ACT_NONE,
                 x_in, sc, false, 1, eps);
        Op& o = h->ops.back();
        o.Hout = Hin / stride; o.Wout = Win / stride;
        o.flops = 2.0 * o.Hout * o.Wout * o.Cout * Cin;
        P.H = Hin; P.W = Win; P.C = Cin;  // the main branch restarts from the block input
      }
      int t1 = P.pick({x_in, sc});
      if (basic) {
        // _1_conv: dense SAME 3x3 sampled at shift::stride, i.e. a strided conv with begin pad dil - shift
        P.conv_k(b + "_1_conv", b + "_1_conv.weight", "", b + "_1_bn", f, 3, stride, dil - shift, 2 * dil, ACT_RELU, x_in, t1,
                 false, dil, eps);
        Op& o = h->ops.back();
        o.Hout = Hin / stride; o.Wout = Win / stride;
        o.flops = 2.0 * o.Hout * o.Wout * o.Cout * Cin * 9;
        P.H = o.Hout; P.W = o.Wout;
        const int dil2 = (st > 0 && first) ? dil * strides_train[st - 1] / strides[st - 1] : dil;
        int t2 = P.pick({sc, t1});
        Op& o2 = P.conv_k(b + "_2_conv", b + "_2_conv.weight", "", b + "_2_bn", f, 3, 1, dil2, 2 * dil2, ACT_RELU, t1,
                          last ? BUF_FEATURES : t2, false, dil2, eps);
        o2.res_buf = sc;
        o2.res_first = true;  // relu(shortcut + x)
        P.cur = t2;
        continue;
      }
      int t2 = P.pick({x_in, sc, t1});
      if (v1_5) {
        P.conv_k(b + "_1_conv", b + "_1_conv.weight", bias(1), b + "_1_bn", f, 1, 1, 0, 0, ACT_RELU, x_in, t1, false, 1, eps);
        // _2_conv: dense SAME 3x3 sampled at shift::stride, i.e. a strided conv with begin pad dil - shift
        const int dil2 = (st > 0 && first) ? dil_in[st - 1] : dil;
        Op& o = P.conv_k(b + "_2_conv", b + "_2_conv.weight", bias(2), b + "_2_bn", f, 3, stride, dil2 - shift, 2 * dil2, ACT_RELU,
                         t1, t2, false, dil2, eps);
        o.Hout = Hin / stride; o.Wout = Win / stride;
        o.flops = 2.0 * o.Hout * o.Wout * f * f * 9;
        P.H = o.Hout; P.W = o.Wout;
      } else {
        P.conv_k(b + "_1_conv", b + "_1_conv.weight", bias(1), b + "_1_bn", f, 1, stride, -shift, 0, ACT_RELU, x_in, t1, false, 1,
                 eps);
        Op& o = h->ops.back();
        o.Hout = Hin / stride; o.Wout = Win / stride;
        o.flops = 2.0 * o.Hout * o.Wout * o.Cout * Cin;
        P.H = o.Hout; P.W = o.Wout;
        P.conv_k(b + "_2_conv", b + "_2_conv.weight", bias(2), b + "_2_bn", f, 3, 1, dil, 2 * dil, ACT_RELU, t1, t2, false, dil,
                 eps);
      }
      int t3 = P.pick({sc, t2});
      Op& o3 = P.conv_k(b + "_3_conv", b + "_3_conv.weight", bias(3), b + "_3_bn", 4 * f, 1, 1, 0, 0, ACT_RELU, t2,
                        last ? BUF_FEATURES : t3, false, 1, eps);
      o3.res_buf = sc;
      o3.res_first = true;  // relu(shortcut + x)
      P.cur = t3;
    }
  }
  h->feat_side = P.H;
  h->feat_c = P.C;
  h->big_elems_per_crop = P.max_elems;
  h->small_c = 4;
  return MTB_OK;
}

// The pre-activation ResNets (ResNetUnifiedV2, metrabs_tf/backbones/resnet.py:710-745; ResNet :160-193 with preact=True,
// use_bias=True; block2_dense :391-456; stack2_dense :558-580; BN eps 1e-5 :52) at output stride `stride_test`, `counts`
// blocks in conv2..conv5, preprocessing tf_preproc 2x - 1 (builder.py:111-113):
// * stem: conv1_conv 7x7 stride 2 with bias, no BN and no ReLU; zero pad 1 + 3x3 stride-2 max pool of the signed values;
// * block: preact = relu(_preact_bn(x)) (a 1x1 depthwise op, BN only); shortcut _0_conv(preact) (1x1 with bias, block1 of a
//   stack), x[c::2, c::2] (a 1x1 max pool with stride 2 and begin pad -c, the strided last block of conv2..conv4) or x;
//   _1_conv (1x1, BN, ReLU) and _2_conv (3x3 dense SAME sampled at c::s, dilated, BN, ReLU) without biases; out = shortcut
//   + _3_conv (1x1 with bias, no BN, no activation);
// * stride plan: the stride sits on the LAST block of conv2..conv4 (dilation dil_in of its stack, shift brs), the other
//   blocks of those stacks have stride 1 and dil_in; conv5 uses dil_out[2] throughout;
// * features: relu(post_bn(x)).
// Keys: "backbone.conv1_conv.{weight,bias}", "backbone.conv<k>_block<i>_preact_bn.*", "_0_conv.{weight,bias}",
// "_1_conv.weight", "_1_bn.*", "_2_conv.weight", "_2_bn.*", "_3_conv.{weight,bias}", "backbone.post_bn.*".
int plan_resnet_v2(mtb_handle* h, const int counts[4]) {
  const mtb_config& c = h->cfg;
  if (c.stride_test != 8 && c.stride_test != 16 && c.stride_test != 32)
    return fail(h, MTB_ERR_UNSUPPORTED, "ResNet V2: stride_test must be 8, 16 or 32 (got %d)", c.stride_test);
  int strides[3], dil_in[3], dil_out[3];
  bool brs[3];
  resnet_stride_plan(c.stride_test, c.centered_stride, strides, dil_in, dil_out, brs);
  Planner P{h, c.proc_side, c.proc_side, 3};
  const std::string pre = "backbone.";
  const float eps = 1e-5f;
  // relu(BN(x)) of the tensor in `in`, as a 1x1 depthwise op with no conv weight
  auto preact = [&](const std::string& name, int in, int out) {
    P.conv_k(name, "", "", name, P.C, 1, 1, 0, 0, ACT_RELU, in, out, true, 1, eps);
  };
  {
    Op op;
    op.type = OP_STEM;
    op.name = pre + "conv1_conv";
    op.wkey = op.name + ".weight"; op.biaskey = op.name + ".bias";
    op.Hin = op.Win = c.proc_side; op.Cin = 3; op.Cout = 64;
    op.R = op.S = 7; op.stride = 2; op.pad_t = op.pad_l = 3; op.act = ACT_NONE;  // pre_scale / pre_shift: 2x - 1
    op.Hout = op.Wout = (c.proc_side + 6 - 7) / 2 + 1;
    op.in_buf = BUF_NONE; op.out_buf = 0;
    op.flops = 2.0 * op.Hout * op.Wout * 64 * 147;
    P.H = op.Hout; P.W = op.Wout; P.C = 64;
    P.track(P.H, P.W, P.C);
    h->ops.push_back(op);
    Op mp;
    mp.type = OP_MAXPOOL; mp.name = pre + "pool1_pool";
    mp.Hin = P.H; mp.Win = P.W; mp.Cin = mp.Cout = 64; mp.R = mp.S = 3; mp.stride = 2; mp.pad_t = mp.pad_l = 1;
    mp.Hout = (P.H + 2 - 3) / 2 + 1; mp.Wout = (P.W + 2 - 3) / 2 + 1;
    mp.in_buf = 0; mp.out_buf = 1;
    P.H = mp.Hout; P.W = mp.Wout; P.cur = 1;
    h->ops.push_back(mp);
  }
  const int filters[4] = {64, 128, 256, 512};
  // the previous block's _3_conv reads these while a fused launch writes the pre-activation: keep it out of them
  int prev_in = BUF_NONE, prev_res = BUF_NONE;
  for (int st = 0; st < 4; ++st) {
    for (int bi = 0; bi < counts[st]; ++bi) {
      const bool first = bi == 0, last_of_stack = bi == counts[st] - 1;
      const bool strided = st < 3 && last_of_stack && strides[st] == 2;
      const int stride = strided ? 2 : 1;
      const int shift = (st < 3 && last_of_stack && brs[st]) ? 1 : 0;
      const int dil = st < 3 ? dil_in[st] : dil_out[2];
      const int f = filters[st];
      char nm[64];
      snprintf(nm, sizeof(nm), "conv%d_block%d", st + 2, bi + 1);
      const std::string b = pre + nm;
      const int x_in = P.cur;
      const int Hin = P.H, Win = P.W, Cin = P.C;
      const int pa = P.pick({x_in, prev_in, prev_res});
      preact(b + "_preact_bn", x_in, pa);
      int sc = x_in;
      if (first) {
        sc = P.pick({x_in, pa});
        P.conv_k(b + "_0_conv", b + "_0_conv.weight", b + "_0_conv.bias", "", 4 * f, 1, 1, 0, 0, ACT_NONE, pa, sc, false, 1, eps);
        P.H = Hin; P.W = Win; P.C = Cin;  // the main branch restarts from the pre-activation
      } else if (stride > 1 || shift) {  // x[c::2, c::2]: Cropping2D(c) + MaxPooling2D(1, 2)
        sc = P.pick({x_in, pa});
        Op mp;
        mp.type = OP_MAXPOOL; mp.name = b + "_shortcut_pool";
        mp.Hin = Hin; mp.Win = Win; mp.Cin = mp.Cout = Cin; mp.stride = stride; mp.pad_t = mp.pad_l = -shift;
        mp.Hout = Hin / stride; mp.Wout = Win / stride;
        mp.in_buf = x_in; mp.out_buf = sc;
        P.track(mp.Hout, mp.Wout, Cin);
        h->ops.push_back(mp);
      }
      const int t1 = P.pick({pa, sc});
      P.conv_k(b + "_1_conv", b + "_1_conv.weight", "", b + "_1_bn", f, 1, 1, 0, 0, ACT_RELU, pa, t1, false, 1, eps);
      const int t2 = P.pick({sc, t1});
      // _2_conv: dense SAME 3x3 sampled at shift::stride, i.e. a strided conv with begin pad dil - shift
      Op& o2 = P.conv_k(b + "_2_conv", b + "_2_conv.weight", "", b + "_2_bn", f, 3, stride, dil - shift, 2 * dil, ACT_RELU, t1, t2,
                        false, dil, eps);
      o2.Hout = Hin / stride; o2.Wout = Win / stride;
      o2.flops = 2.0 * o2.Hout * o2.Wout * f * f * 9;
      P.H = o2.Hout; P.W = o2.Wout;
      const int t3 = P.pick({sc, t2});
      Op& o3 = P.conv_k(b + "_3_conv", b + "_3_conv.weight", b + "_3_conv.bias", "", 4 * f, 1, 1, 0, 0, ACT_NONE, t2, t3, false, 1, eps);
      o3.res_buf = sc;
      P.cur = t3;
      prev_in = t2; prev_res = sc;
    }
  }
  preact(pre + "post_bn", P.cur, BUF_FEATURES);
  h->feat_side = P.H;
  h->feat_c = P.C;
  h->big_elems_per_crop = P.max_elems;
  h->small_c = 4;
  return MTB_OK;
}

// One row of a MobileNetV3 table: _inverted_res_block(x, expansion, filters, kernel, stride, se_ratio, activation, ...)
// with the expanded width already rounded by _depth
struct MbV3Row { int exp_ch, filters, k, stride; bool se; int act; bool br; };
// MobileNetV3-Small (metrabs_tf/backbones/mobilenet_v3.py:364-384)
const MbV3Row kMobileNetV3Small[] = {
    {16, 16, 3, 2, true, ACT_RELU, false},     {72, 24, 3, 2, false, ACT_RELU, false},
    {88, 24, 3, 1, false, ACT_RELU, false},    {96, 40, 5, 2, true, ACT_HSWISH, false},
    {240, 40, 5, 1, true, ACT_HSWISH, false},  {240, 40, 5, 1, true, ACT_HSWISH, false},
    {120, 48, 5, 1, true, ACT_HSWISH, false},  {144, 48, 5, 1, true, ACT_HSWISH, false},
    {288, 96, 5, 2, true, ACT_HSWISH, true},   {576, 96, 5, 1, true, ACT_HSWISH, false},
    {576, 96, 5, 1, true, ACT_HSWISH, false}};
// MobileNetV3-Large (:403-428): block 0 has no expand, the ReLU blocks 3-5 use 5x5 kernels with SE
const MbV3Row kMobileNetV3Large[] = {
    {16, 16, 3, 1, false, ACT_RELU, false},     {64, 24, 3, 2, false, ACT_RELU, false},
    {72, 24, 3, 1, false, ACT_RELU, false},     {72, 40, 5, 2, true, ACT_RELU, false},
    {120, 40, 5, 1, true, ACT_RELU, false},     {120, 40, 5, 1, true, ACT_RELU, false},
    {240, 80, 3, 2, false, ACT_HSWISH, false},  {200, 80, 3, 1, false, ACT_HSWISH, false},
    {184, 80, 3, 1, false, ACT_HSWISH, false},  {184, 80, 3, 1, false, ACT_HSWISH, false},
    {480, 112, 3, 1, true, ACT_HSWISH, false},  {672, 112, 3, 1, true, ACT_HSWISH, false},
    {672, 160, 5, 2, true, ACT_HSWISH, true},   {960, 160, 5, 1, true, ACT_HSWISH, false},
    {960, 160, 5, 1, true, ACT_HSWISH, false}};
// the minimalistic forms (minimalistic=True, :250-257): the same expanded widths, strides and bottom-right rows with every
// kernel 3, every activation ReLU and no squeeze-excitation
const MbV3Row kMobileNetV3SmallMini[] = {
    {16, 16, 3, 2, false, ACT_RELU, false},   {72, 24, 3, 2, false, ACT_RELU, false},
    {88, 24, 3, 1, false, ACT_RELU, false},   {96, 40, 3, 2, false, ACT_RELU, false},
    {240, 40, 3, 1, false, ACT_RELU, false},  {240, 40, 3, 1, false, ACT_RELU, false},
    {120, 48, 3, 1, false, ACT_RELU, false},  {144, 48, 3, 1, false, ACT_RELU, false},
    {288, 96, 3, 2, false, ACT_RELU, true},   {576, 96, 3, 1, false, ACT_RELU, false},
    {576, 96, 3, 1, false, ACT_RELU, false}};
const MbV3Row kMobileNetV3LargeMini[] = {
    {16, 16, 3, 1, false, ACT_RELU, false},   {64, 24, 3, 2, false, ACT_RELU, false},
    {72, 24, 3, 1, false, ACT_RELU, false},   {72, 40, 3, 2, false, ACT_RELU, false},
    {120, 40, 3, 1, false, ACT_RELU, false},  {120, 40, 3, 1, false, ACT_RELU, false},
    {240, 80, 3, 2, false, ACT_RELU, false},  {200, 80, 3, 1, false, ACT_RELU, false},
    {184, 80, 3, 1, false, ACT_RELU, false},  {184, 80, 3, 1, false, ACT_RELU, false},
    {480, 112, 3, 1, false, ACT_RELU, false}, {672, 112, 3, 1, false, ACT_RELU, false},
    {672, 160, 3, 2, false, ACT_RELU, true},  {960, 160, 3, 1, false, ACT_RELU, false},
    {960, 160, 3, 1, false, ACT_RELU, false}};

// MobileNetV3 (metrabs_tf/backbones/mobilenet_v3.py:490-553 block, :465-487 SE, :258-296 stem and Conv_1 / Conv_2,
// :556-575 correct_pad; preprocessing 255*x then Rescaling(1/127.5, -1) = 2x-1, builder.py:116-117), `n_rows` rows of
// `rows` and a last point conv (Conv_2) of `last_point_ch` channels: 1024 for Small, 1280 for Large.  `act` is the
// activation of the stem, Conv_1 and Conv_2: hard-swish, or ReLU in the minimalistic form.
int plan_mobilenetv3(mtb_handle* h, const MbV3Row* rows, int n_rows, int last_point_ch, int act) {
  const mtb_config& c = h->cfg;
  Planner P{h, c.proc_side, c.proc_side, 3};
  const std::string pre = "backbone.";
  {
    Op op;
    op.type = OP_STEM;
    op.name = pre + "Conv";
    op.wkey = op.name + ".weight"; op.bnkey = op.name + ".BatchNorm";
    op.Hin = op.Win = c.proc_side; op.Cin = 3; op.Cout = 16;
    op.R = op.S = 3; op.stride = 2; op.act = act;
    op.Hout = op.Wout = (c.proc_side + 1) / 2;
    // TF 'same' with stride 2: pad_total = max((out-1)*2 + 3 - in, 0), begin = pad_total / 2  (even input: (0,1))
    const int pad_total = std::max((op.Hout - 1) * 2 + 3 - c.proc_side, 0);
    op.pad_t = op.pad_l = pad_total / 2;
    op.in_buf = BUF_NONE; op.out_buf = 0;
    op.flops = 2.0 * op.Hout * op.Wout * 16 * 27;
    P.H = op.Hout; P.W = op.Wout; P.C = 16; P.cur = 0;
    P.track(P.H, P.W, P.C);
    h->ops.push_back(op);
  }
  auto depth8 = [](double v) {  // _depth (:449-456)
    int nv = std::max(8, (int)(v + 4) / 8 * 8);
    if (nv < 0.9 * v) nv += 8;
    return nv;
  };
  for (int bi = 0; bi < n_rows; ++bi) {
    const MbV3Row& r = rows[bi];
    const std::string b = pre + (bi == 0 ? std::string("expanded_conv") : "expanded_conv_" + std::to_string(bi));
    const int x_in = P.cur, cin = P.C;
    int t1 = x_in;
    if (bi != 0) {
      t1 = P.pick({x_in});
      P.conv_k(b + ".expand", b + ".expand.weight", "", b + ".expand.BatchNorm", r.exp_ch, 1, 1, 0, 0, r.act, x_in, t1);
    }
    int t2 = P.pick({x_in, t1});
    const int shift = (r.br && c.centered_stride) ? 1 : 0;
    const int pad_total = r.k - 1, pad_beg = (r.k - 1) / 2 - (r.stride == 2 ? shift : 0);
    P.conv_k(b + ".depthwise", b + ".depthwise.weight", "", b + ".depthwise.BatchNorm", r.exp_ch, r.k, r.stride, pad_beg, pad_total,
             r.act, t1, t2, true);
    if (r.se)
      P.squeeze_excite(b + ".squeeze_excite", b + ".squeeze_excite.Conv", b + ".squeeze_excite.Conv_1", depth8(r.exp_ch * 0.25), t2,
                       ACT_RELU, ACT_HSIGMOID);
    int t3 = P.pick({x_in, t2});
    Op& pr = P.conv_k(b + ".project", b + ".project.weight", "", b + ".project.BatchNorm", r.filters, 1, 1, 0, 0, ACT_NONE, t2, t3);
    if (r.se) pr.scale_buf = BUF_SMALL0 + 2;
    if (r.stride == 1 && cin == r.filters) pr.res_buf = x_in;
    P.cur = t3;
  }
  {
    int t1 = P.pick({P.cur});
    P.conv_k(pre + "Conv_1", pre + "Conv_1.weight", "", pre + "Conv_1.BatchNorm", depth8(P.C * 6), 1, 1, 0, 0, act, P.cur, t1);
    P.conv_k(pre + "Conv_2", pre + "Conv_2.weight", pre + "Conv_2.bias", "", last_point_ch, 1, 1, 0, 0, act, t1, BUF_FEATURES);
  }
  h->feat_side = P.H;
  h->feat_c = P.C;
  h->big_elems_per_crop = P.max_elems;
  h->small_c = std::max(P.max_small, 4);
  return MTB_OK;
}

// block counts of conv2..conv5 (resnet.py:746-788, V1.5 :791-800)
struct ResNetArch { int arch; int counts[4]; bool basic; bool v1_5 = false; };
const ResNetArch kResNets[] = {{MTB_ARCH_RESNET18, {2, 2, 2, 2}, true},    {MTB_ARCH_RESNET34, {3, 4, 6, 3}, true},
                               {MTB_ARCH_RESNET50, {3, 4, 6, 3}, false},   {MTB_ARCH_RESNET101, {3, 4, 23, 3}, false},
                               {MTB_ARCH_RESNET152, {3, 8, 36, 3}, false},
                               {MTB_ARCH_RESNET50V1_5, {3, 4, 6, 3}, false, true},
                               {MTB_ARCH_RESNET101V1_5, {3, 4, 23, 3}, false, true},
                               {MTB_ARCH_RESNET152V1_5, {3, 8, 36, 3}, false, true}};
// block counts of the pre-activation nets (resnet.py:803-831)
const ResNetArch kResNetsV2[] = {{MTB_ARCH_RESNET50V2, {3, 4, 6, 3}, false}, {MTB_ARCH_RESNET101V2, {3, 4, 23, 3}, false},
                                 {MTB_ARCH_RESNET152V2, {3, 8, 36, 3}, false}};

int plan(mtb_handle* h) {
  const mtb_config& c = h->cfg;
  h->ops.clear();
  const ResNetArch* resnet = nullptr;
  for (const ResNetArch& r : kResNets)
    if (c.arch == r.arch) resnet = &r;
  const ResNetArch* resnet_v2 = nullptr;
  for (const ResNetArch& r : kResNetsV2)
    if (c.arch == r.arch) resnet_v2 = &r;
  if (resnet) {
    int rc = plan_resnet(h, resnet->counts, resnet->basic, resnet->v1_5);
    if (rc) return rc;
  } else if (resnet_v2) {
    int rc = plan_resnet_v2(h, resnet_v2->counts);
    if (rc) return rc;
  } else switch (c.arch) {
    case MTB_ARCH_EFFNET: plan_effnet(h, 1e-3f); break;
    case MTB_ARCH_EFFNET_EPS1E5: plan_effnet(h, 1e-5f); break;
    case MTB_ARCH_MOBILENETV3_SMALL: { int rc = plan_mobilenetv3(h, kMobileNetV3Small, (int)std::size(kMobileNetV3Small), 1024, ACT_HSWISH); if (rc) return rc; break; }
    case MTB_ARCH_MOBILENETV3_LARGE: { int rc = plan_mobilenetv3(h, kMobileNetV3Large, (int)std::size(kMobileNetV3Large), 1280, ACT_HSWISH); if (rc) return rc; break; }
    case MTB_ARCH_MOBILENETV3_SMALL_MINI: { int rc = plan_mobilenetv3(h, kMobileNetV3SmallMini, (int)std::size(kMobileNetV3SmallMini), 1024, ACT_RELU); if (rc) return rc; break; }
    case MTB_ARCH_MOBILENETV3_LARGE_MINI: { int rc = plan_mobilenetv3(h, kMobileNetV3LargeMini, (int)std::size(kMobileNetV3LargeMini), 1280, ACT_RELU); if (rc) return rc; break; }
    case MTB_ARCH_HEAD_ONLY:
      h->feat_side = c.proc_side / c.stride_test;
      h->feat_c = c.feature_channels;
      h->big_elems_per_crop = 0;
      h->small_c = 4;
      break;
    default: return fail(h, MTB_ERR_UNSUPPORTED, "arch %d is not built yet", c.arch);
  }
  h->flops_per_crop = 0;
  for (auto& op : h->ops) h->flops_per_crop += op.flops;
  // head: MetrabsHeads.conv_final, 1x1 conv with bias (models/metrabs.py:73)
  Op& hd = h->head;
  hd = Op();
  hd.type = OP_CONV;
  hd.name = "heatmap_heads.conv_final";
  hd.wkey = hd.name + ".weight";
  hd.biaskey = hd.name + ".bias";
  hd.Hin = hd.Win = hd.Hout = hd.Wout = h->feat_side;
  hd.Cin = h->feat_c;
  hd.act = ACT_NONE;
  size_head(h);
  return MTB_OK;
}

// ------------------------------------------------------------------------------------------------ weights
const HostTensor* find(const mtb_handle* h, const std::string& k) {
  auto it = h->raw.find(k);
  return it == h->raw.end() ? nullptr : &it->second;
}

int upload(mtb_handle* h, const void* host, size_t bytes, void** dev) {
  const char* e = upload_dev(h->dev_allocs, dev, host, bytes);
  return e ? fail(h, MTB_ERR_CUDA, "weight upload: %s", e) : MTB_OK;
}

int prepare_op_weights(mtb_handle* h, Op& op) {
  if (op.type == OP_POOL || op.type == OP_MAXPOOL) return MTB_OK;
  // a BatchNorm alone (ResNet V2 pre-activation): a 1x1 depthwise op whose conv weight is 1
  HostTensor ones;
  if (op.wkey.empty() && op.depthwise && op.R == 1 && op.S == 1) ones = {std::vector<float>(op.Cout, 1.f), {op.Cout, 1, 1, 1}};
  const HostTensor* w = op.wkey.empty() ? &ones : find(h, op.wkey);
  if (!w || w->data.empty()) return fail(h, MTB_ERR_MISSING_WEIGHT, "missing weight '%s'", op.wkey.c_str());
  const int cin_g = op.depthwise ? 1 : op.Cin;
  const int64_t expect[4] = {op.Cout, cin_g, op.R, op.S};
  bool shape_ok = w->shape.size() == 4 && std::equal(expect, expect + 4, w->shape.begin());
  if (!shape_ok && op.pad_ok && w->shape.size() == 4 && w->shape[2] == op.R && w->shape[3] == op.S &&
      w->shape[0] <= op.Cout && w->shape[0] > op.Cout - 4 && w->shape[1] <= cin_g && w->shape[1] > cin_g - 4)
    shape_ok = true;
  if (!shape_ok)
    return fail(h, MTB_ERR_INVALID_ARG, "weight '%s' has the wrong shape (want [%d,%d,%d,%d])", op.wkey.c_str(),
                op.Cout, cin_g, op.R, op.S);
  const int n_real = (int)w->shape[0], c_real = (int)w->shape[1];
  std::vector<double> scale(op.Cout, 1.0), shift(op.Cout, 0.0);
  if (!op.biaskey.empty()) {
    const HostTensor* b = find(h, op.biaskey);
    if (!b) return fail(h, MTB_ERR_MISSING_WEIGHT, "missing weight '%s'", op.biaskey.c_str());
    if ((int)b->data.size() != n_real) return fail(h, MTB_ERR_INVALID_ARG, "bias '%s' has the wrong size", op.biaskey.c_str());
    for (int n = 0; n < n_real; ++n) shift[n] = b->data[n];
  }
  if (!op.bnkey.empty()) {
    const HostTensor *g = find(h, op.bnkey + ".weight"), *b = find(h, op.bnkey + ".bias"),
                     *m = find(h, op.bnkey + ".running_mean"), *v = find(h, op.bnkey + ".running_var");
    if (!g || !b || !m || !v) return fail(h, MTB_ERR_MISSING_WEIGHT, "missing batch-norm tensors '%s.*'", op.bnkey.c_str());
    for (const HostTensor* t : {g, b, m, v})
      if ((int)t->data.size() != n_real)
        return fail(h, MTB_ERR_INVALID_ARG, "batch-norm tensors '%s.*' must have %d elements (got %zu)", op.bnkey.c_str(), n_real,
                    t->data.size());
    for (int n = 0; n < n_real; ++n) {
      double s = (double)g->data[n] / std::sqrt((double)v->data[n] + (double)op.bn_eps);
      scale[n] = s;
      shift[n] = (shift[n] - (double)m->data[n]) * s + (double)b->data[n];
    }
  }
  const int K = op.R * op.S * cin_g;
  std::vector<float> wk((size_t)K * op.Cout, 0.f), bias(op.Cout, 0.f);
  for (int n = 0; n < n_real; ++n) {
    bias[n] = (float)shift[n];
    for (int c = 0; c < c_real; ++c)
      for (int r = 0; r < op.R; ++r)
        for (int s = 0; s < op.S; ++s) {
          double v = (double)w->data[(((size_t)n * c_real + c) * op.R + r) * op.S + s] * scale[n];
          wk[((size_t)(r * op.S + s) * cin_g + c) * op.Cout + n] = (float)v;
        }
  }
  const bool tc_like = tc_eligible(op.type == OP_CONV, op.depthwise, op.small_io, op.R, op.stride, op.Cin, op.Cout);
  if (storage(h) == ST_BF16 && tc_like)  // both bf16 modes see the same bf16-rounded GEMM weights
    for (float& v : wk) v = __bfloat162float(host_bf16(v));
  if (storage(h) == ST_F16 && tc_like)  // both fp16 modes see the same fp16-rounded GEMM weights
    for (float& v : wk) v = __half2float(host_f16(v));
  int rc = upload(h, wk.data(), wk.size() * 4, (void**)&op.d_w);
  if (rc) return rc;
  rc = upload(h, bias.data(), bias.size() * 4, (void**)&op.d_bias);
  if (rc) return rc;
  // the tensor-core kernels' own weight copies (the fused head prepares its own in mtb_finalize_weights)
  if (kKernels[op.kernel].cls == KC_TC_GEMM) {
    const char* e = with_storage16(h, [&](auto* tag) {
      return tc_prepare_weights<std::remove_pointer_t<decltype(tag)>>(op.tc, wk.data(), bias.data(), K, op.Cout, op.R, op.S, op.Cin,
                                                                      h->dev_allocs);
    });
    if (e) return fail(h, MTB_ERR_CUDA, "tensor-core weight prep for '%s': %s", op.name.c_str(), e);
  }
  if (kKernels[op.kernel].cls == KC_TC32) {
    const char* e = tc32_prepare_weights(op.tc32, wk.data(), bias.data(), K, op.Cout, op.R, op.S, op.Cin, h->dev_allocs);
    if (e) return fail(h, MTB_ERR_CUDA, "3xTF32 weight prep for '%s': %s", op.name.c_str(), e);
  }
  return MTB_OK;
}

// --------------------------------------------------------------------------------------------- workspace
struct Workspace {
  char* base;
  size_t big_stride, small_stride;
  size_t off_small, off_features, off_logits, off_c2d, off_c3d, off_n2d, off_partial, off_latents, off_bones, total;
};

// scratch of bone_solve_kernel for B crops: per-bone coefficients [B][E] float4, then z, z_new and the objective [B]
struct BoneScratch {
  float4* coef;
  float *z, *z_new, *obj;
};
size_t bone_scratch_bytes(const mtb_handle* h, int B) {
  return align_up((size_t)B * h->bone_len.size() * 16, 256) + 3 * align_up((size_t)B * 4, 256);
}
BoneScratch bone_scratch(const mtb_handle* h, int B, void* base) {
  char* p = (char*)base;
  BoneScratch s;
  s.coef = (float4*)p; p += align_up((size_t)B * h->bone_len.size() * 16, 256);
  s.z = (float*)p;     p += align_up((size_t)B * 4, 256);
  s.z_new = (float*)p; p += align_up((size_t)B * 4, 256);
  s.obj = (float*)p;
  return s;
}

Workspace layout(const mtb_handle* h, int B, void* base) {
  Workspace w;
  w.base = (char*)base;
  const size_t es = elem_size(h);
  w.big_stride = align_up(h->big_elems_per_crop * (size_t)B * es, 1024);
  w.small_stride = align_up((size_t)h->small_c * B * 4 * kPoolSlices, 1024);
  size_t o = w.big_stride * kNumBig;
  w.off_small = o; o += w.small_stride * kNumSmall;
  const size_t P = (size_t)h->feat_side * h->feat_side;
  w.off_features = o; o += align_up(P * h->feat_c * B * es, 1024);
  const size_t J = (size_t)head_points(h);
  const int N = (head_channels(h) + 3) / 4 * 4;
  w.off_logits = o; o += align_up(std::max<size_t>(P, 4) * N * B * 4, 1024);  // also the fused head's state scratch
  w.off_c2d = o; o += align_up((size_t)B * J * 2 * 4, 1024);
  w.off_c3d = o; o += align_up((size_t)B * J * 3 * 4, 1024);
  w.off_n2d = o; o += align_up((size_t)B * J * 2 * 4, 1024);
  w.off_partial = o; o += align_up((size_t)B * 2 * 8, 1024);
  w.off_latents = o;  // latent-point model: absolute latents [B,L,3] between the reconstruction and the recombination
  if (h->n_latents > 0) o += align_up((size_t)B * J * 3 * 4, 1024);
  w.off_bones = o;  // Model25D: the bone-length solve's scratch
  if (h->model_class == MTB_MODEL_25D) o += align_up(bone_scratch_bytes(h, B), 1024);
  w.total = o;
  return w;
}

void* buf_ptr(const Workspace& w, int id, void* features) {
  if (id == BUF_FEATURES) return features;
  if (id < 0) return nullptr;
  if (id < kNumBig) return w.base + w.big_stride * id;
  return w.base + w.off_small + w.small_stride * (id - BUF_SMALL0);
}

// ---------------------------------------------------------------------------------------------- profiler
struct ProfScope {
  mtb_handle* h;
  cudaStream_t st;
  bool on;
  // per_op = false keeps the launch out of the per-op table (the in-place SE scale pass is a class of its own; counting it
  // under the projection GEMM's op index made that GEMM look twice as slow as it is)
  ProfScope(mtb_handle* h_, int cls, double flops, double bytes, cudaStream_t st_, bool per_op = true) : h(h_), st(st_) {
    on = (h->prof_mask >> cls) & 1u;
    if (!on) return;
    if (h->prof_used + 2 > h->prof_events.size()) {
      for (int i = 0; i < 2; ++i) {
        cudaEvent_t e;
        cudaEventCreate(&e);
        h->prof_events.push_back(e);
      }
    }
    h->prof_cls.push_back(cls);
    h->prof_op.push_back(per_op ? h->prof_cur_op : -1);
    h->prof_flops.push_back(flops);
    h->prof_bytes.push_back(bytes);
    cudaEventRecord(h->prof_events[h->prof_used], st);
  }
  ~ProfScope() {
    if (!on) return;
    cudaEventRecord(h->prof_events[h->prof_used + 1], st);
    h->prof_used += 2;
  }
};

// shapes covered by the strip depthwise kernels (dwconv3x3_pool_16b_kernel / dwconv3x3_pool_f32_kernel)
bool dw_strip_eligible(const Op& op) {
  return op.type == OP_DW && op.R == 3 && op.S == 3 && op.dil == 1 && op.Cout % 8 == 0 && (op.stride == 1 || op.stride == 2) &&
         (op.act == ACT_SILU || op.act == ACT_RELU || op.act == ACT_HSWISH);
}

// shapes covered by dwconv5x5_16b_kernel
bool dw5x5_eligible(const Op& op) {
  return op.type == OP_DW && op.R == 5 && op.S == 5 && op.dil == 1 && op.Cout % 8 == 0 && (op.stride == 1 || op.stride == 2) &&
         (op.act == ACT_SILU || op.act == ACT_RELU || op.act == ACT_HSWISH);
}

constexpr int kDwOW = 4;  // outputs per thread along W in dwconv3x3_pool_16b_kernel (measured: 4 -> 3.65 ms, 2 -> 4.25 ms per 128 crops)
constexpr int kDw5OW = 4;  // outputs per thread along W in dwconv5x5_16b_kernel

// block shape of the pooling dwconv5x5_16b_kernel for C channels: gridDim.x chunks of cb channel vectors, `groups` groups of
// cb threads per block.  The fewest chunks that keep at least 192 of a block's 256 threads busy (C = 1152: 2 chunks of 72
// vectors x 3 groups = 216 threads instead of 144 x 1).
struct Dw5PoolShape { int chunks, cb, groups; };
Dw5PoolShape dw5_pool_shape(int C) {
  const int cv = C / 8;
  for (int n = (cv + 255) / 256;; ++n) {
    const int cb = (cv + n - 1) / n, groups = 256 / cb;
    if (cb * groups >= 192 || n >= cv) return {n, cb, groups};
  }
}

// f(stride, act) with both compile-time constants (stride 1 or 2, act one of ACTS): the launch of a templated depthwise kernel
template <int... ACTS, typename F>
cudaError_t dw_dispatch(const Op& op, F&& f) {
  return with_const<1, 2>(op.stride, cudaErrorNotSupported, [&](auto s) {
    return with_const<ACTS...>(op.act, cudaErrorNotSupported, [&](auto a) { return f(s, a); });
  });
}

// ---------------------------------------------------------------------------------------------- kernel choice
bool stem_fast_enabled() {  // MTB_STEM_FAST=0: the generic stem kernel (A/B runs, bit-equality test)
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("MTB_STEM_FAST");
    v = (e && e[0] == '0') ? 0 : 1;
  }
  return v == 1;
}

// Picks the kernel of a depthwise op and the number of partial pooling slices it writes (fc1 sums that many).  bf16 and fp16
// tensor-core modes: 5x5 ops run dwconv5x5_16b_kernel, which pools for SiLU (EfficientNet-B) and does not pool for ReLU /
// hard-swish (MobileNetV3); 3x3 stride-1 ops run the TMA-staged kernel when a plan fits, the other 3x3 ops the 16-bit strip
// kernel; 3x3 stride-1 SiLU ops with dilation 2 or 4 and SAME padding (the dilated EfficientNetV2 stages) run the TMA-staged
// kernel phase by phase when a plan fits.  3xTF32 mode: the fp32 strip kernel (exact activation) for undilated 3x3 ops.  Other
// modes and shapes: the generic kernel, which does not pool.
mtb_kernel choose_dw(const mtb_handle* h, Op& op) {
  if (op.R == 3 && op.S == 3 && (op.dil == 2 || op.dil == 4)) {
    if (!is_tc16(h) || op.stride != 1 || op.act != ACT_SILU || op.Cout % 8 != 0 || op.pad_t != op.dil || op.pad_l != op.dil ||
        op.Hin != op.Hout || op.Win != op.Wout)
      return MTB_DW_GENERIC;
    const DwTmaPlan pl = dw_tma_plan((op.Hout + op.dil - 1) / op.dil, (op.Wout + op.dil - 1) / op.dil, op.dil);
    if (!pl.ok || pl.n_rb > kPoolSlices) return MTB_DW_GENERIC;
    op.dw_plan = pl;
    op.pool_slices = pl.n_rb;
    return MTB_DW_TMA_DIL;
  }
  if (dw5x5_eligible(op)) {
    if (!is_tc16(h)) return MTB_DW_GENERIC;
    if (op.act != ACT_SILU) return MTB_DW_5X5_16B;
    const int strips = op.Hout * ((op.Wout + kDw5OW - 1) / kDw5OW);
    const int groups = dw5_pool_shape(op.Cout).groups;
    op.pool_slices = std::min((strips + groups - 1) / groups, kPoolSlices);
    return MTB_DW_5X5_POOL_16B;
  }
  if (!dw_strip_eligible(op) || !(is_tc16(h) || h->cfg.precision == MTB_PRECISION_TF32X3)) return MTB_DW_GENERIC;
  if (is_tc16(h) && op.stride == 1 && op.Hin == op.Hout && op.Win == op.Wout) {
    const DwTmaPlan pl = dw_tma_plan(op.Hout, op.Wout);
    if (pl.ok && pl.n_rb <= kPoolSlices) {
      op.dw_plan = pl;
      op.pool_slices = pl.n_rb;
      return MTB_DW_TMA;
    }
  }
  const int strips = op.Hout * ((op.Wout + kDwOW - 1) / kDwOW);
  op.pool_slices = std::min((strips + 7) / 8, kPoolSlices);
  return is_tc16(h) ? MTB_DW_STRIP_16B : MTB_DW_STRIP_F32;
}

// A conv or GEMM op: the SE fully-connected layers run conv_igemm_kernel in fp32; the bf16 and fp16 tensor-core modes run
// tc_conv_kernel where tc_eligible, with the SE scale inside the GEMM or in se_scale_kernel ahead of it (tc_se_in_gemm), or
// tc_conv3x3s1_kernel for the shapes it takes; the 3xTF32 mode runs tc32_conv_kernel where tc32_eligible; everything else
// runs conv_igemm_kernel.
mtb_kernel choose_conv(const mtb_handle* h, const Op& op) {
  if (op.small_io) return MTB_SE_FC;
  if (is_tc16(h) && tc_eligible(true, op.depthwise, op.small_io, op.R, op.stride, op.Cin, op.Cout)) {
    if (op.scale_buf != BUF_NONE) return tc_se_in_gemm(op.Cout) ? MTB_TC_CONV_SE : MTB_SE_SCALE_TC_CONV;
    return tc3x3s1_eligible(op.R, op.S, op.stride, op.dil, op.Cin, op.Cout, op.act) ? MTB_TC_CONV3X3S1 : MTB_TC_CONV;
  }
  if (h->cfg.precision == MTB_PRECISION_TF32X3 && tc32_eligible(true, op.depthwise, op.small_io, op.R, op.stride, op.Cin, op.Cout))
    return MTB_TC32;
  return MTB_IGEMM;
}

// Sets Op::kernel of every backbone op and of the head, and which depthwise ops pool for the SE op behind them.  (Whether a
// FusedMBConv pair runs as one fmb_kernel launch is decided once its tensor-core weights exist, in mtb_finalize_weights.)
void choose_kernels(mtb_handle* h) {
  for (size_t i = 0; i < h->ops.size(); ++i) {
    Op& op = h->ops[i];
    switch (op.type) {
      case OP_STEM: {
        // stem3x3s2_kernel: EfficientNet's 3x3 stride-2 stem with 24 or 32 channels; stem_conv_wide_kernel: a multiple of 32,
        // 24 or 16 channels
        const bool s2 = op.R == 3 && op.S == 3 && op.Cin == 3 && op.stride == 2 && (op.Cout == 32 || op.Cout == 24);
        op.kernel = s2 && stem_fast_enabled()                                  ? MTB_STEM_3X3S2
                    : op.Cout % 32 == 0 || op.Cout % 24 == 0 || op.Cout % 16 == 0 ? MTB_STEM_WIDE
                                                                                 : MTB_STEM_GENERIC;
        break;
      }
      case OP_MAXPOOL: op.kernel = MTB_MAXPOOL; break;
      case OP_POOL: op.kernel = i > 0 && h->ops[i - 1].fused_pool ? MTB_POOL_FUSED : MTB_POOL_MEAN; break;
      case OP_DW: op.kernel = choose_dw(h, op); break;
      case OP_CONV: op.kernel = choose_conv(h, op); break;
    }
    op.fused_pool = kKernels[op.kernel].pools && i + 1 < h->ops.size() && h->ops[i + 1].type == OP_POOL;
  }
  // the head: tc_head_kernel when a fused tile fits the feature map, else a GEMM into logits (tc32_conv_kernel where a conv
  // of its shape runs it) and softargmax_bhwn_kernel
  Op& hd = h->head;
  int bnp, cpt, npt;
  if (is_tc16(h) && tc_head_plan(h->feat_side * h->feat_side, &bnp, &cpt, &npt)) hd.kernel = MTB_HEAD_FUSED;
  else if (choose_conv(h, hd) == MTB_TC32) hd.kernel = MTB_HEAD_TC32;
  else hd.kernel = MTB_HEAD_IGEMM;
}

// profiler class of a backbone op: fmb_kernel for the first op of a fused FusedMBConv block
int op_class(const Op& op) { return op.fmb.ready ? KC_FMB : op.preact_next ? KC_TC_PREACT : kKernels[op.kernel].cls; }

double op_weight_bytes(const Op& op) {
  if (op.type == OP_POOL || op.type == OP_MAXPOOL) return 0.0;
  return (double)op.R * op.S * (op.depthwise ? 1 : op.Cin) * op.Cout * (op.tc.ready ? 2.0 : 4.0);
}

double op_bytes(const mtb_handle* h, const Op& op, int B) {
  const double es = op.small_io ? 4.0 : (double)elem_size(h);
  double in = (double)B * op.Hin * op.Win * op.Cin * (op.type == OP_STEM ? 4.0 : es);
  double out = (double)B * op.Hout * op.Wout * op.Cout * es;
  if (op.type == OP_POOL) out = (double)B * op.Cout * 4.0;
  double res = op.res_buf != BUF_NONE ? out : 0.0;
  return in + out + res + op_weight_bytes(op);
}

// ---------------------------------------------------------------------------------------------- executor
const char* cuda_msg(cudaError_t e) { return e == cudaSuccess ? nullptr : cudaGetErrorString(e); }

// op.kernel's launch for the kernels that exist for every storage element type T (float, __nv_bfloat16 or __half);
// nullptr on success
template <typename T>
const char* launch_op(mtb_handle* h, const Op& op, ConvParams p, const float* crops, float* pooled, const Workspace& ws,
                      void* features, cudaStream_t st) {
  const size_t pixels = (size_t)p.B * op.Hout * op.Wout;
  switch (op.kernel) {
    case MTB_STEM_3X3S2:
    case MTB_STEM_WIDE:
    case MTB_STEM_GENERIC: {
      StemParams s;
      s.in = crops;
      s.out = p.out; s.w = op.d_w; s.bias = op.d_bias;
      for (int i = 0; i < 3; ++i) { s.pre_scale[i] = op.pre_scale[i]; s.pre_shift[i] = op.pre_shift[i]; }
      s.pre_scale[3] = 1.f; s.pre_shift[3] = 0.f;
      s.B = p.B; s.Hin = op.Hin; s.Win = op.Win; s.Cin = op.Cin; s.Hout = op.Hout; s.Wout = op.Wout; s.Cout = op.Cout;
      s.R = op.R; s.S = op.S; s.stride = op.stride; s.pad_t = op.pad_t; s.pad_l = op.pad_l; s.act = op.act;
      const size_t smem = ((size_t)op.R * op.S * op.Cin + 1) * op.Cout * 4;
      const bool s2 = op.kernel == MTB_STEM_3X3S2, wide = op.kernel == MTB_STEM_WIDE;
      if (s2 && op.Cout == 32) launch_k(stem3x3s2_kernel<T, 32>, dim3(grid_for(pixels, 128)), dim3(128), (size_t)28 * 32 * 4, st, s);
      else if (s2) launch_k(stem3x3s2_kernel<T, 24>, dim3(grid_for(pixels, 128)), dim3(128), (size_t)28 * 24 * 4, st, s);
      else if (wide && op.Cout % 32 == 0) launch_k(stem_conv_wide_kernel<T, 32>, dim3(grid_for(pixels * (op.Cout / 32), 128)), dim3(128), smem, st, s);
      else if (wide && op.Cout % 24 == 0) launch_k(stem_conv_wide_kernel<T, 24>, dim3(grid_for(pixels * (op.Cout / 24), 128)), dim3(128), smem, st, s);
      else if (wide) launch_k(stem_conv_wide_kernel<T, 16>, dim3(grid_for(pixels * (op.Cout / 16), 128)), dim3(128), smem, st, s);
      else launch_k(stem_conv_kernel<T>, dim3(grid_for(pixels * (op.Cout / 4), 256)), dim3(256), smem, st, s);
      return nullptr;
    }
    case MTB_MAXPOOL:
      launch_k(maxpool_kernel<T>, dim3(grid_for(pixels * (op.Cout / 4), 256)), dim3(256), 0, st, p);
      return nullptr;
    case MTB_POOL_MEAN:
      launch_k(pool_mean_kernel<T>, dim3((op.Cin + 127) / 128, p.B), dim3(32, 8), 0, st, (const T*)p.in, (float*)p.out,
               op.Hin * op.Win, op.Cin);
      return nullptr;
    case MTB_SE_FC: {
      if (op.pool_src > 0 && h->ops[op.pool_src].kernel == MTB_POOL_FUSED) {  // input = partial pooling slices of the depthwise kernel
        p.a_splits = h->ops[op.pool_src - 1].pool_slices;
        p.a_split_stride = (size_t)p.B * op.Cin;
      }
      if (op.ksplit == 1) return cuda_msg(launch_conv_igemm<float, float>(p, st));
      // split-K partial slices go to the (still unused) scale buffer, then one tiny reduce kernel
      float* final_out = (float*)p.out;
      p.ksplit = op.ksplit;
      p.out = buf_ptr(ws, BUF_SMALL0 + 2, features);
      if (const char* e = cuda_msg(launch_conv_igemm<float, float>(p, st))) return e;
      const int n = p.B * op.Cout;
      launch_k(se_reduce_kernel, dim3((n + 255) / 256), dim3(256), 0, st, (const float*)p.out, (const float*)op.d_bias, final_out, n,
               op.Cout, op.ksplit, op.act);
      h->launches++;
      return nullptr;
    }
    case MTB_IGEMM: return cuda_msg(launch_conv_igemm<T, T>(p, st));
    case MTB_TC32: return tc32_conv_launch(op.tc32, p, op.res_first, st);  // SE scale (p.a_scale) applied by the splitter warps
    case MTB_DW_GENERIC:
      launch_k(dwconv_kernel<T>, dim3(grid_for(pixels * (op.Cout / 4), 256)), dim3(256), 0, st, p);
      return nullptr;
    case MTB_DW_STRIP_F32:  // 4 channels x 4 pixels per thread, SE squeeze fused (partial slices summed by fc1)
      return cuda_msg(dw_dispatch<ACT_SILU, ACT_RELU, ACT_HSWISH>(op, [&](auto s, auto a) {
        return launch_k(dwconv3x3_pool_f32_kernel<s, a, kDwOW>, dim3((op.Cout / 4 + 31) / 32, op.pool_slices, p.B), dim3(32, 8), 0,
                        st, p, pooled);
      }));
    default: return "not a backbone kernel";
  }
}

// op.kernel's launch for the kernels that exist for 16-bit storage only (T: __nv_bfloat16 or __half): the tensor-core and
// 16-bit depthwise kernels; nullptr on success
template <typename T>
const char* launch_op16(const Op& op, const ConvParams& p, float* pooled, cudaStream_t st) {
  switch (op.kernel) {
    case MTB_TC_CONV:
    case MTB_TC_CONV_SE:
    case MTB_SE_SCALE_TC_CONV: return tc_conv_launch<T>(op.tc, p, op.res_first, false, st);
    case MTB_TC_CONV3X3S1: return tc_conv_launch<T>(op.tc, p, op.res_first, true, st);
    case MTB_DW_TMA:
    case MTB_DW_TMA_DIL:
      return dw_tma_launch<T>(op.dw_maps, op.dw_plan, p.in, p.out, op.d_w, op.d_bias, pooled, p.B, op.Hout, op.Wout, op.Cout,
                              op.pad_t, op.pad_l, op.act, op.kernel == MTB_DW_TMA ? 1 : op.dil, st);
    case MTB_DW_STRIP_16B:
      return cuda_msg(dw_dispatch<ACT_SILU, ACT_RELU, ACT_HSWISH>(op, [&](auto s, auto a) {
        return launch_k(dwconv3x3_pool_16b_kernel<T, s, a, kDwOW>, dim3((op.Cout / 8 + 31) / 32, op.pool_slices, p.B), dim3(32, 8),
                        0, st, p, pooled);
      }));
    case MTB_DW_5X5_16B: {
      const size_t items = (size_t)p.B * op.Hout * ((op.Wout + kDw5OW - 1) / kDw5OW) * (op.Cout / 8);
      return cuda_msg(dw_dispatch<ACT_RELU, ACT_HSWISH>(op, [&](auto s, auto a) {
        return launch_k(dwconv5x5_16b_kernel<T, s, a, kDw5OW>, dim3(grid_for(items, 256)), dim3(256), 0, st, p, nullptr);
      }));
    }
    case MTB_DW_5X5_POOL_16B: {
      const Dw5PoolShape sh = dw5_pool_shape(op.Cout);
      return cuda_msg(dw_dispatch<ACT_SILU>(op, [&](auto s, auto a) {
        return launch_k(dwconv5x5_16b_kernel<T, s, a, kDw5OW, true>, dim3(sh.chunks, op.pool_slices, p.B), dim3(sh.cb * sh.groups),
                        0, st, p, pooled);
      }));
    }
    default: return "not a 16-bit backbone kernel";
  }
}

int run_op(mtb_handle* h, const Op& op, const float* crops, int B, const Workspace& ws, void* features, cudaStream_t st) {
  if (op.kernel == MTB_POOL_FUSED) return MTB_OK;  // produced by the preceding depthwise kernel
  const bool only16 = kKernels[op.kernel].only16;
  if (only16 && !is_16b(h)) return fail(h, MTB_ERR_CUDA, "%s: 16-bit kernel chosen for fp32 storage", op.name.c_str());
  ConvParams p;
  p.in = buf_ptr(ws, op.in_buf, features);
  p.out = buf_ptr(ws, op.out_buf, features);
  p.res = buf_ptr(ws, op.res_buf, features);
  p.a_scale = (const float*)buf_ptr(ws, op.scale_buf, features);
  p.w = op.d_w; p.bias = op.d_bias;
  p.B = B; p.Hin = op.Hin; p.Win = op.Win; p.Cin = op.Cin; p.Hout = op.Hout; p.Wout = op.Wout; p.Cout = op.Cout;
  p.R = op.R; p.S = op.S; p.stride = op.stride; p.dil = op.dil; p.pad_t = op.pad_t; p.pad_l = op.pad_l; p.act = op.act;
  p.res_first = op.res_first ? 1 : 0;
  if (op.kernel == MTB_SE_SCALE_TC_CONV) {
    // squeeze-excitation scale applied in place ahead of the tensor-core conv, which then runs without it
    const double bytes = 2.0 * B * op.Hin * op.Win * op.Cin * elem_size(h);
    ProfScope ps(h, KC_SE_SCALE, 0.0, bytes, st, false);
    const char* e = with_storage16(h, [&](auto* tag) {
      return tc_se_scale_launch<std::remove_pointer_t<decltype(tag)>>(buf_ptr(ws, op.in_buf, features), p.a_scale, B, op.Hin * op.Win,
                                                                      op.Cin, st);
    });
    if (e) return fail(h, MTB_ERR_CUDA, "se scale %s: %s", op.name.c_str(), e);
    h->launches++;
    p.a_scale = nullptr;
  }
  float* pooled = op.fused_pool ? (float*)buf_ptr(ws, BUF_SMALL0, features) : nullptr;
  ProfScope prof(h, op_class(op), op.flops * B, op_bytes(h, op, B), st);
  const char* e = only16 ? with_storage16(h, [&](auto* tag) { return launch_op16<std::remove_pointer_t<decltype(tag)>>(op, p, pooled, st); })
                         : with_storage(h, [&](auto* tag) {
                             return launch_op<std::remove_pointer_t<decltype(tag)>>(h, op, p, crops, pooled, ws, features, st);
                           });
  if (!e) e = cuda_msg(cudaGetLastError());
  if (e) return fail(h, MTB_ERR_CUDA, "launch %s: %s", op.name.c_str(), e);
  h->launches++;
  return MTB_OK;
}

// The executor runs every op on the whole batch: running a stage crop chunk by crop chunk (intermediates resident in L2)
// makes smaller launches, and these kernels are latency / issue bound at small batches rather than bandwidth bound.
// one fmb_kernel launch for the FusedMBConv block (a = 3x3 expand, b = 1x1 projection [+ residual = a's input])
int run_fused_block(mtb_handle* h, const Op& a, const Op& b, int B, const Workspace& ws, void* features, cudaStream_t st) {
  const void* in = buf_ptr(ws, a.in_buf, features);
  void* out = buf_ptr(ws, b.out_buf, features);
  const double bytes = 2.0 * B * a.Hin * a.Win * (a.Cin + b.Cout) + 2.0 * (9.0 * a.Cin * a.Cout + (double)b.Cin * b.Cout);
  ProfScope prof(h, KC_FMB, (a.flops + b.flops) * B, bytes, st);
  const char* e = with_storage16(h, [&](auto* tag) {
    return fmb_launch<std::remove_pointer_t<decltype(tag)>>(a.fmb, in, out, B, a.Hin, a.Win, a.pad_t, a.pad_l, b.res_buf != BUF_NONE, st);
  });
  if (e) return fail(h, MTB_ERR_CUDA, "fused FusedMBConv launch %s: %s", a.name.c_str(), e);
  h->launches++;
  return MTB_OK;
}

// one tc_conv_preact_kernel launch for a 1x1 GEMM (a) and the pre-activation op behind it (b)
int run_preact_pair(mtb_handle* h, const Op& a, const Op& b, int B, const Workspace& ws, void* features, cudaStream_t st) {
  ConvParams p;
  p.in = buf_ptr(ws, a.in_buf, features);
  p.out = buf_ptr(ws, a.out_buf, features);
  p.res = buf_ptr(ws, a.res_buf, features);
  p.a_scale = nullptr;
  p.w = a.d_w; p.bias = a.d_bias;
  p.B = B; p.Hin = a.Hin; p.Win = a.Win; p.Cin = a.Cin; p.Hout = a.Hout; p.Wout = a.Wout; p.Cout = a.Cout;
  p.R = a.R; p.S = a.S; p.stride = a.stride; p.dil = a.dil; p.pad_t = a.pad_t; p.pad_l = a.pad_l; p.act = a.act;
  p.res_first = 0;
  ProfScope prof(h, KC_TC_PREACT, (a.flops + b.flops) * B, op_bytes(h, a, B) + (double)B * b.Hout * b.Wout * b.Cout * elem_size(h), st);
  const char* e = with_storage16(h, [&](auto* tag) {
    return tc_conv_launch<std::remove_pointer_t<decltype(tag)>>(a.tc, p, false, false, st, buf_ptr(ws, b.out_buf, features),
                                                                TcPreact{b.d_w, b.d_bias});
  });
  if (!e) e = cuda_msg(cudaGetLastError());
  if (e) return fail(h, MTB_ERR_CUDA, "fused pre-activation launch %s: %s", a.name.c_str(), e);
  h->launches++;
  return MTB_OK;
}

// ops [first, last): fusable pairs that lie inside the range run fused
int run_ops_range(mtb_handle* h, size_t first, size_t last, const float* crops, int B, const Workspace& ws, void* features,
                  cudaStream_t st) {
  for (size_t k = first; k < last; ++k) {
    h->prof_cur_op = (int)k;
    int rc;
    if (h->ops[k].fmb.ready && k + 1 < last) {
      rc = run_fused_block(h, h->ops[k], h->ops[k + 1], B, ws, features, st);
      ++k;
    } else if (h->ops[k].preact_next && k + 1 < last) {
      rc = run_preact_pair(h, h->ops[k], h->ops[k + 1], B, ws, features, st);
      ++k;
    } else {
      rc = run_op(h, h->ops[k], crops, B, ws, features, st);
    }
    if (rc) return rc;
  }
  h->prof_cur_op = -1;
  return MTB_OK;
}

int run_backbone(mtb_handle* h, const float* crops, int B, Workspace& ws, void* features, cudaStream_t st) {
  return run_ops_range(h, 0, h->ops.size(), crops, B, ws, features, st);
}

int check_common(mtb_handle* h, int B, size_t ws_bytes, const void* workspace) {
  if (!h) return fail(nullptr, MTB_ERR_INVALID_ARG, "null handle");
  if (!h->finalized) return fail(h, MTB_ERR_NOT_FINALIZED, "mtb_finalize_weights has not been called");
  if (B <= 0) return fail(h, MTB_ERR_INVALID_ARG, "batch must be positive (got %d)", B);
  if (!workspace || ws_bytes < layout(h, B, nullptr).total)
    return fail(h, MTB_ERR_WORKSPACE, "workspace too small: need %zu bytes for batch %d, got %zu",
                layout(h, B, nullptr).total, B, ws_bytes);
  return MTB_OK;
}

DecodeScale make_scale(const mtb_config& c) {
  // heatmap_to_image / heatmap_to_metric (models/util.py:6-33), inference => stride_test
  DecodeScale s;
  int last = c.proc_side - 1;
  int last_rc = last - (last % c.stride_test);
  float add = 0.f;
  if (c.centered_stride) add += (float)(c.stride_test / 2);
  if (c.legacy_centered_stride_bug) add += (float)(c.stride_test / 2);
  s.img_mul = (float)last_rc;
  s.img_add = add;
  s.met_mul = (float)last_rc * c.box_size_mm / (float)c.proc_side;
  s.met_add = add * c.box_size_mm / (float)c.proc_side;
  s.z_mul = c.box_size_mm;
  s.apply = 1;
  return s;
}

template <typename T, bool HEAD3D = false>
const char* launch_softargmax_bhwn(const void* logits, float* out2d, float* out3d, int B, int J, int D, int H, int W,
                                   int ld, DecodeScale sc, cudaStream_t st) {
  const int smem = (J * (HEAD3D ? D : 1 + D) + 4 * 128) * (int)sizeof(float4);
  return launch_smem(softargmax_bhwn_kernel<T, HEAD3D>, dim3(B), dim3(512), smem, st, (const T*)logits, out2d, out3d, J, D, H, W,
                     ld, sc);
}

// the decode scale of the handle's head: heatmap_to_image / heatmap_to_metric for MeTRAbs and Metro, heatmap_to_25d
// (metrabs_tf/models/util.py:21-23: image pixels for x and y, mm for z) for Model25D
DecodeScale head_scale(const mtb_handle* h) {
  DecodeScale s = make_scale(h->cfg);
  if (h->model_class == MTB_MODEL_25D) {
    s.met_mul = s.img_mul;
    s.met_add = s.img_add;
  }
  return s;
}

int head_decode_impl(mtb_handle* h, const void* features, int B, float* c2d, float* c3d, const Workspace& ws,
                     cudaStream_t st) {
  const mtb_config& c = h->cfg;
  const Op& op = h->head;
  const double P = (double)h->feat_side * h->feat_side;
  const double feat_bytes = (double)B * P * op.Cin * elem_size(h);
  const int J = head_points(h);
  const double out_bytes = (double)B * J * 5 * 4;
  if (op.kernel == MTB_HEAD_FUSED) {
    // fused: 1x1-conv GEMM on the tensor cores with the soft-argmax reduction in the epilogue; logits never reach HBM
    ProfScope prof(h, KC_HEAD_FUSED, op.flops * B, feat_bytes + (double)op.Cin * op.Cout * 2 + out_bytes, st);
    const char* e = with_storage16(h, [&](auto* tag) {
      return tc_head_launch<std::remove_pointer_t<decltype(tag)>>(op.tc, features, B, h->feat_side, h->feat_side, J, c.depth,
                                                                  head3d(h), head_scale(h), c2d, c3d, ws.base + ws.off_logits, st);
    });
    if (e) return fail(h, MTB_ERR_CUDA, "fused head: %s", e);
    h->launches += 2;
    return MTB_OK;
  }
  ConvParams p;
  p.in = features; p.out = ws.base + ws.off_logits; p.res = nullptr; p.a_scale = nullptr;
  p.w = op.d_w; p.bias = op.d_bias;
  p.B = B; p.Hin = p.Hout = op.Hin; p.Win = p.Wout = op.Win; p.Cin = op.Cin; p.Cout = op.Cout;
  p.R = p.S = 1; p.stride = 1; p.dil = 1; p.pad_t = p.pad_l = 0; p.act = ACT_NONE;
  const double logit_bytes = (double)B * P * op.Cout * 4;
  {
    // HEAD_TC32: 3xTF32 GEMM, HEAD_IGEMM: conv_igemm_kernel -> fp32 NHWC logits
    ProfScope prof(h, kKernels[op.kernel].cls, op.flops * B, feat_bytes + (double)op.Cin * op.Cout * 4 + logit_bytes, st);
    const char* e = op.kernel == MTB_HEAD_TC32
                        ? tc32_conv_launch(op.tc32, p, false, st)
                        : cuda_msg(with_storage(h, [&](auto* tag) { return launch_conv_igemm<std::remove_pointer_t<decltype(tag)>, float>(p, st); }));
    if (e) return fail(h, MTB_ERR_CUDA, "head conv: %s", e);
  }
  ProfScope prof(h, KC_SOFTARGMAX, 0.0, logit_bytes + out_bytes, st);
  const char* se = head3d(h) ? launch_softargmax_bhwn<float, true>(p.out, c2d, c3d, B, J, c.depth, op.Hin, op.Win, op.Cout, head_scale(h), st)
                             : launch_softargmax_bhwn<float>(p.out, c2d, c3d, B, J, c.depth, op.Hin, op.Win, op.Cout, make_scale(c), st);
  if (se) return fail(h, MTB_ERR_CUDA, "softargmax: %s", se);
  h->launches += 2;
  return MTB_OK;
}

int recon_impl(mtb_handle* h, const float* c2d, const float* c3d, const float* K, int B, float* out, float* n2d,
               double* partial, cudaStream_t st) {
  const mtb_config& c = h->cfg;
  ReconParams p;
  p.c2d = c2d; p.c3d = c3d; p.K = K; p.out = out; p.partial = partial; p.n2d = n2d;
  p.B = B; p.J = head_points(h);
  float offset = c.centered_stride ? 0.f : -(float)c.stride_train / 2.f;  // is_within_fov (ptu3d.py:113-121)
  p.fov_lower = (float)c.stride_train * 0.75f + offset;
  p.fov_upper = (float)c.proc_side - (float)c.stride_train * 0.75f + offset;
  p.use_mix = c.mix_3d_inside_fov >= 0.f;
  p.mix = c.mix_3d_inside_fov;
  ProfScope prof(h, KC_RECON, 0.0, (double)B * p.J * 8 * 4 + (double)B * 36, st);
  launch_k(recon_pass1_kernel, dim3(B), dim3(128), 0, st, p);
  launch_k(recon_pass2_kernel, dim3(B), dim3(128), 0, st, p);
  h->launches += 2;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(h, MTB_ERR_CUDA, "reconstruct: %s", cudaGetErrorString(e));
  return MTB_OK;
}

// Model25D: coords25d [B,J,3] -> absolute joints [B,J,3] (bone_solve_kernel, one CTA over the whole batch)
int bone_solve_impl(mtb_handle* h, const float* c25, const float* K, int B, float* out, void* scratch, cudaStream_t st) {
  const mtb_config& c = h->cfg;
  const BoneScratch sc = bone_scratch(h, B, scratch);
  BoneSolveParams p;
  p.c25 = c25; p.K = K; p.edges = h->d_edges; p.len = h->d_len; p.out = out;
  p.coef = sc.coef; p.z = sc.z; p.z_new = sc.z_new; p.obj = sc.obj;
  p.B = B; p.J = c.n_joints; p.E = (int)h->bone_len.size();
  const float offset = c.centered_stride ? 0.f : -(float)c.stride_train / 2.f;  // is_within_fov (tfu3d.py:210-216)
  p.fov_lower = (float)c.stride_train * 0.75f + offset;
  p.fov_upper = (float)c.proc_side - (float)c.stride_train * 0.75f + offset;
  p.mean_relative = h->mean_relative;
  // per iteration: 2 residual passes + the Jacobian over every bone (about 30 flops per bone)
  ProfScope prof(h, KC_BONE_SOLVE, (double)B * p.E * 30.0 * (BONE_ITERS + 1),
                 (double)B * p.J * 6 * 4 + (double)B * 36 + (double)B * p.E * 16 * (2 * BONE_ITERS + 1), st);
  launch_k(bone_solve_kernel, dim3(1), dim3(BONE_THREADS), 0, st, p);
  h->launches += 1;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(h, MTB_ERR_CUDA, "bone-length solve: %s", cudaGetErrorString(e));
  return MTB_OK;
}

// points [B,L,3] @ w [L,n_out] -> out [B,n_out,3] (combine_points_kernel; the forward and mtb_linear_combine_points)
int launch_combine(const float* pts, int B, int L, const float* w, int n_out, float* out, cudaStream_t st) {
  launch_k(combine_points_kernel, dim3(B, (n_out + 127) / 128), dim3(128), (size_t)L * 3 * sizeof(float), st, pts, w, out, L,
           n_out);
  return (int)cudaGetLastError();
}

// the recombination of a latent-point model: absolute latents [B,L,3] -> joints [B,n_out,3]
int combine_impl(mtb_handle* h, const float* latents, int B, float* out, cudaStream_t st) {
  const double L = h->n_latents, n = h->n_out;
  ProfScope prof(h, KC_COMBINE, 2.0 * B * L * n * 3, (double)B * (L + n) * 3 * 4 + L * n * 4, st);
  int e = launch_combine(latents, B, h->n_latents, h->d_recomb, h->n_out, out, st);
  h->launches += 1;
  if (e) return fail(h, MTB_ERR_CUDA, "combine points: %s", cudaGetErrorString((cudaError_t)e));
  return MTB_OK;
}

// reconstruction into the caller's output, or (latent-point model) into `latents` and then recombined into the output
int recon_and_combine(mtb_handle* h, const float* c2d, const float* c3d, const float* K, int B, float* out, float* n2d,
                      double* partial, float* latents, cudaStream_t st) {
  if (h->n_latents == 0) return recon_impl(h, c2d, c3d, K, B, out, n2d, partial, st);
  int rc = recon_impl(h, c2d, c3d, K, B, latents, n2d, partial, st);
  if (rc) return rc;
  return combine_impl(h, latents, B, out, st);
}

// 16-bit (bf16 / fp16) <-> fp32 copies of the debug entry points; fp32 from_float rounds to nearest even
template <typename T>
__global__ void to_float_kernel(const T* in, float* out, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    out[i] = load1<T>(in + i);
}

template <typename T>
__global__ void from_float_kernel(const float* in, T* out, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    store1<T>(out + i, in[i]);
}

// storage -> fp32 copy of n elements (a plain copy for fp32 storage)
void copy_to_float(const mtb_handle* h, const void* src, float* out, size_t n, cudaStream_t st) {
  with_storage(h, [&](auto* tag) {
    using T = std::remove_pointer_t<decltype(tag)>;
    if constexpr (std::is_same<T, float>::value) return cudaMemcpyAsync(out, src, n * 4, cudaMemcpyDeviceToDevice, st);
    else return launch_k(to_float_kernel<T>, dim3(grid_for(n, 256)), dim3(256), 0, st, (const T*)src, out, n);
  });
}
// fp32 -> storage copy of n elements
void copy_from_float(const mtb_handle* h, const float* src, void* out, size_t n, cudaStream_t st) {
  with_storage(h, [&](auto* tag) {
    using T = std::remove_pointer_t<decltype(tag)>;
    if constexpr (std::is_same<T, float>::value) return cudaMemcpyAsync(out, src, n * 4, cudaMemcpyDeviceToDevice, st);
    else return launch_k(from_float_kernel<T>, dim3(grid_for(n, 256)), dim3(256), 0, st, src, (T*)out, n);
  });
}

// [b,J,2] + [b,J,3] -> [b,J,5] (what travels in the all-gather) and back
__global__ void pack_decoded_kernel(const float* __restrict__ c2d, const float* __restrict__ c3d, float* __restrict__ packed, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    packed[(size_t)i * 5 + 0] = c2d[(size_t)i * 2 + 0];
    packed[(size_t)i * 5 + 1] = c2d[(size_t)i * 2 + 1];
    packed[(size_t)i * 5 + 2] = c3d[(size_t)i * 3 + 0];
    packed[(size_t)i * 5 + 3] = c3d[(size_t)i * 3 + 1];
    packed[(size_t)i * 5 + 4] = c3d[(size_t)i * 3 + 2];
  }
}
__global__ void unpack_decoded_kernel(const float* __restrict__ packed, float* __restrict__ c2d, float* __restrict__ c3d, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    c2d[(size_t)i * 2 + 0] = packed[(size_t)i * 5 + 0];
    c2d[(size_t)i * 2 + 1] = packed[(size_t)i * 5 + 1];
    c3d[(size_t)i * 3 + 0] = packed[(size_t)i * 5 + 2];
    c3d[(size_t)i * 3 + 1] = packed[(size_t)i * 5 + 3];
    c3d[(size_t)i * 3 + 2] = packed[(size_t)i * 5 + 4];
  }
}

struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    cudaGetDevice(&prev);
    if (prev != dev) cudaSetDevice(dev);
    else prev = -1;
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

}  // namespace

// =================================================================================================== C ABI
extern "C" {

const char* mtb_version(void) { return "metrabs_b200 0.1 (sm_90a)"; }

const char* mtb_last_error(const mtb_handle* h) { return h ? h->err.c_str() : g_error.c_str(); }

int mtb_create(const mtb_config* cfg, mtb_handle** out) {
  if (!cfg || !out) return fail(nullptr, MTB_ERR_INVALID_ARG, "null argument");
  if (cfg->abi_version != MTB_ABI_VERSION)
    return fail(nullptr, MTB_ERR_INVALID_ARG, "ABI version mismatch: header %d, caller %d", MTB_ABI_VERSION, cfg->abi_version);
  if (cfg->weak_perspective)
    return fail(nullptr, MTB_ERR_UNSUPPORTED, "weak_perspective reconstruction is not functional in the reference (ptu.py:30,42)");
  if (cfg->n_joints <= 0 || cfg->depth < 1 || cfg->proc_side <= 0 || cfg->stride_test <= 0 || cfg->stride_train <= 0)
    return fail(nullptr, MTB_ERR_INVALID_ARG, "invalid geometry (n_joints=%d depth=%d proc_side=%d stride=%d)", cfg->n_joints,
                cfg->depth, cfg->proc_side, cfg->stride_test);
  const bool effnet = cfg->arch == MTB_ARCH_EFFNET || cfg->arch == MTB_ARCH_EFFNET_EPS1E5;
  if (effnet && (cfg->n_stages <= 0 || cfg->n_stages > MTB_MAX_STAGES))
    return fail(nullptr, MTB_ERR_INVALID_ARG, "n_stages out of range");
  if (cfg->arch == MTB_ARCH_EFFNET_EPS1E5)  // the EfficientNet-B grammar: MBConv rows with 3x3 or 5x5 kernels
    for (int i = 0; i < cfg->n_stages; ++i) {
      const mtb_stage& s = cfg->stages[i];
      if (s.block != 1 || (s.kernel != 3 && s.kernel != 5) || (s.stride != 1 && s.stride != 2))
        return fail(nullptr, MTB_ERR_UNSUPPORTED, "MTB_ARCH_EFFNET_EPS1E5 stage %d: only MBConv rows with kernel 3 or 5 and "
                    "stride 1 or 2 (got block %d, kernel %d, stride %d)", i, s.block, s.kernel, s.stride);
    }
  if (effnet) {
    int out_stride = 2;
    for (int i = 0; i < cfg->n_stages; ++i) {
      const mtb_stage& s = cfg->stages[i];
      if (s.dilation_in < 1 || s.dilation_in > 8 || s.dilation_out < 1 || s.dilation_out > 8)
        return fail(nullptr, MTB_ERR_UNSUPPORTED, "stage %d: dilation %d / %d outside 1..8", i, s.dilation_in, s.dilation_out);
      if (s.block == 0 && (s.dilation_in > 1 || s.dilation_out > 1))
        return fail(nullptr, MTB_ERR_UNSUPPORTED, "stage %d: FusedMBConv rows are not dilated (dilation %d / %d); only the "
                    "output strides 32, 16 and 8 of EfficientNetV2 are built", i, s.dilation_in, s.dilation_out);
      out_stride *= s.stride;
    }
    // stride-32 tables run whatever stride_test says (as before dilation existed); a dilated table decodes its finer heatmap
    // with the geometry of stride_test, so the two must agree
    if (out_stride < 32 && out_stride != cfg->stride_test)
      return fail(nullptr, MTB_ERR_INVALID_ARG, "the stage table has output stride %d but stride_test is %d: set "
                  "Config(stride_test=%d) for this backbone", out_stride, cfg->stride_test, out_stride);
  }
  if (cfg->precision < MTB_PRECISION_FP32 || cfg->precision > MTB_PRECISION_F16_SIMT)
    return fail(nullptr, MTB_ERR_INVALID_ARG, "unknown precision %d", cfg->precision);
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail(nullptr, MTB_ERR_CUDA, "no CUDA device: this library has no CPU fallback");
  if (cfg->device < 0 || cfg->device >= ndev) return fail(nullptr, MTB_ERR_INVALID_ARG, "device %d out of range", cfg->device);
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, cfg->device) != cudaSuccess || prop.major != 9 || prop.minor != 0)
    return fail(nullptr, MTB_ERR_CUDA, "device %d is not sm_90 (compute capability %d.%d)", cfg->device, prop.major, prop.minor);
  mtb_handle* h = new mtb_handle();
  h->cfg = *cfg;
  int rc = plan(h);
  if (rc) {
    g_error = h->err;
    delete h;
    return rc;
  }
  *out = h;
  return MTB_OK;
}

int mtb_destroy(mtb_handle* h) {
  if (!h) return MTB_OK;
  {
    DeviceGuard g(h->cfg.device);
    for (void* p : h->dev_allocs) cudaFree(p);
    if (h->stage) cudaFree(h->stage);
    for (auto& sl : h->slots) {
      if (sl.buf) cudaFree(sl.buf);
      if (sl.h2d_done) cudaEventDestroy(sl.h2d_done);
      if (sl.done) cudaEventDestroy(sl.done);
    }
    for (auto& e : h->graphs)
      if (e.exec) cudaGraphExecDestroy(e.exec);
    if (h->pipe_ws) cudaFree(h->pipe_ws);
    if (h->copy_stream) cudaStreamDestroy(h->copy_stream);
    if (h->graph_stream) cudaStreamDestroy(h->graph_stream);
    if (h->graph_in) cudaEventDestroy(h->graph_in);
    if (h->graph_out) cudaEventDestroy(h->graph_out);
    cudaGetLastError();
    for (size_t i = 0; i < h->prof_events.size(); ++i) {
      if (cudaEventDestroy(h->prof_events[i]) != cudaSuccess) {  // e.g. cudaErrorContextIsDestroyed during process teardown: the driver owns them now
        cudaGetLastError();
        break;
      }
    }
    if (h->nccl_comm && h->nccl_lib) {
      typedef int (*destroy_t)(void*);
      destroy_t f = (destroy_t)dlsym(h->nccl_lib, "ncclCommDestroy");
      if (f) f(h->nccl_comm);
    }
  }
  delete h;
  return MTB_OK;
}

int mtb_load_weight(mtb_handle* h, const char* name, const void* data, int dtype, const int64_t* shape, int ndim) {
  if (!h || !name || !data || (ndim > 0 && !shape)) return fail(h, MTB_ERR_INVALID_ARG, "null argument");
  HostTensor t;
  size_t n = 1;
  for (int i = 0; i < ndim; ++i) {
    t.shape.push_back(shape[i]);
    n *= (size_t)shape[i];
  }
  t.data.resize(n);
  switch (dtype) {
    case MTB_DTYPE_F32: memcpy(t.data.data(), data, n * 4); break;
    case MTB_DTYPE_BF16: {
      const uint16_t* s = (const uint16_t*)data;
      for (size_t i = 0; i < n; ++i) {
        uint32_t u = (uint32_t)s[i] << 16;
        memcpy(&t.data[i], &u, 4);
      }
      break;
    }
    case MTB_DTYPE_F16: {
      const __half* s = (const __half*)data;
      for (size_t i = 0; i < n; ++i) t.data[i] = __half2float(s[i]);
      break;
    }
    case MTB_DTYPE_I64: {
      const int64_t* s = (const int64_t*)data;
      for (size_t i = 0; i < n; ++i) t.data[i] = (float)s[i];
      break;
    }
    default: return fail(h, MTB_ERR_INVALID_ARG, "unknown dtype %d for '%s'", dtype, name);
  }
  h->raw[name] = std::move(t);
  h->finalized = false;
  return MTB_OK;
}

int mtb_finalize_weights(mtb_handle* h) {
  if (!h) return fail(nullptr, MTB_ERR_INVALID_ARG, "null handle");
  DeviceGuard g(h->cfg.device);
  for (auto& e : h->graphs)  // captured forwards hold the old weight pointers
    if (e.exec) cudaGraphExecDestroy(e.exec);
  h->graphs.clear();
  for (void* p : h->dev_allocs) cudaFree(p);
  h->dev_allocs.clear();
  choose_kernels(h);
  for (auto& op : h->ops) {
    int rc = prepare_op_weights(h, op);
    if (rc) return rc;
  }
  // FusedMBConv blocks (3x3 expand + SiLU -> 1x1 projection + residual, stride 1): one fused kernel per block (tc_fmb.cuh)
  for (size_t i = 0; i + 1 < h->ops.size(); ++i) {
    Op& a = h->ops[i];
    const Op& b = h->ops[i + 1];
    a.fmb.ready = false;
    if (!is_tc16(h) || !a.tc.ready || !b.tc.ready) continue;
    if (a.type != OP_CONV || b.type != OP_CONV || a.small_io || b.small_io) continue;
    if (a.R != 3 || a.S != 3 || a.stride != 1 || a.dil != 1 || a.act != ACT_SILU || a.res_buf != BUF_NONE || a.scale_buf != BUF_NONE) continue;
    if (b.R != 1 || b.stride != 1 || b.act != ACT_NONE || b.scale_buf != BUF_NONE || b.res_first || b.in_buf != a.out_buf) continue;
    if (b.res_buf != BUF_NONE && b.res_buf != a.in_buf) continue;
    if (a.Hin != a.Hout || a.Win != a.Wout || b.out_buf == a.in_buf) continue;
    fmb_prepare(a.fmb, a.tc, b.tc);
  }
  // ResNet V2: a block's _3_conv and the pre-activation behind it (the next block's, or post_bn): one tc_conv_preact_kernel.
  // Its tiles store the pre-activation while later tiles still read the GEMM's input and residual, so b writes neither.
  for (size_t i = 0; i + 1 < h->ops.size(); ++i) {
    Op& a = h->ops[i];
    const Op& b = h->ops[i + 1];
    a.preact_next = a.kernel == MTB_TC_CONV && b.kernel == MTB_DW_GENERIC && b.R == 1 && b.S == 1 && b.stride == 1 &&
                    b.act == ACT_RELU && b.Cout == a.Cout && b.in_buf == a.out_buf && b.out_buf != a.out_buf &&
                    b.out_buf != a.in_buf && b.out_buf != a.res_buf && a.scale_buf == BUF_NONE && !a.res_first &&
                    tc_preact_eligible(a.R, a.stride, a.Cout, a.act, a.res_buf != BUF_NONE);
  }
  {
    Op& hd = h->head;
    const HostTensor* w = find(h, hd.wkey);
    if (!w) return fail(h, MTB_ERR_MISSING_WEIGHT, "missing weight '%s'", hd.wkey.c_str());
    const int n_raw = h->cfg.n_joints, D = h->cfg.depth;
    const int n_ch = n_raw * (head3d(h) ? D : 1 + D);  // the checkpoint's channels (all raw points)
    if (w->shape.size() != 4 || w->shape[0] != n_ch || w->shape[1] != hd.Cin)
      return fail(h, MTB_ERR_INVALID_ARG, "'%s' must be [%d,%d,1,1]", hd.wkey.c_str(), n_ch, hd.Cin);
    const HostTensor* hb = find(h, hd.biaskey);
    if (!hb || (int)hb->data.size() != n_ch)
      return fail(h, MTB_ERR_MISSING_WEIGHT, "missing weight '%s'", hd.biaskey.c_str());
    const int P = head_points(h);
    if (P < n_raw) {
      // predict_all_and_latents: the forward reconstructs only points [0, P) (models/metrabs.py:53-55), so keep just their
      // channels - 2D row j and 3D row n_raw + d*n_raw + j - repacked as a P-point head (channel P + d*P + j).  Every
      // channel is an independent dot product, so this is the reference computation minus the discarded points.
      HostTensor ws, bs;
      ws.shape = {(int64_t)P * (1 + D), hd.Cin, 1, 1};
      bs.shape = {(int64_t)P * (1 + D)};
      ws.data.resize((size_t)P * (1 + D) * hd.Cin);
      bs.data.resize((size_t)P * (1 + D));
      for (int d = -1; d < D; ++d)
        for (int j = 0; j < P; ++j) {
          const size_t src = d < 0 ? (size_t)j : (size_t)n_raw + (size_t)d * n_raw + j;
          const size_t dst = d < 0 ? (size_t)j : (size_t)P + (size_t)d * P + j;
          std::copy_n(w->data.begin() + src * hd.Cin, hd.Cin, ws.data.begin() + dst * hd.Cin);
          bs.data[dst] = hb->data[src];
        }
      h->raw[hd.wkey] = std::move(ws);
      h->raw[hd.biaskey] = std::move(bs);
      w = find(h, hd.wkey);
      hb = find(h, hd.biaskey);
    }
    const int n_real = head_channels(h);
    if (n_real != hd.Cout) {  // zero-pad the output channels
      HostTensor wp = *w, bp = *hb;
      wp.data.resize((size_t)hd.Cout * hd.Cin, 0.f);
      wp.shape[0] = hd.Cout;
      bp.data.resize(hd.Cout, 0.f);
      bp.shape[0] = hd.Cout;
      h->raw[hd.wkey] = wp;
      h->raw[hd.biaskey] = bp;
      w = find(h, hd.wkey);
    }
    int rc = prepare_op_weights(h, hd);
    if (rc) return rc;
    if (hd.kernel == MTB_HEAD_FUSED) {
      // the ORIGINAL (unpadded) [n_real][C] weight: the fused kernel masks rows itself
      std::vector<float> w0((size_t)n_real * hd.Cin), b0(n_real);
      for (int n = 0; n < n_real; ++n) {
        b0[n] = find(h, hd.biaskey)->data[n];
        for (int cc = 0; cc < hd.Cin; ++cc) w0[(size_t)n * hd.Cin + cc] = w->data[(size_t)n * hd.Cin + cc];
      }
      const char* e = with_storage16(h, [&](auto* tag) {
        return tc_prepare_head<std::remove_pointer_t<decltype(tag)>>(hd.tc, w0.data(), b0.data(), hd.Cin, n_real, h->dev_allocs);
      });
      if (e) return fail(h, MTB_ERR_CUDA, "tensor-core head weight prep: %s", e);
    }
  }
  h->d_recomb = nullptr;
  if (h->n_latents > 0) {
    int rc = upload(h, h->recomb.data(), h->recomb.size() * sizeof(float), (void**)&h->d_recomb);
    if (rc) return rc;
  }
  h->d_edges = nullptr;
  h->d_len = nullptr;
  if (h->model_class == MTB_MODEL_25D) {
    int rc = upload(h, h->bone_edges.data(), h->bone_edges.size() * sizeof(int32_t), (void**)&h->d_edges);
    if (!rc) rc = upload(h, h->bone_len.data(), h->bone_len.size() * sizeof(float), (void**)&h->d_len);
    if (rc) return rc;
  }
  h->raw.clear();
  h->finalized = true;
  return MTB_OK;
}

int mtb_set_latent_recombination(mtb_handle* h, const float* weights, int n_latents, int n_out) {
  if (!h) return fail(nullptr, MTB_ERR_INVALID_ARG, "null handle");
  if (!weights) return fail(h, MTB_ERR_INVALID_ARG, "null recombination weights");
  if (h->finalized)
    return fail(h, MTB_ERR_INVALID_ARG, "the latent recombination must be set before mtb_finalize_weights (load the weights again first)");
  if (h->cfg.arch == MTB_ARCH_HEAD_ONLY) return fail(h, MTB_ERR_INVALID_ARG, "a head-only handle has no forward to recombine");
  if (h->model_class != MTB_MODEL_METRABS)
    return fail(h, MTB_ERR_INVALID_ARG, "latent points are a MeTRAbs feature: this handle is a Metro or Model25D model");
  if (n_latents < 1 || n_latents > h->cfg.n_joints)
    return fail(h, MTB_ERR_INVALID_ARG, "n_latents must be in [1, %d] (the head's points), got %d", h->cfg.n_joints, n_latents);
  if (n_out < 1 || n_out > kMaxCombinePoints)
    return fail(h, MTB_ERR_INVALID_ARG, "n_out must be in [1, %d], got %d", kMaxCombinePoints, n_out);
  const size_t n = (size_t)n_latents * n_out;
  for (size_t i = 0; i < n; ++i)
    if (!std::isfinite(weights[i])) return fail(h, MTB_ERR_INVALID_ARG, "recombination weight %zu is not finite", i);
  h->recomb.assign(weights, weights + n);
  h->n_latents = n_latents;
  h->n_out = n_out;
  size_head(h);
  return MTB_OK;
}

int mtb_set_model_class(mtb_handle* h, int model_class, const int32_t* edges, const float* bone_lengths, int n_bones,
                        int mean_relative) {
  if (!h) return fail(nullptr, MTB_ERR_INVALID_ARG, "null handle");
  if (h->finalized)
    return fail(h, MTB_ERR_INVALID_ARG, "the model class must be set before mtb_finalize_weights (load the weights again first)");
  if (h->cfg.arch == MTB_ARCH_HEAD_ONLY) return fail(h, MTB_ERR_INVALID_ARG, "a head-only handle has no model class");
  if (model_class != MTB_MODEL_METRABS && model_class != MTB_MODEL_METRO && model_class != MTB_MODEL_25D)
    return fail(h, MTB_ERR_INVALID_ARG, "unknown model class %d", model_class);
  if (h->n_latents > 0)
    return fail(h, MTB_ERR_INVALID_ARG, "this handle has a latent recombination, which only MeTRAbs models have");
  if (model_class != MTB_MODEL_METRABS && h->cfg.legacy_centered_stride_bug)
    return fail(h, MTB_ERR_INVALID_ARG, "legacy_centered_stride_bug does not exist in the TF heatmap_to_image that Metro and "
                "Model25D decode with (metrabs_tf/models/util.py:8-18)");
  std::vector<int32_t> e;
  std::vector<float> len;
  if (model_class == MTB_MODEL_25D) {
    if (!edges || !bone_lengths) return fail(h, MTB_ERR_INVALID_ARG, "a Model25D needs its bone edges and lengths");
    if (n_bones < 1 || n_bones > kMaxCombinePoints)
      return fail(h, MTB_ERR_INVALID_ARG, "n_bones must be in [1, %d], got %d", kMaxCombinePoints, n_bones);
    for (int i = 0; i < n_bones; ++i) {
      for (int k = 0; k < 2; ++k)
        if (edges[2 * i + k] < 0 || edges[2 * i + k] >= h->cfg.n_joints)
          return fail(h, MTB_ERR_INVALID_ARG, "bone %d: joint index %d outside [0, %d)", i, edges[2 * i + k], h->cfg.n_joints);
      if (!std::isfinite(bone_lengths[i]) || !(bone_lengths[i] > 0.f))
        return fail(h, MTB_ERR_INVALID_ARG, "bone %d: length %g is not finite and positive", i, (double)bone_lengths[i]);
    }
    e.assign(edges, edges + 2 * (size_t)n_bones);
    len.assign(bone_lengths, bone_lengths + n_bones);
  }
  h->model_class = model_class;
  h->bone_edges = std::move(e);
  h->bone_len = std::move(len);
  h->mean_relative = mean_relative ? 1 : 0;
  // the TF heads' key schema: metrabs_tf/models/{metro,twofive}.py name the head `heatmap_head`
  Op& hd = h->head;
  hd.name = head3d(h) ? "heatmap_head.conv_final" : "heatmap_heads.conv_final";
  hd.wkey = hd.name + ".weight";
  hd.biaskey = hd.name + ".bias";
  size_head(h);
  return MTB_OK;
}

int mtb_output_joints(const mtb_handle* h) { return h ? output_joints(h) : 0; }

int mtb_linear_combine_points(const float* points, int batch, int n_in, const float* weights, int n_out, float* out, void* stream) {
  if (!points || !weights || !out) return fail(nullptr, MTB_ERR_INVALID_ARG, "null argument");
  if (batch <= 0 || n_in < 1 || n_in > kMaxCombinePoints || n_out < 1 || n_out > kMaxCombinePoints)
    return fail(nullptr, MTB_ERR_INVALID_ARG, "invalid sizes (batch=%d n_in=%d n_out=%d; n_in and n_out must be in [1, %d])", batch,
                n_in, n_out, kMaxCombinePoints);
  int e = launch_combine(points, batch, n_in, weights, n_out, out, (cudaStream_t)stream);
  if (e) return fail(nullptr, MTB_ERR_CUDA, "combine points launch: %s", cudaGetErrorString((cudaError_t)e));
  return MTB_OK;
}

size_t mtb_workspace_bytes(const mtb_handle* h, int batch) {
  if (!h || batch <= 0) return 0;
  return layout(h, batch, nullptr).total;
}

int mtb_feature_shape(const mtb_handle* h, int* hw_side, int* channels) {
  if (!h) return fail(nullptr, MTB_ERR_INVALID_ARG, "null handle");
  if (hw_side) *hw_side = h->feat_side;
  if (channels) *channels = h->feat_c;
  return MTB_OK;
}

int mtb_backbone_forward(mtb_handle* h, const float* crops, int batch, void* features, void* workspace,
                         size_t workspace_bytes, void* stream) {
  int rc = check_common(h, batch, workspace_bytes, workspace);
  if (rc) return rc;
  if (!crops || !features) return fail(h, MTB_ERR_INVALID_ARG, "null crops/features");
  if (h->ops.empty()) return fail(h, MTB_ERR_UNSUPPORTED, "this handle has no backbone (head-only)");
  DeviceGuard g(h->cfg.device);
  h->launches = 0;
  Workspace ws = layout(h, batch, workspace);
  return run_backbone(h, crops, batch, ws, features, (cudaStream_t)stream);
}

int mtb_head_decode(mtb_handle* h, const void* features, int batch, float* coords2d, float* coords3d_rel,
                    void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_common(h, batch, workspace_bytes, workspace);
  if (rc) return rc;
  if (!features || !coords3d_rel || (!coords2d && !head3d(h))) return fail(h, MTB_ERR_INVALID_ARG, "null argument");
  DeviceGuard g(h->cfg.device);
  h->launches = 0;
  Workspace ws = layout(h, batch, workspace);
  return head_decode_impl(h, features, batch, coords2d, coords3d_rel, ws, (cudaStream_t)stream);
}

int mtb_softargmax(const void* logits, int dtype, int layout_, int batch, int n_joints, int depth, int height,
                   int width, float* out2d, float* out3d, void* stream) {
  if (!logits || batch <= 0 || n_joints <= 0 || depth < 0 || height <= 0 || width <= 0)
    return fail(nullptr, MTB_ERR_INVALID_ARG, "invalid soft-argmax arguments");
  if (dtype != MTB_DTYPE_F32 && dtype != MTB_DTYPE_BF16 && dtype != MTB_DTYPE_F16)
    return fail(nullptr, MTB_ERR_UNSUPPORTED, "soft-argmax dtype must be f32, bf16 or f16");
  if (dtype == MTB_DTYPE_F16 && layout_ != MTB_LAYOUT_BDJHW)
    return fail(nullptr, MTB_ERR_UNSUPPORTED, "f16 logits are supported in the reference layout (BDJHW) only");
  cudaStream_t st = (cudaStream_t)stream;
  if (layout_ == MTB_LAYOUT_BDJHW) {
    const bool two_d = depth == 0;
    float* out = two_d ? out2d : out3d;
    if (!out) return fail(nullptr, MTB_ERR_INVALID_ARG, "null output");
    const int D = two_d ? 1 : depth;
    const int vw = dtype == MTB_DTYPE_F32 ? 4 : 8;  // elements per 16-byte vector
    const bool vec = (width % vw == 0) && (((uintptr_t)logits) % 16 == 0);
    const int rows = batch * n_joints;
    const int hw = height * width;
    const bool pow2 = (hw & (hw - 1)) == 0 && (width & (width - 1)) == 0;
    int hw_shift = 0, w_shift = 0;
    while ((1 << hw_shift) < hw) ++hw_shift;
    while ((1 << w_shift) < width) ++w_shift;
    // loads: 0 scalar, 1 vector, 2 vector with power-of-two shapes (shift indexing)
    const int loads = vec ? (pow2 ? 2 : 1) : 0;
    auto launch = [&](auto* tag) {
      using TT = std::remove_pointer_t<decltype(tag)>;
      with_const<0, 1, 2>(loads, cudaErrorNotSupported, [&](auto l) {
        return launch_k(softargmax_bdjhw_kernel<TT, l == 0 ? 1 : 16 / (int)sizeof(TT), l == 2>, dim3(rows), dim3(256), 0, st,
                        (const TT*)logits, out, n_joints, D, height, width, (int)two_d, hw_shift, w_shift);
      });
    };
    if (dtype == MTB_DTYPE_F32) launch((float*)nullptr);
    else if (dtype == MTB_DTYPE_BF16) launch((__nv_bfloat16*)nullptr);
    else launch((__half*)nullptr);  // fp16: what the reference's head emits under its autocast (multiperson_model.py:241, models/metrabs.py:80)
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(nullptr, MTB_ERR_CUDA, "softargmax launch: %s", cudaGetErrorString(e));
    return MTB_OK;
  }
  if (layout_ == MTB_LAYOUT_BHWN) {
    DecodeScale sc{};
    sc.apply = 0;
    const char* e = dtype == MTB_DTYPE_F32
                 ? launch_softargmax_bhwn<float>(logits, out2d, out3d, batch, n_joints, depth, height, width, n_joints * (1 + depth), sc, st)
                 : launch_softargmax_bhwn<__nv_bfloat16>(logits, out2d, out3d, batch, n_joints, depth, height, width, n_joints * (1 + depth), sc, st);
    if (e) return fail(nullptr, MTB_ERR_CUDA, "softargmax launch: %s", e);
    return MTB_OK;
  }
  return fail(nullptr, MTB_ERR_INVALID_ARG, "unknown layout %d", layout_);
}

size_t mtb_reconstruct_scratch_bytes(int batch) {
  return batch <= 0 ? 0 : align_up((size_t)batch * 2 * 8, 256) + (size_t)batch * 4096 * 2 * 4;
}

int mtb_reconstruct_absolute(mtb_handle* h, const float* coords2d, const float* coords3d_rel, const float* intrinsics,
                             int batch, float* coords3d_abs, void* scratch, void* stream) {
  if (!h) return fail(nullptr, MTB_ERR_INVALID_ARG, "null handle");
  if (!coords2d || !coords3d_rel || !intrinsics || !coords3d_abs || !scratch || batch <= 0)
    return fail(h, MTB_ERR_INVALID_ARG, "null/invalid argument");
  if (head_points(h) > 4096) return fail(h, MTB_ERR_UNSUPPORTED, "more than 4096 joints");
  if (head3d(h))
    return fail(h, MTB_ERR_UNSUPPORTED, "a Metro or Model25D handle has no MeTRAbs reconstruction (Model25D: "
                "mtb_reconstruct_by_bone_lengths)");
  DeviceGuard g(h->cfg.device);
  h->launches = 0;
  double* partial = (double*)scratch;
  float* n2d = (float*)((char*)scratch + align_up((size_t)batch * 2 * 8, 256));
  return recon_impl(h, coords2d, coords3d_rel, intrinsics, batch, coords3d_abs, n2d, partial, (cudaStream_t)stream);
}

size_t mtb_bone_lengths_scratch_bytes(const mtb_handle* h, int batch) {
  if (!h || batch <= 0 || h->model_class != MTB_MODEL_25D) return 0;
  return bone_scratch_bytes(h, batch);
}

int mtb_reconstruct_by_bone_lengths(mtb_handle* h, const float* coords25d, const float* intrinsics, int batch, float* coords3d_abs,
                                    void* scratch, void* stream) {
  if (!h) return fail(nullptr, MTB_ERR_INVALID_ARG, "null handle");
  if (h->model_class != MTB_MODEL_25D) return fail(h, MTB_ERR_INVALID_ARG, "not a Model25D handle (mtb_set_model_class)");
  if (!h->finalized) return fail(h, MTB_ERR_NOT_FINALIZED, "mtb_finalize_weights has not been called");
  if (!coords25d || !intrinsics || !coords3d_abs || !scratch || batch <= 0)
    return fail(h, MTB_ERR_INVALID_ARG, "null/invalid argument");
  DeviceGuard g(h->cfg.device);
  h->launches = 0;
  return bone_solve_impl(h, coords25d, intrinsics, batch, coords3d_abs, scratch, (cudaStream_t)stream);
}

// the forward proper: every launch of one step on `st` (no allocation, no synchronisation: capturable)
static int forward_body(mtb_handle* h, const float* crops, const float* intrinsics, int batch, float* coords3d_abs, void* workspace,
                        cudaStream_t st) {
  h->launches = 0;
  Workspace ws = layout(h, batch, workspace);
  void* features = ws.base + ws.off_features;
  int rc = run_backbone(h, crops, batch, ws, features, st);
  if (rc) return rc;
  float* c2d = (float*)(ws.base + ws.off_c2d);
  float* c3d = (float*)(ws.base + ws.off_c3d);
  if (h->model_class == MTB_MODEL_METRO) return head_decode_impl(h, features, batch, nullptr, coords3d_abs, ws, st);
  rc = head_decode_impl(h, features, batch, head3d(h) ? nullptr : c2d, c3d, ws, st);
  if (rc) return rc;
  if (h->model_class == MTB_MODEL_25D) return bone_solve_impl(h, c3d, intrinsics, batch, coords3d_abs, ws.base + ws.off_bones, st);
  return recon_and_combine(h, c2d, c3d, intrinsics, batch, coords3d_abs, (float*)(ws.base + ws.off_n2d),
                           (double*)(ws.base + ws.off_partial), (float*)(ws.base + ws.off_latents), st);
}

// mtb_forward captures its own launches into a CUDA graph the second time it sees the same (buffers, batch, stream) and
// replays that graph from then on: the ~465 launches of a step cost less as one graph launch than as stream submissions
// (measured, round 2: 12.28 k vs 11.83 k crops/s end to end through mtb_forward_host_submit/_wait, EfficientNetV2-L@256, 256
// crops).  A profiling window bypasses it (events cannot be timed inside a graph), a caller that is itself capturing the
// stream just records our launches, any capture failure falls back to plain launches for that key.
static void drop_graphs_on(mtb_handle* h, const void* ws) {
  for (size_t i = 0; i < h->graphs.size();) {
    if (ws == nullptr || h->graphs[i].ws == ws) {
      if (h->graphs[i].exec) cudaGraphExecDestroy(h->graphs[i].exec);
      h->graphs.erase(h->graphs.begin() + (long)i);
    } else {
      ++i;
    }
  }
}

int mtb_forward(mtb_handle* h, const float* crops, const float* intrinsics, int batch, float* coords3d_abs,
                void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_common(h, batch, workspace_bytes, workspace);
  if (rc) return rc;
  if (!crops || (!intrinsics && h->model_class != MTB_MODEL_METRO) || !coords3d_abs)
    return fail(h, MTB_ERR_INVALID_ARG, "null argument");
  if (h->ops.empty()) return fail(h, MTB_ERR_UNSUPPORTED, "this handle has no backbone (head-only)");
  DeviceGuard g(h->cfg.device);
  cudaStream_t st = (cudaStream_t)stream;
  if (h->prof_mask == 0) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    cudaStreamIsCapturing(st, &cs);
    if (cs == cudaStreamCaptureStatusNone) {  // (a caller capturing this stream itself just records our launches)
      // the legacy default stream cannot be captured: fork to an internal stream and join back with events
      const bool side = st == nullptr || st == cudaStreamLegacy || st == cudaStreamPerThread;
      cudaStream_t gs = st;
      if (side) {
        if (!h->graph_stream) {
          CUDA_TRY(h, cudaStreamCreateWithFlags(&h->graph_stream, cudaStreamNonBlocking));
          CUDA_TRY(h, cudaEventCreateWithFlags(&h->graph_in, cudaEventDisableTiming));
          CUDA_TRY(h, cudaEventCreateWithFlags(&h->graph_out, cudaEventDisableTiming));
        }
        gs = h->graph_stream;
      }
      auto launch = [&](cudaGraphExec_t ex) -> cudaError_t {
        cudaError_t e = cudaSuccess;
        if (side) {
          if ((e = cudaEventRecord(h->graph_in, st)) != cudaSuccess) return e;
          if ((e = cudaStreamWaitEvent(gs, h->graph_in, 0)) != cudaSuccess) return e;
        }
        if ((e = cudaGraphLaunch(ex, gs)) != cudaSuccess) return e;
        if (side) {
          if ((e = cudaEventRecord(h->graph_out, gs)) != cudaSuccess) return e;
          if ((e = cudaStreamWaitEvent(st, h->graph_out, 0)) != cudaSuccess) return e;
        }
        return e;
      };
      mtb_handle::GraphEntry* ent = nullptr;
      for (auto& e : h->graphs)
        if (e.crops == crops && e.k == intrinsics && e.out == coords3d_abs && e.ws == workspace && e.batch == batch && e.st == st) ent = &e;
      if (ent && ent->exec) {
        CUDA_TRY(h, launch(ent->exec));
        h->launches = ent->launches;
        return MTB_OK;
      }
      if (ent && !ent->failed) {  // second sighting of this key: capture
        if (side) cudaStreamSynchronize(st);  // (once per key) everything the capture stream must see has completed
        if (cudaStreamBeginCapture(gs, cudaStreamCaptureModeRelaxed) == cudaSuccess) {
          rc = forward_body(h, crops, intrinsics, batch, coords3d_abs, workspace, gs);
          cudaGraph_t gr = nullptr;
          cudaError_t ce = cudaStreamEndCapture(gs, &gr);
          cudaGraphExec_t ex = nullptr;
          if (rc == MTB_OK && ce == cudaSuccess && gr && cudaGraphInstantiate(&ex, gr, 0) == cudaSuccess) {
            cudaGraphDestroy(gr);
            ent->exec = ex;
            ent->launches = h->launches;
            CUDA_TRY(h, launch(ent->exec));
            return MTB_OK;
          }
          if (gr) cudaGraphDestroy(gr);
        }
        cudaGetLastError();  // a refused capture leaves a sticky error behind: clear it before the plain launches
        ent->failed = true;  // plain launches for this key from now on
      } else if (!ent) {
        if (h->graphs.size() >= 8) drop_graphs_on(h, nullptr);  // a caller cycling through many buffers: bounded state
        mtb_handle::GraphEntry e;
        e.crops = crops; e.k = intrinsics; e.out = coords3d_abs; e.ws = workspace; e.batch = batch; e.st = st;
        h->graphs.push_back(e);
      }
    }
  }
  return forward_body(h, crops, intrinsics, batch, coords3d_abs, workspace, st);
}

int mtb_forward_host(mtb_handle* h, const float* host_crops, const float* host_intrinsics, int batch,
                     float* host_coords3d_abs, void* stream) {
  if (!h) return fail(nullptr, MTB_ERR_INVALID_ARG, "null handle");
  if (!h->finalized) return fail(h, MTB_ERR_NOT_FINALIZED, "mtb_finalize_weights has not been called");
  if (!host_crops || (!host_intrinsics && h->model_class != MTB_MODEL_METRO) || !host_coords3d_abs || batch <= 0)
    return fail(h, MTB_ERR_INVALID_ARG, "null/invalid argument");
  DeviceGuard g(h->cfg.device);
  cudaStream_t st = (cudaStream_t)stream;
  const size_t S = h->cfg.proc_side;
  const size_t crops_b = align_up((size_t)batch * 3 * S * S * 4, 1024), k_b = align_up((size_t)batch * 9 * 4, 1024),
               out_b = align_up((size_t)batch * output_joints(h) * 3 * 4, 1024);
  const size_t ws_b = layout(h, batch, nullptr).total;
  const size_t need = crops_b + k_b + out_b + ws_b;
  if (need > h->stage_bytes) {  // grows only when a larger batch than ever before arrives
    CUDA_TRY(h, cudaStreamSynchronize(st));
    if (h->stage) drop_graphs_on(h, (char*)h->stage + (h->stage_bytes - h->stage_ws_bytes));
    if (h->stage) cudaFree(h->stage);
    h->stage = nullptr;
    h->stage_bytes = 0;
    CUDA_TRY(h, cudaMalloc(&h->stage, need));
    h->stage_bytes = need;
    h->stage_ws_bytes = ws_b;
  }
  char* base = (char*)h->stage;
  float* d_crops = (float*)base;
  float* d_k = (float*)(base + crops_b);
  float* d_out = (float*)(base + crops_b + k_b);
  void* d_ws = base + crops_b + k_b + out_b;
  CUDA_TRY(h, cudaMemcpyAsync(d_crops, host_crops, (size_t)batch * 3 * S * S * 4, cudaMemcpyHostToDevice, st));
  if (host_intrinsics) CUDA_TRY(h, cudaMemcpyAsync(d_k, host_intrinsics, (size_t)batch * 9 * 4, cudaMemcpyHostToDevice, st));
  int rc = mtb_forward(h, d_crops, d_k, batch, d_out, d_ws, ws_b, stream);
  if (rc) return rc;
  CUDA_TRY(h, cudaMemcpyAsync(host_coords3d_abs, d_out, (size_t)batch * output_joints(h) * 3 * 4, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(h, cudaStreamSynchronize(st));
  return MTB_OK;
}

int mtb_forward_host_submit(mtb_handle* h, const float* host_crops, const float* host_intrinsics, int batch,
                            float* host_coords3d_abs, int slot, void* stream) {
  if (!h) return fail(nullptr, MTB_ERR_INVALID_ARG, "null handle");
  if (!h->finalized) return fail(h, MTB_ERR_NOT_FINALIZED, "mtb_finalize_weights has not been called");
  if (!host_crops || (!host_intrinsics && h->model_class != MTB_MODEL_METRO) || !host_coords3d_abs || batch <= 0 || slot < 0 ||
      slot > 1)
    return fail(h, MTB_ERR_INVALID_ARG, "null/invalid argument");
  DeviceGuard g(h->cfg.device);
  cudaStream_t st = (cudaStream_t)stream;
  const size_t S = h->cfg.proc_side;
  const size_t crops_b = align_up((size_t)batch * 3 * S * S * 4, 1024), k_b = align_up((size_t)batch * 9 * 4, 1024),
               out_b = align_up((size_t)batch * output_joints(h) * 3 * 4, 1024);
  const size_t ws_b = layout(h, batch, nullptr).total;
  mtb_handle::HostSlot& sl = h->slots[slot];
  if (!h->copy_stream) CUDA_TRY(h, cudaStreamCreateWithFlags(&h->copy_stream, cudaStreamNonBlocking));
  if (!sl.h2d_done) {
    CUDA_TRY(h, cudaEventCreateWithFlags(&sl.h2d_done, cudaEventDisableTiming));
    CUDA_TRY(h, cudaEventCreateWithFlags(&sl.done, cudaEventDisableTiming));
  }
  if (crops_b + k_b + out_b > sl.bytes || ws_b > h->pipe_ws_bytes) {  // grows only when a larger batch than ever before arrives
    CUDA_TRY(h, cudaDeviceSynchronize());
    if (crops_b + k_b + out_b > sl.bytes) {
      if (sl.buf) cudaFree(sl.buf);
      sl.buf = nullptr; sl.bytes = 0;
      CUDA_TRY(h, cudaMalloc(&sl.buf, crops_b + k_b + out_b));
      sl.bytes = crops_b + k_b + out_b;
    }
    if (ws_b > h->pipe_ws_bytes) {
      drop_graphs_on(h, h->pipe_ws);  // captured forwards that write into the old pipeline workspace
      if (h->pipe_ws) cudaFree(h->pipe_ws);
      h->pipe_ws = nullptr; h->pipe_ws_bytes = 0;
      CUDA_TRY(h, cudaMalloc(&h->pipe_ws, ws_b));
      h->pipe_ws_bytes = ws_b;
    }
  }
  char* base = (char*)sl.buf;
  float* d_crops = (float*)base;
  float* d_k = (float*)(base + crops_b);
  float* d_out = (float*)(base + crops_b + k_b);
  // copy stream: this slot's staging is free once its previous forward + read-back have completed
  if (sl.used) CUDA_TRY(h, cudaStreamWaitEvent(h->copy_stream, sl.done, 0));
  CUDA_TRY(h, cudaMemcpyAsync(d_crops, host_crops, (size_t)batch * 3 * S * S * 4, cudaMemcpyHostToDevice, h->copy_stream));
  if (host_intrinsics)
    CUDA_TRY(h, cudaMemcpyAsync(d_k, host_intrinsics, (size_t)batch * 9 * 4, cudaMemcpyHostToDevice, h->copy_stream));
  CUDA_TRY(h, cudaEventRecord(sl.h2d_done, h->copy_stream));
  // compute stream: forward of this step behind its own copy (and behind the previous step's forward: one workspace)
  CUDA_TRY(h, cudaStreamWaitEvent(st, sl.h2d_done, 0));
  int rc = mtb_forward(h, d_crops, d_k, batch, d_out, h->pipe_ws, h->pipe_ws_bytes, stream);
  if (rc) return rc;
  CUDA_TRY(h, cudaMemcpyAsync(host_coords3d_abs, d_out, (size_t)batch * output_joints(h) * 3 * 4, cudaMemcpyDeviceToHost, st));
  CUDA_TRY(h, cudaEventRecord(sl.done, st));
  sl.used = true;
  return MTB_OK;
}

int mtb_forward_host_wait(mtb_handle* h, int slot) {
  if (!h || slot < 0 || slot > 1) return fail(h, MTB_ERR_INVALID_ARG, "null handle / invalid slot");
  DeviceGuard g(h->cfg.device);
  if (!h->slots[slot].used) return MTB_OK;
  CUDA_TRY(h, cudaEventSynchronize(h->slots[slot].done));
  return MTB_OK;
}

// ------------------------------------------------------------------------------------------------- NCCL
typedef struct { char internal[128]; } nccl_uid;
static void* open_nccl() {
  const char* names[] = {"libnccl.so.2", "libnccl.so"};
  for (const char* n : names) {
    void* l = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
    if (l) return l;
  }
  return nullptr;
}

int mtb_comm_unique_id(void* id128) {
  if (!id128) return fail(nullptr, MTB_ERR_INVALID_ARG, "null id");
  void* lib = open_nccl();
  if (!lib) return fail(nullptr, MTB_ERR_NCCL, "cannot dlopen libnccl.so.2: %s", dlerror());
  typedef int (*fn_t)(nccl_uid*);
  fn_t f = (fn_t)dlsym(lib, "ncclGetUniqueId");
  if (!f) return fail(nullptr, MTB_ERR_NCCL, "ncclGetUniqueId not found");
  int rc = f((nccl_uid*)id128);
  if (rc) return fail(nullptr, MTB_ERR_NCCL, "ncclGetUniqueId failed (%d)", rc);
  return MTB_OK;
}

int mtb_comm_init(mtb_handle* h, const void* id128, int rank, int world_size) {
  if (!h || !id128 || rank < 0 || rank >= world_size) return fail(h, MTB_ERR_INVALID_ARG, "invalid communicator arguments");
  DeviceGuard g(h->cfg.device);
  if (!h->nccl_lib) h->nccl_lib = open_nccl();
  if (!h->nccl_lib) return fail(h, MTB_ERR_NCCL, "cannot dlopen libnccl.so.2: %s", dlerror());
  typedef int (*fn_t)(void**, int, nccl_uid, int);
  fn_t f = (fn_t)dlsym(h->nccl_lib, "ncclCommInitRank");
  if (!f) return fail(h, MTB_ERR_NCCL, "ncclCommInitRank not found");
  nccl_uid id;
  memcpy(&id, id128, sizeof(id));
  int rc = f(&h->nccl_comm, world_size, id, rank);
  if (rc) return fail(h, MTB_ERR_NCCL, "ncclCommInitRank failed (%d)", rc);
  h->nccl_world = world_size;
  return MTB_OK;
}

int mtb_allgather_joints(mtb_handle* h, const float* local, int floats_per_rank, float* all, void* stream) {
  if (!h || !local || !all || floats_per_rank <= 0) return fail(h, MTB_ERR_INVALID_ARG, "invalid all-gather arguments");
  if (!h->nccl_comm) return fail(h, MTB_ERR_NCCL, "mtb_comm_init has not been called");
  DeviceGuard g(h->cfg.device);
  typedef int (*fn_t)(const void*, void*, size_t, int, void*, cudaStream_t);
  static fn_t f = nullptr;
  if (!f) f = (fn_t)dlsym(h->nccl_lib, "ncclAllGather");
  if (!f) return fail(h, MTB_ERR_NCCL, "ncclAllGather not found");
  int rc = f(local, all, (size_t)floats_per_rank, /*ncclFloat32*/ 7, h->nccl_comm, (cudaStream_t)stream);
  if (rc) return fail(h, MTB_ERR_NCCL, "ncclAllGather failed (%d)", rc);
  return MTB_OK;
}

// ------------------------------------------------------------------------------------ multiperson (SURVEY 8f)
int mtb_image_pyramid(const uint8_t* images, int n_images, int height, int width, float* level1, float* level2, void* stream) {
  if (!images || !level1 || !level2 || n_images <= 0 || height < 4 || width < 4)
    return fail(nullptr, MTB_ERR_INVALID_ARG, "invalid pyramid arguments");
  cudaStream_t st = (cudaStream_t)stream;
  const int planes = n_images * 3;
  const size_t t1 = (size_t)planes * (height / 2) * (width / 2), t2 = (size_t)planes * (height / 4) * (width / 4);
  launch_k(pyramid_level1_kernel, dim3(grid_for(t1, 256)), dim3(256), 0, st, images, level1, planes, height, width);
  launch_k(pyramid_down_kernel, dim3(grid_for(t2, 256)), dim3(256), 0, st, (const float*)level1, level2, planes, height / 2, width / 2);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(nullptr, MTB_ERR_CUDA, "pyramid launch: %s", cudaGetErrorString(e));
  return MTB_OK;
}

int mtb_crop_setup(const mtb_crop_setup_args* a, void* stream) {
  if (!a || !a->boxes || !a->intrinsics || !a->camspace_up || !a->aug_rotflipmat || !a->aug_scales || !a->new_intrinsics ||
      !a->rotations || !a->inv_projections || !a->pyramid_levels || (a->n_dist > 0 && !a->distortion))
    return fail(nullptr, MTB_ERR_INVALID_ARG, "null crop-setup argument");
  if (a->n_boxes <= 0 || a->num_aug <= 0 || a->num_aug > MP_MAX_AUG || a->box_stride < 4 || a->n_dist < 0 || a->n_dist > MP_NDIST ||
      a->resolution <= 0)
    return fail(nullptr, MTB_ERR_INVALID_ARG, "invalid crop-setup sizes (n_boxes=%d num_aug=%d n_dist=%d)", a->n_boxes, a->num_aug, a->n_dist);
  if (a->antialias_factor != 1 && a->antialias_factor != 2 && a->antialias_factor != 4)
    return fail(nullptr, MTB_ERR_UNSUPPORTED, "antialias_factor must be 1, 2 or 4 (got %d)", a->antialias_factor);
  CropSetupParams p;
  p.boxes = a->boxes; p.box_stride = a->box_stride; p.K = a->intrinsics; p.dist = a->distortion; p.ncoef = a->n_dist;
  p.up = a->camspace_up; p.rotflip = a->aug_rotflipmat; p.aug_scales = a->aug_scales;
  p.n_box = a->n_boxes; p.num_aug = a->num_aug; p.res = a->resolution; p.antialias = a->antialias_factor;
  p.new_K = a->new_intrinsics; p.R = a->rotations; p.invproj = a->inv_projections; p.level = a->pyramid_levels;
  launch_k(crop_setup_kernel, dim3((a->n_boxes + 127) / 128), dim3(128), 0, (cudaStream_t)stream, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(nullptr, MTB_ERR_CUDA, "crop setup launch: %s", cudaGetErrorString(e));
  return MTB_OK;
}

int mtb_warp_crops(const mtb_warp_args* a, void* stream) {
  if (!a || !a->images || !a->level1 || !a->level2 || !a->intrinsics || !a->image_ids || !a->inv_projections ||
      !a->pyramid_levels || !a->gamma_exponents || !a->crops || (a->n_dist > 0 && !a->distortion))
    return fail(nullptr, MTB_ERR_INVALID_ARG, "null warp argument");
  if (a->n_boxes <= 0 || a->num_aug <= 0 || a->num_aug > MP_MAX_AUG || a->n_dist < 0 || a->n_dist > MP_NDIST || a->resolution <= 0 ||
      a->height < 4 || a->width < 4 || a->n_images <= 0)
    return fail(nullptr, MTB_ERR_INVALID_ARG, "invalid warp sizes");
  if (a->antialias_factor != 1 && a->antialias_factor != 2 && a->antialias_factor != 4)
    return fail(nullptr, MTB_ERR_UNSUPPORTED, "antialias_factor must be 1, 2 or 4 (got %d)", a->antialias_factor);
  if ((long long)a->n_boxes * a->num_aug > 65535) return fail(nullptr, MTB_ERR_UNSUPPORTED, "more than 65535 crops per call");
  WarpParams p;
  p.img = a->images; p.l1 = a->level1; p.l2 = a->level2; p.N = a->n_images; p.H = a->height; p.W = a->width;
  p.K = a->intrinsics; p.dist = a->distortion; p.ncoef = a->n_dist; p.image_ids = a->image_ids; p.invproj = a->inv_projections;
  p.level = a->pyramid_levels; p.gamma_exp = a->gamma_exponents; p.n_box = a->n_boxes; p.num_aug = a->num_aug;
  p.res = a->resolution; p.antialias = a->antialias_factor; p.crops = a->crops;
  const int npix = a->resolution * a->resolution;
  launch_k(warp_crops_kernel, dim3((npix + 255) / 256, a->n_boxes * a->num_aug), dim3(256), 0, (cudaStream_t)stream, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(nullptr, MTB_ERR_CUDA, "warp launch: %s", cudaGetErrorString(e));
  return MTB_OK;
}

int mtb_tta_merge(const mtb_tta_args* a, void* stream) {
  if (!a || !a->poses || !a->rotations || !a->aug_should_flip || !a->mirror_mapping || !a->intrinsics || !a->extrinsics_inv ||
      !a->poses3d || !a->poses2d || (a->n_dist > 0 && !a->distortion))
    return fail(nullptr, MTB_ERR_INVALID_ARG, "null TTA-merge argument");
  if (a->n_boxes <= 0 || a->num_aug <= 0 || a->n_joints <= 0 || a->n_dist < 0 || a->n_dist > MP_NDIST)
    return fail(nullptr, MTB_ERR_INVALID_ARG, "invalid TTA-merge sizes");
  TtaParams p;
  p.poses = a->poses; p.R = a->rotations; p.flip = a->aug_should_flip; p.mirror = a->mirror_mapping; p.jt = a->joint_transform;
  p.skel = a->skeleton; p.K = a->intrinsics; p.dist = a->distortion; p.ncoef = a->n_dist; p.ext_inv = a->extrinsics_inv;
  p.n_box = a->n_boxes; p.num_aug = a->num_aug; p.J = a->n_joints;
  p.J2 = a->joint_transform ? a->n_joints_transformed : a->n_joints;
  p.Js = a->skeleton ? a->n_skeleton : p.J2;
  p.average = a->average_aug ? 1 : 0;
  p.poses3d = a->poses3d; p.poses2d = a->poses2d;
  if (p.J2 <= 0 || p.Js <= 0) return fail(nullptr, MTB_ERR_INVALID_ARG, "invalid joint counts");
  launch_k(tta_merge_kernel, dim3(a->n_boxes), dim3(128), 0, (cudaStream_t)stream, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(nullptr, MTB_ERR_CUDA, "TTA merge launch: %s", cudaGetErrorString(e));
  return MTB_OK;
}

int mtb_filter_poses(const mtb_filter_args* a, void* stream) {
  if (!a || !a->poses3d || !a->poses2d || !a->boxes || !a->image_start || !a->plausible || !a->keep || !a->scratch ||
      (a->n_bones > 0 && (!a->bones || !a->mean_bones)))
    return fail(nullptr, MTB_ERR_INVALID_ARG, "null pose-filter argument");
  if (a->n_images <= 0 || a->n_boxes <= 0 || a->num_aug < 2 || a->num_aug > MP_MAX_AUG || a->n_joints < 4 || a->box_stride < 5)
    return fail(nullptr, MTB_ERR_INVALID_ARG, "invalid pose-filter sizes (num_aug must be 2..16, boxes need a score column)");
  FilterParams p;
  p.poses3d = a->poses3d; p.poses2d = a->poses2d; p.boxes = a->boxes; p.box_stride = a->box_stride; p.bones = a->bones;
  p.mean_bones = a->mean_bones; p.n_bones = a->n_bones; p.image_start = a->image_start; p.num_aug = a->num_aug; p.J = a->n_joints;
  p.plausible = a->plausible; p.keep = a->keep; p.scratch = a->scratch;
  // every image's box count is at most n_boxes, so per-box state for n_boxes boxes covers the most crowded image
  p.max_boxes = a->n_boxes;
  int dev = 0, optin = 0;
  cudaFuncAttributes fa;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, pose_filter_kernel);
  if (e != cudaSuccess) return fail(nullptr, MTB_ERR_CUDA, "pose filter setup: %s", cudaGetErrorString(e));
  const long long smem = (long long)a->n_boxes * MP_FILTER_SMEM_PER_BOX;
  if (smem > (long long)optin - (long long)fa.sharedSizeBytes)
    return fail(nullptr, MTB_ERR_UNSUPPORTED, "pose filter: %d boxes need %lld B of shared memory, the device holds %d B per block "
                "(at most %d boxes per call)", a->n_boxes, smem, optin - (int)fa.sharedSizeBytes,
                (optin - (int)fa.sharedSizeBytes) / MP_FILTER_SMEM_PER_BOX);
  if (const char* err = launch_smem(pose_filter_kernel, dim3(a->n_images), dim3(FILTER_THREADS), (int)smem, (cudaStream_t)stream, p))
    return fail(nullptr, MTB_ERR_CUDA, "pose filter launch: %s", err);
  return MTB_OK;
}

// Data-parallel forward (SURVEY.md 8e): local crops -> backbone -> head decode, ONE all-gather of [coords2d | coords3d_rel]
// (5 floats per joint), absolute reconstruction of the FULL batch on every rank - reconstruct_ref_fullpersp normalises with
// batch-global RMS scalars (ptu3d.py:71-74), so only a full-batch solve reproduces the unsharded result exactly.
size_t mtb_sharded_scratch_bytes(const mtb_handle* h, int batch_local) {
  if (!h || batch_local <= 0 || h->nccl_world <= 0) return 0;
  const size_t J = (size_t)head_points(h), bl = (size_t)batch_local, bt = bl * (size_t)h->nccl_world;
  if (head3d(h))  // the gathered coords25d [bt,J,3] and the solve's scratch (a Metro handle gathers into the output)
    return align_up(bt * J * 3 * 4, 256) + (h->model_class == MTB_MODEL_25D ? bone_scratch_bytes(h, (int)bt) : 0);
  return align_up(bl * J * 5 * 4, 256) + align_up(bt * J * 5 * 4, 256) + align_up(bt * J * 2 * 4, 256) + align_up(bt * J * 3 * 4, 256) +
         align_up(bt * J * 2 * 4, 256) + align_up(bt * 2 * 8, 256) + (h->n_latents > 0 ? align_up(bt * J * 3 * 4, 256) : 0);
}

int mtb_forward_sharded(mtb_handle* h, const float* crops_local, int batch_local, const float* intrinsics_all, float* coords3d_abs_all,
                        void* scratch, void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_common(h, batch_local, workspace_bytes, workspace);
  if (rc) return rc;
  if (!crops_local || (!intrinsics_all && h->model_class != MTB_MODEL_METRO) || !coords3d_abs_all ||
      (!scratch && h->model_class != MTB_MODEL_METRO))
    return fail(h, MTB_ERR_INVALID_ARG, "null argument");
  if (!h->nccl_comm) return fail(h, MTB_ERR_NCCL, "mtb_comm_init has not been called");
  if (h->ops.empty()) return fail(h, MTB_ERR_UNSUPPORTED, "this handle has no backbone (head-only)");
  DeviceGuard g(h->cfg.device);
  cudaStream_t st = (cudaStream_t)stream;
  const size_t J = (size_t)head_points(h), bl = (size_t)batch_local, bt = bl * (size_t)h->nccl_world;
  char* sp = (char*)scratch;
  float* packed_local = (float*)sp; sp += align_up(bl * J * 5 * 4, 256);
  float* packed_all = (float*)sp;   sp += align_up(bt * J * 5 * 4, 256);
  float* c2d_all = (float*)sp;      sp += align_up(bt * J * 2 * 4, 256);
  float* c3d_all = (float*)sp;      sp += align_up(bt * J * 3 * 4, 256);
  float* n2d = (float*)sp;          sp += align_up(bt * J * 2 * 4, 256);
  double* partial = (double*)sp;    sp += align_up(bt * 2 * 8, 256);
  float* latents = (float*)sp;      // [bt,L,3], latent-point models only
  h->launches = 0;
  Workspace ws = layout(h, batch_local, workspace);
  void* features = ws.base + ws.off_features;
  rc = run_backbone(h, crops_local, batch_local, ws, features, st);
  if (rc) return rc;
  float* c2d = (float*)(ws.base + ws.off_c2d);
  float* c3d = (float*)(ws.base + ws.off_c3d);
  if (head3d(h)) {
    // Metro: the decoded joints are the output, gathered in rank order.  Model25D: ONE all-gather of coords25d (3 floats per
    // joint), then the batch-coupled bone-length solve on the full batch on every rank, as the unsharded forward runs it.
    float* all = h->model_class == MTB_MODEL_METRO ? coords3d_abs_all : (float*)scratch;
    rc = head_decode_impl(h, features, batch_local, nullptr, c3d, ws, st);
    if (rc) return rc;
    rc = mtb_allgather_joints(h, c3d, (int)(bl * J * 3), all, stream);
    if (rc) return rc;
    h->launches += 1;
    if (h->model_class == MTB_MODEL_METRO) return MTB_OK;
    return bone_solve_impl(h, all, intrinsics_all, (int)bt, coords3d_abs_all, (char*)scratch + align_up(bt * J * 3 * 4, 256), st);
  }
  rc = head_decode_impl(h, features, batch_local, c2d, c3d, ws, st);
  if (rc) return rc;
  const int64_t before = h->launches;
  launch_k(pack_decoded_kernel, dim3(grid_for(bl * J, 256)), dim3(256), 0, st, (const float*)c2d, (const float*)c3d, packed_local,
           (int)(bl * J));
  rc = mtb_allgather_joints(h, packed_local, (int)(bl * J * 5), packed_all, stream);
  if (rc) return rc;
  launch_k(unpack_decoded_kernel, dim3(grid_for(bt * J, 256)), dim3(256), 0, st, (const float*)packed_all, c2d_all, c3d_all, (int)(bt * J));
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(h, MTB_ERR_CUDA, "pack/unpack launch: %s", cudaGetErrorString(e));
  rc = recon_and_combine(h, c2d_all, c3d_all, intrinsics_all, (int)bt, coords3d_abs_all, n2d, partial, latents, st);
  h->launches = before + 3 + 2 + (h->n_latents > 0 ? 1 : 0);  // pack, all-gather, unpack, reconstruction passes, recombination
  return rc;
}

// ---------------------------------------------------------------------------------------- introspection
int mtb_num_ops(const mtb_handle* h) { return h ? (int)h->ops.size() : 0; }

const char* mtb_op_name(const mtb_handle* h, int op) {
  if (!h || op < 0 || op >= (int)h->ops.size()) return "";
  return h->ops[op].name.c_str();
}

int mtb_op_output_shape(const mtb_handle* h, int op, int* height, int* width, int* channels) {
  if (!h || op < 0 || op >= (int)h->ops.size()) return fail(h, MTB_ERR_INVALID_ARG, "op index out of range");
  const Op& o = h->ops[op];
  if (height) *height = (o.type == OP_POOL || o.small_io) ? 1 : o.Hout;
  if (width) *width = (o.type == OP_POOL || o.small_io) ? 1 : o.Wout;
  if (channels) *channels = o.Cout;
  return MTB_OK;
}

int mtb_debug_run_ops(mtb_handle* h, const float* crops, int batch, int n_ops, float* out, size_t out_floats,
                      void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_common(h, batch, workspace_bytes, workspace);
  if (rc) return rc;
  if (n_ops <= 0 || n_ops > (int)h->ops.size() || !out || !crops) return fail(h, MTB_ERR_INVALID_ARG, "invalid debug arguments");
  DeviceGuard g(h->cfg.device);
  cudaStream_t st = (cudaStream_t)stream;
  Workspace ws = layout(h, batch, workspace);
  void* features = ws.base + ws.off_features;
  rc = run_ops_range(h, 0, (size_t)n_ops, crops, batch, ws, features, st);
  if (rc) return rc;
  const Op& o = h->ops[n_ops - 1];
  const bool small = o.type == OP_POOL || o.small_io;
  size_t n = (size_t)batch * (small ? 1 : (size_t)o.Hout * o.Wout) * o.Cout;
  if (n > out_floats) return fail(h, MTB_ERR_INVALID_ARG, "debug output buffer too small (%zu > %zu)", n, out_floats);
  void* src = buf_ptr(ws, o.out_buf, features);
  if (small) CUDA_TRY(h, cudaMemcpyAsync(out, src, n * 4, cudaMemcpyDeviceToDevice, st));
  else copy_to_float(h, src, out, n, st);
  CUDA_TRY(h, cudaGetLastError());
  return MTB_OK;
}

int mtb_profile_begin(mtb_handle* h, unsigned class_mask) {
  if (!h) return fail(nullptr, MTB_ERR_INVALID_ARG, "null handle");
  h->prof_mask = class_mask;
  h->prof_used = 0;
  h->prof_cls.clear();
  h->prof_op.clear();
  h->prof_flops.clear();
  h->prof_bytes.clear();
  return MTB_OK;
}

int mtb_profile_end(mtb_handle* h, double* ms, double* flops, double* bytes, int64_t* launches) {
  if (!h || !ms || !flops || !bytes || !launches) return fail(h, MTB_ERR_INVALID_ARG, "null argument");
  DeviceGuard g(h->cfg.device);
  for (int i = 0; i < KC_COUNT; ++i) { ms[i] = 0; flops[i] = 0; bytes[i] = 0; launches[i] = 0; }
  h->prof_op_ms.assign(h->ops.size(), 0.0);
  for (size_t i = 0; i < h->prof_cls.size(); ++i) {
    CUDA_TRY(h, cudaEventSynchronize(h->prof_events[2 * i + 1]));
    float t = 0.f;
    CUDA_TRY(h, cudaEventElapsedTime(&t, h->prof_events[2 * i], h->prof_events[2 * i + 1]));
    int cls = h->prof_cls[i];
    ms[cls] += t;
    if (h->prof_op[i] >= 0 && h->prof_op[i] < (int)h->prof_op_ms.size()) h->prof_op_ms[h->prof_op[i]] += t;
    flops[cls] += h->prof_flops[i];
    bytes[cls] += h->prof_bytes[i];
    launches[cls] += (cls == KC_RECON) ? 2 : 1;
  }
  h->prof_mask = 0;
  h->prof_used = 0;
  h->prof_cls.clear();
  h->prof_op.clear();
  h->prof_flops.clear();
  h->prof_bytes.clear();
  return MTB_OK;
}

/* per-op device time (ms) accumulated by the last mtb_profile_begin/end window, plus each op's algorithmic FLOPs and
 * bytes PER CROP and its kernel class */
int mtb_profile_op_times(const mtb_handle* h, double* ms, double* flops_per_crop, double* bytes_per_crop, int* cls, int n) {
  if (!h || !ms || n < (int)h->ops.size()) return fail(h, MTB_ERR_INVALID_ARG, "invalid arguments");
  for (size_t i = 0; i < h->ops.size(); ++i) {
    ms[i] = i < h->prof_op_ms.size() ? h->prof_op_ms[i] : 0.0;
    if (flops_per_crop) flops_per_crop[i] = h->ops[i].flops;
    if (bytes_per_crop) bytes_per_crop[i] = op_bytes(h, h->ops[i], 1) - op_weight_bytes(h->ops[i]);  // activations only
    if (cls) cls[i] = op_class(h->ops[i]);
  }
  return MTB_OK;
}

double mtb_op_weight_bytes(const mtb_handle* h, int op) {
  if (!h || op < 0 || op >= (int)h->ops.size()) return 0.0;
  return op_weight_bytes(h->ops[op]);
}

int mtb_num_kernel_classes(void) { return KC_COUNT; }
const char* mtb_kernel_class_name(int cls) { return (cls >= 0 && cls < KC_COUNT) ? kKClassNames[cls] : ""; }

int mtb_op_input_shape(const mtb_handle* h, int op, int* height, int* width, int* channels, int* has_residual, int* has_scale) {
  if (!h || op < 0 || op >= (int)h->ops.size()) return fail(h, MTB_ERR_INVALID_ARG, "op index out of range");
  const Op& o = h->ops[op];
  if (height) *height = o.Hin;
  if (width) *width = o.Win;
  if (channels) *channels = o.Cin;
  if (has_residual) *has_residual = o.res_buf != BUF_NONE;
  if (has_scale) *has_scale = o.scale_buf != BUF_NONE;
  return MTB_OK;
}

int mtb_debug_run_op(mtb_handle* h, int op_index, const float* in, const float* res, const float* scale, int batch,
                     float* out, size_t out_floats, void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_common(h, batch, workspace_bytes, workspace);
  if (rc) return rc;
  if (op_index < 0 || op_index >= (int)h->ops.size() || !in || !out) return fail(h, MTB_ERR_INVALID_ARG, "invalid debug arguments");
  DeviceGuard g(h->cfg.device);
  cudaStream_t st = (cudaStream_t)stream;
  Workspace ws = layout(h, batch, workspace);
  Op o = h->ops[op_index];  // copy with overridden buffers
  const bool small = o.type == OP_POOL || o.small_io;
  const size_t n_in = (size_t)batch * o.Hin * o.Win * o.Cin;
  const size_t n_out = (size_t)batch * (o.type == OP_POOL ? 1 : (size_t)o.Hout * o.Wout) * o.Cout;
  if (n_out > out_floats) return fail(h, MTB_ERR_INVALID_ARG, "debug output buffer too small");
  if ((o.res_buf != BUF_NONE) != (res != nullptr) || (o.scale_buf != BUF_NONE) != (scale != nullptr))
    return fail(h, MTB_ERR_INVALID_ARG, "op %d: residual/scale inputs do not match the op (see mtb_op_input_shape)", op_index);
  auto put = [&](const float* src, int buf, size_t n, bool as_f32) {
    void* dst = buf_ptr(ws, buf, nullptr);
    if (as_f32) cudaMemcpyAsync(dst, src, n * 4, cudaMemcpyDeviceToDevice, st);
    else copy_from_float(h, src, dst, n, st);
  };
  const float* crops = nullptr;
  if (o.type == OP_STEM) {
    crops = in;
  } else if (o.small_io) {
    o.in_buf = BUF_SMALL0;
    put(in, o.in_buf, n_in, true);
  } else {
    o.in_buf = 0;
    put(in, 0, n_in, false);
  }
  if (res) { o.res_buf = 1; put(res, 1, n_out, false); }
  if (scale) { o.scale_buf = BUF_SMALL0 + 2; put(scale, o.scale_buf, (size_t)batch * o.Cin, true); }
  o.out_buf = (o.type == OP_POOL || o.small_io) ? BUF_SMALL0 + 1 : 2;
  o.fused_pool = false;  // in isolation a depthwise op does not pool and a pool op runs its own kernel
  if (o.kernel == MTB_POOL_FUSED) o.kernel = MTB_POOL_MEAN;
  rc = run_op(h, o, crops, batch, ws, nullptr, st);
  if (rc) return rc;
  void* src = buf_ptr(ws, o.out_buf, nullptr);
  if (small) CUDA_TRY(h, cudaMemcpyAsync(out, src, n_out * 4, cudaMemcpyDeviceToDevice, st));
  else copy_to_float(h, src, out, n_out, st);
  CUDA_TRY(h, cudaGetLastError());
  return MTB_OK;
}

int mtb_op_kernel(const mtb_handle* h, int op) {
  if (!h || op < 0 || op >= (int)h->ops.size()) return fail(h, MTB_ERR_INVALID_ARG, "op index out of range");
  if (!h->finalized) return fail(h, MTB_ERR_NOT_FINALIZED, "mtb_finalize_weights has not been called");
  return h->ops[op].kernel;
}

int mtb_op_is_fused_block(const mtb_handle* h, int op_index) {
  return (h && op_index >= 0 && op_index + 1 < (int)h->ops.size() && h->ops[op_index].fmb.ready) ? 1 : 0;
}

int mtb_debug_op_buffers(const mtb_handle* h, int op, int* in_buf, int* out_buf, int* res_buf, int* scale_buf) {
  if (!h || op < 0 || op >= (int)h->ops.size()) return fail(h, MTB_ERR_INVALID_ARG, "op index out of range");
  const Op& o = h->ops[op];
  if (in_buf) *in_buf = o.in_buf;
  if (out_buf) *out_buf = o.out_buf;
  if (res_buf) *res_buf = o.res_buf;
  if (scale_buf) *scale_buf = o.scale_buf;
  return MTB_OK;
}

int mtb_debug_run_fused_block(mtb_handle* h, int op_index, const float* in, int batch, float* out, size_t out_floats, void* workspace,
                              size_t workspace_bytes, void* stream) {
  int rc = check_common(h, batch, workspace_bytes, workspace);
  if (rc) return rc;
  if (op_index < 0 || op_index + 1 >= (int)h->ops.size() || !in || !out) return fail(h, MTB_ERR_INVALID_ARG, "invalid debug arguments");
  if (!h->ops[op_index].fmb.ready) return fail(h, MTB_ERR_UNSUPPORTED, "op %d does not start a fused FusedMBConv block", op_index);
  DeviceGuard g(h->cfg.device);
  cudaStream_t st = (cudaStream_t)stream;
  Workspace ws = layout(h, batch, workspace);
  Op a = h->ops[op_index], b = h->ops[op_index + 1];
  const size_t n_in = (size_t)batch * a.Hin * a.Win * a.Cin, n_out = (size_t)batch * b.Hout * b.Wout * b.Cout;
  if (n_out > out_floats) return fail(h, MTB_ERR_INVALID_ARG, "debug output buffer too small");
  copy_from_float(h, in, buf_ptr(ws, 0, nullptr), n_in, st);
  a.in_buf = 0; a.out_buf = 1; b.in_buf = 1; b.out_buf = 2;
  if (b.res_buf != BUF_NONE) b.res_buf = 0;
  rc = run_fused_block(h, a, b, batch, ws, nullptr, st);
  if (rc) return rc;
  copy_to_float(h, buf_ptr(ws, 2, nullptr), out, n_out, st);
  CUDA_TRY(h, cudaGetLastError());
  return MTB_OK;
}

int mtb_op_is_preact_pair(const mtb_handle* h, int op_index) {
  return (h && op_index >= 0 && op_index + 1 < (int)h->ops.size() && h->ops[op_index].preact_next) ? 1 : 0;
}

int mtb_debug_run_preact_pair(mtb_handle* h, int op_index, const float* in, const float* res, int batch, float* out, float* out_preact,
                              size_t out_floats, void* workspace, size_t workspace_bytes, void* stream) {
  int rc = check_common(h, batch, workspace_bytes, workspace);
  if (rc) return rc;
  if (op_index < 0 || op_index + 1 >= (int)h->ops.size() || !in || !res || !out || !out_preact)
    return fail(h, MTB_ERR_INVALID_ARG, "invalid debug arguments");
  if (!h->ops[op_index].preact_next) return fail(h, MTB_ERR_UNSUPPORTED, "op %d does not run fused with the pre-activation after it", op_index);
  DeviceGuard g(h->cfg.device);
  cudaStream_t st = (cudaStream_t)stream;
  Workspace ws = layout(h, batch, workspace);
  Op a = h->ops[op_index], b = h->ops[op_index + 1];
  const size_t n_in = (size_t)batch * a.Hin * a.Win * a.Cin, n_out = (size_t)batch * a.Hout * a.Wout * a.Cout;
  if (n_out > out_floats) return fail(h, MTB_ERR_INVALID_ARG, "debug output buffer too small");
  copy_from_float(h, in, buf_ptr(ws, 0, nullptr), n_in, st);
  copy_from_float(h, res, buf_ptr(ws, 1, nullptr), n_out, st);
  a.in_buf = 0; a.res_buf = 1; a.out_buf = 2; b.in_buf = 2; b.out_buf = 3;
  rc = run_preact_pair(h, a, b, batch, ws, nullptr, st);
  if (rc) return rc;
  copy_to_float(h, buf_ptr(ws, 2, nullptr), out, n_out, st);
  copy_to_float(h, buf_ptr(ws, 3, nullptr), out_preact, n_out, st);
  CUDA_TRY(h, cudaGetLastError());
  return MTB_OK;
}

int64_t mtb_last_launch_count(const mtb_handle* h) { return h ? h->launches : 0; }
double mtb_backbone_flops_per_crop(const mtb_handle* h) { return h ? h->flops_per_crop : 0.0; }

int mtb_debug_dw_plan(int height, int width, int* crops_per_item, int* rows_per_item, int* row_bands, int* stage_bytes) {
  if (height <= 0 || width <= 0 || !crops_per_item || !rows_per_item || !row_bands || !stage_bytes)
    return fail(nullptr, MTB_ERR_INVALID_ARG, "invalid arguments");
  const DwTmaPlan pl = dw_tma_plan(height, width);
  if (!pl.ok) { *crops_per_item = *rows_per_item = *row_bands = *stage_bytes = 0; return MTB_OK; }
  *crops_per_item = pl.G;
  *rows_per_item = pl.BH;
  *row_bands = pl.n_rb;
  *stage_bytes = 128 * (width + 2) * (pl.BH + 2) * pl.G;
  return MTB_OK;
}

}  // extern "C"
