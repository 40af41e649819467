// DCSCN engine: graph plan, parameter storage / packing, workspace, launch orchestration and the C-ABI
// declared in include/dcscn_b200.h.  Stands in for what `sess.run(self.y_)` executed in the reference
// (DCSCN.py:565; graph built by DCSCN.py:222-332 and helper/tf_graph.py:104-249).
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include "../../include/dcscn_b200.h"
#include "common.h"
#include "conv_aux.cuh"
#include "conv_tc.cuh"
#include "conv_ds_tile.cuh"
#include "train.cuh"
#include "wgrad_tc.cuh"
#include "train_ds.cuh"
#include "tile.cuh"
#include "eval.cuh"

using namespace dcscn;

// ----------------------------------------------------------------------------------------- errors ----
static thread_local std::string g_last_error;

static int fail(const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_last_error = buf;
  return 1;
}

#define CUDA_TRY(expr)                                                                         \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess)                                                                     \
      return fail("%s failed at %s:%d: %s", #expr, __FILE__, __LINE__, cudaGetErrorString(_e)); \
  } while (0)

// ---------------------------------------------------------------------------------- device memory ----
// The one owner of a cudaMalloc allocation of size() elements of T: the destructor frees it.  Pointers taken from get()
// (kernel parameters, launch plans, tensor maps) do not own it.
template <typename T>
class DeviceArray {
 public:
  DeviceArray() = default;
  DeviceArray(const DeviceArray&) = delete;
  DeviceArray& operator=(const DeviceArray&) = delete;
  DeviceArray(DeviceArray&& o) noexcept : p_(o.p_), n_(o.n_) { o.p_ = nullptr; o.n_ = 0; }
  DeviceArray& operator=(DeviceArray&& o) noexcept {
    if (this != &o) {
      release();
      std::swap(p_, o.p_);
      std::swap(n_, o.n_);
    }
    return *this;
  }
  ~DeviceArray() { release(); }

  T* get() const { return p_; }
  size_t size() const { return n_; }

  // Frees, then allocates n elements (n = 0 leaves the array empty), zero-filled when asked.
  int alloc(size_t n, bool zero = false) {
    release();
    if (n == 0) return 0;
    void* p = nullptr;
    CUDA_TRY(cudaMalloc(&p, n * sizeof(T)));
    p_ = static_cast<T*>(p);
    n_ = n;
    if (zero) CUDA_TRY(cudaMemset(p_, 0, n * sizeof(T)));
    return 0;
  }
  // Grow-only staging: reallocates, without zero-filling, only when n exceeds the current size.
  int grow(size_t n) { return n > n_ ? alloc(n) : 0; }
  // Copies `host` in.  An allocation of the same size is reused, so the pointers cached launch plans embed stay valid
  // across weight updates; otherwise it is replaced and *moved is set.
  int upload(const std::vector<T>& host, bool* moved = nullptr) {
    if (host.size() != n_) {
      if (moved) *moved = true;
      if (alloc(host.size())) return 1;
    }
    if (n_) CUDA_TRY(cudaMemcpy(p_, host.data(), n_ * sizeof(T), cudaMemcpyHostToDevice));
    return 0;
  }

 private:
  void release() {
    if (p_) cudaFree(p_);
    p_ = nullptr;
    n_ = 0;
  }
  T* p_ = nullptr;
  size_t n_ = 0;
};

// The hi and lo fp16 planes of one tensor (hi + lo = the value) at some channel offset.  In f16x1 there is no lo plane:
// lo stays null at every offset.
struct PlaneView {
  __half* hi = nullptr;
  __half* lo = nullptr;
  PlaneView at(size_t off) const { return {hi ? hi + off : nullptr, lo ? lo + off : nullptr}; }
};
struct Planes {
  DeviceArray<__half> hi, lo;
  // n zero-filled elements per plane; lo stays empty unless `two`
  int alloc(size_t n, bool two) { return hi.alloc(n, true) || lo.alloc(two ? n : 0, true); }
  PlaneView at(size_t off) const { return PlaneView{hi.get(), lo.get()}.at(off); }
  int64_t bytes() const { return (int64_t)((hi.size() + lo.size()) * sizeof(__half)); }
};

struct StreamDeleter { void operator()(cudaStream_t s) const { cudaStreamDestroy(s); } };
struct EventDeleter { void operator()(cudaEvent_t e) const { cudaEventDestroy(e); } };
using Stream = std::unique_ptr<std::remove_pointer_t<cudaStream_t>, StreamDeleter>;
using Event = std::unique_ptr<std::remove_pointer_t<cudaEvent_t>, EventDeleter>;

static inline int pad16(int v) { return (v + 15) & ~15; }

// ------------------------------------------------------------------------------------- graph plan ----
struct LayerDef {
  std::string scope;  // TF variable scope, e.g. "CNN3", "Up-PS/Up-PS_CNN"
  int k, cin, cout;
  bool bias;
  bool act;           // activated (--activator, then dropout): CNN1..CNNL, A1, B1, B2
};

struct ParamDef {
  std::string name;
  std::vector<int64_t> shape;
  std::vector<float> host;
  std::vector<float> shadow;    // flat index + 2 of every element (float-coded), see build_refresh_maps
  int64_t numel() const {
    int64_t n = 1;
    for (auto d : shape) n *= d;
    return n;
  }
};

// device-side packed form of one tensor-core layer (possibly a fusion of several TF layers)
struct TcLayer {
  std::string name;
  int ksz = 3;
  int cin_pad = 0;              // channel extent of the source region
  int n_tiles = 1, n_pad = 16;  // column tiling
  int n_valid = 0;
  std::vector<int> in_map;      // logical cin -> channel position in the source region
  std::vector<float> w_host;    // fused HWIO fp32 [taps][cin][cout]
  std::vector<float> bias_host, alpha_host;  // [n_tiles*n_pad]
  int cin = 0, cout = 0;
  float wscale = 1.f;
  DeviceArray<__half> d_wpack;
  DeviceArray<float> d_bias;
  DeviceArray<float> d_alpha;
  DeviceArray<float> d_wref;    // fp32 HWIO for the validation kernel
  DeviceArray<int> d_in_map;
  int packed_planes = 0;
  DeviceArray<int> d_img_map;   // training: flat parameter index behind every hi-plane element of d_wpack (-1 = zero)
  // wide depthwise-separable graphs: the k x k depthwise step that runs in front of this 1x1 pointwise layer
  int dw_ksz = 0;               // 0 = none
  std::vector<float> dw_host;   // [taps][cin_pad] by source position, zero where no channel maps
  DeviceArray<float> d_dw;
};

struct GatherJob {   // training: dst[i] = d_w[map[i]] where map[i] >= 0 (biases, PReLU slopes, CNN1 / R-CNN1 filters)
  float* dst;
  int* map;
  int n;
};

// The buffers a named activation lives in: the fp16 planes dcscn_handle::feat / nin / b1 / mid and the fp32 hr of the
// tensor-core graphs, or the fp32 ds_* buffers of forward_ds_tile.
enum ActBuf { BUF_FEAT, BUF_NIN, BUF_B1, BUF_MID, BUF_HR };

// A named activation (act_view): where it lives, and the dropout stream the forward, the backward and the CPU oracles
// (dcscn_dropout_mask) must agree on.
struct ActView {
  ActBuf buf;
  PlaneView planes;               // tensor-core layouts: the planes at the tensor's first channel
  const float* f32;               // fp32 buffers: the tensor's first channel
  int pitch, off, ch;             // channels per pixel of the buffer, the tensor's first channel, its logical channels
  int px_mul;                     // pixels per LR pixel
  uint32_t drop_layer;            // dropout stream (0: no dropout); keep-mask element px * drop_stride + drop_col0 + channel
  int drop_stride, drop_col0;
};

struct TcLaunch {
  int layer_index = -1;          // index into dcscn_handle::tcl (forward) or ::bwd (dgrad twins): the layer whose CURRENT
  bool layer_bwd = false;        // power-of-two weight scale the epilogue has to undo (it changes when a layer is re-packed)
  bool layer_fold = false;       // the layer is dcscn_handle::fold
  const ActView* act[kMaxSegments] = {};  // activated layers: the tensor behind each epilogue segment (in Plan::act), else null
  CUtensorMap tm_hi, tm_lo;
  ConvTCParams p;
  ConvRefParams ref;
  int grid = 0;
  int a_slots = 0, w_slots = 0;  // activation / weight ring depths of conv_tc_kernel
  size_t smem = 0;
};

struct Plan {
  int n = 0, h = 0, w = 0;
  std::vector<ActView> act;      // per entry of dcscn_handle::layers: the activated layers' outputs (act_view)
  ConvFirstParams first;
  std::vector<TcLaunch> tc;      // in execution order
  std::vector<DwParams> dw;      // depthwise step in front of tc[i] (ksz 0: none; wide depthwise-separable graphs)
  int dw_count = 0;              // depthwise launches per forward
  ConvLastParams last;
  bool fused_last = false;       // Up-PS epilogue computes the per-pixel half of R-CNN1 (EPI_D2S_RDOT)
  int fused_index = -1;          // index into tc of the launch that carries the fused epilogue
  TcLaunch unfused;              // same layer with the plain depth_to_space epilogue (validation path)
  ConvGatherParams gather;
  bool ran_fused = false;
  std::vector<TcLaunch> bwd;     // dgrad launches (built lazily by the train step)
  bool bwd_built = false;
  // CUDA graph of CNN1 + the tensor-core layers (everything but the last kernel, the only one that reads x2 / writes y):
  // instantiated after the plan ran eagerly once, replayed while the input pointer and the option epoch stay the same
  cudaGraphExec_t gexec = nullptr;
  const float* g_x = nullptr;
  uint64_t g_epoch = 0;
  bool g_fused = false;
  int g_launches = 0;
  int eager_runs = 0;
  const float* last_x = nullptr; // input of the previous forward on this plan: a graph is only built for a pointer seen twice in a row
  ~Plan() { if (gexec) cudaGraphExecDestroy(gexec); }
};

struct TrainState;                    // train_engine.inc

struct dcscn_handle {
  dcscn_config cfg;
  int sm_count = 132;
  std::vector<int> filters;          // feature-extraction filter schedule
  std::vector<LayerDef> layers;      // graph-construction order (self.Weights order)
  std::vector<ParamDef> params;
  std::map<std::string, int> param_index;
  bool params_dirty = true;

  // layout
  std::vector<int> feat_off, feat_w;
  int feat_pitch = 0;
  int a1_w = 0, b1_w = 0, nin_pitch = 0;
  int ps_out = 0;                    // channels after the last depth_to_space
  int mid_pitch = 0;                 // x4: channels after the first depth_to_space (padded)

  // packed layers
  std::vector<TcLayer> tcl;          // CNN2..CNNL, A1+B1, B2, Up-PS [, Up-PS2]
  std::vector<TcLayer> bwd;          // data-gradient twins (transposed, flipped filters), see build_bwd_layers
  TcLayer fold;                      // the last depth_to_space layer folded with R-CNN1 (build_fold; cout == 0: none)
  bool train_enabled = false;
  DeviceArray<float> ens_x, ens_x2, ens_y;   // self-ensemble: transformed copies / per-flip outputs
  DeviceArray<float> ensio_x, ensio_x2;      // host-call staging of the ensemble entry point
  DeviceArray<double> ensio_y;
  int l1_loss = 0;                   // --use_l1_loss: image_loss = mean |y_ - y| (DCSCN.py:342-344)
  int wgrad_impl = 0;                // 0 = wgmma (wgrad_tc.cuh), 1 = CUDA cores (validation)
  bool shadow_mode = false;          // P() returns index-coded shadows (build_refresh_maps)
  bool refresh_ready = false;        // device-side weight refresh maps are valid for the current packing
  std::vector<struct GatherJob> gather_jobs;
  std::unique_ptr<TrainState> train;
  DeviceArray<float> d_first_w;      // CNN1 [taps][n_pad]
  DeviceArray<float> d_first_bias;
  DeviceArray<float> d_first_alpha;
  DeviceArray<float> d_last_w;       // R-CNN1 [taps][C]

  // workspace (grow-only)
  size_t cap_px = 0;                 // LR pixels the buffers can hold
  Planes feat, b1, nin, mid;         // the activation buffers (act_view)
  Planes u;                          // wide depthwise-separable graphs: a layer's depthwise output, read by its pointwise
  DeviceArray<float> hr;
  DeviceArray<float> vbuf;           // tap-planar partial products of the fused R-CNN1 [9][N][sH][sW]
  DeviceArray<float> io_x, io_x2, io_y;  // staging for forward_host
  // training patch store (dcscn_patch_store_set): uint8 patches resident in HBM + the mini-batch's index list
  DeviceArray<uint8_t> ps_lr, ps_bic, ps_true;
  int64_t ps_count = 0;
  int ps_h = 0, ps_w = 0;
  DeviceArray<int> ps_idx;
  // random-crop image store (dcscn_image_store_set): the decoded uint8 images and their table (a host copy checks crops),
  // the mini-batch's crop jobs and the resampler staging of the mode-'F' (float) and mode-'L' (uint8) groups
  DeviceArray<uint8_t> is_pixels;
  DeviceArray<ImageEntry> is_table;
  std::vector<ImageEntry> is_host;
  DeviceArray<CropJob> crop_jobs;
  DeviceArray<float> crop_f;
  DeviceArray<uint8_t> crop_u8;
  // evaluation (dcscn_eval_store_set / dcscn_evaluate_image): the decoded test images and their table, the upload of a
  // host image, the per-image planes (fp32 / uint8 / float64), the SSE accumulators; all separate from the training stores
  DeviceArray<uint8_t> ev_pixels;
  std::vector<ImageEntry> ev_host;
  DeviceArray<uint8_t> ev_upload, ev_u8;
  DeviceArray<float> ev_f;
  DeviceArray<double> ev_y64, ev_map;
  DeviceArray<unsigned long long> ev_acc;
  std::vector<Event> eval_ev;        // timing events of the last evaluation (option "timing") and the names of its steps
  int eval_marks = 0;
  std::string eval_names;
  bool eval_timed = false;           // the last call that recorded timings was dcscn_evaluate_image
  // Pillow-bicubic resampling tables per (input size, output size) and the float32 intermediate of the two passes
  struct PilTable { int in = 0, out = 0, ksize = 0; DeviceArray<double> k; DeviceArray<int> bounds; };
  std::vector<PilTable> pil_tables;
  DeviceArray<float> pil_tmp;
  Stream copy_stream;                  // forward_host: x2 (only read by the last kernel) rides in beside the conv stack
  Event x2_ready;
  bool wait_x2 = false;                // the next forward's last kernel waits for x2_ready
  // tiled inference (option "workspace_mb"): staging buffers of one batch of windows, grow-only
  int64_t workspace_mb = 0;          // 0 = whole-image forwards only
  DeviceArray<float> tile_x, tile_x2, tile_y;
  bool tiling = false;               // a tiled forward is issuing its batches (forward_impl keeps the timing events)
  bool tile_vec4 = false;            // while tiling: the four-pixel R-CNN1 kernel the whole-image forward would pick
  bool tiled_last = false;           // the last forward ran tiled: the activation buffers hold its last batch
  int tiled_batches = 0;             // batches of the last tiled forward (timing names)

  // Depthwise-separable graphs run one of two ways, chosen from the graph's shape alone (ds_tile_fits):
  //   * ds_wide = false: every layer on the fp32 CUDA-core kernels of conv_ds_tile.cuh, in the ds_* buffers below;
  //   * ds_wide = true: the tensor-core graph's buffers, plans and kernels, each k x k separable layer as
  //     depthwise_planes_kernel followed by a 1x1 conv_tc_kernel layer (see construct_tc_layers).
  bool ds_wide = false;
  // depthwise-separable graphs on the CUDA-core kernels: fp32 buffers + per-layer device filters
  struct DsDev { DeviceArray<float> dw, pw, bias, alpha; };
  std::vector<DsDev> ds;             // same order as `layers`
  DsDev ds_ab;                       // fused A1 | B1 1x1 layer of the tile kernels: [concat positions][A1 cols | B1 cols], scales folded
  DeviceArray<float> ds_feat, ds_b1, ds_nin, ds_mid, ds_hr;
  int ds_total = 0;                  // channels of the concat buffer (4-aligned slots at ds_off, see build_graph)
  int ds_n = 0, ds_h = 0, ds_w = 0;  // geometry of the last DS forward
  std::vector<int> ds_off;

  std::vector<std::unique_ptr<Plan>> plans;
  Plan* last_plan = nullptr;
  int use_graph = 1;                 // option "graph": replay the per-(n,h,w) launch sequence of a forward as one CUDA graph
  uint64_t graph_epoch = 1;          // bumped by everything a captured launch bakes in (options, weight re-packs)
  Stream cap_stream;                 // capture happens on a private stream (the caller's may be the legacy default stream)
  int64_t graph_replays = 0;

  int conv_impl = 0;
  int seg_chunks = 0;                // pipeline stages per fp32-promotion segment; 0 = automatic
  int act_grad_impl = 0;             // 0: 16-byte activation-gradient kernel, 1: channel-pair kernel (cross-check)
  int grad_capture = 0;              // 1: the train step copies its gradient tensors out (dcscn_get_train_tensor)
  int timing = 0;
  int fuse_last = 1;                 // fold the per-pixel half of R-CNN1 into the last Up-PS epilogue
  std::vector<Event> ev;             // timing events (launch boundaries of the last forward)
  int ev_used = 0;
  int64_t launches = 0;
  PFN_cuTensorMapEncodeTiled_v12000 encode = nullptr;
};

static int planes(const dcscn_handle* h) { return h->cfg.precision == DCSCN_PRECISION_F16X1 ? 1 : 2; }

// A depthwise-separable graph whose layers all run on the fp32 CUDA-core kernels (forward_ds_tile).
static bool uses_ds_tile(const dcscn_handle* h) { return h->cfg.depthwise_separable && !h->ds_wide; }

// --pixel_shuffler=false: the upsampler is Up-TCNN, one stride-s conv2d_transpose (tf_graph.py build_transposed_conv),
// computed as a 3x3 LR convolution into s*s*C columns (tconv_filter) followed by depth_to_space(s).
static bool tconv(const dcscn_handle* h) { return h->cfg.transposed_upsampler != 0; }
// Whether the upsampler is two x2 pixel-shuffler stages (Up-PS at LR, Up-PS2 at 2x): x4 with the pixel shuffler.
static bool two_stage_up(const dcscn_handle* h) { return h->cfg.scale == 4 && !tconv(h); }
// The scope of the layer that reads Concat2 = [B2 | A1].
static std::string up_scope(const dcscn_handle* h) { return tconv(h) ? "Up-TCNN" : "Up-PS/Up-PS_CNN"; }
static int tconv_ksize(int s) { return 2 * s - s % 2; }   // util.get_upscale_filter_size

// Filter-count schedule of the feature-extraction stack (DCSCN.py:240-244).
static std::vector<int> feature_filters(const dcscn_config& c) {
  std::vector<int> out;
  const int minf = std::min(c.filters, c.min_filters);  // DCSCN.py:37
  int n = c.filters;
  for (int i = 0; i < c.layers; ++i) {
    if (minf != 0 && i > 0) {
      double x1 = (double)i / (double)(c.layers - 1);
      double y1 = std::pow(x1, 1.0 / (double)c.filters_decay_gamma);
      n = (int)((c.filters - minf) * (1 - y1) + minf);
    }
    out.push_back(n);
  }
  return out;
}

static void add_param(dcscn_handle* h, const std::string& name, std::vector<int64_t> shape, float fill) {
  ParamDef p;
  p.name = name;
  p.shape = shape;
  p.host.assign((size_t)p.numel(), fill);
  h->param_index[name] = (int)h->params.size();
  h->params.push_back(std::move(p));
}

// Name of an activated layer's PReLU slope variable (tf_graph.py:89-91); only --activator=prelu creates it.
static std::string prelu_name(const std::string& scope) {
  const size_t k = scope.find_last_of('/');
  return scope + "/prelu/" + (k == std::string::npos ? scope : scope.substr(k + 1)) + "_prelu";
}
static bool has_slope_variable(const dcscn_handle* h, const LayerDef& l) {
  return l.act && h->cfg.activator == DCSCN_ACTIVATOR_PRELU;
}
static const std::vector<float>& P(const dcscn_handle* h, const std::string& name);

// The slope below zero that the forward kernels apply to an activated layer's channels: the PReLU variable, relu's 0 or
// leaky_relu's 0.1f (whose product 0.1f * z is the value tf.maximum(z, 0.1 * z) returns).  sigmoid, tanh and selu use
// no slope (EpiParams::act); their entries keep the linear 1.
static void layer_slopes(const dcscn_handle* h, const LayerDef& l, float* dst) {
  const int a = h->cfg.activator;
  for (int co = 0; co < l.cout; ++co)
    dst[co] = a == DCSCN_ACTIVATOR_RELU ? 0.f : a == DCSCN_ACTIVATOR_LEAKY_RELU ? 0.1f : 1.f;
  if (a == DCSCN_ACTIVATOR_PRELU) {
    const std::vector<float>& A = P(h, prelu_name(l.scope));
    std::copy(A.begin(), A.begin() + l.cout, dst);
  }
}

// Shared memory launch_ds_tile gives ds_tile_kernel for a layer (the template's column count sizes the carve-up).
static size_t ds_tile_launch_smem(int ksz, int cin, int cout) {
  const int cols = cout < 32 ? ((cout + 3) & ~3) : 32;
  const int tcols = cols <= 4 ? 4 : cols <= 8 ? 8 : cols <= 16 ? 16 : cols <= 24 ? 24 : 32;
  const size_t in_px = ksz == 3 ? (size_t)(kDtT + 2) * kDtS : (size_t)kDtThreads;
  const size_t cache = ds_tile_caches_depthwise(ksz, cin, cout) ? (size_t)kDtThreads * kDtCP : 0;   // private depthwise rows
  return (in_px * kDtCP + (size_t)cin * tcols + (size_t)ksz * ksz * cin + cache) * sizeof(float);
}
static bool ds_tile_accepts(int ksz, int cin, int cout) {
  return (ksz == 1 || ksz == 3) && !(cout > 32 && cin > kDtCC) && ds_tile_launch_smem(ksz, cin, cout) <= 200 * 1024;
}

// Whether forward_ds_tile runs every layer of the depthwise-separable graph: the one statement of the choice between
// the fp32 CUDA-core kernels and the wide path (dcscn_handle::ds_wide).
static bool ds_tile_fits(const dcscn_handle* h) {
  const dcscn_config& c = h->cfg;
  if (tconv(h)) return false;   // Up-TCNN is a dense conv2d_transpose even here: it runs on the tensor cores
  int T = 0;   // concat channels with 4-aligned slots (finalize_params_ds)
  for (int f : h->filters) T += (f + 3) & ~3;
  const int cps = c.nin_filters + c.nin_filters2;
  if (cps > 32 || !ds_tile_accepts(1, T, cps)) return false;   // the fused A1 | B1 launch
  for (const LayerDef& l : h->layers) {
    if (l.scope == "A1" || l.scope == "B1") continue;
    if (l.cin == 1 && l.cout == 1) {                              // R-CNN1 on ds_single(4)_kernel
      if (l.k != 1 && l.k != 3) return false;
    } else if (!ds_tile_accepts(l.k, l.cin, l.cout)) {
      return false;
    }
  }
  return true;
}

static int build_graph(dcscn_handle* h) {
  const dcscn_config& c = h->cfg;
  if (c.activator < DCSCN_ACTIVATOR_PRELU || c.activator > DCSCN_ACTIVATOR_SELU) return fail("activator %d is not one of DCSCN_ACTIVATOR_*", c.activator);
  if (c.optimizer < DCSCN_OPTIMIZER_ADAM || c.optimizer > DCSCN_OPTIMIZER_RMSPROP) return fail("optimizer %d is not one of DCSCN_OPTIMIZER_*", c.optimizer);
  if (!std::isfinite(c.momentum)) return fail("momentum must be finite");
  if (!c.use_nin) return fail("use_nin=false is not supported (no shipped checkpoint uses it)");
  if (c.channels != 1) return fail("channels must be 1 (helper/args.py: 'Now it should be 1')");
  if (std::max(c.reconstruct_layers, 1) != 1) return fail("reconstruct_layers > 1 is not supported");
  // x4 is two x2 stages; every other factor is one Up-PS / Up-TCNN into s*s columns (DCSCN.py:293-311).  x8 is the
  // largest factor the tests verify.
  if (c.scale < 2 || c.scale > 8) return fail("scale must be in 2..8 (got %d)", c.scale);
  if (c.cnn_size != 3 && c.cnn_size != 1 && c.cnn_size != 5) return fail("cnn_size %d is not supported", c.cnn_size);
  if (c.layers < 2) return fail("layers must be >= 2");

  h->filters = feature_filters(c);
  int cin = c.channels, total = 0;
  for (int i = 0; i < c.layers; ++i) {
    h->layers.push_back({"CNN" + std::to_string(i + 1), c.cnn_size, cin, h->filters[i], true, true});
    cin = h->filters[i];
    total += cin;
  }
  h->layers.push_back({"A1", 1, total, c.nin_filters, true, true});
  h->layers.push_back({"B1", 1, total, c.nin_filters2, true, true});
  h->layers.push_back({"B2", 3, c.nin_filters2, c.nin_filters2, true, true});
  cin = c.nin_filters + c.nin_filters2;
  h->ps_out = c.pixel_shuffler_filters != 0 && !c.transposed_upsampler ? c.pixel_shuffler_filters : cin;
  if (c.transposed_upsampler) {  // DCSCN.py:310-311: C -> C at s x the resolution, no bias, no activation
    h->layers.push_back({"Up-TCNN", 3, cin, c.scale * c.scale * cin, false, false});
  } else if (c.scale == 4) {  // DCSCN.py:298-304
    h->layers.push_back({"Up-PS/Up-PS_CNN", c.cnn_size, cin, 4 * cin, true, false});
    h->layers.push_back({"Up-PS2/Up-PS2_CNN", c.cnn_size, cin, 4 * h->ps_out, true, false});
  } else {
    h->layers.push_back({"Up-PS/Up-PS_CNN", c.cnn_size, cin, c.scale * c.scale * h->ps_out, true, false});
  }
  h->layers.push_back({"R-CNN1", c.cnn_size, h->ps_out, 1, false, false});

  for (const LayerDef& l : h->layers) {
    std::string base = l.scope.substr(l.scope.find_last_of('/') == std::string::npos ? 0 : l.scope.find_last_of('/') + 1);
    if (l.scope == "Up-TCNN") {   // util.upscale_weight: [K, K, out, in]
      const int K = tconv_ksize(c.scale);
      add_param(h, "Up-TCNN/Tconv_W", {K, K, l.cin, l.cin}, 0.f);
      continue;
    }
    add_param(h, l.scope + "/conv_W", {l.k, l.k, l.cin, l.cout}, 0.f);
    if (c.depthwise_separable) {  // tf_graph.py:157-160; conv_W stays as the (dead) variable the reference also creates
      add_param(h, l.scope + "/depthwise_W", {l.k, l.k, l.cin, 1}, 0.f);
      add_param(h, l.scope + "/pointwise_W", {1, 1, l.cin, l.cout}, 0.f);
    }
    if (l.bias) add_param(h, l.scope + "/conv_B", {l.cout}, 0.f);                 // util.bias: zeros
    if (has_slope_variable(h, l)) add_param(h, prelu_name(l.scope), {l.cout}, 0.1f);  // tf_graph.py:91
  }

  // channel layout of the shared feature ("concat") buffer: 16-aligned slot per CNN layer
  int off = 0;
  for (int f : h->filters) {
    h->feat_off.push_back(off);
    h->feat_w.push_back(pad16(f));
    off += pad16(f);
  }
  h->feat_pitch = off;
  h->b1_w = pad16(c.nin_filters2);
  h->a1_w = pad16(c.nin_filters);
  h->nin_pitch = h->b1_w + h->a1_w;  // [B2 | A1]  (Concat2 order, DCSCN.py:281)
  h->mid_pitch = pad16(cin);
  // the fp32 concat buffer of forward_ds_tile: every CNNi slot starts on a multiple of 4 channels (16-byte loads /
  // stores); the pad channels are never written (the buffer is zero-filled once) and meet zero rows in the A1 / B1 filters
  off = 0;
  for (int f : h->filters) {
    h->ds_off.push_back(off);
    off += (f + 3) & ~3;
  }
  h->ds_total = off;
  h->ds_wide = c.depthwise_separable && !ds_tile_fits(h);
  return 0;
}

// Resolves an activation name of the C ABI (CNNi, A1, B1, B2, Up-PS, Up-PS2 at x4, Up-TCNN; the pixel-shuffler output
// is named after the layer that writes it) against the buffers the graph runs on.  False: no such tensor.
// The dropout streams are stated here and nowhere else.  The tensor-core layout numbers them CNNi = i, A1 = B1 = L+1
// (one keep mask over the fused A1+B1 GEMM's a1_w + b1_w columns, B1 from column a1_w), B2 = L+2; forward_ds_tile's
// dense [px][C] layout numbers A1 = L+1, B2 = L+2, B1 = L+3.
static bool act_view(const dcscn_handle* h, const std::string& name, ActView* v) {
  const dcscn_config& c = h->cfg;
  const int L = c.layers, na = c.nin_filters, nb = c.nin_filters2, cps = na + nb;
  const bool ds = uses_ds_tile(h);
  if (name.rfind("CNN", 0) == 0) {
    const int i = atoi(name.c_str() + 3) - 1;
    if (i < 0 || i >= L) return false;
    *v = ds ? ActView{BUF_FEAT, {}, nullptr, h->ds_total, h->ds_off[i], h->filters[i], 1, (uint32_t)(i + 1), h->filters[i], 0}
            : ActView{BUF_FEAT, {}, nullptr, h->feat_pitch, h->feat_off[i], h->filters[i], 1, (uint32_t)(i + 1), h->feat_w[i], 0};
  } else if (name == "A1") {
    *v = ds ? ActView{BUF_NIN, {}, nullptr, cps, nb, na, 1, (uint32_t)(L + 1), na, 0}
            : ActView{BUF_NIN, {}, nullptr, h->nin_pitch, h->b1_w, na, 1, (uint32_t)(L + 1), h->a1_w + h->b1_w, 0};
  } else if (name == "B1") {
    *v = ds ? ActView{BUF_B1, {}, nullptr, nb, 0, nb, 1, (uint32_t)(L + 3), nb, 0}
            : ActView{BUF_B1, {}, nullptr, h->b1_w, 0, nb, 1, (uint32_t)(L + 1), h->a1_w + h->b1_w, h->a1_w};
  } else if (name == "B2") {
    *v = ActView{BUF_NIN, {}, nullptr, ds ? cps : h->nin_pitch, 0, nb, 1, (uint32_t)(L + 2), ds ? nb : h->b1_w, 0};
  } else if (name == "Up-PS" && two_stage_up(h)) {
    *v = ActView{BUF_MID, {}, nullptr, ds ? cps : h->mid_pitch, 0, cps, 4, 0, 0, 0};
  } else if (name == (tconv(h) ? "Up-TCNN" : two_stage_up(h) ? "Up-PS2" : "Up-PS")) {
    *v = ActView{BUF_HR, {}, nullptr, h->ps_out, 0, h->ps_out, c.scale * c.scale, 0, 0, 0};
  } else {
    return false;
  }
  auto at = [&](auto* base) { return base ? base + v->off : nullptr; };
  if (ds) {
    const DeviceArray<float>* bufs[] = {&h->ds_feat, &h->ds_nin, &h->ds_b1, &h->ds_mid, &h->ds_hr};
    v->f32 = at(bufs[v->buf]->get());
  } else if (v->buf == BUF_HR) {
    v->f32 = at(h->hr.get());
  } else {
    const Planes* bufs[] = {&h->feat, &h->nin, &h->b1, &h->mid};
    v->planes = bufs[v->buf]->at(v->off);
  }
  return true;
}

static const LayerDef* find_layer(const dcscn_handle* h, const std::string& scope) {
  for (const LayerDef& l : h->layers)
    if (l.scope == scope) return &l;
  return nullptr;
}
static const std::vector<float>& P(const dcscn_handle* h, const std::string& name) {
  const ParamDef& p = h->params[h->param_index.at(name)];
  return h->shadow_mode ? p.shadow : p.host;
}

// ------------------------------------------------------------------------------ weight packing ----
// Whether a layer of a wide depthwise-separable graph runs as depthwise_planes_kernel + a 1x1 pointwise layer.  The
// other layers fold their depthwise filter into a dense one (layer_filter): 1x1 layers (a per-channel scale), CNN1
// (one input channel) and R-CNN1 (one output channel).
// Once a handle trains, every layer is composed instead: the dense train step differentiates the composed k x k filters.
static bool ds_split(const dcscn_handle* h, const LayerDef& l) {
  return h->ds_wide && !h->train_enabled && l.k > 1 && l.cin > 1 && l.cout > 1 && l.scope != "Up-TCNN";
}

// Index in Up-TCNN/Tconv_W W[K][K][C][C] ([h, w, out, in]) behind every entry of its 3x3 LR filter
// F[3][3][C][s*s*C] (HWIO), or -1 for a structural zero.  With SAME padding, pad_top = (K - s) / 2 and
//   out[s*m + p] = sum_d in[m + d] * W[p + pad_top - s*d]   per axis,
// and for every s >= 2 every used offset d lies in {-1, 0, 1}: F[dy+1][dx+1][ci][(py*s + px)*C + co] =
// W[py + pad_top - s*dy][px + pad_top - s*dx][co][ci].  (phase, offset) -> tap is a bijection onto [0, K), so each
// W entry appears in F exactly once and the map inverts without sums (tconv gradient, train_engine.inc).
static std::vector<int> tconv_filter_map(int s, int C) {
  const int K = tconv_ksize(s), pad = (K - s) / 2, cols = s * s * C;
  std::vector<int> m((size_t)9 * C * cols, -1);
  for (int dy = -1; dy <= 1; ++dy)
    for (int dx = -1; dx <= 1; ++dx)
      for (int py = 0; py < s; ++py)
        for (int px = 0; px < s; ++px) {
          const int ky = py + pad - s * dy, kx = px + pad - s * dx;
          if (ky < 0 || ky >= K || kx < 0 || kx >= K) continue;
          const int tap = (dy + 1) * 3 + (dx + 1);
          for (int ci = 0; ci < C; ++ci)
            for (int co = 0; co < C; ++co)
              m[((size_t)tap * C + ci) * cols + (py * s + px) * C + co] = ((ky * K + kx) * C + co) * C + ci;
        }
  return m;
}

// The HWIO filter the packed form of layer `l` computes with: conv_W; Up-TCNN's 3x3 form of Tconv_W (tconv_filter_map,
// a pure gather); on the wide depthwise-separable path the pointwise filter alone for a split layer, else
// W[t][ci][co] = dw[t][ci] pw[ci][co] in `tmp` (exact in real arithmetic: one side of the product has a single channel
// or a single tap).
static const std::vector<float>& layer_filter(const dcscn_handle* h, const LayerDef& l, std::vector<float>& tmp) {
  if (l.scope == "Up-TCNN") {   // shadow mode too: structural zeros stay 0, i.e. "no source" in the refresh maps
    const std::vector<float>& W = P(h, "Up-TCNN/Tconv_W");
    const std::vector<int> m = tconv_filter_map(h->cfg.scale, l.cin);
    tmp.assign(m.size(), 0.f);
    for (size_t i = 0; i < m.size(); ++i)
      if (m[i] >= 0) tmp[i] = W[m[i]];
    return tmp;
  }
  // shadow mode (build_refresh_maps): a composed filter lives in the layer's conv_W slot of TrainState::d_wc
  if (!h->ds_wide || h->shadow_mode) return P(h, l.scope + "/conv_W");
  const std::vector<float>& pw = P(h, l.scope + "/pointwise_W");
  if (ds_split(h, l)) return pw;
  const std::vector<float>& dw = P(h, l.scope + "/depthwise_W");
  const int taps = l.k * l.k;
  tmp.assign((size_t)taps * l.cin * l.cout, 0.f);
  for (int tp = 0; tp < taps; ++tp)
    for (int ci = 0; ci < l.cin; ++ci)
      for (int co = 0; co < l.cout; ++co)
        tmp[((size_t)tp * l.cin + ci) * l.cout + co] = dw[(size_t)tp * l.cin + ci] * pw[(size_t)ci * l.cout + co];
  return tmp;
}

// Filter size of the tensor-core layer that computes `l`.
static int tc_ksz(const dcscn_handle* h, const LayerDef& l) { return ds_split(h, l) ? 1 : l.k; }

// Appends the TF layer `scope` as columns [col0, col0+cout) of a fused tensor-core layer (t.in_map set).  A split layer
// of a wide depthwise-separable graph also gets its depthwise filter, by source position.
static void fuse_columns(const dcscn_handle* h, TcLayer& t, const std::string& scope, int col0, int n_total_pad) {
  const LayerDef* l = find_layer(h, scope);
  std::vector<float> tmp;
  const std::vector<float>& W = layer_filter(h, *l, tmp);
  const int taps = t.ksz * t.ksz;
  if (ds_split(h, *l)) {
    const std::vector<float>& D = P(h, scope + "/depthwise_W");
    const int dtaps = l->k * l->k;
    t.dw_ksz = l->k;
    t.dw_host.assign((size_t)dtaps * t.cin_pad, 0.f);
    for (int tp = 0; tp < dtaps; ++tp)
      for (int ci = 0; ci < l->cin; ++ci) t.dw_host[(size_t)tp * t.cin_pad + t.in_map[ci]] = D[(size_t)tp * l->cin + ci];
  }
  for (int tp = 0; tp < taps; ++tp)
    for (int ci = 0; ci < l->cin; ++ci)
      for (int co = 0; co < l->cout; ++co)
        t.w_host[((size_t)tp * t.cin + ci) * t.cout + col0 + co] = W[((size_t)tp * l->cin + ci) * l->cout + co];
  (void)n_total_pad;
  if (l->bias) {
    const std::vector<float>& B = P(h, scope + "/conv_B");
    for (int co = 0; co < l->cout; ++co) t.bias_host[col0 + co] = B[co];
  }
  if (l->act) layer_slopes(h, *l, t.alpha_host.data() + col0);
}

static void choose_tiling(int n_total_pad16, int* n_tiles, int* n_pad, int cap = kMaxTileN) {
  int nt = (n_total_pad16 + cap - 1) / cap;
  int np = pad16((n_total_pad16 + nt - 1) / nt);
  *n_tiles = nt;
  *n_pad = np;
}

// Values (unscaled fp32) of the operand image of a layer, one per hi-plane element, in image order:
// [n_tile][tap][chunk][n_pad rows x 64 halves], the shared-memory image of a K-major SWIZZLE_128B wgmma operand tile
// (16-byte chunk j of row r at chunk j ^ (r & 7)).
static void tile_image(const TcLayer& t, std::vector<float>& img) {
  const int taps = t.ksz * t.ksz, chunks = (t.cin_pad + kTcKC - 1) / kTcKC, n_total = t.n_tiles * t.n_pad;
  std::vector<float> wq((size_t)taps * t.cin_pad * n_total, 0.f);   // dense, channel-position-indexed  Wq[tap][q][n]
  for (int tp = 0; tp < taps; ++tp)
    for (int ci = 0; ci < t.cin; ++ci) {
      const int q = t.in_map[ci];
      for (int co = 0; co < t.cout; ++co)
        wq[((size_t)tp * t.cin_pad + q) * n_total + co] = t.w_host[((size_t)tp * t.cin + ci) * t.cout + co];
    }
  const size_t tile_elems = (size_t)t.n_pad * kTcKC;
  img.assign((size_t)t.n_tiles * taps * chunks * tile_elems, 0.f);
  for (int nt = 0; nt < t.n_tiles; ++nt)
    for (int tp = 0; tp < taps; ++tp)
      for (int ch = 0; ch < chunks; ++ch) {
        float* base = img.data() + (((size_t)nt * taps + tp) * chunks + ch) * tile_elems;
        for (int r = 0; r < t.n_pad; ++r) {
          const int n = nt * t.n_pad + r;
          const int sw = r & 7;
          for (int kk = 0; kk < kTcKC; ++kk) {
            const int q = ch * kTcKC + kk;
            if (q < t.cin_pad) base[(size_t)r * kTcKC + (size_t)((kk / 8) ^ sw) * 8 + kk % 8] = wq[((size_t)tp * t.cin_pad + q) * n_total + n];
          }
        }
      }
}

// Sets *moved when a device array of the layer was reallocated.
static int pack_tc_layer(dcscn_handle* h, TcLayer& t, bool* moved) {
  const int NPL = planes(h);
  float maxw = 0.f;
  for (float v : t.w_host) maxw = std::max(maxw, std::fabs(v));
  t.wscale = 1.f;
  if (maxw > 0.f) t.wscale = std::ldexp(1.0f, (int)std::floor(std::log2(16384.0 / (double)maxw)));

  const size_t tile_elems = (size_t)t.n_pad * kTcKC;
  std::vector<float> img;
  tile_image(t, img);
  std::vector<__half> pack(img.size() * NPL);
  for (size_t i = 0; i < img.size(); ++i) {
    const size_t blk = i / tile_elems, pos = i - blk * tile_elems;
    const float v = img[i] * t.wscale;
    const __half hi = __float2half_rn(v);
    pack[blk * NPL * tile_elems + pos] = hi;
    if (NPL == 2) pack[blk * NPL * tile_elems + tile_elems + pos] = __float2half_rn(v - __half2float(hi));
  }
  if (t.d_wpack.upload(pack, moved) || t.d_bias.upload(t.bias_host, moved) || t.d_alpha.upload(t.alpha_host, moved) ||
      t.d_wref.upload(t.w_host, moved) || t.d_in_map.upload(t.in_map, moved) || t.d_dw.upload(t.dw_host, moved))
    return 1;
  t.packed_planes = NPL;
  return 0;
}

// Whether a column tile of n_pad columns lets the fused R-CNN1 epilogue (EPI_D2S_RDOT, see get_plan) run for sub-pixels
// of `cout` channels: tiles start on sub-pixel boundaries, and each epilogue thread's n_pad / kColSplit columns are whole
// sub-pixels or an equal share of one.
static bool rdot_fusable(int n_pad, int cout) {
  if (cout <= 0 || cout % 16 || cout > kMaxTileN || n_pad % cout || (n_pad >> 4) % kColSplit) return false;
  const int per16 = (n_pad >> 4) / kColSplit * 16;
  return per16 % cout == 0 || cout % per16 == 0;
}

// `fuse_unit` > 0: the layer is the last depth_to_space and R-CNN1 can be fused into its epilogue for sub-pixels of
// fuse_unit channels.  When the default tiling does not allow that, the widest tile that does is taken (fewest tiles;
// columns past cout_cols are padding that the epilogue drops).
static TcLayer make_tc(const std::string& name, int ksz, int cin, int cout_cols, int cin_pad, int fuse_unit = 0) {
  TcLayer t;
  t.name = name;
  t.ksz = ksz;
  t.cin = cin;
  t.cout = cout_cols;
  t.cin_pad = cin_pad;
  choose_tiling(pad16(cout_cols), &t.n_tiles, &t.n_pad);
  if (fuse_unit > 0 && cout_cols % fuse_unit == 0 && !rdot_fusable(t.n_pad, fuse_unit)) {
    for (int np = kMaxTileN / fuse_unit * fuse_unit; np >= fuse_unit; np -= fuse_unit) {
      if (rdot_fusable(np, fuse_unit)) {
        t.n_pad = np;
        t.n_tiles = (cout_cols + np - 1) / np;
        break;
      }
    }
  }
  t.n_valid = cout_cols;
  t.w_host.assign((size_t)ksz * ksz * cin * cout_cols, 0.f);
  t.bias_host.assign((size_t)t.n_tiles * t.n_pad, 0.f);
  t.alpha_host.assign((size_t)t.n_tiles * t.n_pad, 1.f);
  return t;
}

// (Re)builds every device-side weight image from the host fp32 parameters.
static int finalize_params_ds(dcscn_handle* h) {
  h->ds_ab = dcscn_handle::DsDev();
  h->ds.clear();
  h->ds.resize(h->layers.size());
  const int T = h->ds_total, L = h->cfg.layers;
  std::vector<float> ab_pw, ab_bias, ab_alpha;
  const int na = h->cfg.nin_filters, nb = h->cfg.nin_filters2;
  ab_pw.assign((size_t)T * (na + nb), 0.f);
  ab_bias.assign(na + nb, 0.f);
  ab_alpha.assign(na + nb, 1.f);
  // slope vectors for prelu / relu / leaky_relu; sigmoid, tanh and selu have none (ds_activate)
  const bool slopes = h->cfg.activator <= DCSCN_ACTIVATOR_LEAKY_RELU;
  for (size_t i = 0; i < h->layers.size(); ++i) {
    const LayerDef& l = h->layers[i];
    const std::vector<float>& dwv = P(h, l.scope + "/depthwise_W");   // [k,k,cin,1] == [taps][cin]
    const std::vector<float>& pwv = P(h, l.scope + "/pointwise_W");   // [1,1,cin,cout] == [cin][cout]
    if (l.scope == "A1" || l.scope == "B1") {
      // both run as the one fused layer ds_ab over the whole concat buffer: their rows go to the 4-aligned slot
      // positions, with the per-channel depthwise scale folded in
      const int col0 = l.scope == "A1" ? 0 : na;
      int ci = 0;
      for (int li = 0; li < L; ++li)
        for (int k = 0; k < h->filters[li]; ++k, ++ci) {
          const int pos = h->ds_off[li] + k;
          for (int co = 0; co < l.cout; ++co)
            if (l.k == 1) ab_pw[(size_t)pos * (na + nb) + col0 + co] = dwv[ci] * pwv[(size_t)ci * l.cout + co];
        }
      const auto& B = P(h, l.scope + "/conv_B");
      for (int co = 0; co < l.cout; ++co) ab_bias[col0 + co] = B[co];
      layer_slopes(h, l, ab_alpha.data() + col0);
      continue;
    }
    if (h->ds[i].dw.upload(dwv) || h->ds[i].pw.upload(pwv)) return 1;
    if (l.bias && h->ds[i].bias.upload(P(h, l.scope + "/conv_B"))) return 1;
    if (l.act) {
      std::vector<float> a(l.cout);
      layer_slopes(h, l, a.data());
      if (slopes && h->ds[i].alpha.upload(a)) return 1;
    }
  }
  if (h->ds_ab.pw.upload(ab_pw) || h->ds_ab.bias.upload(ab_bias)) return 1;
  if (slopes && h->ds_ab.alpha.upload(ab_alpha)) return 1;
  h->params_dirty = false;
  return 0;
}

static int build_bwd_layers(dcscn_handle* h);
static int sync_host_params(dcscn_handle* h);   // train_engine.inc: device master copy -> host, when newer

// CNN1's device vectors (CUDA cores): filter [taps][n_pad], bias, slope (layer_slopes), padded to the slot width.
static void first_layer_vectors(const dcscn_handle* h, std::vector<float>& w, std::vector<float>& b, std::vector<float>& a) {
  const LayerDef* l = find_layer(h, "CNN1");
  const int taps = l->k * l->k, np = h->feat_w[0];
  w.assign((size_t)taps * np, 0.f);
  b.assign(np, 0.f);
  a.assign(np, 1.f);
  std::vector<float> tmp;
  const std::vector<float>& W = layer_filter(h, *l, tmp);
  for (int tp = 0; tp < taps; ++tp)
    for (int co = 0; co < l->cout; ++co) w[(size_t)tp * np + co] = W[(size_t)tp * l->cout + co];
  const auto& B = P(h, "CNN1/conv_B");
  for (int co = 0; co < l->cout; ++co) b[co] = B[co];
  layer_slopes(h, *l, a.data());
}

// Fills h->tcl (forward tensor-core layers) and, when training, h->bwd (their dgrad twins) from the parameters P().
static int construct_tc_layers(dcscn_handle* h) {
  const dcscn_config& c = h->cfg;
  const int L = c.layers;
  // CNN2..CNNL
  for (int i = 1; i < L; ++i) {
    const std::string scope = "CNN" + std::to_string(i + 1);
    const LayerDef* l = find_layer(h, scope);
    TcLayer t = make_tc(scope, tc_ksz(h, *l), l->cin, l->cout, h->feat_w[i - 1]);
    for (int ci = 0; ci < l->cin; ++ci) t.in_map.push_back(ci);
    fuse_columns(h, t, scope, 0, 0);
    h->tcl.push_back(std::move(t));
  }
  // A1 || B1 fused 1x1 over the whole concat buffer: columns [A1 (padded to 16) | B1]
  {
    const LayerDef* a1 = find_layer(h, "A1");
    const LayerDef* b1 = find_layer(h, "B1");
    TcLayer t = make_tc("A1+B1", 1, a1->cin, h->a1_w + b1->cout, h->feat_pitch);
    for (int li = 0; li < L; ++li)
      for (int ci = 0; ci < h->filters[li]; ++ci) t.in_map.push_back(h->feat_off[li] + ci);
    fuse_columns(h, t, "A1", 0, 0);
    fuse_columns(h, t, "B1", h->a1_w, 0);
    h->tcl.push_back(std::move(t));
  }
  // B2
  {
    const LayerDef* l = find_layer(h, "B2");
    TcLayer t = make_tc("B2", tc_ksz(h, *l), l->cin, l->cout, h->b1_w);
    for (int ci = 0; ci < l->cin; ++ci) t.in_map.push_back(ci);
    fuse_columns(h, t, "B2", 0, 0);
    h->tcl.push_back(std::move(t));
  }
  // Up-PS (+ Up-PS2) or Up-TCNN: input = Concat2 = [B2 | A1]
  {
    const std::string scope = up_scope(h);
    const LayerDef* l = find_layer(h, scope);
    // the LAST depth_to_space layer carries the fused R-CNN1 epilogue (3x3 R-CNN1 only)
    const int fuse_unit = find_layer(h, "R-CNN1")->k == 3 ? h->ps_out : 0;
    TcLayer t = make_tc(tconv(h) ? "Up-TCNN" : "Up-PS", tc_ksz(h, *l), l->cin, l->cout, h->nin_pitch,
                        two_stage_up(h) ? 0 : fuse_unit);
    for (int ci = 0; ci < c.nin_filters2; ++ci) t.in_map.push_back(ci);
    for (int ci = 0; ci < c.nin_filters; ++ci) t.in_map.push_back(h->b1_w + ci);
    fuse_columns(h, t, scope, 0, 0);
    h->tcl.push_back(std::move(t));
    if (two_stage_up(h)) {
      const LayerDef* l2 = find_layer(h, "Up-PS2/Up-PS2_CNN");
      TcLayer t2 = make_tc("Up-PS2", tc_ksz(h, *l2), l2->cin, l2->cout, h->mid_pitch, fuse_unit);
      for (int ci = 0; ci < l2->cin; ++ci) t2.in_map.push_back(ci);
      fuse_columns(h, t2, "Up-PS2/Up-PS2_CNN", 0, 0);
      h->tcl.push_back(std::move(t2));
    }
  }
  // forward_ds_tile graphs train on the fp32 step of train_ds.inc, which needs no dgrad twins
  if (h->train_enabled && !uses_ds_tile(h) && build_bwd_layers(h)) return 1;
  return 0;
}

// Partial plane sets of the fused R-CNN1 epilogue: an epilogue thread owns n_pad / kColSplit GEMM columns; when that share
// is a fraction of one sub-pixel's `cout` channels, `cout / share` threads each write their own tap-planar partials.
static int rdot_parts(int n_pad, int cout) {
  const int nch = n_pad >> 4, per16 = ((nch + kColSplit - 1) / kColSplit) * 16;
  if (cout <= 0 || per16 % cout == 0) return 1;
  return (cout % per16 == 0) ? cout / per16 : 1;
}

// Whether get_plan fuses R-CNN1 into the last depth_to_space layer, whose column tiles are n_pad wide: a 3x3 R-CNN1 and
// epilogue threads that own whole sub-pixels or an equal share of one.
static bool last_fuses(const dcscn_handle* h, int n_pad) {
  const int cout = h->ps_out, nch = n_pad >> 4, per = (nch + kColSplit - 1) / kColSplit;
  return find_layer(h, "R-CNN1")->k == 3 && cout % 16 == 0 && cout <= 128 && nch % kColSplit == 0 &&
         ((per * 16) % cout == 0 || (rdot_parts(n_pad, cout) > 1 && n_pad % (per * 16) == 0));
}

// sum over c of a[c] w[c]: exact products of fp32 values, added in fp64 in ascending c.  fold_kernel (train.cuh) forms
// the same sum, so host and device folds round to the same fp32 value.
static double fold_dot(const float* a, const float* w, int C) {
  double s = 0.0;
  for (int c = 0; c < C; ++c) s += (double)a[c] * (double)w[c];
  return s;
}

// The shape of the fold of `up` (s^2 sub-pixels of C channels) with a 3x3 R-CNN1: s^2 * 9 columns in `up`'s column-tile
// width, same input, taps and depthwise step; no activation.
static TcLayer fold_shape(const TcLayer& up, int C) {
  TcLayer f;
  f.name = up.name;
  f.ksz = up.ksz;
  f.cin = up.cin;
  f.cin_pad = up.cin_pad;
  f.in_map = up.in_map;
  f.cout = f.n_valid = up.cout / C * 9;
  f.n_pad = up.n_pad;
  f.n_tiles = (f.cout + f.n_pad - 1) / f.n_pad;
  f.w_host.assign((size_t)f.ksz * f.ksz * f.cin * f.cout, 0.f);
  f.bias_host.assign((size_t)f.n_tiles * f.n_pad, 0.f);
  f.alpha_host.assign((size_t)f.n_tiles * f.n_pad, 1.f);
  f.dw_ksz = up.dw_ksz;
  f.dw_host = up.dw_host;
  return f;
}

// The last depth_to_space layer (Up-PS, Up-PS2 at x4, Up-TCNN) and R-CNN1 are both linear at inference, so where get_plan
// fuses them and the operands are f16x3, R-CNN1's reduction over the C channels of a sub-pixel is done once, on the
// weights:
//   W'[tap][ci][ij * 9 + t] = sum_c W[tap][ci][ij * C + c] w_r[t][c],   b'[ij * 9 + t] = sum_c b[ij * C + c] w_r[t][c]
// and the layer computes s^2 * 9 columns instead of s^2 * C.  Column (ij, t) at LR pixel (y, x) is R-CNN1 tap t's
// product at HR pixel (s y + i, s x + j), the value EPI_D2S_RDOT writes.  f16x1 keeps EPI_D2S_RDOT: that mode is each
// layer on its own fp16-rounded weights, and a folded filter rounded to fp16 would be a different quantised model.
static void build_fold(dcscn_handle* h) {
  h->fold = TcLayer();
  const TcLayer& up = h->tcl.back();
  if (planes(h) != 2 || !last_fuses(h, up.n_pad)) return;
  std::vector<float> tmp;
  const std::vector<float>& wr = layer_filter(h, *find_layer(h, "R-CNN1"), tmp);   // [9][C]
  const int C = h->ps_out, sub = up.cout / C;
  TcLayer f = fold_shape(up, C);
  const size_t rows = (size_t)up.ksz * up.ksz * up.cin;
  for (size_t r = 0; r < rows; ++r)
    for (int ij = 0; ij < sub; ++ij)
      for (int t = 0; t < 9; ++t)
        f.w_host[r * f.cout + ij * 9 + t] = (float)fold_dot(&up.w_host[r * up.cout + (size_t)ij * C], &wr[(size_t)t * C], C);
  for (int ij = 0; ij < sub; ++ij)
    for (int t = 0; t < 9; ++t) f.bias_host[ij * 9 + t] = (float)fold_dot(&up.bias_host[(size_t)ij * C], &wr[(size_t)t * C], C);
  h->fold = std::move(f);
}

// A re-built layer keeps the device allocations of its previous packing.
static void adopt_arrays(TcLayer& t, TcLayer& old) {
  t.d_wpack = std::move(old.d_wpack); t.d_bias = std::move(old.d_bias); t.d_alpha = std::move(old.d_alpha);
  t.d_wref = std::move(old.d_wref); t.d_in_map = std::move(old.d_in_map); t.d_img_map = std::move(old.d_img_map);
  t.d_dw = std::move(old.d_dw);
}

static int finalize_params(dcscn_handle* h) {
  const dcscn_config& c = h->cfg;
  if (sync_host_params(h)) return 1;
  if (uses_ds_tile(h)) return finalize_params_ds(h);
  std::vector<TcLayer> old_tcl = std::move(h->tcl);
  std::vector<TcLayer> old_bwd = std::move(h->bwd);
  TcLayer old_fold = std::move(h->fold);
  h->tcl.clear();
  h->bwd.clear();
  h->refresh_ready = false;
  bool moved = false;
  {
    std::vector<float> w, b, a;
    first_layer_vectors(h, w, b, a);
    if (h->d_first_w.upload(w, &moved) || h->d_first_bias.upload(b, &moved) || h->d_first_alpha.upload(a, &moved)) return 1;
  }
  if (construct_tc_layers(h)) return 1;
  // each layer keeps the device allocations of its previous packing; those of layers that no longer exist are freed with
  // old_tcl / old_bwd
  auto repack = [&](std::vector<TcLayer>& cur, std::vector<TcLayer>& old) {
    for (size_t i = 0; i < cur.size(); ++i) {
      TcLayer& t = cur[i];
      if (i < old.size()) adopt_arrays(t, old[i]);
      if (pack_tc_layer(h, t, &moved)) return 1;
    }
    return 0;
  };
  if (repack(h->tcl, old_tcl) || repack(h->bwd, old_bwd)) return 1;
  build_fold(h);
  if (h->fold.cout > 0) {
    adopt_arrays(h->fold, old_fold);
    if (pack_tc_layer(h, h->fold, &moved)) return 1;
  }
  // R-CNN1 (CUDA cores): [taps][C]
  {
    std::vector<float> tmp;
    if (h->d_last_w.upload(layer_filter(h, *find_layer(h, "R-CNN1"), tmp), &moved)) return 1;
  }
  if (moved) {  // some device pointer moved: cached plans embed stale pointers
    h->plans.clear();
    h->last_plan = nullptr;
  }
  h->graph_epoch++;          // captured launches bake the epilogue's 1 / weight-scale
  h->params_dirty = false;
  return 0;
}

// ----------------------------------------------------------------------------------- workspace ----
// Elements per LR pixel of every buffer ensure_workspace allocates: the one statement of their sizes, shared by the
// allocation and by the tile planner's workspace budget (valid once the parameters are finalised).
struct WorkspaceShape {
  size_t feat, b1, nin, mid;   // fp16 elements per plane (tensor-core graphs) or fp32 (forward_ds_tile)
  size_t u;                    // fp16 elements per plane: the widest depthwise output of a wide depthwise-separable graph
  size_t hr, vbuf;             // fp32
  int planes;                  // fp16 planes (tensor-core graphs)
  size_t bytes_per_px(bool ds) const {
    return ds ? 4 * (feat + b1 + nin + mid + hr) : 2 * (size_t)planes * (feat + b1 + nin + mid + u) + 4 * (hr + vbuf);
  }
};

static WorkspaceShape workspace_shape(const dcscn_handle* h) {
  const dcscn_config& c = h->cfg;
  const size_t s2 = (size_t)c.scale * c.scale;
  WorkspaceShape w;
  w.u = 0;
  if (uses_ds_tile(h)) {
    const int cps = c.nin_filters + c.nin_filters2;
    w.feat = h->ds_total;
    w.b1 = c.nin_filters2;
    w.nin = cps;
    w.mid = c.scale == 4 ? 4 * (size_t)cps : 0;
    w.hr = s2 * h->ps_out;
    w.vbuf = 0;
    w.planes = 1;
    return w;
  }
  w.feat = h->feat_pitch;
  w.b1 = h->b1_w;
  w.nin = h->nin_pitch;
  w.mid = two_stage_up(h) ? 4 * (size_t)h->mid_pitch : 0;
  w.hr = s2 * h->ps_out;
  w.vbuf = s2 * 9 * (size_t)rdot_parts(h->tcl.empty() ? 16 : h->tcl.back().n_pad, h->ps_out);
  w.planes = planes(h);
  if (h->ds_wide) {   // u of a split layer has its source region's pitch; Up-PS2 runs at 2x the LR resolution
    for (const LayerDef& l : h->layers) {
      if (!ds_split(h, l)) continue;
      const std::string& sc = l.scope;
      const size_t per_px = sc == "B2" ? w.b1 : sc == "Up-PS/Up-PS_CNN" ? w.nin : sc == "Up-PS2/Up-PS2_CNN" ? w.mid
                                                                          : (size_t)pad16(l.cin);
      w.u = std::max(w.u, per_px);
    }
  }
  return w;
}

static int ensure_workspace(dcscn_handle* h, size_t lr_px) {
  if (lr_px <= h->cap_px) return 0;
  const dcscn_config& c = h->cfg;
  const WorkspaceShape ws = workspace_shape(h);
  if (uses_ds_tile(h)) {
    if (h->ds_feat.alloc(lr_px * ws.feat, true)) return 1;   // pad channels must stay zero
    if (h->ds_b1.alloc(lr_px * ws.b1) || h->ds_nin.alloc(lr_px * ws.nin)) return 1;
    if (c.scale == 4 && h->ds_mid.alloc(lr_px * ws.mid)) return 1;
    if (h->ds_hr.alloc(lr_px * ws.hr)) return 1;
    h->cap_px = lr_px;
    return 0;
  }
  h->plans.clear();
  h->last_plan = nullptr;
  const bool two = ws.planes == 2;
  if (h->feat.alloc(lr_px * ws.feat, two) || h->b1.alloc(lr_px * ws.b1, two) || h->nin.alloc(lr_px * ws.nin, two) ||
      h->mid.alloc(lr_px * ws.mid, two) || h->u.alloc(lr_px * ws.u, two))
    return 1;
  if (h->hr.alloc(lr_px * ws.hr, true) || h->vbuf.alloc(lr_px * ws.vbuf, true)) return 1;
  h->cap_px = lr_px;
  return 0;
}

// Device bytes of the activation workspace and the tiled-inference staging buffers (dcscn_device_bytes).
static int64_t workspace_bytes(const dcscn_handle* h) {
  auto bytes = [](const auto&... a) { return (int64_t)(0 + ... + (a.size() * sizeof(*a.get()))); };
  return h->feat.bytes() + h->b1.bytes() + h->nin.bytes() + h->mid.bytes() + h->u.bytes() +
         bytes(h->hr, h->vbuf, h->ds_feat, h->ds_b1, h->ds_nin, h->ds_mid, h->ds_hr, h->tile_x, h->tile_x2, h->tile_y);
}

// --------------------------------------------------------------------------------------- plans ----
// Shared memory of conv_tc_kernel: at most kTcSmemMax per CTA, of which its barriers, 1 KB of alignment slack and the
// fp32 hand-off tile of an n_pad-column tile leave the rest for the activation and weight rings.  The patch
// (tc_patch_fits) and the ring depths (add_tc_launch) are both chosen against this budget.  The epilogue's copy of the
// bias and slopes only takes what the rings leave over (add_tc_launch); the R-CNN1 taps of a launch that fuses R-CNN1
// take it from there too, or from one weight tile (get_plan).
constexpr size_t kTcSmemMax = 227 * 1024;
static size_t tc_ring_budget(int n_pad) { return kTcSmemMax - 1024 - kTcBarrierBytes - tc_stage_bytes(n_pad); }

// Whether a k x k layer (k > 1) can load one activation box of (TW + k - 1) x (TH + k - 1) pixels per 64-channel chunk
// for all k x k taps (ConvTCParams::chunk_box): the patch's 8-pixel rows must each be one 8-row operand group (TW = 8),
// and two such boxes must fit beside three weight tiles (with two, 112-column layers ran 17-20 % slower than with
// (chunk, kx) boxes).  At k = 3 a chunk then fills 10 x 18 = 180 pixels instead of the 3 x 16 x 10 = 480 of an 8 x 16
// patch's three (chunk, kx) boxes.
static bool tc_chunk_box(int nplanes, int n_pad, int ksz, int TH, int TW) {
  if (ksz == 1 || TW != 8) return false;
  return 2 * (size_t)nplanes * tc_a_plane_bytes(tc_box_w(TW, ksz, 1), TH, ksz) +
             3 * (size_t)tc_w_tile_bytes(nplanes, n_pad) <= tc_ring_budget(n_pad);
}

// Whether a k x k layer (k > 1) can run on a TH x TW patch: with a chunk box (tc_chunk_box), or else with one box of
// TW x (TH + k - 1) pixels per (chunk, kx) whose ky taps are read at row offsets of TW pixels, which the swizzled
// operand descriptors allow only in whole 8-row groups (TW a multiple of 8); two such boxes plus two weight tiles must
// fit in shared memory.
static bool tc_patch_fits(int nplanes, int n_pad, int ksz, int TH, int TW) {
  if (ksz == 1 || tc_chunk_box(nplanes, n_pad, ksz, TH, TW)) return true;
  if (TW % 8 != 0) return false;
  return 2 * (size_t)nplanes * tc_a_plane_bytes(TW, TH, ksz) + 2 * (size_t)tc_w_tile_bytes(nplanes, n_pad) <=
         tc_ring_budget(n_pad);
}

// 128-pixel rectangular patches; minimise padded area, prefer wide patches (contiguous TMA rows).  A k x k layer
// (k > 1) takes the 16 x 8 patch with a chunk box unless another patch pads less.  Returns false when no patch suits
// the layer.
static bool choose_patch(int H, int W, int nplanes, int n_pad, int ksz, int* TH, int* TW) {
  static const int cand[][2] = {{8, 16}, {4, 32}, {16, 8}, {2, 64}, {32, 4}, {1, 128}, {64, 2}, {128, 1}};
  long long best = -1;
  auto area = [&](int th, int tw) { return (long long)((H + th - 1) / th) * th * ((W + tw - 1) / tw) * tw; };
  if (tc_chunk_box(nplanes, n_pad, ksz, 16, 8)) {
    best = area(16, 8);
    *TH = 16;
    *TW = 8;
  }
  for (auto& c : cand) {
    const int th = c[0], tw = c[1];
    if (!tc_patch_fits(nplanes, n_pad, ksz, th, tw)) continue;
    if (best < 0 || area(th, tw) < best) {
      best = area(th, tw);
      *TH = th;
      *TW = tw;
    }
  }
  return best >= 0;
}

// Tensor map of an NHWC fp16 plane whose boxes are 64 channels x TW x TH pixels, swizzled as the wgmma operands expect.
static int encode_map(dcscn_handle* h, CUtensorMap* tm, const __half* base, int cin_pad, int pitch, int n, int H,
                      int W, int TH, int TW) {
  cuuint64_t dims[4] = {(cuuint64_t)cin_pad, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)n};
  cuuint64_t strides[3] = {(cuuint64_t)pitch * 2, (cuuint64_t)W * pitch * 2, (cuuint64_t)H * W * pitch * 2};
  cuuint32_t box[4] = {(cuuint32_t)kTcKC, (cuuint32_t)TW, (cuuint32_t)TH, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = h->encode(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, (void*)base, dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return fail("cuTensorMapEncodeTiled failed (%d) cin_pad=%d pitch=%d n=%d H=%d W=%d box=%dx%d", (int)r, cin_pad,
                pitch, n, H, W, TH, TW);
  return 0;
}

// The epilogue's copy of a launch's bias and slopes (fp32, every column tile) in conv_tc_kernel's shared memory.
static size_t tc_bias_bytes(const ConvTCParams& p) { return 2 * sizeof(float) * (size_t)p.n_tiles * p.n_pad; }

static int add_tc_launch(dcscn_handle* h, Plan* pl, const TcLayer& t, PlaneView src, int src_pitch, int n, int H, int W,
                         const EpiParams& epi) {
  TcLaunch L;
  memset(&L, 0, sizeof(L));
  int TH = 0, TW = 0;
  if (!choose_patch(H, W, planes(h), t.n_pad, t.ksz, &TH, &TW))
    return fail("layer %s: no pixel patch fits a %dx%d filter in shared memory", t.name.c_str(), t.ksz, t.ksz);
  const int chunk_box = tc_chunk_box(planes(h), t.n_pad, t.ksz, TH, TW);
  // without a chunk box the kernel's ky taps start TW pixels apart inside the box: whole 8-row operand groups, or the
  // operands are misread
  if (t.ksz > 1 && !chunk_box && TW % 8 != 0)
    return fail("internal: layer %s: patch width %d is not a whole number of swizzle atoms", t.name.c_str(), TW);
  ConvGeom g{n, H, W, (W + TW - 1) / TW, (H + TH - 1) / TH, TW, TH};
  const int box_rows = TH + t.ksz - 1;   // a k x k layer's box carries the rows of all k ky taps
  const int box_w = tc_box_w(TW, t.ksz, chunk_box);   // and with a chunk box the columns of all k kx taps
  if (encode_map(h, &L.tm_hi, src.hi, t.cin_pad, src_pitch, n, H, W, box_rows, box_w)) return 1;
  if (planes(h) == 2) {
    if (encode_map(h, &L.tm_lo, src.lo, t.cin_pad, src_pitch, n, H, W, box_rows, box_w)) return 1;
  } else {
    L.tm_lo = L.tm_hi;
  }
  L.p.g = g;
  L.p.ksz = t.ksz;
  L.p.chunk_box = chunk_box;
  L.p.cin_pad = t.cin_pad;
  L.p.chunks = (t.cin_pad + kTcKC - 1) / kTcKC;
  L.p.n_tiles = t.n_tiles;
  L.p.n_pad = t.n_pad;
  // weight tiles per promotion segment; 1 = promote every 16-channel K slice.  The automatic lengths keep the dominant
  // chain as short as the earlier two-pass scheme had it (2 tiles for wide layers, 3 for thin ones).
  L.p.seg_chunks = h->seg_chunks > 0 ? h->seg_chunks : (t.n_pad > 64 ? 2 : 3);
  L.p.wpack = t.d_wpack.get();
  L.p.epi = epi;
  L.p.epi.bias = t.d_bias.get();
  L.p.epi.alpha = t.d_alpha.get();
  L.p.epi.out_scale = 1.0f / t.wscale;   // refreshed at every launch (launch_tc): a re-pack may pick another scale
  if (!h->tcl.empty() && &t >= h->tcl.data() && &t < h->tcl.data() + h->tcl.size()) {
    L.layer_index = (int)(&t - h->tcl.data());
    L.layer_bwd = false;
  } else if (!h->bwd.empty() && &t >= h->bwd.data() && &t < h->bwd.data() + h->bwd.size()) {
    L.layer_index = (int)(&t - h->bwd.data());
    L.layer_bwd = true;
  }
  L.p.epi.n_valid = t.n_valid;

  // Ring depths.  The consumers release a slot one weight tile late, so each ring needs at least two slots.  With a
  // chunk box a k x k layer reads k x k weight tiles per activation slot: two activation slots (one chunk ahead) and
  // the rest in weight tiles.  Without one it reads k weight tiles per activation slot: three activation slots when
  // four weight tiles still fit, else two.  A 1x1 layer pairs one activation slot with one weight tile.
  const size_t a_slot = (size_t)planes(h) * tc_a_plane_bytes(box_w, TH, t.ksz);
  const size_t w_tile = tc_w_tile_bytes(planes(h), t.n_pad);
  const size_t budget = tc_ring_budget(t.n_pad);
  int a_slots, w_slots;
  if (t.ksz == 1) {
    a_slots = w_slots = (int)std::min<size_t>(kMaxASlots, budget / (a_slot + w_tile));
  } else if (chunk_box) {
    a_slots = 2;
    w_slots = (int)std::min<size_t>(kMaxWSlots, (budget - a_slots * a_slot) / w_tile);
  } else {
    a_slots = 3;
    if (budget < a_slots * a_slot + 4 * w_tile) a_slots = 2;
    w_slots = budget < a_slots * a_slot ? 0 : (int)std::min<size_t>(kMaxWSlots, (budget - a_slots * a_slot) / w_tile);
  }
  if (a_slots < 2 || w_slots < 2)
    return fail("layer %s: two %zu-byte activation slots and two %zu-byte weight tiles do not fit in shared memory",
                t.name.c_str(), a_slot, w_tile);
  L.a_slots = a_slots;
  L.w_slots = w_slots;
  L.smem = a_slots * a_slot + w_slots * w_tile + 1024 + kTcBarrierBytes + tc_stage_bytes(t.n_pad);
  // the epilogue warps read bias and slopes from shared memory when what the rings leave over holds them; a layer
  // never gives up a ring slot for them (wide layers, e.g. the x5 ... x8 pixel shufflers, read them from global memory)
  L.p.bias_smem = L.smem + tc_bias_bytes(L.p) <= kTcSmemMax;
  if (L.p.bias_smem) L.smem += tc_bias_bytes(L.p);
  const long long tiles = (long long)n * g.tiles_x * g.tiles_y;
  const long long items = tiles * t.n_tiles;
  L.grid = (int)std::min<long long>(items, h->sm_count);

  // validation twin
  L.ref.g = g;
  L.ref.ksz = t.ksz;
  L.ref.cin = t.cin;
  L.ref.cout = t.cout;
  L.ref.src_hi = src.hi;
  L.ref.src_lo = src.lo;
  L.ref.src_pitch = src_pitch;
  L.ref.in_map = t.d_in_map.get();
  L.ref.w = t.d_wref.get();
  L.ref.n_total_pad = t.n_tiles * t.n_pad;
  L.ref.epi = L.p.epi;
  L.ref.epi.out_scale = 1.0f;
  pl->tc.push_back(L);
  return 0;
}

// A forward layer: its depthwise step when it has one (the 1x1 pointwise then reads u instead of the source), then
// its tensor-core launch.  pl->dw stays parallel to pl->tc.
static int add_layer_launch(dcscn_handle* h, Plan* pl, const TcLayer& t, PlaneView src, int src_pitch, int n, int H, int W,
                            const EpiParams& epi) {
  DwParams d;
  memset(&d, 0, sizeof(d));
  if (t.dw_ksz) {
    const PlaneView u = h->u.at(0);
    d = DwParams{n, H, W, t.dw_ksz, t.cin_pad, src.hi, src.lo, src_pitch, t.d_dw.get(), u.hi, u.lo};
    src = u;
    src_pitch = t.cin_pad;
    pl->dw_count++;
  }
  pl->dw.push_back(d);
  return add_tc_launch(h, pl, t, src, src_pitch, n, H, W, epi);
}

// One EPI_PLANES segment: GEMM columns [0, cols) to `dst`.
static EpiParams epi_planes(PlaneView dst, int pitch, int cols) {
  EpiParams e;
  memset(&e, 0, sizeof(e));
  e.mode = EPI_PLANES;
  e.num_seg = 1;
  e.seg[0] = {0, cols, dst.hi, dst.lo, pitch};
  e.keep_prob = 1.0f;
  e.out_scale = 1.0f;
  return e;
}

// The epilogue of an activated layer: one segment per output tensor, over the GEMM columns its keep mask indexes.
static EpiParams epi_activated(const dcscn_handle* h, std::initializer_list<const ActView*> outs) {
  EpiParams e = epi_planes({}, 0, 0);
  e.num_seg = 0;
  for (const ActView* v : outs) {
    e.seg[e.num_seg++] = {v->drop_col0, v->drop_col0 + pad16(v->ch), v->planes.hi, v->planes.lo, v->pitch};
    e.drop_ntotal = v->drop_stride;
  }
  e.act = h->cfg.activator;
  return e;
}

static int add_activated_launch(dcscn_handle* h, Plan* pl, const TcLayer& t, const ActView& src, int n, int H, int W,
                                std::initializer_list<const ActView*> outs) {
  if (add_layer_launch(h, pl, t, src.planes, src.pitch, n, H, W, epi_activated(h, outs))) return 1;
  std::copy(outs.begin(), outs.end(), pl->tc.back().act);
  return 0;
}

static Plan* get_plan(dcscn_handle* h, int n, int H, int W) {
  for (auto& p : h->plans)
    if (p->n == n && p->h == H && p->w == W) return p.get();
  const dcscn_config& c = h->cfg;
  const int L = c.layers;
  std::unique_ptr<Plan> pl(new Plan());
  pl->n = n;
  pl->h = H;
  pl->w = W;
  pl->act.resize(h->layers.size());
  for (size_t li = 0; li < h->layers.size(); ++li)
    if (h->layers[li].act) act_view(h, h->layers[li].scope, &pl->act[li]);
  const ActView* a = pl->act.data();   // CNN1 .. CNNL, A1, B1, B2 (build_graph's layer order)

  // CNN1
  memset(&pl->first, 0, sizeof(pl->first));
  pl->first.g = ConvGeom{n, H, W, 1, 1, 1, 1};
  pl->first.ksz = find_layer(h, "CNN1")->k;
  pl->first.n_pad = h->feat_w[0];
  pl->first.w = h->d_first_w.get();
  pl->first.epi = epi_activated(h, {&a[0]});
  pl->first.epi.bias = h->d_first_bias.get();
  pl->first.epi.alpha = h->d_first_alpha.get();
  pl->first.epi.n_valid = h->filters[0];

  size_t ti = 0;
  for (int i = 1; i < L; ++i)
    if (add_activated_launch(h, pl.get(), h->tcl[ti++], a[i - 1], n, H, W, {&a[i]})) return nullptr;
  // A1+B1 reads the whole concat buffer (CNN1's slot starts at channel 0)
  if (add_activated_launch(h, pl.get(), h->tcl[ti++], a[0], n, H, W, {&a[L], &a[L + 1]})) return nullptr;
  if (add_activated_launch(h, pl.get(), h->tcl[ti++], a[L + 1], n, H, W, {&a[L + 2]})) return nullptr;   // B1 -> B2
  int HR_H = H, HR_W = W;
  {  // Up-PS, or Up-TCNN (its 3x3 LR form, then depth_to_space(s) in one step at every scale)
    EpiParams e;
    memset(&e, 0, sizeof(e));
    e.keep_prob = 1.0f;
    if (two_stage_up(h)) {
      e.mode = EPI_D2S_PLANES;
      e.d2s_r = 2;
      e.d2s_cout = c.nin_filters + c.nin_filters2;
      e.num_seg = 1;
      e.seg[0] = {0, 0, h->mid.hi.get(), h->mid.lo.get(), h->mid_pitch};
    } else {
      e.mode = EPI_D2S_F32;
      e.d2s_r = c.scale;
      e.d2s_cout = h->ps_out;
      e.dst_f32 = h->hr.get();
      e.d2s_pitch = h->ps_out;
    }
    if (add_layer_launch(h, pl.get(), h->tcl[ti++], h->nin.at(0), h->nin_pitch, n, H, W, e)) return nullptr;
    HR_H = H * (two_stage_up(h) ? 2 : c.scale);
    HR_W = W * (two_stage_up(h) ? 2 : c.scale);
  }
  if (two_stage_up(h)) {  // Up-PS2 at 2x resolution
    EpiParams e;
    memset(&e, 0, sizeof(e));
    e.keep_prob = 1.0f;
    e.mode = EPI_D2S_F32;
    e.d2s_r = 2;
    e.d2s_cout = h->ps_out;
    e.dst_f32 = h->hr.get();
    e.d2s_pitch = h->ps_out;
    if (add_layer_launch(h, pl.get(), h->tcl[ti++], h->mid.at(0), h->mid_pitch, n, HR_H, HR_W, e)) return nullptr;
    HR_H *= 2;
    HR_W *= 2;
  }
  {  // the last depth_to_space layer can carry the per-pixel half of R-CNN1 in its epilogue
    TcLaunch& L = pl->tc.back();
    const int cout = h->ps_out, nch = L.p.n_pad >> 4, per = (nch + kColSplit - 1) / kColSplit;
    const int klast = find_layer(h, "R-CNN1")->k;
    const int parts = rdot_parts(L.p.n_pad, cout);
    pl->unfused = L;
    pl->fused_index = (int)pl->tc.size() - 1;
    pl->fused_last = last_fuses(h, L.p.n_pad);
    if (pl->fused_last && L.p.bias_smem) {   // the fused epilogues (EPI_D2S_TAPS / EPI_D2S_RDOT) read bias from global
      L.smem -= tc_bias_bytes(L.p);
      L.p.bias_smem = 0;
    }
    if (pl->fused_last && h->fold.cout > 0) {
      // the folded layer (build_fold): same input, patch, rings and column-tile width, fewer column tiles
      const TcLayer& f = h->fold;
      L.layer_index = -1;
      L.layer_fold = true;
      L.p.n_tiles = f.n_tiles;
      L.p.wpack = f.d_wpack.get();
      L.p.epi.bias = f.d_bias.get();
      L.p.epi.alpha = f.d_alpha.get();
      L.p.epi.out_scale = 1.0f / f.wscale;
      L.p.epi.n_valid = f.n_valid;
      L.p.epi.mode = EPI_D2S_TAPS;
      L.p.epi.rdot_out = h->vbuf.get();
      L.p.epi.rdot_taps = 9;
      L.p.epi.rdot_parts = 1;
      L.grid = (int)std::min<long long>((long long)n * L.p.g.tiles_x * L.p.g.tiles_y * f.n_tiles, h->sm_count);
    } else if (pl->fused_last) {
      L.p.epi.rdot_parts = ((per * 16) % cout == 0) ? 1 : parts;
      L.p.epi.mode = EPI_D2S_RDOT;
      L.p.epi.rdot_w = h->d_last_w.get();
      L.p.epi.rdot_out = h->vbuf.get();
      L.p.epi.rdot_taps = klast * klast;
      // the kernel stages the R-CNN1 taps behind the hand-off tile: weight tiles make room for them
      const size_t w_tile = tc_w_tile_bytes(planes(h), L.p.n_pad);
      for (L.smem += kRdotSmemBytes; L.smem > kTcSmemMax && L.w_slots > 2; L.smem -= w_tile) L.w_slots--;
      if (L.smem > kTcSmemMax) {
        fail("the fused R-CNN1 taps do not fit in shared memory beside two weight tiles (column tile %d)", L.p.n_pad);
        return nullptr;
      }
    }
    const int gparts = pl->fused_last ? L.p.epi.rdot_parts : 1;
    memset(&pl->gather, 0, sizeof(pl->gather));
    pl->gather.parts = gparts;
    pl->gather.n_img = n;
    pl->gather.H = HR_H;
    pl->gather.W = HR_W;
    pl->gather.ksz = klast;
    pl->gather.v = h->vbuf.get();
  }
  memset(&pl->last, 0, sizeof(pl->last));
  pl->last.n_img = n;
  pl->last.H = HR_H;
  pl->last.W = HR_W;
  pl->last.ksz = find_layer(h, "R-CNN1")->k;
  pl->last.C = h->ps_out;
  pl->last.pitch = h->ps_out;
  pl->last.src = h->hr.get();
  pl->last.w = h->d_last_w.get();
  pl->last.bias = 0.f;
  if (h->plans.size() >= 64) h->plans.erase(h->plans.begin());
  h->plans.push_back(std::move(pl));
  return h->plans.back().get();
}

// ------------------------------------------------------------------------------------- forward ----
#ifdef DCSCN_TC_PHASES
// Diagnostic build: one stderr line per conv_tc_kernel launch with its phase cycles (g_tc_phase) and its plan; the launch
// is waited for, so the timings of this build are not the product's.
static int tc_phase_report(dcscn_handle* h, const TcLaunch& L, cudaStream_t st) {
  unsigned long long c[4];
  CUDA_TRY(cudaStreamSynchronize(st));
  CUDA_TRY(cudaMemcpyFromSymbol(c, g_tc_phase, sizeof(c)));
  const unsigned long long zero[4] = {};
  CUDA_TRY(cudaMemcpyToSymbol(g_tc_phase, zero, sizeof(zero)));
  std::string name = "?";
  if (L.layer_fold) name = "Up-PS(fold)";
  else if (L.layer_index >= 0 && !L.layer_bwd && L.layer_index < (int)h->tcl.size()) name = h->tcl[L.layer_index].name;
  else if (L.layer_index >= 0 && L.layer_bwd && L.layer_index < (int)h->bwd.size()) name = "bwd:" + h->bwd[L.layer_index].name;
  fprintf(stderr, "tc_phase %s mode=%d n_pad=%d n_tiles=%d patch=%dx%d a_slots=%d w_slots=%d smem=%zu k=%llu epi=%llu "
          "items=%llu epw=%llu chunk_box=%d\n", name.c_str(), L.p.epi.mode, L.p.n_pad, L.p.n_tiles, L.p.g.TH, L.p.g.TW,
          L.a_slots, L.w_slots, L.smem, c[0], c[1], c[2], c[3], L.p.chunk_box);
  return 0;
}
#endif

template <int NPL, int N>
static int launch_tc_inst(dcscn_handle* h, const TcLaunch& L, cudaStream_t st) {
  static bool attr_set_dev[64] = {};   // function attributes are per device
  bool& attr_set = attr_set_dev[h->cfg.device_id & 63];
  if (!attr_set) {
    CUDA_TRY(cudaFuncSetAttribute(conv_tc_kernel<NPL, N>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr_set = true;
  }
  conv_tc_kernel<NPL, N><<<L.grid, kTcThreads, L.smem, st>>>(L.tm_hi, L.tm_lo, L.p, L.a_slots, L.w_slots);
  CUDA_TRY(cudaGetLastError());
#ifdef DCSCN_TC_PHASES
  return tc_phase_report(h, L, st);
#else
  return 0;
#endif
}

// The column-tile width is a template parameter of the kernel (the wgmma width is an immediate of the instruction).
template <int NPL>
static int launch_tc_width(dcscn_handle* h, const TcLaunch& L, cudaStream_t st) {
  switch (L.p.n_pad) {
    case 16: return launch_tc_inst<NPL, 16>(h, L, st);
    case 32: return launch_tc_inst<NPL, 32>(h, L, st);
    case 48: return launch_tc_inst<NPL, 48>(h, L, st);
    case 64: return launch_tc_inst<NPL, 64>(h, L, st);
    case 80: return launch_tc_inst<NPL, 80>(h, L, st);
    case 96: return launch_tc_inst<NPL, 96>(h, L, st);
    case 112: return launch_tc_inst<NPL, 112>(h, L, st);
  }
  return fail("internal: column tile width %d is not a multiple of 16 in [16, %d]", L.p.n_pad, kMaxTileN);
}

static int launch_tc(dcscn_handle* h, const TcLaunch& Lc, cudaStream_t st) {
  h->launches++;
  // Cached plans outlive weight re-packs.  A re-pack keeps the device allocations (so the plan's pointers stay valid) but
  // may choose a different power-of-two weight scale: take the epilogue's 1 / scale from the layer as it is NOW.
  TcLaunch& L = const_cast<TcLaunch&>(Lc);
  if (L.layer_fold) {
    L.p.epi.out_scale = 1.0f / h->fold.wscale;
  } else if (L.layer_index >= 0) {
    const std::vector<TcLayer>& ls = L.layer_bwd ? h->bwd : h->tcl;
    if (L.layer_index < (int)ls.size()) L.p.epi.out_scale = 1.0f / ls[L.layer_index].wscale;
  }
  if (h->conv_impl == 1) {
    const long long total = (long long)L.ref.g.n_img * L.ref.g.H * L.ref.g.W * (L.ref.n_total_pad >> 4);
    const int grid = (int)std::min<long long>((total + 127) / 128, (long long)h->sm_count * 16);
    conv_ref_kernel<<<grid, 128, 0, st>>>(L.ref);
    CUDA_TRY(cudaGetLastError());
    return 0;
  }
  const int npl = planes(h);
  if (L.p.wpack == nullptr) return fail("internal: weight image was not packed for this layer");
  return npl == 2 ? launch_tc_width<2>(h, L, st) : launch_tc_width<1>(h, L, st);
}

static int mark(dcscn_handle* h, cudaStream_t st) {
  if (!h->timing) return 0;
  if (h->ev_used >= (int)h->ev.size()) {
    cudaEvent_t e;
    CUDA_TRY(cudaEventCreate(&e));
    h->ev.emplace_back(e);
  }
  CUDA_TRY(cudaEventRecord(h->ev[h->ev_used++].get(), st));
  return 0;
}

// ---- depthwise-separable kernels (conv_ds_tile.cuh) ----
template <int KSZ>
static int launch_ds_tile_k(dcscn_handle* h, const DsTileParams& p, unsigned grid, size_t smem, cudaStream_t st) {
  const int cols = p.cout < 32 ? ((p.cout + 3) & ~3) : 32;
  static size_t attr_dev[64][2] = {};
  size_t& cur = attr_dev[h->cfg.device_id & 63][KSZ == 3 ? 1 : 0];
  if (cur == 0) cur = 48 * 1024;
  if (smem > cur) {
    const int b = (int)smem;
    CUDA_TRY(cudaFuncSetAttribute(ds_tile_kernel<KSZ, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, b));
    CUDA_TRY(cudaFuncSetAttribute(ds_tile_kernel<KSZ, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, b));
    CUDA_TRY(cudaFuncSetAttribute(ds_tile_kernel<KSZ, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, b));
    CUDA_TRY(cudaFuncSetAttribute(ds_tile_kernel<KSZ, 6>, cudaFuncAttributeMaxDynamicSharedMemorySize, b));
    CUDA_TRY(cudaFuncSetAttribute(ds_tile_kernel<KSZ, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, b));
    cur = smem;
  }
  if (cols <= 4) ds_tile_kernel<KSZ, 1><<<grid, kDtThreads, smem, st>>>(p);
  else if (cols <= 8) ds_tile_kernel<KSZ, 2><<<grid, kDtThreads, smem, st>>>(p);
  else if (cols <= 16) ds_tile_kernel<KSZ, 4><<<grid, kDtThreads, smem, st>>>(p);
  else if (cols <= 24) ds_tile_kernel<KSZ, 6><<<grid, kDtThreads, smem, st>>>(p);
  else ds_tile_kernel<KSZ, 8><<<grid, kDtThreads, smem, st>>>(p);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

static int launch_ds_tile(dcscn_handle* h, DsTileParams p, int ksz, cudaStream_t st) {
  if (ksz != 1 && ksz != 3) return fail("depthwise-separable layer: kernel size %d is not supported (1 or 3)", ksz);
  if (p.cout > 32 && p.cin > kDtCC) return fail("depthwise-separable layer %d -> %d: more than 32 output columns need <= 32 input channels", p.cin, p.cout);
  const size_t smem = ds_tile_launch_smem(ksz, p.cin, p.cout);
  if (smem > 200 * 1024) return fail("depthwise-separable layer %d -> %d exceeds the kernel's shared memory", p.cin, p.cout);
  unsigned grid;
  if (ksz == 3) {
    p.tiles_x = (p.W + kDtT - 1) / kDtT;
    p.tiles_y = (p.H + kDtT - 1) / kDtT;
    grid = (unsigned)((long long)p.n_img * p.tiles_x * p.tiles_y);
  } else {
    grid = (unsigned)(((long long)p.n_img * p.H * p.W + kDtThreads - 1) / kDtThreads);
  }
  const int rc = ksz == 3 ? launch_ds_tile_k<3>(h, p, grid, smem, st) : launch_ds_tile_k<1>(h, p, grid, smem, st);
  if (rc) return rc;
  h->launches++;
  return mark(h, st);
}

static DsTileParams ds_tile_params(const LayerDef& l, const dcscn_handle::DsDev& d, const float* src, int src_pitch, float* dst,
                                   int dst_pitch, int dst_off, int n, int H, int W) {
  DsTileParams p;
  memset(&p, 0, sizeof(p));
  p.n_img = n; p.H = H; p.W = W; p.cin = l.cin; p.cout = l.cout;
  p.src = src; p.src_pitch = src_pitch; p.dw = d.dw.get(); p.pw = d.pw.get(); p.bias = d.bias.get(); p.alpha = d.alpha.get();
  p.dst = dst; p.dst_pitch = dst_pitch; p.dst_off = dst_off;
  return p;
}

// sigmoid / tanh / selu of an activated depthwise-separable layer (see ds_act_kernel); nothing for the other activators.
static int ds_activate(dcscn_handle* h, float* buf, long long npx, int pitch, int off, int C, cudaStream_t st) {
  if (h->cfg.activator < DCSCN_ACTIVATOR_SIGMOID) return 0;
  const long long total = npx * C;
  ds_act_kernel<<<(int)std::min<long long>((total + 255) / 256, (long long)h->sm_count * 16), 256, 0, st>>>(buf, npx, pitch, off, C,
                                                                                                          h->cfg.activator);
  CUDA_TRY(cudaGetLastError());
  h->launches++;
  return 0;
}

// Depthwise-separable graph (DCSCN.py:246-249, 264-271, 318-320; tf_graph.py:240-243): fp32 NHWC, CUDA cores.
static int forward_ds_tile(dcscn_handle* h, const float* x, const float* x2, float* y, int n, int H, int W, cudaStream_t st) {
  const dcscn_config& c = h->cfg;
  const int L = c.layers, T = h->ds_total, na = c.nin_filters, nb = c.nin_filters2, cps = na + nb;
  if (!h->tiling) {   // a tiled forward keeps one event sequence over all its batches
    h->ev_used = 0;
    if (mark(h, st)) return 1;
  }
  size_t li = 0;
  for (int i = 0; i < L; ++i, ++li) {
    const float* src = i == 0 ? x : h->ds_feat.get() + h->ds_off[i - 1];
    DsTileParams p = ds_tile_params(h->layers[li], h->ds[li], src, i == 0 ? c.channels : T, h->ds_feat.get(), T, h->ds_off[i], n, H, W);
    if (launch_ds_tile(h, p, h->layers[li].k, st)) return 1;
    if (ds_activate(h, h->ds_feat.get(), (long long)n * H * W, T, h->ds_off[i], h->filters[i], st)) return 1;
  }
  {  // A1 | B1: both are 1x1 over the whole concat buffer -> ONE pass; the per-channel depthwise scales are folded into the
     // pointwise rows.  Columns [0, na) = A1 -> [B2 | A1] buffer at channel nb; columns [na, na+nb) = B1 -> B1 buffer.
    if (h->layers[li].k != 1 || h->layers[li + 1].k != 1) return fail("depthwise-separable A1 / B1 must be 1x1");
    LayerDef ab = h->layers[li];
    ab.k = 1; ab.cin = T; ab.cout = cps;
    DsTileParams p = ds_tile_params(ab, h->ds_ab, h->ds_feat.get(), T, h->ds_nin.get(), cps, nb, n, H, W);
    p.dw = nullptr;
    p.split = na;
    p.dst2 = h->ds_b1.get(); p.dst2_pitch = nb; p.dst2_off = 0;
    if (cps > 32) return fail("depthwise-separable graph: nin_filters + nin_filters2 = %d > 32 is not supported by the fused A1|B1 kernel", cps);
    if (launch_ds_tile(h, p, 1, st)) return 1;
    if (ds_activate(h, h->ds_nin.get(), (long long)n * H * W, cps, nb, na, st) || ds_activate(h, h->ds_b1.get(), (long long)n * H * W, nb, 0, nb, st))
      return 1;
    li += 2;
  }
  {  // B2
    DsTileParams p = ds_tile_params(h->layers[li], h->ds[li], h->ds_b1.get(), nb, h->ds_nin.get(), cps, 0, n, H, W);
    if (launch_ds_tile(h, p, h->layers[li].k, st)) return 1;
    if (ds_activate(h, h->ds_nin.get(), (long long)n * H * W, cps, 0, nb, st)) return 1;
    ++li;
  }
  int HH = H, WW = W;
  if (c.scale == 4) {
    DsTileParams p = ds_tile_params(h->layers[li], h->ds[li], h->ds_nin.get(), cps, h->ds_mid.get(), cps, 0, n, H, W);
    p.d2s_r = 2; p.d2s_cout = cps;
    if (launch_ds_tile(h, p, h->layers[li].k, st)) return 1;
    ++li;
    HH = 2 * H; WW = 2 * W;
    DsTileParams q = ds_tile_params(h->layers[li], h->ds[li], h->ds_mid.get(), cps, h->ds_hr.get(), h->ps_out, 0, n, HH, WW);
    q.d2s_r = 2; q.d2s_cout = h->ps_out;
    if (launch_ds_tile(h, q, h->layers[li].k, st)) return 1;
    ++li;
    HH *= 2; WW *= 2;
  } else {
    DsTileParams p = ds_tile_params(h->layers[li], h->ds[li], h->ds_nin.get(), cps, h->ds_hr.get(), h->ps_out, 0, n, H, W);
    p.d2s_r = c.scale; p.d2s_cout = h->ps_out;
    if (launch_ds_tile(h, p, h->layers[li].k, st)) return 1;
    ++li;
    HH = c.scale * H; WW = c.scale * W;
  }
  if (h->wait_x2) {
    CUDA_TRY(cudaStreamWaitEvent(st, h->x2_ready.get(), 0));
    h->wait_x2 = false;
  }
  // R-CNN1 (no bias / activation) + x2
  const LayerDef& lr = h->layers[li];
  const dcscn_handle::DsDev& d = h->ds[li];
  if (lr.cin == 1 && lr.cout == 1) {
    if (lr.k != 1 && lr.k != 3) return fail("depthwise-separable R-CNN1: kernel size %d is not supported (1 or 3)", lr.k);
    const long long total = (long long)n * HH * WW;
    // four pixels per thread when the row width and the x2 / y alignment allow it, else one
    // (a tiled forward takes the kernel the whole image would take: they sum the taps in different orders)
    const bool vec4 = lr.k == 3 && (WW & 3) == 0 && total < (1ll << 32) &&
                      ((reinterpret_cast<uintptr_t>(y) | reinterpret_cast<uintptr_t>(x2)) & 15) == 0 &&
                      (!h->tiling || h->tile_vec4);
    const int grid = (int)std::min<long long>(((vec4 ? total / 4 : total) + 255) / 256, (long long)h->sm_count * 16);
    if (vec4) ds_single4_kernel<<<grid, 256, 0, st>>>(h->ds_hr.get(), x2, y, n, HH, WW, d.dw.get(), d.pw.get(), d.bias.get(), d.alpha.get());
    else if (lr.k == 3) ds_single_kernel<3><<<grid, 256, 0, st>>>(h->ds_hr.get(), x2, y, n, HH, WW, d.dw.get(), d.pw.get(), d.bias.get(), d.alpha.get());
    else ds_single_kernel<1><<<grid, 256, 0, st>>>(h->ds_hr.get(), x2, y, n, HH, WW, d.dw.get(), d.pw.get(), d.bias.get(), d.alpha.get());
    CUDA_TRY(cudaGetLastError());
    h->launches++;
    return mark(h, st);
  }
  DsTileParams p = ds_tile_params(lr, d, h->ds_hr.get(), h->ps_out, y, 1, 0, n, HH, WW);
  p.add = x2;
  return launch_ds_tile(h, p, lr.k, st);
}

static int launch_depthwise(dcscn_handle* h, const DwParams& p, cudaStream_t st) {
  const long long total = (long long)p.n_img * p.H * p.W * (p.cpad >> 3);
  const int grid = (int)std::min<long long>((total + 255) / 256, (long long)h->sm_count * 16);
  if (p.ksz == 3) depthwise_planes_kernel<3><<<grid, 256, 0, st>>>(p);
  else if (p.ksz == 5) depthwise_planes_kernel<5><<<grid, 256, 0, st>>>(p);
  else return fail("depthwise step: kernel size %d is not supported (3 or 5)", p.ksz);
  CUDA_TRY(cudaGetLastError());
  h->launches++;
  return mark(h, st);
}

// CNN1 (the forward's and the train step's): the 3x3 fast path, storing min(z, 0) when the epilogue asks for it, or the
// general kernel.
static int launch_first(dcscn_handle* h, const ConvFirstParams& p, cudaStream_t st) {
  if (p.ksz > 5) return fail("cnn_size %d is not supported by the first-layer kernel", p.ksz);
  const long long total = (long long)p.g.n_img * p.g.H * p.g.W;
  if (p.ksz == 3 && p.n_pad <= 256) {
    const int grid = (int)std::min<long long>((total + 7) / 8, (long long)h->sm_count * 8);
    if (p.epi.seg[0].dst_zneg != nullptr) conv_first3x3_kernel<true><<<grid, 256, 0, st>>>(p);
    else conv_first3x3_kernel<false><<<grid, 256, 0, st>>>(p);
  } else {
    const int grid = (int)std::min<long long>((total + 255) / 256, (long long)h->sm_count * 8);
    conv_first_kernel<<<grid, 256, (size_t)p.ksz * p.ksz * p.n_pad * sizeof(float), st>>>(p);
  }
  CUDA_TRY(cudaGetLastError());
  h->launches++;
  return 0;
}

// CNN1 and the tensor-core layers of one forward, in execution order, on `st` (a capturing stream when the plan's graph is
// being built).  The last kernel (R-CNN1 gather / R-CNN1) is issued by forward_impl: it alone touches x2 and y.
static int issue_front(dcscn_handle* h, Plan* pl, const float* x, bool fused, cudaStream_t st) {
  ConvFirstParams first = pl->first;
  first.x = x;
  if (launch_first(h, first, st) || mark(h, st)) return 1;
  for (size_t i = 0; i < pl->tc.size(); ++i) {
    if (pl->dw[i].ksz && launch_depthwise(h, pl->dw[i], st)) return 1;
    const TcLaunch& L = ((int)i == pl->fused_index && !fused) ? pl->unfused : pl->tc[i];
    if (launch_tc(h, L, st)) return 1;
    if (mark(h, st)) return 1;
  }
  return 0;
}

static int forward_impl(dcscn_handle* h, const float* x, const float* x2, float* y, int n, int H, int W,
                        cudaStream_t st) {
  if (n <= 0 || H <= 0 || W <= 0) return fail("forward: bad shape n=%d h=%d w=%d", n, H, W);
  CUDA_TRY(cudaSetDevice(h->cfg.device_id));
  if (h->params_dirty && finalize_params(h)) return 1;
  if (ensure_workspace(h, (size_t)n * H * W)) return 1;
  if (!h->tiling) h->tiled_last = false;
  if (uses_ds_tile(h)) {
    h->ds_n = n; h->ds_h = H; h->ds_w = W;
    return forward_ds_tile(h, x, x2, y, n, H, W, st);
  }
  Plan* pl = get_plan(h, n, H, W);
  if (!pl) return 1;
  h->last_plan = pl;
  if (!h->tiling) {
    h->ev_used = 0;
    if (mark(h, st)) return 1;
  }
  const bool fused = pl->fused_last && h->fuse_last && h->conv_impl == 0;

  // ---- graph replay / capture of the launches in front of the last kernel (SURVEY 7 step 5: 15 launches per step)
  const bool graphable = h->use_graph && !h->timing && h->conv_impl == 0;
  if (graphable && pl->gexec && pl->g_x == x && pl->g_epoch == h->graph_epoch && pl->g_fused == fused) {
    CUDA_TRY(cudaGraphLaunch(pl->gexec, st));
    h->launches += pl->g_launches;
    h->graph_replays++;
  } else if (graphable && pl->eager_runs >= 1 && pl->last_x == x) {
    if (!h->cap_stream) {
      cudaStream_t s;
      CUDA_TRY(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
      h->cap_stream.reset(s);
    }
    if (pl->gexec) { cudaGraphExecDestroy(pl->gexec); pl->gexec = nullptr; }
    const int64_t before = h->launches;
    CUDA_TRY(cudaStreamBeginCapture(h->cap_stream.get(), cudaStreamCaptureModeThreadLocal));
    const int rc = issue_front(h, pl, x, fused, h->cap_stream.get());
    cudaGraph_t g = nullptr;
    const cudaError_t ce = cudaStreamEndCapture(h->cap_stream.get(), &g);
    h->launches = before;
    if (rc) { if (g) cudaGraphDestroy(g); return 1; }
    if (ce != cudaSuccess || g == nullptr) return fail("forward: stream capture failed: %s", cudaGetErrorString(ce));
    const cudaError_t ie = cudaGraphInstantiate(&pl->gexec, g, 0);
    cudaGraphDestroy(g);
    if (ie != cudaSuccess) { pl->gexec = nullptr; return fail("forward: cudaGraphInstantiate failed: %s", cudaGetErrorString(ie)); }
    pl->g_x = x; pl->g_epoch = h->graph_epoch; pl->g_fused = fused;
    pl->g_launches = 1 + pl->dw_count + (int)pl->tc.size();
    CUDA_TRY(cudaGraphLaunch(pl->gexec, st));
    h->launches += pl->g_launches;
    h->graph_replays++;
  } else {
    if (issue_front(h, pl, x, fused, st)) return 1;
    pl->eager_runs++;
  }
  pl->last_x = x;
  pl->ran_fused = fused;
  if (h->wait_x2) {  // forward_host: x2 was copied on the side stream
    CUDA_TRY(cudaStreamWaitEvent(st, h->x2_ready.get(), 0));
    h->wait_x2 = false;
  }
  if (fused) {  // R-CNN1 second half: 9-tap gather of the tap-planar partial products + x2
    ConvGatherParams p = pl->gather;
    p.x2 = x2;
    p.y = y;
    const size_t total = (size_t)p.n_img * p.H * p.W;
    // (a tiled forward takes the kernel the whole image would take: they can differ in the sign of a zero)
    const bool vec4 = p.ksz == 3 && (p.W & 3) == 0 && ((reinterpret_cast<uintptr_t>(x2) | reinterpret_cast<uintptr_t>(y)) & 15) == 0 &&
                      (!h->tiling || h->tile_vec4);
    if (vec4) {
      const int grid = (int)std::min<size_t>((total / 4 + 255) / 256, (size_t)h->sm_count * 16);
      conv_last_gather4_kernel<<<grid, 256, 0, st>>>(p);
    } else {
      const int grid = (int)std::min<size_t>((total + 255) / 256, (size_t)h->sm_count * 16);
      conv_last_gather_kernel<<<grid, 256, 0, st>>>(p);
    }
    CUDA_TRY(cudaGetLastError());
    h->launches++;
    if (mark(h, st)) return 1;
    return 0;
  }
  {  // R-CNN1 + x2
    ConvLastParams p = pl->last;
    p.x2 = x2;
    p.y = y;
    const int half = p.ksz >> 1;
    const int tiles = ((p.W + kLastTW - 1) / kLastTW) * ((p.H + kLastTH - 1) / kLastTH) * p.n_img;
    const size_t smem = ((size_t)p.ksz * p.ksz * p.C + (size_t)(kLastTH + 2 * half) * (kLastTW + 2 * half) * kLastCC) * sizeof(float);
    conv_last_kernel<<<tiles, 256, smem, st>>>(p);
    CUDA_TRY(cudaGetLastError());
    h->launches++;
    if (mark(h, st)) return 1;
  }
  return 0;
}

// ------------------------------------------------------------------------------ tiled inference ----
// LR pixels of context a window core needs: the longest dependency path CNN1 .. CNNL -> B1 (1x1) -> B2 -> Up-PS
// [-> Up-PS2 at 2x] -> R-CNN1 at HR resolution, walked back from an LR core edge.  An HR reach of q pixels past an edge
// of s-times upscaled pixels is ceil(q / s) pixels before the upscale.  Up-TCNN and R-CNN1 are walked back together
// (tconv_halo): the 3x3 LR form of Up-TCNN reads only one side of each LR pixel per output phase.
static int tconv_halo(int s, int hr) {
  const int K = tconv_ksize(s), pad = (K - s) / 2;
  int reach = 0;
  for (int o = -hr; o < s + hr; ++o) {   // HR pixels R-CNN1 reads around the s outputs of LR pixel 0
    const int m = o >= 0 ? o / s : -((-o + s - 1) / s), p = o - m * s;
    for (int d = -1; d <= 1; ++d) {
      const int k = p + pad - s * d;
      if (k >= 0 && k < K) reach = std::max(reach, std::abs(m + d));
    }
  }
  return reach;
}

static int tile_halo(const dcscn_handle* h) {
  auto half = [](int k) { return (k - 1) / 2; };
  auto k_of = [h](const std::string& scope) { return find_layer(h, scope)->k; };
  int r = 0;
  for (int i = 0; i < h->cfg.layers; ++i) r += half(k_of("CNN" + std::to_string(i + 1)));
  r += half(k_of("B1")) + half(k_of("B2"));
  const int hr = half(k_of("R-CNN1"));
  if (tconv(h)) return r + tconv_halo(h->cfg.scale, hr);
  r += half(k_of("Up-PS/Up-PS_CNN"));
  if (two_stage_up(h)) r += (half(k_of("Up-PS2/Up-PS2_CNN")) + (hr + 1) / 2 + 1) / 2;
  else r += (hr + h->cfg.scale - 1) / h->cfg.scale;
  return r;
}

constexpr int kTileMinCore = 16;   // smallest window core (LR pixels per side) the planner uses

struct TilePlan {
  int th = 0, tw = 0;   // window, LR pixels
  int my = 0, mx = 0;   // windows per image along y / x
  int batch = 0;        // windows per batch
};

// Windows of one size per forward, clamped inside the image.  Of the window shapes whose pixels fit the budget, the one
// with the fewest window pixels per image is taken (a dimension that fits whole is spanned: no halo along it), ties going
// to the larger window; then as many windows of all n images as still fit form one batch.  When the whole image would run
// R-CNN1 on its four-pixel kernel, a window narrower than the image is a multiple of 4 wide so that its batch does too.
static int plan_tiles(dcscn_handle* h, int n, int H, int W, size_t px_bytes, TilePlan* tp) {
  const int r = tile_halo(h);
  const long long max_px = (h->workspace_mb << 20) / (long long)px_bytes;
  const int min_th = std::min(H, kTileMinCore + 2 * r);
  const int min_tw = std::min(W, h->tile_vec4 ? (kTileMinCore + 2 * r + 3) & ~3 : kTileMinCore + 2 * r);
  if ((long long)min_th * min_tw > max_px) {
    const long long need = ((long long)min_th * min_tw * (long long)px_bytes + (1 << 20) - 1) >> 20;
    return fail("forward: option workspace_mb = %lld cannot hold one %dx%d window (a %dx%d core plus a %d-pixel halo); this "
                "graph needs at least workspace_mb = %lld for this image", (long long)h->workspace_mb, min_th, min_tw,
                kTileMinCore, kTileMinCore, r, need);
  }
  long long best = -1, best_area = 0;
  for (int th = min_th; th <= H && (long long)th * min_tw <= max_px; ++th) {
    int tw = (int)std::min<long long>(W, max_px / th);
    if (tw < W && h->tile_vec4) tw &= ~3;
    if (tw < min_tw) continue;
    const int my = tile_count(H, th, r), mx = tile_count(W, tw, r);
    const long long cost = (long long)my * mx * th * tw, area = (long long)th * tw;
    if (best < 0 || cost < best || (cost == best && area > best_area)) {
      best = cost;
      best_area = area;
      tp->th = th; tp->tw = tw; tp->my = my; tp->mx = mx;
    }
  }
  const long long windows = (long long)n * tp->my * tp->mx;
  tp->batch = (int)std::max<long long>(1, std::min<long long>(windows, max_px / best_area));
  return 0;
}

// Runs the forward as batches of windows (plan_tiles) through forward_impl on the staging buffers: every full batch
// shares one (batch, th, tw) plan and one staging pointer, so its front launches are captured and replayed like any
// repeated forward; the last, partial batch has a plan of its own.
static int forward_tiled(dcscn_handle* h, const float* x, const float* x2, float* y, int n, int H, int W,
                         const TilePlan& tp, cudaStream_t st) {
  const int s = h->cfg.scale;
  const size_t lr_px = (size_t)tp.batch * tp.th * tp.tw, hr_px = lr_px * s * s;
  if (h->tile_x.grow(lr_px) || h->tile_x2.grow(hr_px) || h->tile_y.grow(hr_px)) return 1;
  struct Scope {
    dcscn_handle* h;
    ~Scope() { h->tiling = false; }
  } scope{h};
  h->tiling = true;
  h->ev_used = 0;
  if (mark(h, st)) return 1;
  if (h->wait_x2) {  // forward_host: x2 was copied on the side stream, and the first gather reads it
    CUDA_TRY(cudaStreamWaitEvent(st, h->x2_ready.get(), 0));
    h->wait_x2 = false;
  }
  const long long windows = (long long)n * tp.my * tp.mx;
  int batches = 0;
  for (long long first = 0; first < windows; first += tp.batch, ++batches) {
    const int count = (int)std::min<long long>(tp.batch, windows - first);
    const TileGeom g{n, H, W, s, tp.th, tp.tw, tile_halo(h), tp.my, tp.mx, first, count};
    const long long elems = (long long)count * tp.th * tp.tw * (1 + s * s);
    tile_gather_kernel<<<(int)std::min<long long>((elems + 255) / 256, (long long)h->sm_count * 8), 256, 0, st>>>(
        g, x, x2, h->tile_x.get(), h->tile_x2.get());
    CUDA_TRY(cudaGetLastError());
    h->launches++;
    if (mark(h, st)) return 1;
    if (forward_impl(h, h->tile_x.get(), h->tile_x2.get(), h->tile_y.get(), count, tp.th, tp.tw, st)) return 1;
    const long long hr_elems = (long long)count * tp.th * tp.tw * s * s;
    tile_stitch_kernel<<<(int)std::min<long long>((hr_elems + 255) / 256, (long long)h->sm_count * 8), 256, 0, st>>>(
        g, h->tile_y.get(), y);
    CUDA_TRY(cudaGetLastError());
    h->launches++;
    if (mark(h, st)) return 1;
  }
  h->tiled_last = true;
  h->tiled_batches = batches;
  return 0;
}

// Every inference forward: whole-image (forward_impl) unless option workspace_mb is set and the image's workspace
// would exceed it.
static int forward_any(dcscn_handle* h, const float* x, const float* x2, float* y, int n, int H, int W, cudaStream_t st) {
  h->eval_timed = false;
  if (h->workspace_mb <= 0) return forward_impl(h, x, x2, y, n, H, W, st);
  if (n <= 0 || H <= 0 || W <= 0) return fail("forward: bad shape n=%d h=%d w=%d", n, H, W);
  CUDA_TRY(cudaSetDevice(h->cfg.device_id));
  if (h->params_dirty && finalize_params(h)) return 1;
  const bool ds = uses_ds_tile(h);
  const size_t ws_px = workspace_shape(h).bytes_per_px(ds);
  const long long budget = h->workspace_mb << 20;
  const long long lr_total = (long long)n * H * W;
  if (lr_total <= budget / (long long)ws_px) return forward_impl(h, x, x2, y, n, H, W, st);
  const int s = h->cfg.scale;
  h->tile_vec4 = find_layer(h, "R-CNN1")->k == 3 && (((long long)s * W) & 3) == 0 &&
                 ((reinterpret_cast<uintptr_t>(x2) | reinterpret_cast<uintptr_t>(y)) & 15) == 0 &&
                 (!ds || lr_total * s * s < (1ll << 32));
  TilePlan tp;
  if (plan_tiles(h, n, H, W, ws_px + sizeof(float) * (1 + 2 * (size_t)s * s), &tp)) return 1;
  return forward_tiled(h, x, x2, y, n, H, W, tp, st);
}

// ------------------------------------------------------------------------- Pillow bicubic on the device ----
static double pil_bicubic_filter(double x) {   // Pillow Resample.c bicubic_filter, a = -0.5
  const double a = -0.5;
  if (x < 0.0) x = -x;
  if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
  if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
  return 0.0;
}

// Pillow's precompute_coeffs for one axis (helper/pil_resample.py is the Python statement of the same arithmetic).
static int pil_axis(dcscn_handle* h, int in_size, int out_size, PilAxis* ax) {
  for (const auto& t : h->pil_tables)
    if (t.in == in_size && t.out == out_size) {
      *ax = PilAxis{t.k.get(), t.bounds.get(), t.ksize};
      return 0;
    }
  double scale = (double)in_size / (double)out_size, filterscale = scale;
  if (filterscale < 1.0) filterscale = 1.0;
  const double support = 2.0 * filterscale;
  const int ksize = (int)std::ceil(support) * 2 + 1;
  std::vector<double> kk((size_t)out_size * ksize, 0.0);
  std::vector<int> bounds((size_t)out_size * 2, 0);
  const double ss = 1.0 / filterscale;
  for (int xx = 0; xx < out_size; ++xx) {
    const double center = (xx + 0.5) * scale;
    int xmin = (int)(center - support + 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = (int)(center + support + 0.5);
    if (xmax > in_size) xmax = in_size;
    xmax -= xmin;
    double* k = kk.data() + (size_t)xx * ksize;
    double ww = 0.0;
    for (int x = 0; x < xmax; ++x) {
      const double w = pil_bicubic_filter((x + xmin - center + 0.5) * ss);
      k[x] = w;
      ww += w;
    }
    for (int x = 0; x < xmax; ++x)
      if (ww != 0.0) k[x] /= ww;
    bounds[2 * xx] = xmin;
    bounds[2 * xx + 1] = xmax;
  }
  dcscn_handle::PilTable t;
  t.in = in_size; t.out = out_size; t.ksize = ksize;
  if (t.k.upload(kk) || t.bounds.upload(bounds)) return 1;
  *ax = PilAxis{t.k.get(), t.bounds.get(), t.ksize};
  if (h->pil_tables.size() >= 64) h->pil_tables.erase(h->pil_tables.begin());
  h->pil_tables.push_back(std::move(t));
  return 0;
}

// dst [n, OH, OW] = Pillow-bicubic resize of src [n, H, W] (both fp32 device tensors), horizontal pass first.
static int pil_resize_impl(dcscn_handle* h, const float* src, float* dst, int n, int H, int W, int OH, int OW, cudaStream_t st) {
  if (n <= 0 || H <= 0 || W <= 0 || OH <= 0 || OW <= 0) return fail("bicubic_resize: bad shape");
  PilAxis ax, ay;
  if (pil_axis(h, W, OW, &ax) || pil_axis(h, H, OH, &ay)) return 1;
  const size_t need = (size_t)n * H * OW;
  if (h->pil_tmp.grow(need)) return 1;
  const long long t1 = (long long)need, t2 = (long long)n * OH * OW;
  pil_resample_h_kernel<<<(int)std::min<long long>((t1 + 255) / 256, (long long)h->sm_count * 16), 256, 0, st>>>(
      src, h->pil_tmp.get(), (long long)n * H, W, OW, ax);
  pil_resample_v_kernel<<<(int)std::min<long long>((t2 + 255) / 256, (long long)h->sm_count * 16), 256, 0, st>>>(
      h->pil_tmp.get(), dst, n, H, OH, OW, ay);
  CUDA_TRY(cudaGetLastError());
  h->launches += 2;
  return 0;
}

#include "train_engine.inc"
#include "train_ds.inc"

// --------------------------------------------------------------------------------------- C ABI ----
extern "C" {

const char* dcscn_last_error(void) { return g_last_error.c_str(); }

int dcscn_create(const dcscn_config* cfg, dcscn_handle** out) {
  if (!cfg || !out) return fail("dcscn_create: null argument");
  if (cfg->struct_size != (int32_t)sizeof(dcscn_config))
    return fail("dcscn_create: dcscn_config size mismatch (got %d, expected %d)", cfg->struct_size, (int)sizeof(dcscn_config));
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return fail("dcscn_create: no CUDA device available (%s); this library has no CPU path", cudaGetErrorString(e));
  if (cfg->device_id < 0 || cfg->device_id >= ndev) return fail("dcscn_create: device %d out of range (%d devices)", cfg->device_id, ndev);
  CUDA_TRY(cudaSetDevice(cfg->device_id));
  cudaDeviceProp prop;
  CUDA_TRY(cudaGetDeviceProperties(&prop, cfg->device_id));
  if (prop.major != 9) return fail("dcscn_create: device %d is sm_%d%d; this library is built for sm_90a (H100) only", cfg->device_id, prop.major, prop.minor);

  std::unique_ptr<dcscn_handle> h(new dcscn_handle());
  h->cfg = *cfg;
  h->sm_count = prop.multiProcessorCount;
  if (build_graph(h.get())) return 1;

  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  CUDA_TRY(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
  if (qres != cudaDriverEntryPointSuccess || fn == nullptr) return fail("cuTensorMapEncodeTiled is not available in this driver");
  h->encode = (PFN_cuTensorMapEncodeTiled_v12000)fn;
  *out = h.release();
  return 0;
}

int dcscn_destroy(dcscn_handle* h) {
  if (!h) return 0;
  cudaSetDevice(h->cfg.device_id);
  cudaDeviceSynchronize();
  delete h;
  return 0;
}

int dcscn_num_params(dcscn_handle* h) { return h ? (int)h->params.size() : 0; }

int dcscn_param_info(dcscn_handle* h, int index, char* name_buf, int name_buf_len, int64_t* dims4, int* ndim) {
  if (!h || index < 0 || index >= (int)h->params.size()) return fail("dcscn_param_info: bad index %d", index);
  const ParamDef& p = h->params[index];
  if (name_buf && name_buf_len > 0) snprintf(name_buf, name_buf_len, "%s", p.name.c_str());
  if (ndim) *ndim = (int)p.shape.size();
  if (dims4)
    for (size_t i = 0; i < p.shape.size() && i < 4; ++i) dims4[i] = p.shape[i];
  return 0;
}

int dcscn_set_param(dcscn_handle* h, const char* name, const float* host_data, int64_t numel) {
  if (!h || !name || !host_data) return fail("dcscn_set_param: null argument");
  auto it = h->param_index.find(name);
  if (it == h->param_index.end()) return fail("dcscn_set_param: unknown variable '%s'", name);
  if (sync_host_params(h)) return 1;
  ParamDef& p = h->params[it->second];
  if (numel != p.numel()) return fail("dcscn_set_param: '%s' has %lld elements, got %lld", name, (long long)p.numel(), (long long)numel);
  memcpy(p.host.data(), host_data, (size_t)numel * sizeof(float));
  h->params_dirty = true;
  if (h->train) h->train->w_synced = false;
  return 0;
}

int dcscn_get_param(dcscn_handle* h, const char* name, float* host_data, int64_t numel) {
  if (!h || !name || !host_data) return fail("dcscn_get_param: null argument");
  auto it = h->param_index.find(name);
  if (it == h->param_index.end()) return fail("dcscn_get_param: unknown variable '%s'", name);
  if (sync_host_params(h)) return 1;
  const ParamDef& p = h->params[it->second];
  if (numel != p.numel()) return fail("dcscn_get_param: '%s' has %lld elements, got %lld", name, (long long)p.numel(), (long long)numel);
  memcpy(host_data, p.host.data(), (size_t)numel * sizeof(float));
  return 0;
}

int dcscn_forward(dcscn_handle* h, const float* x_dev, const float* x2_dev, float* y_dev, int n, int height, int width,
                  void* stream) {
  if (!h || !x_dev || !x2_dev || !y_dev) return fail("dcscn_forward: null argument");
  return forward_any(h, x_dev, x2_dev, y_dev, n, height, width, (cudaStream_t)stream);
}

int dcscn_bicubic_resize(dcscn_handle* h, const float* src_dev, float* dst_dev, int n, int height, int width, int out_height,
                         int out_width, void* stream) {
  if (!h || !src_dev || !dst_dev) return fail("dcscn_bicubic_resize: null argument");
  CUDA_TRY(cudaSetDevice(h->cfg.device_id));
  return pil_resize_impl(h, src_dev, dst_dev, n, height, width, out_height, out_width, (cudaStream_t)stream);
}

int dcscn_forward_host(dcscn_handle* h, const float* x, const float* x2, float* y, int n, int height, int width) {
  if (!h || !x || !y) return fail("dcscn_forward_host: null argument");
  CUDA_TRY(cudaSetDevice(h->cfg.device_id));
  const size_t lr = (size_t)n * height * width;
  const size_t hr = lr * h->cfg.scale * h->cfg.scale;
  if (h->io_x.grow(lr) || h->io_x2.grow(hr) || h->io_y.grow(hr)) return 1;
  cudaStream_t st = 0;
  if (!h->copy_stream) {
    cudaStream_t s;
    cudaEvent_t e;
    CUDA_TRY(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    h->copy_stream.reset(s);
    CUDA_TRY(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    h->x2_ready.reset(e);
  }
  // x feeds the first kernel; x2 (4x / 9x / 16x the bytes) is only read by the very last one, so it is copied on a second
  // stream while the conv stack runs and the last kernel waits for it
  CUDA_TRY(cudaMemcpyAsync(h->io_x.get(), x, lr * sizeof(float), cudaMemcpyHostToDevice, st));
  if (x2) {
    CUDA_TRY(cudaMemcpyAsync(h->io_x2.get(), x2, hr * sizeof(float), cudaMemcpyHostToDevice, h->copy_stream.get()));
    CUDA_TRY(cudaEventRecord(h->x2_ready.get(), h->copy_stream.get()));
    h->wait_x2 = true;
  } else {
    // x2 = Pillow-bicubic up-scale of x, formed in HBM (what util.resize_image_by_pil does on the host, bit for bit)
    const int s = h->cfg.scale;
    if (pil_resize_impl(h, h->io_x.get(), h->io_x2.get(), n, height, width, s * height, s * width, st)) return 1;
  }
  const int rc = forward_any(h, h->io_x.get(), h->io_x2.get(), h->io_y.get(), n, height, width, st);
  h->wait_x2 = false;
  if (rc) {
    cudaStreamSynchronize(h->copy_stream.get());
    return 1;
  }
  CUDA_TRY(cudaMemcpyAsync(y, h->io_y.get(), hr * sizeof(float), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  return 0;
}

// Self-ensemble entirely on the device (DCSCN.py:547-586 `do` with self_ensemble = flips): the transformed copies of x
// and x2 are produced by a kernel, transforms 0..3 run as ONE batched forward (n = up to 4, shape [h][w]) and 4..7 as
// another (shape [w][h]), and the inverse transforms + the float64 mean are one more kernel.
static int ensemble_impl(dcscn_handle* h, const float* x, const float* x2, double* y, int height, int width, int mask,
                         double divisor, cudaStream_t st) {
  if (mask <= 0 || mask > 255) return fail("forward_ensemble: transform mask must select 1..8 of the 8 transforms (got 0x%x)", mask);
  if (height <= 0 || width <= 0) return fail("forward_ensemble: bad shape h=%d w=%d", height, width);
  CUDA_TRY(cudaSetDevice(h->cfg.device_id));
  const int s = h->cfg.scale;
  const size_t lr = (size_t)height * width, hr = lr * s * s;
  if (h->ens_x.grow(4 * lr) || h->ens_x2.grow(4 * hr) || h->ens_y.grow(8 * hr)) return 1;
  const int grid_lr = (int)std::min<size_t>((4 * lr + 255) / 256, (size_t)h->sm_count * 8);
  const int grid_hr = (int)std::min<size_t>((4 * hr + 255) / 256, (size_t)h->sm_count * 8);
  for (int grp = 0; grp < 2; ++grp) {
    EnsembleSel sel;
    memset(&sel, 0, sizeof(sel));
    for (int t = 4 * grp; t < 4 * grp + 4; ++t)
      if ((mask >> t) & 1) sel.t[sel.count++] = t;
    if (sel.count == 0) continue;
    ensemble_flip_kernel<<<grid_lr, 256, 0, st>>>(x, h->ens_x.get(), height, width, sel);
    ensemble_flip_kernel<<<grid_hr, 256, 0, st>>>(x2, h->ens_x2.get(), s * height, s * width, sel);
    CUDA_TRY(cudaGetLastError());
    h->launches += 2;
    const int fh = grp == 0 ? height : width, fw = grp == 0 ? width : height;
    if (forward_any(h, h->ens_x.get(), h->ens_x2.get(), h->ens_y.get() + (size_t)grp * 4 * hr, sel.count, fh, fw, st)) return 1;
  }
  ensemble_reduce_kernel<<<(int)std::min<size_t>((hr + 255) / 256, (size_t)h->sm_count * 8), 256, 0, st>>>(
      h->ens_y.get(), h->ens_y.get() + 4 * hr, y, s * height, s * width, mask, divisor);
  CUDA_TRY(cudaGetLastError());
  h->launches++;
  return 0;
}

int dcscn_forward_ensemble(dcscn_handle* h, const float* x_dev, const float* x2_dev, double* y_dev, int height, int width,
                           int flips, void* stream) {
  if (!h || !x_dev || !x2_dev || !y_dev) return fail("dcscn_forward_ensemble: null argument");
  if (flips < 1 || flips > 8) return fail("forward_ensemble: flips must be 1..8 (got %d)", flips);
  return ensemble_impl(h, x_dev, x2_dev, y_dev, height, width, (1 << flips) - 1, (double)flips, (cudaStream_t)stream);
}

int dcscn_forward_ensemble_partial(dcscn_handle* h, const float* x_dev, const float* x2_dev, double* y_dev, int height,
                                   int width, int transform_mask, void* stream) {
  if (!h || !x_dev || !x2_dev || !y_dev) return fail("dcscn_forward_ensemble_partial: null argument");
  return ensemble_impl(h, x_dev, x2_dev, y_dev, height, width, transform_mask, 1.0, (cudaStream_t)stream);
}

int dcscn_forward_ensemble_host(dcscn_handle* h, const float* x, const float* x2, double* y, int height, int width, int flips) {
  if (!h || !x || !y) return fail("dcscn_forward_ensemble_host: null argument");
  CUDA_TRY(cudaSetDevice(h->cfg.device_id));
  const size_t lr = (size_t)height * width;
  const size_t hr = lr * h->cfg.scale * h->cfg.scale;
  if (h->ensio_x.grow(lr) || h->ensio_x2.grow(hr) || h->ensio_y.grow(hr)) return 1;
  cudaStream_t st = 0;
  CUDA_TRY(cudaMemcpyAsync(h->ensio_x.get(), x, lr * sizeof(float), cudaMemcpyHostToDevice, st));
  if (x2) {
    CUDA_TRY(cudaMemcpyAsync(h->ensio_x2.get(), x2, hr * sizeof(float), cudaMemcpyHostToDevice, st));
  } else if (pil_resize_impl(h, h->ensio_x.get(), h->ensio_x2.get(), 1, height, width, h->cfg.scale * height, h->cfg.scale * width, st)) {
    return 1;
  }
  if (flips < 1 || flips > 8) return fail("forward_ensemble: flips must be 1..8 (got %d)", flips);
  if (ensemble_impl(h, h->ensio_x.get(), h->ensio_x2.get(), h->ensio_y.get(), height, width, (1 << flips) - 1, (double)flips, st)) return 1;
  CUDA_TRY(cudaMemcpyAsync(y, h->ensio_y.get(), hr * sizeof(double), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  return 0;
}

int dcscn_get_activation(dcscn_handle* h, const char* tensor, float* host_data, int64_t numel) {
  if (!h || !tensor || !host_data) return fail("dcscn_get_activation: null argument");
  if (h->tiled_last)
    return fail("dcscn_get_activation: the last forward ran tiled (option workspace_mb): the buffers hold its last batch "
                "of windows, not the image");
  const bool ds = uses_ds_tile(h);
  const Plan* pl = h->last_plan;
  if (ds ? h->ds_n == 0 : !pl) return fail("dcscn_get_activation: no forward has run yet");
  CUDA_TRY(cudaSetDevice(h->cfg.device_id));
  CUDA_TRY(cudaDeviceSynchronize());
  const std::string t(tensor);
  const size_t lr_px = ds ? (size_t)h->ds_n * h->ds_h * h->ds_w : (size_t)pl->n * pl->h * pl->w;
  if (!ds && pl->ran_fused && t == "R-CNN1/taps") {   // the fused R-CNN1's tap-planar products [parts][9][N][sH][sW]
    const size_t count = lr_px * h->cfg.scale * h->cfg.scale * 9 * pl->gather.parts;
    if (numel != (int64_t)count) return fail("dcscn_get_activation: '%s' has %lld elements, got %lld", tensor, (long long)count, (long long)numel);
    CUDA_TRY(cudaMemcpy(host_data, h->vbuf.get(), count * sizeof(float), cudaMemcpyDeviceToHost));
    return 0;
  }
  ActView v;
  if (!act_view(h, t, &v)) return fail("dcscn_get_activation: no tensor '%s'", tensor);
  if (!ds && pl->ran_fused && v.buf == BUF_HR)
    return fail("dcscn_get_activation: '%s' is not materialised when the R-CNN1 fusion is on (set option fuse_last=0)", tensor);
  const size_t px = lr_px * v.px_mul;
  if (numel != (int64_t)(px * v.ch)) return fail("dcscn_get_activation: '%s' has %lld elements, got %lld", tensor, (long long)(px * v.ch), (long long)numel);
  const float* src = v.f32;
  DeviceArray<float> tmp;
  if (!src) {   // fp16 planes: hi + lo in fp32, from the tensor's first channel on
    const size_t count = px * v.pitch - v.off;
    if (tmp.alloc(count)) return 1;
    planes_to_f32_kernel<<<1024, 256>>>(v.planes.hi, v.planes.lo, tmp.get(), count);
    src = tmp.get();
  }
  const size_t row = v.ch * sizeof(float);
  CUDA_TRY(cudaMemcpy2D(host_data, row, src, v.pitch * sizeof(float), row, px, cudaMemcpyDeviceToHost));
  return 0;
}

int dcscn_set_option(dcscn_handle* h, const char* key, int64_t value) {
  if (!h || !key) return fail("dcscn_set_option: null argument");
  const std::string k(key);
  h->graph_epoch++;          // whatever changes, captured launch sequences are rebuilt
  if (k == "graph") {
    h->use_graph = value ? 1 : 0;
    return 0;
  }
  if (k == "conv_impl") {
    if (value != 0 && value != 1) return fail("conv_impl must be 0 (wgmma) or 1 (CUDA-core validation)");
    h->conv_impl = (int)value;
  } else if (k == "fuse_last") {
    h->fuse_last = value ? 1 : 0;
  } else if (k == "timing") {
    h->timing = value ? 1 : 0;
  } else if (k == "wgrad_impl") {
    if (value != 0 && value != 1) return fail("wgrad_impl must be 0 (tensor cores) or 1 (CUDA cores)");
    h->wgrad_impl = (int)value;
  } else if (k == "l1_loss") {
    h->l1_loss = value ? 1 : 0;
  } else if (k == "act_grad_impl") {
    if (value < 0 || value > 1) return fail("act_grad_impl must be 0 or 1");
    h->act_grad_impl = (int)value;
  } else if (k == "grad_capture") {
    if (value < 0 || value > 1) return fail("grad_capture must be 0 or 1");
    h->grad_capture = (int)value;
  } else if (k == "workspace_mb") {
    if (value < 0 || value > (int64_t(1) << 40)) return fail("workspace_mb must be >= 0 MiB (0 = no limit), got %lld", (long long)value);
    h->workspace_mb = value;
  } else if (k == "seg_chunks") {
    if (value < 0 || value > 4096) return fail("seg_chunks must be >= 0 (0 = automatic)");
    h->seg_chunks = (int)value;
    h->params_dirty = true;     // the streaming kernel's stage tables carry the segment boundaries
    h->plans.clear();
    h->last_plan = nullptr;
  } else {
    return fail("dcscn_set_option: unknown option '%s'", key);
  }
  return 0;
}

int dcscn_get_timings(dcscn_handle* h, float* ms, int capacity, int* count, char* names, int names_len) {
  if (!h || !count) return fail("dcscn_get_timings: null argument");
  *count = 0;
  if (h->eval_timed) {   // the last timed call was dcscn_evaluate_image: its steps, the forward or ensemble as one
    if (h->eval_marks < 2) return 0;
    CUDA_TRY(cudaEventSynchronize(h->eval_ev[h->eval_marks - 1].get()));
    const int n = h->eval_marks - 1;
    for (int i = 0; i < n && i < capacity; ++i) CUDA_TRY(cudaEventElapsedTime(&ms[i], h->eval_ev[i].get(), h->eval_ev[i + 1].get()));
    *count = n;
    if (names && names_len > 0) snprintf(names, names_len, "%s", h->eval_names.c_str());
    return 0;
  }
  if (h->ev_used < 2) return 0;
  CUDA_TRY(cudaEventSynchronize(h->ev[h->ev_used - 1].get()));
  const int n = h->ev_used - 1;
  for (int i = 0; i < n && i < capacity; ++i) CUDA_TRY(cudaEventElapsedTime(&ms[i], h->ev[i].get(), h->ev[i + 1].get()));
  *count = n;
  if (names && names_len > 0) {
    std::string s = "CNN1";
    if (uses_ds_tile(h)) {
      s = "";
      for (const LayerDef& l : h->layers) {
        std::string nm = l.scope.substr(0, l.scope.find('/'));
        if (nm == "B1") continue;          // A1 | B1 run as one launch
        if (nm == "A1") nm = "A1+B1";
        s += (s.empty() ? "" : ",") + nm;
      }
    } else {
      for (const TcLayer& t : h->tcl) s += (t.dw_ksz ? ",dw:" + t.name : "") + "," + t.name;
      s += ",R-CNN1";
    }
    if (h->tiled_last) {   // every batch of windows: gather, the layers, stitch
      const std::string layers = s;
      s = "";
      for (int b = 0; b < h->tiled_batches; ++b) s += (b ? "," : "") + std::string("tile_gather,") + layers + ",tile_stitch";
    }
    snprintf(names, names_len, "%s", s.c_str());
  }
  return 0;
}

int dcscn_train_step(dcscn_handle* h, const float* x_dev, const float* x2_dev, const float* y_dev, int n, int height, int width,
                     float lr, uint32_t seed, int apply_update, float* out_loss, float* out_mse, void* stream) {
  if (!h || !x_dev || !x2_dev || !y_dev) return fail("dcscn_train_step: null argument");
  return train_step_impl(h, x_dev, x2_dev, y_dev, n, height, width, lr, seed, apply_update, out_loss, out_mse, (cudaStream_t)stream);
}

int dcscn_train_step_host(dcscn_handle* h, const float* x, const float* x2, const float* y, int n, int height, int width, float lr,
                          uint32_t seed, int apply_update, float* out_loss, float* out_mse) {
  if (!h || !x || !x2 || !y) return fail("dcscn_train_step_host: null argument");
  CUDA_TRY(cudaSetDevice(h->cfg.device_id));
  const size_t lr_px = (size_t)n * height * width;
  const size_t hr_px = lr_px * h->cfg.scale * h->cfg.scale;
  if (h->io_x.grow(lr_px) || h->io_x2.grow(hr_px) || h->io_y.grow(hr_px)) return 1;
  cudaStream_t st = 0;
  CUDA_TRY(cudaMemcpyAsync(h->io_x.get(), x, lr_px * sizeof(float), cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(h->io_x2.get(), x2, hr_px * sizeof(float), cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(h->io_y.get(), y, hr_px * sizeof(float), cudaMemcpyHostToDevice, st));
  return train_step_impl(h, h->io_x.get(), h->io_x2.get(), h->io_y.get(), n, height, width, lr, seed, apply_update, out_loss, out_mse, st);
}

int dcscn_patch_store_set(dcscn_handle* h, const uint8_t* lr, const uint8_t* bicubic, const uint8_t* truth, int64_t count,
                          int patch_height, int patch_width) {
  if (!h || !lr || !bicubic || !truth) return fail("dcscn_patch_store_set: null argument");
  if (count <= 0 || count > 0x7FFFFFFF || patch_height <= 0 || patch_width <= 0) return fail("dcscn_patch_store_set: bad size");
  CUDA_TRY(cudaSetDevice(h->cfg.device_id));
  h->ps_count = 0;
  const size_t s2 = (size_t)h->cfg.scale * h->cfg.scale;
  const size_t lr_b = (size_t)count * patch_height * patch_width, hr_b = lr_b * s2;
  if (h->ps_lr.alloc(lr_b) || h->ps_bic.alloc(hr_b) || h->ps_true.alloc(hr_b)) return 1;
  CUDA_TRY(cudaMemcpy(h->ps_lr.get(), lr, lr_b, cudaMemcpyHostToDevice));
  CUDA_TRY(cudaMemcpy(h->ps_bic.get(), bicubic, hr_b, cudaMemcpyHostToDevice));
  CUDA_TRY(cudaMemcpy(h->ps_true.get(), truth, hr_b, cudaMemcpyHostToDevice));
  h->ps_count = count;
  h->ps_h = patch_height;
  h->ps_w = patch_width;
  return 0;
}

// Gathers the indexed patches into the fp32 staging tensors io_x / io_x2 / io_y (shared with the host-buffer calls).
static int patch_gather(dcscn_handle* h, const int32_t* indices, int n, float max_value, cudaStream_t st) {
  if (h->ps_count == 0) return fail("train_step_indexed: no patch store (call dcscn_patch_store_set first)");
  if (n <= 0) return fail("train_step_indexed: empty mini-batch");
  for (int i = 0; i < n; ++i) {
    const int64_t k = indices[i] & 0x7FFFFFFF;
    if (k >= h->ps_count) return fail("train_step_indexed: patch index %lld out of range (%lld patches)", (long long)k, (long long)h->ps_count);
  }
  const int s = h->cfg.scale;
  const size_t lr_px = (size_t)n * h->ps_h * h->ps_w, hr_px = lr_px * s * s;
  if (h->io_x.grow(lr_px) || h->io_x2.grow(hr_px) || h->io_y.grow(hr_px) || h->ps_idx.grow(n)) return 1;
  CUDA_TRY(cudaMemcpyAsync(h->ps_idx.get(), indices, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, st));
  const double scale = (double)max_value / 255.0;
  const int grid_lr = (int)std::min<size_t>((lr_px + 255) / 256, (size_t)h->sm_count * 8);
  const int grid_hr = (int)std::min<size_t>((hr_px + 255) / 256, (size_t)h->sm_count * 8);
  patch_gather_kernel<<<grid_lr, 256, 0, st>>>(h->ps_lr.get(), h->ps_idx.get(), h->io_x.get(), n, h->ps_h, h->ps_w, scale);
  patch_gather_kernel<<<grid_hr, 256, 0, st>>>(h->ps_bic.get(), h->ps_idx.get(), h->io_x2.get(), n, s * h->ps_h, s * h->ps_w, scale);
  patch_gather_kernel<<<grid_hr, 256, 0, st>>>(h->ps_true.get(), h->ps_idx.get(), h->io_y.get(), n, s * h->ps_h, s * h->ps_w, scale);
  CUDA_TRY(cudaGetLastError());
  h->launches += 3;
  return 0;
}

int dcscn_train_step_indexed(dcscn_handle* h, const int32_t* indices, int n, float max_value, float lr, uint32_t seed,
                             int apply_update, float* out_loss, float* out_mse) {
  if (!h || !indices) return fail("dcscn_train_step_indexed: null argument");
  CUDA_TRY(cudaSetDevice(h->cfg.device_id));
  cudaStream_t st = 0;
  if (patch_gather(h, indices, n, max_value, st)) return 1;
  return train_step_impl(h, h->io_x.get(), h->io_x2.get(), h->io_y.get(), n, h->ps_h, h->ps_w, lr, seed, apply_update, out_loss, out_mse, st);
}

int dcscn_patch_gather(dcscn_handle* h, const int32_t* indices, int n, float max_value, float* x, float* x2, float* y) {
  if (!h || !indices || !x || !x2 || !y) return fail("dcscn_patch_gather: null argument");
  CUDA_TRY(cudaSetDevice(h->cfg.device_id));
  cudaStream_t st = 0;
  if (patch_gather(h, indices, n, max_value, st)) return 1;
  const int s = h->cfg.scale;
  const size_t lr_px = (size_t)n * h->ps_h * h->ps_w, hr_px = lr_px * s * s;
  CUDA_TRY(cudaMemcpyAsync(x, h->io_x.get(), lr_px * sizeof(float), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaMemcpyAsync(x2, h->io_x2.get(), hr_px * sizeof(float), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaMemcpyAsync(y, h->io_y.get(), hr_px * sizeof(float), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  return 0;
}

int dcscn_image_store_set(dcscn_handle* h, const uint8_t* pixels, int64_t bytes, const int64_t* offsets, const int32_t* heights,
                          const int32_t* widths, const int32_t* channels, int count) {
  if (!h || !pixels || !offsets || !heights || !widths || !channels) return fail("dcscn_image_store_set: null argument");
  if (count <= 0 || bytes <= 0) return fail("dcscn_image_store_set: empty store");
  std::vector<ImageEntry> table((size_t)count);
  for (int i = 0; i < count; ++i) {
    if (heights[i] <= 0 || widths[i] <= 0 || (channels[i] != 1 && channels[i] != 3))
      return fail("dcscn_image_store_set: image %d is %d x %d x %d (1 or 3 channels expected)", i, heights[i], widths[i], channels[i]);
    const int64_t size = (int64_t)heights[i] * widths[i] * channels[i];
    if (offsets[i] < 0 || offsets[i] > bytes - size)
      return fail("dcscn_image_store_set: image %d (%lld bytes at offset %lld) lies outside the %lld-byte store", i,
                  (long long)size, (long long)offsets[i], (long long)bytes);
    table[i] = ImageEntry{(long long)offsets[i], heights[i], widths[i], channels[i]};
  }
  CUDA_TRY(cudaSetDevice(h->cfg.device_id));
  h->is_host.clear();
  if (h->is_pixels.alloc((size_t)bytes) || h->is_table.upload(table)) return 1;
  CUDA_TRY(cudaMemcpy(h->is_pixels.get(), pixels, (size_t)bytes, cudaMemcpyHostToDevice));
  h->is_host = std::move(table);
  return 0;
}

// Builds the fp32 mini-batch tensors of the crops into io_x / io_x2 / io_y (shared with the host-buffer calls): crop
// gather, the mode-'F' group through pil_resize_impl (e -> p -> e), the mode-'L' group through the 8-bit resampler, place.
static int crop_gather(dcscn_handle* h, const int32_t* crops, int n, int patch_size, float max_value, cudaStream_t st) {
  if (h->is_host.empty()) return fail("train_step_crops: no image store (call dcscn_image_store_set first)");
  if (n <= 0) return fail("train_step_crops: empty mini-batch");
  const int s = h->cfg.scale;
  if (patch_size <= 0 || patch_size > 4096) return fail("train_step_crops: bad patch size %d", patch_size);
  const int e = s * patch_size;
  // util.resize_image_by_pil(truth, 1 / scale) makes int(e * (1 / scale)) pixels
  if ((int)(e * (1.0 / s)) != patch_size) return fail("train_step_crops: a %d-pixel crop does not shrink to %d at scale %d", e, patch_size, s);
  std::vector<CropJob> jobs((size_t)n);
  int n8 = 0;
  for (int i = 0; i < n; ++i) {
    const int32_t* c = crops + 4 * (size_t)i;
    if (c[0] < 0 || c[0] >= (int)h->is_host.size())
      return fail("train_step_crops: crop %d names image %d (%d images)", i, c[0], (int)h->is_host.size());
    const ImageEntry& im = h->is_host[c[0]];
    if (c[1] < 0 || c[1] > im.height - e || c[2] < 0 || c[2] > im.width - e)
      return fail("train_step_crops: crop %d at (%d, %d) of %d x %d does not fit image %d (%d x %d)", i, c[1], c[2], e, e, c[0],
                  im.height, im.width);
    if (c[3] != 0 && c[3] != 1) return fail("train_step_crops: crop %d has mirror %d (0 or 1)", i, c[3]);
    jobs[i] = CropJob{c[0], c[1], c[2], c[3], im.channels == 1, 0};
    n8 += im.channels == 1;
  }
  const int nf = n - n8;
  for (int i = 0, kf = 0, k8 = 0; i < n; ++i) jobs[i].slot = jobs[i].mode8 ? k8++ : kf++;
  const size_t hr = (size_t)e * e, lr = (size_t)patch_size * patch_size, mid = (size_t)e * patch_size;
  // crop_f: input, down-scaled, up-scaled of the mode-'F' group; crop_u8: input, h-pass, down-scaled, h-pass, up-scaled
  if (h->io_x.grow(lr * n) || h->io_x2.grow(hr * n) || h->io_y.grow(hr * n) || h->crop_jobs.grow(n) ||
      h->crop_f.grow((2 * hr + lr) * nf) || h->crop_u8.grow((2 * hr + 2 * mid + lr) * n8))
    return 1;
  CUDA_TRY(cudaMemcpyAsync(h->crop_jobs.get(), jobs.data(), (size_t)n * sizeof(CropJob), cudaMemcpyHostToDevice, st));
  const double scale = (double)max_value / 255.0;
  float* f_in = h->crop_f.get();
  float* f_small = f_in + hr * nf;
  float* f_big = f_small + lr * nf;
  uint8_t* l_in = h->crop_u8.get();
  uint8_t* l_tmp1 = l_in + hr * n8;
  uint8_t* l_small = l_tmp1 + mid * n8;
  uint8_t* l_tmp2 = l_small + lr * n8;
  uint8_t* l_big = l_tmp2 + mid * n8;
  auto grid = [&](size_t total) { return (int)std::min<size_t>((total + 255) / 256, (size_t)h->sm_count * 16); };
  crop_gather_kernel<<<grid(hr * n), 256, 0, st>>>(h->is_pixels.get(), h->is_table.get(), h->crop_jobs.get(), n, e, scale,
                                                   h->io_y.get(), f_in, l_in);
  CUDA_TRY(cudaGetLastError());
  h->launches += 1;
  if (nf > 0 && (pil_resize_impl(h, f_in, f_small, nf, e, e, patch_size, patch_size, st) ||
                 pil_resize_impl(h, f_small, f_big, nf, patch_size, patch_size, e, e, st)))
    return 1;
  if (n8 > 0) {
    PilAxis down, up;
    if (pil_axis(h, e, patch_size, &down) || pil_axis(h, patch_size, e, &up)) return 1;
    pil_resample8_h_kernel<<<grid(mid * n8), 256, 0, st>>>(l_in, l_tmp1, (long long)n8 * e, e, patch_size, down);
    pil_resample8_v_kernel<<<grid(lr * n8), 256, 0, st>>>(l_tmp1, l_small, n8, e, patch_size, patch_size, down);
    pil_resample8_h_kernel<<<grid(mid * n8), 256, 0, st>>>(l_small, l_tmp2, (long long)n8 * patch_size, patch_size, e, up);
    pil_resample8_v_kernel<<<grid(hr * n8), 256, 0, st>>>(l_tmp2, l_big, n8, patch_size, e, e, up);
    CUDA_TRY(cudaGetLastError());
    h->launches += 4;
  }
  crop_place_kernel<<<grid(lr * n), 256, 0, st>>>(h->crop_jobs.get(), f_small, l_small, h->io_x.get(), n, patch_size, patch_size, scale);
  crop_place_kernel<<<grid(hr * n), 256, 0, st>>>(h->crop_jobs.get(), f_big, l_big, h->io_x2.get(), n, e, e, scale);
  CUDA_TRY(cudaGetLastError());
  h->launches += 2;
  return 0;
}

int dcscn_train_step_crops(dcscn_handle* h, const int32_t* crops, int n, int patch_size, float max_value, float lr, uint32_t seed,
                           int apply_update, float* out_loss, float* out_mse) {
  if (!h || !crops) return fail("dcscn_train_step_crops: null argument");
  CUDA_TRY(cudaSetDevice(h->cfg.device_id));
  cudaStream_t st = 0;
  if (crop_gather(h, crops, n, patch_size, max_value, st)) return 1;
  return train_step_impl(h, h->io_x.get(), h->io_x2.get(), h->io_y.get(), n, patch_size, patch_size, lr, seed, apply_update,
                         out_loss, out_mse, st);
}

int dcscn_crop_gather(dcscn_handle* h, const int32_t* crops, int n, int patch_size, float max_value, float* x, float* x2, float* y) {
  if (!h || !crops || !x || !x2 || !y) return fail("dcscn_crop_gather: null argument");
  CUDA_TRY(cudaSetDevice(h->cfg.device_id));
  cudaStream_t st = 0;
  if (crop_gather(h, crops, n, patch_size, max_value, st)) return 1;
  const size_t lr_px = (size_t)n * patch_size * patch_size, hr_px = lr_px * h->cfg.scale * h->cfg.scale;
  CUDA_TRY(cudaMemcpyAsync(x, h->io_x.get(), lr_px * sizeof(float), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaMemcpyAsync(x2, h->io_x2.get(), hr_px * sizeof(float), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaMemcpyAsync(y, h->io_y.get(), hr_px * sizeof(float), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  return 0;
}

// ------------------------------------------------------------------------------------------ evaluation ----
// What DCSCN._evaluation_set -> do(lr, bicubic) -> util.compute_psnr_and_ssim compute for one test image (DCSCN.py:672-703,
// :705-725), on the device.  The store holds the decoded test images (util.load_image), one upload per test set.
int dcscn_eval_store_set(dcscn_handle* h, const uint8_t* pixels, int64_t bytes, const int64_t* offsets, const int32_t* heights,
                         const int32_t* widths, const int32_t* channels, int count) {
  if (!h || !pixels || !offsets || !heights || !widths || !channels) return fail("dcscn_eval_store_set: null argument");
  if (count <= 0 || bytes <= 0) return fail("dcscn_eval_store_set: empty store");
  std::vector<ImageEntry> table((size_t)count);
  for (int i = 0; i < count; ++i) {
    if (heights[i] <= 0 || widths[i] <= 0 || (channels[i] != 1 && channels[i] != 3))
      return fail("dcscn_eval_store_set: image %d is %d x %d x %d (1 or 3 channels expected)", i, heights[i], widths[i], channels[i]);
    const int64_t size = (int64_t)heights[i] * widths[i] * channels[i];
    if (offsets[i] < 0 || offsets[i] > bytes - size)
      return fail("dcscn_eval_store_set: image %d (%lld bytes at offset %lld) lies outside the %lld-byte store", i,
                  (long long)size, (long long)offsets[i], (long long)bytes);
    table[i] = ImageEntry{(long long)offsets[i], heights[i], widths[i], channels[i]};
  }
  CUDA_TRY(cudaSetDevice(h->cfg.device_id));
  h->ev_host.clear();
  if (h->ev_pixels.alloc((size_t)bytes)) return 1;
  CUDA_TRY(cudaMemcpy(h->ev_pixels.get(), pixels, (size_t)bytes, cudaMemcpyHostToDevice));
  h->ev_host = std::move(table);
  return 0;
}

static int eval_mark(dcscn_handle* h, const char* name, cudaStream_t st) {
  if (!h->timing) return 0;
  if (h->eval_marks >= (int)h->eval_ev.size()) {
    cudaEvent_t e;
    CUDA_TRY(cudaEventCreate(&e));
    h->eval_ev.emplace_back(e);
  }
  CUDA_TRY(cudaEventRecord(h->eval_ev[h->eval_marks++].get(), st));
  if (name) h->eval_names += (h->eval_names.empty() ? "" : ",") + std::string(name);
  return 0;
}

static int evaluate_impl(dcscn_handle* h, const EvalImage& im, int lh, int lw, int flips, double max_value, int border,
                         const double* ssim_params, uint64_t* sse, int64_t* pixels, int64_t* nan_pixels, double* ssim_map,
                         int64_t map_capacity) {
  const int s = h->cfg.scale;
  const int ah = im.height / s * s, aw = im.width / s * s;   // util.set_image_alignment
  if (ah <= 0 || aw <= 0) return fail("evaluate_image: a %d x %d image is smaller than the scale %d", im.height, im.width, s);
  if ((long long)lh * s != ah || (long long)lw * s != aw)
    return fail("evaluate_image: an LR image of %d x %d does not up-scale to the aligned %d x %d at scale %d", lh, lw, ah, aw, s);
  if (flips < 0 || flips > 8) return fail("evaluate_image: flips must be 0 (bicubic) or 1..8 (got %d)", flips);
  if (!(max_value > 0.0)) return fail("evaluate_image: max_value must be positive (got %g)", max_value);
  const int b = border > 0 ? border : 0;                   // the host shaves only a positive border
  const int hs = std::max(ah - 2 * b, 0), ws = std::max(aw - 2 * b, 0);
  const int64_t map_n = hs >= 11 ? (int64_t)(hs - 10) * ws : 0;
  if (map_n > 0 && (!ssim_map || !ssim_params || map_capacity < map_n))
    return fail("evaluate_image: the SSIM map needs %lld doubles and the filter weights (capacity %lld)", (long long)map_n,
                (long long)map_capacity);
  CUDA_TRY(cudaSetDevice(h->cfg.device_id));
  const size_t hr = (size_t)ah * aw, lr = (size_t)lh * lw;
  // fp32 planes: truth, mode-'F' input, down-scaled, up-scaled, x, x2, forward output, trimmed output (16-byte aligned)
  auto up = [](size_t n) { return (n + 63) & ~(size_t)63; };
  const size_t fsz[8] = {hr, hr, lr, hr, lr, hr, hr, hr};
  size_t foff[8], ftotal = 0;
  for (int i = 0; i < 8; ++i) { foff[i] = ftotal; ftotal += up(fsz[i]); }
  // uint8 planes: mode-'L' input, horizontal pass down, down-scaled, horizontal pass up, up-scaled
  const size_t usz[5] = {hr, (size_t)ah * lw, lr, (size_t)lh * aw, hr};
  size_t uoff[5], utotal = 0;
  for (int i = 0; i < 5; ++i) { uoff[i] = utotal; utotal += up(usz[i]); }
  const bool rgb = im.channels == 3;
  if (h->ev_f.grow(ftotal) || (!rgb && h->ev_u8.grow(utotal)) || (flips > 1 && h->ev_y64.grow(hr)) ||
      (map_n > 0 && h->ev_map.grow((size_t)map_n)) || h->ev_acc.grow(2))
    return 1;
  float* F = h->ev_f.get();
  float *truth = F + foff[0], *f_in = F + foff[1], *f_small = F + foff[2], *f_big = F + foff[3];
  float *x = F + foff[4], *x2 = F + foff[5], *y32 = F + foff[6], *out = F + foff[7];
  uint8_t* U = h->ev_u8.get();
  uint8_t *l_in = rgb ? nullptr : U + uoff[0], *l_t1 = rgb ? nullptr : U + uoff[1], *l_small = rgb ? nullptr : U + uoff[2];
  uint8_t *l_t2 = rgb ? nullptr : U + uoff[3], *l_big = rgb ? nullptr : U + uoff[4];
  auto grid = [&](size_t total) { return (int)std::min<size_t>((total + 255) / 256, (size_t)h->sm_count * 16); };
  cudaStream_t st = 0;
  h->eval_marks = 0;
  h->eval_names.clear();
  if (eval_mark(h, nullptr, st)) return 1;

  // 1. aligned crop, Y and the truth
  eval_prepare_kernel<<<grid(hr), 256, 0, st>>>(im, ah, aw, truth, f_in, l_in);
  CUDA_TRY(cudaGetLastError());
  h->launches++;
  if (eval_mark(h, "eval_prepare", st)) return 1;
  // 2. LR = Pillow bicubic down by 1 / scale, bicubic = the LR up by scale (mode 'F' for Y, the 8-bit path for 'L')
  if (rgb) {
    if (pil_resize_impl(h, f_in, f_small, 1, ah, aw, lh, lw, st) || pil_resize_impl(h, f_small, f_big, 1, lh, lw, ah, aw, st)) return 1;
  } else {
    PilAxis dx, dy, ux, uy;
    if (pil_axis(h, aw, lw, &dx) || pil_axis(h, ah, lh, &dy) || pil_axis(h, lw, aw, &ux) || pil_axis(h, lh, ah, &uy)) return 1;
    pil_resample8_h_kernel<<<grid(usz[1]), 256, 0, st>>>(l_in, l_t1, ah, aw, lw, dx);
    pil_resample8_v_kernel<<<grid(lr), 256, 0, st>>>(l_t1, l_small, 1, ah, lh, lw, dy);
    pil_resample8_h_kernel<<<grid(usz[3]), 256, 0, st>>>(l_small, l_t2, lh, lw, aw, ux);
    pil_resample8_v_kernel<<<grid(hr), 256, 0, st>>>(l_t2, l_big, 1, lh, ah, aw, uy);
    CUDA_TRY(cudaGetLastError());
    h->launches += 4;
  }
  if (eval_mark(h, "eval_resize", st)) return 1;
  // 3.-4. forward or self-ensemble, then trim_image_as_file of its output (the bicubic baseline trims the up-scale)
  if (flips > 0) {
    const double scale = max_value / 255.0;
    eval_place_kernel<<<grid(lr), 256, 0, st>>>(f_small, l_small, x, (long long)lr, scale);
    eval_place_kernel<<<grid(hr), 256, 0, st>>>(f_big, l_big, x2, (long long)hr, scale);
    CUDA_TRY(cudaGetLastError());
    h->launches += 2;
    if (eval_mark(h, "eval_place", st)) return 1;
    if (flips == 1) {
      if (forward_any(h, x, x2, y32, 1, lh, lw, st)) return 1;
    } else if (ensemble_impl(h, x, x2, h->ev_y64.get(), lh, lw, (1 << flips) - 1, (double)flips, st)) {
      return 1;
    }
    if (eval_mark(h, flips == 1 ? "forward" : "ensemble", st)) return 1;
    const double back = 255.0 / max_value;
    eval_trim_kernel<<<grid(hr), 256, 0, st>>>(flips > 1 ? h->ev_y64.get() : nullptr, flips == 1 ? y32 : nullptr, nullptr, out,
                                               (long long)hr, back);
  } else {
    eval_trim_kernel<<<grid(hr), 256, 0, st>>>(nullptr, rgb ? f_big : nullptr, l_big, out, (long long)hr, 1.0);
  }
  CUDA_TRY(cudaGetLastError());
  h->launches++;
  if (eval_mark(h, "eval_trim", st)) return 1;
  // 5. the metric on the region left after shaving the border
  CUDA_TRY(cudaMemsetAsync(h->ev_acc.get(), 0, 2 * sizeof(unsigned long long), st));
  if ((size_t)hs * ws > 0) {
    eval_sse_kernel<<<grid((size_t)hs * ws), 256, 0, st>>>(truth, out, aw, b, hs, ws, h->ev_acc.get());
    CUDA_TRY(cudaGetLastError());
    h->launches++;
    if (eval_mark(h, "eval_sse", st)) return 1;
  }
  if (map_n > 0) {
    EvalSsim p;
    for (int i = 0; i < 6; ++i) p.w[i] = ssim_params[i];
    p.c1 = ssim_params[6];
    p.c2 = ssim_params[7];
    eval_ssim_kernel<<<grid((size_t)map_n), 256, 0, st>>>(truth, out, aw, b, hs, ws, p, h->ev_map.get());
    CUDA_TRY(cudaGetLastError());
    h->launches++;
    if (eval_mark(h, "eval_ssim", st)) return 1;
    CUDA_TRY(cudaMemcpyAsync(ssim_map, h->ev_map.get(), (size_t)map_n * sizeof(double), cudaMemcpyDeviceToHost, st));
  }
  unsigned long long acc[2];
  CUDA_TRY(cudaMemcpyAsync(acc, h->ev_acc.get(), sizeof(acc), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  *sse = acc[0];
  *pixels = (int64_t)hs * ws;
  *nan_pixels = (int64_t)acc[1];
  h->eval_timed = h->timing != 0;
  return 0;
}

int dcscn_evaluate_image(dcscn_handle* h, int index, const uint8_t* pixels, int height, int width, int channels, int lr_height,
                         int lr_width, int flips, double max_value, int border, const double* ssim_params, uint64_t* sse,
                         int64_t* pixel_count, int64_t* nan_pixels, double* ssim_map, int64_t map_capacity) {
  if (!h || !sse || !pixel_count || !nan_pixels) return fail("dcscn_evaluate_image: null argument");
  EvalImage im;
  if (index >= 0) {
    if (index >= (int)h->ev_host.size())
      return fail("dcscn_evaluate_image: image %d of an evaluation store of %d (call dcscn_eval_store_set first)", index,
                  (int)h->ev_host.size());
    const ImageEntry& e = h->ev_host[index];
    im = EvalImage{h->ev_pixels.get() + e.offset, e.height, e.width, e.channels};
  } else {
    if (!pixels) return fail("dcscn_evaluate_image: null pixels");
    if (height <= 0 || width <= 0 || (channels != 1 && channels != 3))
      return fail("dcscn_evaluate_image: the image is %d x %d x %d (1 or 3 channels expected)", height, width, channels);
    const size_t bytes = (size_t)height * width * channels;
    CUDA_TRY(cudaSetDevice(h->cfg.device_id));
    if (h->ev_upload.grow(bytes)) return 1;
    CUDA_TRY(cudaMemcpyAsync(h->ev_upload.get(), pixels, bytes, cudaMemcpyHostToDevice, 0));
    im = EvalImage{h->ev_upload.get(), height, width, channels};
  }
  return evaluate_impl(h, im, lr_height, lr_width, flips, max_value, border, ssim_params, sse, pixel_count, nan_pixels, ssim_map,
                       map_capacity);
}

int dcscn_get_grad(dcscn_handle* h, const char* name, float* host_data, int64_t numel) {
  if (!h || !name || !host_data) return fail("dcscn_get_grad: null argument");
  if (!h->train || h->train->total == 0) return fail("dcscn_get_grad: no train step has run yet");
  auto it = h->param_index.find(name);
  if (it == h->param_index.end()) return fail("dcscn_get_grad: unknown variable '%s'", name);
  const ParamDef& p = h->params[it->second];
  if (numel != p.numel()) return fail("dcscn_get_grad: '%s' has %lld elements, got %lld", name, (long long)p.numel(), (long long)numel);
  CUDA_TRY(cudaSetDevice(h->cfg.device_id));
  CUDA_TRY(cudaMemcpy(host_data, h->train->d_g.get() + h->train->off[it->second], (size_t)numel * sizeof(float), cudaMemcpyDeviceToHost));
  return 0;
}

int dcscn_get_train_tensor(dcscn_handle* h, const char* name, float* host_data, int64_t numel) {
  if (!h || !name || !host_data) return fail("dcscn_get_train_tensor: null argument");
  TrainState* t = h->train.get();
  if (!t || (t->last_px == 0 && t->last_ds_px == 0)) return fail("dcscn_get_train_tensor: no train step has run yet");
  CUDA_TRY(cudaSetDevice(h->cfg.device_id));
  CUDA_TRY(cudaDeviceSynchronize());
  const std::string s(name);
  std::vector<__half> hi, lo;
  size_t px = 0;
  int ch = 0;
  if (s.rfind("zneg:", 0) == 0) {   // min(z, 0) planes of the last training forward (prelu / leaky_relu only)
    if (!needs_zneg(h)) return fail("dcscn_get_train_tensor: '%s': the activator keeps no min(z, 0) planes", name);
    if (t->last_px == 0) return fail("dcscn_get_train_tensor: '%s': the fp32 depthwise-separable step keeps no min(z, 0) planes (see \"Z:\")", name);
    ActView v;
    if (!act_view(h, s.substr(5), &v) || !v.drop_layer) return fail("dcscn_get_train_tensor: no tensor '%s'", name);   // activated ones only
    px = t->last_px;
    ch = v.ch;
    hi.resize(px * ch);
    CUDA_TRY(cudaMemcpy2D(hi.data(), ch * sizeof(__half), zneg_of(h, v), v.pitch * sizeof(__half), ch * sizeof(__half), px, cudaMemcpyDeviceToHost));
  } else {
    auto it = t->captured.find(s);
    if (it == t->captured.end())
      return fail("dcscn_get_train_tensor: no tensor '%s' (set option grad_capture = 1 before the train step)", name);
    const TrainState::Captured& c = it->second;
    px = c.px; ch = c.ch;
    if (numel != (int64_t)(px * ch)) return fail("dcscn_get_train_tensor: '%s' has %lld elements, got %lld", name, (long long)(px * ch), (long long)numel);
    if (c.f32) {
      CUDA_TRY(cudaMemcpy(host_data, c.hi.get(), px * ch * sizeof(float), cudaMemcpyDeviceToHost));
      return 0;
    }
    hi.resize(px * ch);
    lo.resize(px * ch);
    CUDA_TRY(cudaMemcpy(hi.data(), c.hi.get(), hi.size() * sizeof(__half), cudaMemcpyDeviceToHost));
    CUDA_TRY(cudaMemcpy(lo.data(), c.lo.get(), lo.size() * sizeof(__half), cudaMemcpyDeviceToHost));
  }
  if (numel != (int64_t)(px * ch)) return fail("dcscn_get_train_tensor: '%s' has %lld elements, got %lld", name, (long long)(px * ch), (long long)numel);
  for (size_t i = 0; i < hi.size(); ++i) host_data[i] = __half2float(hi[i]) + (lo.empty() ? 0.f : __half2float(lo[i]));
  return 0;
}

int dcscn_get_adam_slot(dcscn_handle* h, const char* name, int slot, float* host_data, int64_t numel) {
  if (!h || !name || !host_data) return fail("dcscn_get_adam_slot: null argument");
  if (h->cfg.optimizer != DCSCN_OPTIMIZER_ADAM) return fail("dcscn_get_adam_slot: the optimizer is not adam (use dcscn_get_optimizer_slot)");
  if (!h->train || h->train->total == 0) return fail("dcscn_get_adam_slot: no train step has run yet");
  auto it = h->param_index.find(name);
  if (it == h->param_index.end()) return fail("dcscn_get_adam_slot: unknown variable '%s'", name);
  const ParamDef& p = h->params[it->second];
  if (numel != p.numel() || (slot != 0 && slot != 1)) return fail("dcscn_get_adam_slot: bad size or slot");
  CUDA_TRY(cudaSetDevice(h->cfg.device_id));
  const float* src = (slot == 0 ? h->train->d_m.get() : h->train->d_v.get()) + h->train->off[it->second];
  CUDA_TRY(cudaMemcpy(host_data, src, (size_t)numel * sizeof(float), cudaMemcpyDeviceToHost));
  return 0;
}

int dcscn_set_adam_slot(dcscn_handle* h, const char* name, int slot, const float* host_data, int64_t numel) {
  if (!h || !name || !host_data) return fail("dcscn_set_adam_slot: null argument");
  if (h->cfg.optimizer != DCSCN_OPTIMIZER_ADAM) return fail("dcscn_set_adam_slot: the optimizer is not adam (use dcscn_set_optimizer_slot)");
  CUDA_TRY(cudaSetDevice(h->cfg.device_id));
  if (train_init(h)) return 1;
  auto it = h->param_index.find(name);
  if (it == h->param_index.end()) return fail("dcscn_set_adam_slot: unknown variable '%s'", name);
  const ParamDef& p = h->params[it->second];
  if (numel != p.numel() || (slot != 0 && slot != 1)) return fail("dcscn_set_adam_slot: bad size or slot");
  float* dst = (slot == 0 ? h->train->d_m.get() : h->train->d_v.get()) + h->train->off[it->second];
  CUDA_TRY(cudaMemcpy(dst, host_data, (size_t)numel * sizeof(float), cudaMemcpyHostToDevice));
  return 0;
}

int dcscn_get_adam_step(dcscn_handle* h, int64_t* step) {
  if (!h || !step) return fail("dcscn_get_adam_step: null argument");
  *step = h->train ? h->train->step : 0;
  return 0;
}

int dcscn_set_adam_step(dcscn_handle* h, int64_t step) {
  if (!h || step < 0) return fail("dcscn_set_adam_step: bad argument");
  CUDA_TRY(cudaSetDevice(h->cfg.device_id));
  if (train_init(h)) return 1;
  h->train->step = step;
  return 0;
}

int dcscn_optimizer_slot_count(dcscn_handle* h) { return h ? optimizer_slot_count(h->cfg.optimizer) : 0; }

// Resolves (variable, slot) of the configured optimizer to its offset in the flat slot buffers.
static int optimizer_slot_view(dcscn_handle* h, const char* fn, const char* name, int slot, int64_t numel, size_t* off, float** buf) {
  auto it = h->param_index.find(name);
  if (it == h->param_index.end()) return fail("%s: unknown variable '%s'", fn, name);
  const ParamDef& p = h->params[it->second];
  if (numel != p.numel()) return fail("%s: '%s' has %lld elements, got %lld", fn, name, (long long)p.numel(), (long long)numel);
  if (slot < 0 || slot >= optimizer_slot_count(h->cfg.optimizer))
    return fail("%s: optimizer %d has no slot %d", fn, h->cfg.optimizer, slot);
  *off = h->train ? h->train->off[it->second] : 0;
  *buf = !h->train ? nullptr : slot == 0 ? h->train->d_m.get() : h->train->d_v.get();
  return 0;
}

int dcscn_get_optimizer_slot(dcscn_handle* h, const char* name, int slot, float* host_data, int64_t numel) {
  if (!h || !name || !host_data) return fail("dcscn_get_optimizer_slot: null argument");
  size_t off;
  float* buf;
  if (optimizer_slot_view(h, "dcscn_get_optimizer_slot", name, slot, numel, &off, &buf)) return 1;
  if (!h->train || h->train->total == 0) {   // no state allocated yet: the slot holds its initial value
    std::fill(host_data, host_data + numel, optimizer_slot_init(h->cfg.optimizer, slot));
    return 0;
  }
  CUDA_TRY(cudaSetDevice(h->cfg.device_id));
  CUDA_TRY(cudaMemcpy(host_data, buf + off, (size_t)numel * sizeof(float), cudaMemcpyDeviceToHost));
  return 0;
}

int dcscn_set_optimizer_slot(dcscn_handle* h, const char* name, int slot, const float* host_data, int64_t numel) {
  if (!h || !name || !host_data) return fail("dcscn_set_optimizer_slot: null argument");
  CUDA_TRY(cudaSetDevice(h->cfg.device_id));
  if (train_init(h)) return 1;
  size_t off;
  float* buf;
  if (optimizer_slot_view(h, "dcscn_set_optimizer_slot", name, slot, numel, &off, &buf)) return 1;
  CUDA_TRY(cudaMemcpy(buf + off, host_data, (size_t)numel * sizeof(float), cudaMemcpyHostToDevice));
  return 0;
}

int dcscn_reset_optimizer(dcscn_handle* h) {
  if (!h) return fail("dcscn_reset_optimizer: null argument");
  if (!h->train || h->train->total == 0) return 0;   // no optimizer state exists yet: train_init starts the slots right
  CUDA_TRY(cudaSetDevice(h->cfg.device_id));
  if (reset_optimizer_slots(h)) return 1;
  h->train->step = 0;
  return 0;
}

int dcscn_grad_buffer(dcscn_handle* h, float** dev_ptr, int64_t* count) {
  if (!h || !dev_ptr || !count) return fail("dcscn_grad_buffer: null argument");
  if (!h->train || h->train->total == 0) return fail("dcscn_grad_buffer: no train step has run yet");
  *dev_ptr = h->train->d_g.get();
  *count = (int64_t)h->train->total + 2;   // gradients of every trainable, then {image_loss, mse} of the last step
  return 0;
}

int dcscn_apply_gradients(dcscn_handle* h, float lr, void* stream) {
  if (!h) return fail("dcscn_apply_gradients: null argument");
  CUDA_TRY(cudaSetDevice(h->cfg.device_id));
  return apply_gradients_impl(h, lr, true, (cudaStream_t)stream);
}

int dcscn_apply_gradients_avg(dcscn_handle* h, float lr, float grad_scale, float* out_loss, float* out_mse, void* stream) {
  if (!h) return fail("dcscn_apply_gradients_avg: null argument");
  CUDA_TRY(cudaSetDevice(h->cfg.device_id));
  return apply_gradients_impl(h, lr, true, (cudaStream_t)stream, grad_scale, out_loss, out_mse);
}

float dcscn_last_grad_norm(dcscn_handle* h) { return (h && h->train) ? h->train->last_norm : 0.f; }

int dcscn_dropout_mask(dcscn_handle* h, const char* tensor, uint32_t seed, int n, int height, int width, uint8_t* mask, int64_t numel) {
  if (!h || !tensor || !mask) return fail("dcscn_dropout_mask: null argument");
  ActView v;
  if (!act_view(h, tensor, &v) || !v.drop_layer)
    return fail(strncmp(tensor, "CNN", 3) == 0 ? "dcscn_dropout_mask: no tensor '%s'" : "dcscn_dropout_mask: tensor '%s' has no dropout", tensor);
  const size_t px = (size_t)n * height * width;
  const int C = v.ch;
  if (numel != (int64_t)(px * C)) return fail("dcscn_dropout_mask: expected %lld elements", (long long)(px * C));
  for (size_t q = 0; q < px; ++q)
    for (int k = 0; k < C; ++k)
      mask[q * C + k] = dropout_keep(seed, v.drop_layer, (uint64_t)q * (uint64_t)v.drop_stride + v.drop_col0 + k, h->cfg.dropout_keep) ? 1 : 0;
  return 0;
}

int64_t dcscn_launch_count(dcscn_handle* h) { return h ? h->launches : 0; }
int64_t dcscn_device_bytes(dcscn_handle* h) { return h ? workspace_bytes(h) : 0; }

int dcscn_tile_halo(dcscn_handle* h, int* lr_pixels) {
  if (!h || !lr_pixels) return fail("dcscn_tile_halo: null argument");
  *lr_pixels = tile_halo(h);
  return 0;
}
int64_t dcscn_graph_replays(dcscn_handle* h) { return h ? h->graph_replays : 0; }

}  // extern "C"
