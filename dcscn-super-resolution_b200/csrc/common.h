// Shared host/device declarations for the DCSCN sm_90a hot path.
//
// Data layout in HBM (see DESIGN.md "Data layout"):
//   * Activations between tensor-core layers are kept as TWO fp16 planes ("hi" and "lo",
//     value = hi + lo, 22 significand bits) in NHWC order with a padded channel pitch.  Each
//     layer of the feature-extraction stack owns a 16-channel-aligned slot of one shared
//     "concat" buffer, so tf.concat (DCSCN.py:259,281) never materialises.
//   * Weights are pre-packed per layer into the exact shared-memory image a K-major
//     SWIZZLE_128B wgmma operand tile needs (hi and lo fp16 planes, scaled by a power of two).
#pragma once
#include <cstdint>
#include <cuda_fp16.h>

namespace dcscn {

constexpr int kTileM = 128;          // pixels per CTA tile (GEMM M: two m64 wgmma warpgroups)
constexpr int kMaxSegments = 2;

enum EpilogueMode : int {
  EPI_PLANES = 0,      // fp16 hi/lo planes, same resolution (up to 2 column segments)
  EPI_D2S_F32 = 1,     // depth_to_space scatter into an fp32 NHWC buffer
  EPI_D2S_PLANES = 2,  // depth_to_space scatter into fp16 hi/lo planes
  EPI_D2S_RDOT = 3,    // depth_to_space fused with the per-pixel half of the final cout=1 conv (R-CNN1):
                       // writes, per HR pixel and filter tap, dot(h[pixel, :], w_last[tap, :])
  EPI_D2S_TAPS = 4,    // the same tap-planar values from a layer folded with R-CNN1 (engine.cu build_fold): column
                       // ij * rdot_taps + t of sub-pixel ij is tap t, stored at rdot_out[t][N][rH][rW]
};

// Point-wise activation of CNN1..CNNL, A1, B1 and B2 (--activator, tf_graph.py:77-102); values of DCSCN_ACTIVATOR_*.
// The forward kernels apply prelu, relu and leaky_relu as z > 0 ? z : a * z with a per-channel slope vector a (the
// PReLU variable, 0, or 0.1f; linear layers carry act = ACT_PRELU with a = 1) and evaluate the others as functions.
enum Activation : int {
  ACT_NONE = -1,       // linear layer without dropout (train kernels only)
  ACT_PRELU = 0,
  ACT_RELU = 1,
  ACT_LEAKY_RELU = 2,
  ACT_SIGMOID = 3,
  ACT_TANH = 4,
  ACT_SELU = 5,
};

struct EpiSegment {
  int col_begin;       // first GEMM column of this segment (multiple of 16)
  int col_end;         // one past the last column written (multiple of 16)
  __half* dst_hi;      // plane base, already offset to the slot's first channel
  __half* dst_lo;      // may be null in single-plane (fast) mode
  int pitch;           // channels per pixel of the destination buffer (elements)
  __half* dst_zneg;    // training only (else null): fp16 plane, same indexing, of min(z, 0) - the pre-activation's negative
                       // part.  PReLU's backward needs sign(z) and, for d alpha, z itself where z < 0; the post-activation
                       // output cannot give either when the slope alpha is <= 0 (trained checkpoints have many such).
};

struct EpiParams {
  const float* bias;   // [n_total_pad]  (zeros where the layer has no bias / padding)
  const float* alpha;  // [n_total_pad]  PReLU slope; 1.0 == linear layer
  float out_scale;     // 1 / weight_scale (exact power of two)
  int act;             // Activation: ACT_SIGMOID / ACT_TANH / ACT_SELU apply that function (their slope vector is 1)
  int mode;
  int n_valid;         // real output channels (cout) - columns >= n_valid are dropped for D2S
  EpiSegment seg[kMaxSegments];
  int num_seg;
  // depth_to_space
  int d2s_r;           // block size
  int d2s_cout;        // channels after depth_to_space
  float* dst_f32;      // EPI_D2S_F32 destination [N, r*H, r*W, d2s_pitch]
  int d2s_pitch;
  // EPI_D2S_RDOT: final conv weights [taps][d2s_cout] and tap-planar output [taps][N][rH][rW] (EPI_D2S_TAPS: the output
  // and rdot_taps only)
  const float* rdot_w;
  float* rdot_out;
  int rdot_taps;
  int rdot_parts;      // epilogue threads sharing one sub-pixel's channels each write their own partial plane set
                       // [parts][taps][N][rH][rW] (1 when a thread's column share covers whole sub-pixels)
  // inverted dropout (training): keep-mask generated from a counter hash; keep_prob==1 -> off
  float keep_prob;
  uint32_t drop_seed;
  uint32_t drop_layer;
  int drop_ntotal;     // channel count the keep-mask index is built with (the slot width; 0 = the GEMM's padded N)
};

struct ConvGeom {
  int n_img, H, W;       // input == output resolution of this conv
  int tiles_x, tiles_y;  // ceil(W/TW), ceil(H/TH)
  int TW, TH;            // TW*TH == 128
};

struct ConvTCParams {
  ConvGeom g;
  int ksz;               // 1 or 3
  int cin_pad;           // padded input channels of the source slot (multiple of 16)
  int chunks;            // ceil(cin_pad / 64)
  int n_tiles;           // column tiles (N > kMaxTileN is split)
  int n_pad;             // columns per tile, multiple of 16, <= kMaxTileN (112)
  int seg_chunks;        // pipeline stages per accumulation segment (fp32 promotion period)
  int chunk_box;         // k > 1: one (TW + k - 1) x (TH + k - 1) activation box per chunk serves all k x k taps (TW = 8);
                         // 0: one TW x (TH + k - 1) box per (chunk, kx)
  const __half* wpack;   // packed weights [n_tile][tap][chunk][plane][n_pad x 64] (pre-swizzled)
  int bias_smem;         // conv_tc_kernel keeps a copy of epi.bias / epi.alpha in shared memory (add_tc_launch)
  EpiParams epi;
};

// Parameters of the CUDA-core validation convolution (same math in plain fp32 FMAs).
struct ConvRefParams {
  ConvGeom g;
  int ksz;
  int cin;               // logical input channels
  int cout;              // logical output channels
  const __half* src_hi;  // input planes, already offset to the slot
  const __half* src_lo;
  int src_pitch;
  const int* in_map;     // [cin] channel position inside the source buffer
  const float* w;        // HWIO fp32 [k][k][cin][cout]
  int n_total_pad;
  EpiParams epi;         // out_scale must be 1 for this path
};

}  // namespace dcscn
