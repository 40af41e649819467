/*
 * dcscn_b200.h - C-ABI of the H100-native (sm_90a) DCSCN forward / backward hot path.
 *
 * The reference (jiny2001/dcscn-super-resolution) has no FFI: its seam is the Python class
 * DCSCN.SuperResolution and the four `sess.run` call sites.  Each entry point below names the
 * reference interface it stands in for (paths relative to the reference checkout).
 *
 * All tensors are contiguous fp32 NHWC with C == 1 at the boundary (TF placeholders
 * x / x2 / y, DCSCN.py:224-226).  Functions return 0 on success, non-zero on error;
 * dcscn_last_error() returns the message of the last failure on the calling thread.
 * A handle is not re-entrant; use one handle per GPU / host thread.
 */
#ifndef DCSCN_B200_H_
#define DCSCN_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct dcscn_handle dcscn_handle;

/* Arithmetic of the tensor-core layers. */
enum {
  DCSCN_PRECISION_F16X3 = 0, /* fp32-equivalent: fp16 hi/lo split operands, 3 wgmma passes, fp32 accumulate */
  DCSCN_PRECISION_F16X1 = 1  /* single-pass fp16 operands (PSNR-neutral, not 1e-3-pixel exact) */
};

/* Point-wise activation of CNN1..CNNL, A1, B1 and B2 (--activator, helper/tf_graph.py:77-102).  Up-PS, Up-PS2 and R-CNN1
 * stay linear.  Only prelu has a variable (a per-channel slope, initialised to 0.1); leaky_relu is max(z, 0.1 z); selu uses
 * TensorFlow's lambda = 1.0507009873554805 and alpha = 1.6732632423543772.  Gradients follow TensorFlow's gradient ops,
 * also at z = 0: relu' = 0, leaky_relu' = 1, selu' = lambda there. */
enum {
  DCSCN_ACTIVATOR_PRELU = 0,
  DCSCN_ACTIVATOR_RELU = 1,
  DCSCN_ACTIVATOR_LEAKY_RELU = 2,
  DCSCN_ACTIVATOR_SIGMOID = 3,
  DCSCN_ACTIVATOR_TANH = 4,
  DCSCN_ACTIVATOR_SELU = 5
};

/* Update rule of the train step (--optimizer, DCSCN.py:379-413): TF1's training ops at TF's defaults for every argument
 * the reference does not pass, applied to g = the gradient after the L2 term and clip_by_global_norm, in fp32.  lr is
 * the step's learning rate, mu = cfg.momentum.  Slots are listed in creation order: slot i is "<var>/<Name>" for i = 0
 * and "<var>/<Name>_1" for i = 1 in the reference's checkpoints, and starts at the value given.
 *   ADAM      slots m (0), v (0):       the update documented at dcscn_train_step (cfg.beta1 / beta2 / epsilon)
 *   GD        no slot:                  w -= lr * g
 *   MOMENTUM  accum (0):                a = mu * a + g;  w -= lr * a                       (no Nesterov)
 *   ADADELTA  accum (0), accum_update (0), rho = 0.95, eps = 1e-8:
 *             acc = rho * acc + (1 - rho) * g^2;  u = sqrt(acc_u + eps) / sqrt(acc + eps) * g;  w -= lr * u;
 *             acc_u = rho * acc_u + (1 - rho) * u^2                                       (u uses the old acc_u)
 *   ADAGRAD   accumulator (0.1):        acc += g^2;  w -= lr * g / sqrt(acc)               (no epsilon)
 *   RMSPROP   rms (1.0), momentum (0), rho = 0.9, eps = 1e-10:
 *             ms += (g^2 - ms) * (1 - rho);  mom = mu * mom + lr * g / sqrt(ms + eps);  w -= mom   (not centred) */
enum {
  DCSCN_OPTIMIZER_ADAM = 0,
  DCSCN_OPTIMIZER_GD = 1,
  DCSCN_OPTIMIZER_MOMENTUM = 2,
  DCSCN_OPTIMIZER_ADADELTA = 3,
  DCSCN_OPTIMIZER_ADAGRAD = 4,
  DCSCN_OPTIMIZER_RMSPROP = 5
};

/*
 * Graph hyper-parameters: the subset of helper/args.py:16-98 flags that shape the graph built by
 * DCSCN.SuperResolution.__init__ (DCSCN.py:29-106) and build_graph (DCSCN.py:222-332).
 */
typedef struct dcscn_config {
  int32_t struct_size;            /* sizeof(dcscn_config), for ABI checking */
  int32_t scale;                  /* --scale, 2..8: x4 is two x2 pixel-shuffler stages, every other factor one */
  int32_t layers;                 /* --layers */
  int32_t filters;                /* --filters */
  int32_t min_filters;            /* --min_filters */
  float filters_decay_gamma;      /* --filters_decay_gamma */
  int32_t use_nin;                /* --use_nin (only 1 is supported) */
  int32_t nin_filters;            /* --nin_filters  (A1) */
  int32_t nin_filters2;           /* --nin_filters2 (B1, B2) */
  int32_t cnn_size;               /* --cnn_size (3) */
  int32_t reconstruct_layers;     /* --reconstruct_layers (max(flag,1) == 1 supported) */
  int32_t reconstruct_filters;    /* --reconstruct_filters */
  int32_t pixel_shuffler_filters; /* --pixel_shuffler_filters (0 = same as input) */
  int32_t depthwise_separable;    /* --depthwise_separable */
  int32_t channels;               /* --channels (1) */
  float dropout_keep;             /* --dropout_rate (keep probability, training only) */
  float l2_decay;                 /* --l2_decay */
  float clipping_norm;            /* --clipping_norm */
  float beta1, beta2, epsilon;    /* --beta1 --beta2 --epsilon (Adam) */
  int32_t device_id;              /* --gpu_device_id */
  int32_t precision;              /* DCSCN_PRECISION_* */
  int32_t activator;              /* --activator: DCSCN_ACTIVATOR_* (0 = prelu) */
  int32_t optimizer;              /* --optimizer: DCSCN_OPTIMIZER_* (0 = adam) */
  float momentum;                 /* --momentum (momentum and rmsprop) */
  int32_t transposed_upsampler;   /* --pixel_shuffler=false: Up-TCNN, one stride-`scale` conv2d_transpose (0 = Up-PS) */
} dcscn_config;

/* SuperResolution(flags) + build_graph() + init_session (DCSCN.py:29, :222; tf_graph.py:65). */
int dcscn_create(const dcscn_config* cfg, dcscn_handle** out);
/* sess.close() */
int dcscn_destroy(dcscn_handle* h);
const char* dcscn_last_error(void);

/*
 * Variables of the graph, named exactly like the TF variables in the reference's checkpoints
 * (tf.train.Saver, tf_graph.py:263-296): "CNN1/conv_W" [k,k,cin,cout] HWIO, "CNN1/conv_B",
 * "CNN1/prelu/CNN1_prelu", "A1/...", "B1/...", "B2/...", "Up-PS/Up-PS_CNN/conv_W", "R-CNN1/conv_W" ...
 * The "<scope>/prelu/<scope>_prelu" slopes exist only with DCSCN_ACTIVATOR_PRELU; the other activators have no variable.
 * With cfg.transposed_upsampler the Up-PS variables are replaced by "Up-TCNN/Tconv_W" [K,K,C,C] (K = 2*scale - scale%2,
 * C = nin_filters + nin_filters2, TF's conv2d_transpose layout [h, w, out, in]; no bias, not depthwise-separable).
 */
int dcscn_num_params(dcscn_handle* h);
int dcscn_param_info(dcscn_handle* h, int index, char* name_buf, int name_buf_len, int64_t* dims4, int* ndim);
/* saver.restore (tf_graph.py:276): host fp32 -> engine.  numel must match the variable. */
int dcscn_set_param(dcscn_handle* h, const char* name, const float* host_data, int64_t numel);
/* saver.save (tf_graph.py:291): engine -> host fp32. */
int dcscn_get_param(dcscn_handle* h, const char* name, float* host_data, int64_t numel);

/*
 * sess.run(self.y_, {x, x2, dropout: 1.0, is_training: 0})  (DCSCN.py:565, :575).
 * x [n,h,w,1], x2 and y [n,scale*h,scale*w,1]: DEVICE pointers; asynchronous on `stream` (cudaStream_t).
 */
int dcscn_forward(dcscn_handle* h, const float* x_dev, const float* x2_dev, float* y_dev, int n, int height,
                  int width, void* stream);
/* Same call with HOST buffers (pinned or pageable): H2D, forward, D2H, synchronises before returning.  x2 may be NULL:
 * the bicubic up-scale of x is then formed on the device, bit for bit what `util.resize_image_by_pil(x, scale)` returns
 * (dcscn_bicubic_resize), and only x crosses PCIe (the default of `SuperResolution.do`, DCSCN.py:551-553). */
int dcscn_forward_host(dcscn_handle* h, const float* x, const float* x2, float* y, int n, int height, int width);
/* `util.resize_image_by_pil` (helper/utilty.py:211-239) for single-channel float images on the device: Pillow's bicubic
 * `Image.resize` of mode 'F' images restated bit-exactly (two passes, double accumulation, float32 intermediate; up- or
 * down-scaling).  src [n, height, width] -> dst [n, out_height, out_width], fp32 device tensors. */
int dcscn_bicubic_resize(dcscn_handle* h, const float* src_dev, float* dst_dev, int n, int height, int width, int out_height,
                         int out_width, void* stream);

/* The self-ensemble of `SuperResolution.do` (DCSCN.py:547-586) for ONE image, entirely on the device: the first `flips`
 * (1..8) transforms of helper/utilty.py:595-617 are applied to x [height,width] and x2 [scale*height, scale*width],
 * transforms 0..3 and 4..7 each run as one batched forward, and y [scale*height, scale*width] receives the float64 mean
 * of the inverse-transformed outputs, summed in the order 0, 1, ... like the reference's float64 accumulator. */
int dcscn_forward_ensemble(dcscn_handle* h, const float* x_dev, const float* x2_dev, double* y_dev, int height, int width,
                           int flips, void* stream);
int dcscn_forward_ensemble_host(dcscn_handle* h, const float* x, const float* x2, double* y, int height, int width, int flips);
/* (x2 may be NULL in dcscn_forward_ensemble_host as well: formed on the device from x.) */
/* One rank's share of the same ensemble when the 8 transforms are spread over several GPUs (SURVEY.md section 8e): bit t of
 * `transform_mask` selects transform t; y receives the float64 SUM of the selected inverse-transformed outputs (no
 * division), ready for one ncclAllReduce(sum) over the ranks followed by the division by the ensemble size. */
int dcscn_forward_ensemble_partial(dcscn_handle* h, const float* x_dev, const float* x2_dev, double* y_dev, int height,
                                   int width, int transform_mask, void* stream);

/*
 * sess.run([self.training_optimizer, self.image_loss, self.mse], {x, x2, y, lr, dropout: keep, is_training: 1})
 * (DCSCN.py:415-425; graph: build_optimizer / add_optimizer_op, DCSCN.py:334-413): forward with inverted dropout
 * (keep = cfg.dropout_keep, masks from a counter hash of `seed`), mse loss + l2_decay * sum(l2_loss(conv_W)),
 * gradients of every variable, tf.clip_by_global_norm(cfg.clipping_norm), then the cfg.optimizer update
 * (DCSCN_OPTIMIZER_*) with learning rate `lr`; for Adam m = b1*m + (1-b1)*g, v = b2*v + (1-b2)*g^2,
 * w -= lr * sqrt(1-b2^t) / (1-b1^t) * m / (sqrt(v) + eps).
 * `apply_update` = 0 computes loss and gradients only (dcscn_get_grad), leaving the weights untouched.
 * x / x2 / y are DEVICE pointers (dcscn_train_step) or HOST pointers (dcscn_train_step_host); both synchronise.
 */
int dcscn_train_step(dcscn_handle* h, const float* x_dev, const float* x2_dev, const float* y_dev, int n, int height, int width,
                     float lr, uint32_t seed, int apply_update, float* out_loss, float* out_mse, void* stream);
int dcscn_train_step_host(dcscn_handle* h, const float* x, const float* x2, const float* y, int n, int height, int width, float lr,
                          uint32_t seed, int apply_update, float* out_loss, float* out_mse);
/*
 * Training data path on the device (reference: helper/loader.py:70-275 BatchDataSets + DCSCN.py:186-190 build_input_batch,
 * which assemble every mini-batch patch by patch in Python).  dcscn_patch_store_set copies the data set's uint8 patch
 * arrays - LR input [count, ph, pw], its bicubic up-scale and the ground truth [count, scale*ph, scale*pw] - into HBM
 * once.  dcscn_train_step_indexed is dcscn_train_step on the mini-batch {patch indices[i]}: one gather launch per tensor
 * converts uint8 -> fp32 * (max_value / 255) (loader.py:251-255); bit 31 of an index mirrors that patch left-right
 * (the augmentation of loader.py:318-319).  dcscn_patch_gather returns the same gathered fp32 tensors to the host
 * (parity checks against the host loader).
 */
int dcscn_patch_store_set(dcscn_handle* h, const uint8_t* lr, const uint8_t* bicubic, const uint8_t* truth, int64_t count,
                          int patch_height, int patch_width);
int dcscn_train_step_indexed(dcscn_handle* h, const int32_t* indices, int n, float max_value, float lr, uint32_t seed,
                             int apply_update, float* out_loss, float* out_mse);
int dcscn_patch_gather(dcscn_handle* h, const int32_t* indices, int n, float max_value, float* x, float* x2, float* y);
/*
 * Random-crop training data on the device (reference: helper/loader.py:278-355 DynamicDataSets, the data set of train.py
 * without --build_batch, which decodes, crops, converts and resizes every patch of every step in Python).
 * dcscn_image_store_set copies the decoded uint8 images (what util.load_image returns: RGB, 3 interleaved channels, or
 * mode 'L', 1 channel; image i is heights[i] x widths[i] x channels[i] bytes at offsets[i] of `pixels`) into HBM once;
 * it replaces the previous image store and nothing else.  dcscn_train_step_crops is dcscn_train_step on the mini-batch of
 * `n` crop descriptors crops[4 * i ..] = (image, top, left, mirror) (loader.py:332-355 load_random_patch + the mirror of
 * loader.py:318-319): an e x e crop, e = scale * patch_size, at row `top` and column `left`, mirrored left-right when
 * mirror = 1.  Per crop the device forms what load_batch_image returns, bit for bit: the truth y = Y (float64 RGB -> Y,
 * util.convert_rgb_to_y) or the 'L' sample, x = Pillow bicubic of y down by 1 / scale (mode 'F' for Y, Pillow's 8-bit
 * path for 'L'), x2 = x up by scale, each multiplied by max_value / 255 under numpy's dtype rules (loader.py:323-327).
 * Every descriptor is checked before any launch: image in range, 0 <= top <= height - e, 0 <= left <= width - e,
 * mirror 0 or 1.  dcscn_crop_gather returns the same fp32 tensors x [n, ps, ps], x2 / y [n, e, e] to the host.
 */
int dcscn_image_store_set(dcscn_handle* h, const uint8_t* pixels, int64_t bytes, const int64_t* offsets, const int32_t* heights,
                          const int32_t* widths, const int32_t* channels, int count);
int dcscn_train_step_crops(dcscn_handle* h, const int32_t* crops, int n, int patch_size, float max_value, float lr, uint32_t seed,
                           int apply_update, float* out_loss, float* out_mse);
int dcscn_crop_gather(dcscn_handle* h, const int32_t* crops, int n, int patch_size, float max_value, float* x, float* x2, float* y);
/* d loss / d variable of the LAST train step (after the L2 term, before clipping): tf.gradients(loss, trainables). */
int dcscn_get_grad(dcscn_handle* h, const char* name, float* host_data, int64_t numel);
/* Adam slots of a variable ("<var>/Adam" = slot 0, "<var>/Adam_1" = slot 1 in the reference's checkpoints).  Fail for
 * any other cfg.optimizer. */
int dcscn_get_adam_slot(dcscn_handle* h, const char* name, int slot, float* host_data, int64_t numel);
/* Restoring optimizer state from a checkpoint (what tf.train.Saver.restore does for the graph sr.py / train.py build,
 * helper/tf_graph.py:263-280): the slots, and the number of applied updates t (the reference stores it as
 * beta1_power = beta1^(t+1), beta2_power = beta2^(t+1)). */
int dcscn_set_adam_slot(dcscn_handle* h, const char* name, int slot, const float* host_data, int64_t numel);
int dcscn_get_adam_step(dcscn_handle* h, int64_t* step);
int dcscn_set_adam_step(dcscn_handle* h, int64_t step);
/* The slots of cfg.optimizer (DCSCN_OPTIMIZER_*): how many each variable has (0 for gd, 1 for momentum and adagrad, 2 for
 * adam, adadelta and rmsprop), and slot `slot` of variable `name` in the order the enum's comment lists.  Before the first
 * train step, get returns the slot's initial value. */
int dcscn_optimizer_slot_count(dcscn_handle* h);
int dcscn_get_optimizer_slot(dcscn_handle* h, const char* name, int slot, float* host_data, int64_t numel);
int dcscn_set_optimizer_slot(dcscn_handle* h, const char* name, int slot, const float* host_data, int64_t numel);
/* tf.global_variables_initializer() on the optimizer's variables (helper/tf_graph.py:73-75 re-runs it for every trial of
 * train.py:100-103): every slot of every variable back to its initial value (see DCSCN_OPTIMIZER_*) and the update
 * count t to 0. */
int dcscn_reset_optimizer(dcscn_handle* h);
/* Data-parallel training: after dcscn_train_step(..., apply_update = 0) on every rank, all-reduce the flat buffer
 * returned here (device pointer, `count` floats: the gradient of every trainable in dcscn_param_info order followed by
 * this rank's {image_loss, mse}) - ONE ncclAllReduce(sum) over NVLink - then call dcscn_apply_gradients_avg on every
 * rank with grad_scale = 1 / ranks: it scales the summed gradients to their mean, applies the global-norm clip of the
 * averaged gradient + the cfg.optimizer update identically everywhere (SURVEY.md section 8e) and returns the job-wide
 * mean loss / mse.
 * Every rank must hold the same number of patches (each normalises by its own pixel count).
 * dcscn_apply_gradients is the same with grad_scale = 1 (gradients already averaged by the caller). */
int dcscn_grad_buffer(dcscn_handle* h, float** dev_ptr, int64_t* count);
int dcscn_apply_gradients(dcscn_handle* h, float lr, void* stream);
int dcscn_apply_gradients_avg(dcscn_handle* h, float lr, float grad_scale, float* out_loss, float* out_mse, void* stream);
/* Global gradient norm of the last train step (what clip_by_global_norm computed). */
float dcscn_last_grad_norm(dcscn_handle* h);
/* The keep mask (1 = kept) the train step with `seed` applies to `tensor` ("CNNi", "A1", "B1", "B2"), [n,h,w,C] uint8:
 * lets a CPU oracle replay the exact same dropout. */
int dcscn_dropout_mask(dcscn_handle* h, const char* tensor, uint32_t seed, int n, int height, int width, uint8_t* mask, int64_t numel);

/*
 * Parity / debug: output of one layer of the LAST forward as fp32 NHWC [n, H_l, W_l, cout_l]
 * (`tensor` is the reference's self.H entry: "CNN1".."CNNL", "A1", "B1", "B2", "Up-PS", "Up-PS2", or "Up-TCNN"
 * [n, s*H, s*W, C] with cfg.transposed_upsampler).  After a forward that fused R-CNN1 into the last upsampler,
 * "R-CNN1/taps" is its tap-planar products [parts, 9, n, s*H, s*W]: R-CNN1 tap t's contribution from each HR pixel,
 * in `parts` partial sets to be added (1 where the upsampler is folded with R-CNN1, see DESIGN 4.2).
 * Fails after a forward that ran tiled (option "workspace_mb"): the buffers then hold its last batch of windows.
 */
int dcscn_get_activation(dcscn_handle* h, const char* tensor, float* host_data, int64_t numel);
/*
 * Parity / debug: a tensor of the LAST train step as fp32 NHWC; on a tensor-core graph hi + lo of its fp16 planes,
 * logical channels only.  After a train step dcscn_get_activation returns that step's forward, after dropout.  Needs
 * option "grad_capture" = 1 during the step, except for the "zneg:" planes, which every prelu / leaky_relu step keeps:
 *   "y_", "dY"        the prediction and d loss / d y_ * grad_scale, [n, s*H, s*W, 1] (fp32, exact)
 *   "dZ:<layer>"      gradient at the layer's convolution output (before bias / activation), scaled by grad_scale:
 *                     CNNi, A1, B1, B2 [n, H, W, cout]; Up-PS [n, H, W, r*r*C] (x2, x3) or [n, H, W, 4*C] (x4), and at x4
 *                     Up-PS2 [n, 2H, 2W, 4*C], in the space_to_depth column order (i*r + j)*C + c; Up-TCNN
 *                     [n, H, W, s*s*C] in the same order (its equivalent 3x3 convolution, see engine.cu tconv_filter)
 *   "dH:<layer>"      output of the layer's data-gradient twin = gradient at the layer's input: CNNi (i >= 2)
 *                     [.., filters(i-1)], A1+B1 [.., concat channels], B2 [.., nin_filters2], Up-PS and Up-TCNN
 *                     [.., nin_filters2 + nin_filters] (B2 then A1), Up-PS2 [n, 2H, 2W, C]
 *   "zneg:<layer>"    the fp16 min(z, 0) plane the forward stored for CNNi, A1, B1, B2
 * A wide depthwise-separable graph (one that trains through the tensor-core step on composed filters) adds
 *   "Wc:<layer>"      the composed filter fp32(dw * pw) the step read, [k, k, cin, cout] (fp32, exact)
 *   "dWc:<layer>"     the composed filter's gradient before ds_decompose, scaled by grad_scale, [k, k, cin, cout]
 * The fp32 step of a narrow depthwise-separable graph (every other one) has no grad_scale and keeps no "zneg:" planes.
 * Its tensors are fp32 copies, per layer (CNNi, A1, B1, B2, Up-PS/Up-PS_CNN, Up-PS2/Up-PS2_CNN, R-CNN1) at the
 * resolution of the layer's input ([n, h, w, ch]) unless stated:
 *   "y_", "dY"        as above, with grad_scale 1
 *   "U:<layer>"       the depthwise output u = depthwise(input, depthwise_W), [.., cin]
 *   "Z:<layer>"       the pre-activation z = u . pointwise_W + conv_B, [.., cout] (pixel shufflers: before depth_to_space)
 *   "H:<layer>"       the output after activation and dropout, [.., cout]; pixel shufflers the whole depth_to_space
 *                     output [n, r*h, r*w, C] (all but R-CNN1, whose output is "y_")
 *   "dZ:<layer>"      d loss / d z, [.., cout];  "E:<layer>" (prelu) d loss / d h * min(z, 0), whose sums are d alpha
 *   "dU:<layer>"      d loss / d u, [.., cin]
 *   "dH:<layer>"      the gradient buffer at the layer's input as the layer's data-gradient kernel left it, [.., cin]:
 *                     B1 writes the concat gradient, A1 then adds to it, CNNi+1 adds to CNNi's channels of it
 */
int dcscn_get_train_tensor(dcscn_handle* h, const char* name, float* host_data, int64_t numel);

/* Options: "conv_impl" 0 = wgmma tensor cores (default), 1 = CUDA-core fp32 validation kernels;
 *          "seg_chunks" = pipeline stages per fp32-promotion segment (default 0 = automatic: 2, or 3 for thin layers);
 *          "fuse_last" 1 | 0 = compute the per-pixel half of R-CNN1 inside the last Up-PS epilogue (default 1);
 *          "timing" 0 | 1 = record per-launch CUDA events (see dcscn_get_timings);
 *          "act_grad_impl" 0 | 1 = activation gradients with 16-byte (default) or channel-pair accesses (cross-check);
 *          "graph" 1 | 0 = replay the launches of a forward (all but the last kernel) as one CUDA graph per (n, h, w) once
 *          the same input pointer has been seen twice in a row (default 1; off while "timing" = 1 or "conv_impl" = 1);
 *          "l1_loss" 0 | 1 = image_loss of the train step is mean |y_ - y| instead of the MSE (--use_l1_loss,
 *          DCSCN.py:342-344; the returned mse stays the MSE);
 *          "wgrad_impl" 0 | 1 = filter gradients on wgmma tensor cores (default) or on CUDA cores (cross-check);
 *          "grad_capture" 0 | 1 = the train step copies its activation-sized gradient tensors into buffers allocated on
 *          first use, for dcscn_get_train_tensor (default 0: no copy, no allocation);
 *          "workspace_mb" = MiB an inference forward may allocate per batch (default 0 = no limit: the whole batch runs
 *          at once).  Covers dcscn_forward, dcscn_forward_host and the dcscn_forward_ensemble* calls.  The limit counts
 *          the activation workspace and the staging buffers of one batch of windows; an image whose workspace fits runs
 *          exactly as without the option, a larger one runs as batches of overlapping windows (each with
 *          dcscn_tile_halo pixels of context), bit-identical to the whole-image forward.  A limit too small for one
 *          window of a 16 x 16 core plus its halo fails the forward, naming the minimum.  Not counted: the whole-image
 *          buffers of the host-buffer and ensemble calls (their x / x2 / y copies and transformed images, tens of bytes
 *          per LR pixel) and the bicubic scratch.  The workspace only grows: set the option before the first forward.
 *          The train step does not read it (its batches are patches).  Negative values are refused. */
int dcscn_set_option(dcscn_handle* h, const char* key, int64_t value);
/* With option "timing" = 1 every launch of a forward is bracketed by CUDA events on its stream; this returns the
 * device time in ms of each launch of the LAST forward (in launch order) and their comma-separated names.  A tiled
 * forward lists tile_gather, its layers and tile_stitch once per batch of windows.  After dcscn_evaluate_image it lists
 * that call's steps instead (see there), until the next forward. */
int dcscn_get_timings(dcscn_handle* h, float* ms, int capacity, int* count, char* names, int names_len);
/* LR pixels of context a window of a tiled forward carries around its core (option "workspace_mb"): the receptive
 * radius of the graph, walked back from R-CNN1 at HR resolution (15 for the 12-layer 3x3 graphs, 10 for 7 layers).
 * A core computed with this much context is bit-identical to the same pixels of the whole-image forward, which also
 * lets a caller split one image over several GPUs. */
int dcscn_tile_halo(dcscn_handle* h, int* lr_pixels);
/*
 * Evaluation on the device (reference DCSCN.py:672-703 do_for_evaluate, :705-725 evaluate_bicubic): one call computes
 * for one test image what _evaluation_set -> do(lr, bicubic) -> util.compute_psnr_and_ssim compute on the host, bit for
 * bit.  dcscn_eval_store_set copies decoded uint8 test images (layout of dcscn_image_store_set) into HBM once; it
 * replaces the previous evaluation store and touches neither the training stores nor anything else.
 * dcscn_evaluate_image evaluates image `index` of that store, or with index < 0 the height x width x channels image at
 * host `pixels`:
 *   1. crop to the top-left (height / s * s) x (width / s * s) pixels; RGB becomes the float64 Y of
 *      util.convert_rgb_to_y, the truth clip(rint(Y), 0, 255); a mode-'L' pixel is its own truth;
 *   2. LR = Pillow bicubic down to lr_height x lr_width (the host's int(side * (1.0 / s)), passed in; it must up-scale
 *      back to the aligned size), bicubic = the LR up by s: mode 'F' for Y, Pillow's 8-bit path for 'L';
 *   3. flips 1..8: both multiplied by max_value / 255 under numpy's dtype rules, then the forward (flips = 1) or the
 *      self-ensemble of the first `flips` transforms; the output times 255 / max_value (fp32 for one flip, float64 for
 *      the ensemble mean), rint, clip to [0, 255].  flips = 0: the bicubic up-scale itself, rint, clip (no forward);
 *   4. on the region left after shaving `border` pixels from each side (border > 0 only): *sse = the exact sum of
 *      squared differences of the integer-valued planes over the non-NaN output pixels, *pixel_count = the region's
 *      pixels, *nan_pixels = its NaN output pixels; and when the region has at least 11 rows, rows 5 .. rows - 6 of
 *      util._ssim_columns' SSIM map ((rows - 10) x columns float64, row-major) into ssim_map, which must hold that many.
 *      ssim_params = {w0, w1, .. w5, c1, c2}: the centre and side taps of scipy's gaussian_filter1d(sigma 1.5,
 *      truncate 3.5) and the SSIM constants.  The caller finishes PSNR = 10 log10(255^2 / (sse / pixel_count)) and
 *      SSIM = the numpy mean of the map rows.
 * The planes are the handle's own; option "workspace_mb" tiles the forward as usual.  With option "timing" = 1,
 * dcscn_get_timings then lists eval_prepare, eval_resize, eval_place, forward (or ensemble), eval_trim, eval_sse,
 * eval_ssim (the steps that ran), until the next forward.
 */
int dcscn_eval_store_set(dcscn_handle* h, const uint8_t* pixels, int64_t bytes, const int64_t* offsets, const int32_t* heights,
                         const int32_t* widths, const int32_t* channels, int count);
int dcscn_evaluate_image(dcscn_handle* h, int index, const uint8_t* pixels, int height, int width, int channels, int lr_height,
                         int lr_width, int flips, double max_value, int border, const double* ssim_params, uint64_t* sse,
                         int64_t* pixel_count, int64_t* nan_pixels, double* ssim_map, int64_t map_capacity);
/* Number of kernels this handle has launched so far (bench.py "gpu_launches"). */
int64_t dcscn_launch_count(dcscn_handle* h);
/* Forwards served by a CUDA-graph replay so far (option "graph"). */
int64_t dcscn_graph_replays(dcscn_handle* h);
/* Bytes of device memory currently held by the handle. */
int64_t dcscn_device_bytes(dcscn_handle* h);

#ifdef __cplusplus
}
#endif
#endif /* DCSCN_B200_H_ */
