/* libhorizonnet_b200 -- C ABI of the H100-native HorizonNet hot path.
 *
 * The reference (sunset1995/HorizonNet @ c9a7df9) is pure Python and has no FFI of its own, so this
 * ABI sits *beneath* the two Python entry points it keeps drop-in compatible (see INTEGRATION.md):
 *
 *   model.HorizonNet('resnet50', use_rnn=True).forward(x)        reference model.py:254-281
 *   misc.panostretch.pano_stretch(img, corners, kx, ky, order)   reference misc/panostretch.py:81-117
 *
 * Conventions: plain pointers and sizes only (no torch types); the caller owns every buffer;
 * device entry points are asynchronous on the CUstream/cudaStream_t passed as `void* stream`
 * (NULL = legacy default stream); every function returns 0 on success and a negative value on
 * failure, with the message available from hn_last_error() (thread-local).  A handle is bound to
 * one device and is not thread-safe; use one handle per replica (reference train.py:190-192
 * replicates the module per device).  There is no CPU path: without a CUDA device every compute
 * entry point fails.
 */
#ifndef HORIZONNET_B200_H
#define HORIZONNET_B200_H

#ifdef __cplusplus
extern "C" {
#endif

typedef struct hn_model hn_model;

/* Last error message of the calling thread ("" if none). */
const char* hn_last_error(void);
/* ABI version (bumped on any signature change). */
int hn_abi_version(void);
/* Digest of the sources this binary was built from (horizonnet_b200/build.py embeds it; the Python binding
 * refuses to run a binary whose digest differs from the checked-out sources). */
const char* hn_build_digest(void);
/* Number of kernels this library has launched in this process (bench.py "gpu_launches"). */
long long hn_kernel_launches(void);

/* ---- model.HorizonNet (reference model.py:185-281), resnet50 or resnet18 with the bi-LSTM or the MLP head ---- */

/* Creates HorizonNet('resnet50', use_rnn=True) on CUDA device `device`, with activation workspace for up to
 * `max_batch` panoramas per forward.  Replaces HorizonNet.__init__ (model.py:189-246) minus the ImageNet
 * download.  Same as hn_model_create_head(device, max_batch, 1, out). */
int hn_model_create(int device, int max_batch, hn_model** out);
/* use_rnn = 1: the 2-layer bi-LSTM + Linear(1024, 12) head (model.py:222-233); use_rnn = 0: the per-column MLP head
 * Linear(1024, 512), ReLU, Dropout(0.5), Linear(512, 12) (model.py:234-243, what train.py --no_rnn builds), which has
 * 434 state_dict keys: linear.0.* and linear.3.* instead of bi_rnn.* and linear.*.  Every entry point below takes
 * either model. */
int hn_model_create_head(int device, int max_batch, int use_rnn, hn_model** out);
/* Any supported backbone: "resnet50" (torchvision Bottlenecks; what hn_model_create / _head build) or "resnet18"
 * (BasicBlocks, 250 state_dict keys with the bi-LSTM, 236 with the MLP head; the feature sequence is 256 wide instead of
 * 1024, so bi_rnn.weight_ih_l0* is [2048][256] and linear.0.weight [512][256]).  Other names fail. */
int hn_model_create_arch(int device, int max_batch, const char* backbone, int use_rnn, hn_model** out);

/* Number of tensors of the reference checkpoint layout (448, or 434 with the MLP head; misc/utils.py:49-58) and the i-th key
 * with its element count; lets a binding iterate the state_dict without knowing the topology. */
int hn_model_num_tensors(const hn_model* m);
int hn_model_tensor_info(const hn_model* m, int index, const char** key, long long* numel);

/* Uploads one fp32 tensor of the reference state_dict (same key names and PyTorch layouts:
 * conv OIHW, LSTM [4H, in], linear [out, in]).  `data` may be a host (on_device=0) or a device
 * pointer (on_device=1).  `*.num_batches_tracked` keys are accepted and ignored.
 * Replaces nn.Module.load_state_dict for this module (misc/utils.py:64). */
int hn_model_set_tensor(hn_model* m, const char* key, const float* data, long long numel, int on_device);

/* Folds eval-mode BN / conv bias and re-packs all weights into the kernels' layouts.  Fails if a
 * tensor was never set.  Must be called after the last hn_model_set_tensor and before forward. */
int hn_model_finalize(hn_model* m);

/* HorizonNet.forward (model.py:254-281), eval mode.  x: [batch][in_channels >= 3][512][1024] fp32
 * NCHW in [0,1] on the device (only the first 3 channels are read, model.py:252);
 * bon: [batch][2][1024], cor: [batch][1][1024] fp32 on the device (raw: cor is a logit). */
int hn_model_forward(hn_model* m, const float* x_nchw_dev, int batch, int in_channels,
                     float* bon_dev, float* cor_dev, void* stream);

/* Throughput form of hn_model_forward for streams of batches.  The forward is split over two internal streams:
 * the encoder + height reduction of call i+1 (all SMs, tensor-core bound) run while the bi-LSTM recurrence + head
 * of call i (16-CTA clusters on 64 SMs, latency-bound: 512 dependent steps) are still in flight.  Ordering contract
 * on `stream`: x must be ready in stream order at the call; x may be reused by work enqueued on `stream` after the
 * call returns; bon/cor of call i are complete for work enqueued on `stream` after call i+1 returns, or after
 * hn_model_flush(m, stream).  Results are bit-identical to hn_model_forward.  Keep bon/cor of consecutive calls in
 * distinct buffers. */
int hn_model_forward_async(hn_model* m, const float* x_nchw_dev, int batch, int in_channels,
                           float* bon_dev, float* cor_dev, void* stream);
/* Makes `stream` wait for every forward enqueued so far by hn_model_forward_async. */
int hn_model_flush(hn_model* m, void* stream);

/* The BatchNorm2d modules in graph order (hn_train_forward's bn_train / bn_factor index them) and their state_dict
 * prefixes. */
int hn_model_num_bn(const hn_model* m);
const char* hn_model_bn_name(const hn_model* m, int i);
/* The dropout factors (0 or 1/(1-p)) hn_train_forward multiplies with for this seed and `which` (see below). */
int hn_dropout_mask(unsigned long long seed, int which, double p, float* out_dev, long long n, void* stream);
/* Current device copy of a state_dict tensor (e.g. "...bn1.running_mean" after train forwards) -> out
 * (device pointer if on_device, else host; the host form synchronises). */
int hn_model_get_tensor(hn_model* m, const char* key, float* out, long long numel, int on_device, void* stream);

/* Training step (row f1; reference train.py:44-58 feed_forward + :272-281 backward).
 * hn_train_forward is the TRAIN-mode forward: what `net(x)` computes under `net.train()` (reference train.py:52 inside
 * feed_forward, model.py:254-281 with every nn.BatchNorm2d in training mode and the dropouts active), with or without
 * autograd.  It keeps a tape (every conv output and activation) for hn_train_backward; batch <= 64.
 *   - BatchNorm2d i (i < hn_model_num_bn(m), state_dict prefix hn_model_bn_name(m, i)): bn_train[i] = 1 normalises
 *     with the batch mean / biased variance of the raw conv output and moves running_mean / running_var (the device
 *     copies inside the model, read them back with hn_model_get_tensor) by bn_factor[i] (= the module's momentum, or
 *     1/num_batches_tracked for momentum=None; < 0: track_running_stats off) using the unbiased variance;
 *     bn_train[i] = 0 keeps that module in eval mode (train.py:251-256, --freeze_earlier_blocks).
 *   - rnn_dropout: nn.LSTM(dropout=0.5) between the recurrent layers (model.py:226); head_dropout: self.drop_out
 *     (model.py:228, :265); 0 disables.  Masks are Philox4x32-10 functions of (seed, which, element index):
 *     hn_dropout_mask writes the factors (0 or 1/(1-p)) the forward multiplies with, which = 0 inter-layer
 *     [256][batch][1024], 1 head [256][batch][1024].  torch's own generator stream is not reproduced; for parity
 *     against a torch run, rnn_mask_dev / head_mask_dev (same shapes, or NULL) replace the Philox masks.
 *   - MLP head (hn_model_create_head with use_rnn = 0): rnn_dropout must be 0 and rnn_mask_dev NULL; head_dropout is
 *     the p of linear[2] (model.py:240), which acts on the post-ReLU hidden layer: which = 1 over 256*batch*512
 *     elements, head_mask_dev [256][batch][512] (row t*batch + b, the library's order; the reference's own mask is
 *     [batch][256][512]).
 * Eval-mode entry points called afterwards fold the moved running statistics again on their own.
 * hn_train_backward takes d(loss)/d(bon) [batch][2][1024] and d(loss)/d(cor) [batch][1][1024] (device) -- the losses
 * themselves (train.py:53-56: L1 + BCE-with-logits) and the optimizer (train.py:216-223) stay with the caller -- and
 * leaves d(loss)/d(parameter) for every state_dict parameter in the reference's layout (nn.Conv2d OIHW, nn.LSTM
 * [4H][in], ...), read back with hn_model_get_grad (device pointer).  One backward per forward.  With option
 * "tensor_cores" on, the encoder and height-reduction convolutions, their data gradients (hn_conv2d_dgrad_tc) and the
 * weight gradients of those convolutions, the LSTM and the MLP head (hn_conv2d_wgrad_tc) run on the split-fp16 wgmma
 * kernels where those take the shape, everything else on exact fp32 CUDA-core kernels; no loss scaling or gradient
 * all-reduce. */
int hn_train_forward(hn_model* m, const float* x_nchw_dev, int batch, int in_channels, float* bon_dev, float* cor_dev,
                     const unsigned char* bn_train, const double* bn_factor, int n_bn, unsigned long long seed,
                     double rnn_dropout, double head_dropout, const float* rnn_mask_dev, const float* head_mask_dev,
                     void* stream);
int hn_train_backward(hn_model* m, const float* dbon_dev, const float* dcor_dev, void* stream);
int hn_model_get_grad(hn_model* m, const char* key, float* out_dev, long long numel, void* stream);
/* Device time (ms) of the phases of the last hn_train_backward: head, bi-LSTM BPTT, sequence adjoint, the 69 conv units.
 * With the MLP head, ms[0] is the whole MLP backward and ms[1] is 0. */
int hn_train_profile(hn_model* m, double ms[4]);
/* HN_TRAIN_PROF=1 during the last hn_train_backward: the conv-unit phase split into ms[0] BatchNorm backward, ms[1] weight
 * gradients, ms[2] data gradients (device ms, summed over the units); -1 when that backward was not profiled. */
int hn_train_profile_units(hn_model* m, double ms[3]);
/* Tape inspection for tests: conv unit i of the last hn_train_forward (graph order: stem, blocks, height reduction);
 * what = 0 activation, 1 raw conv output, 2 gradient of the activation; halo-1 NHWC copy, dims = {B, H, W, C}. */
int hn_train_debug_unit(hn_model* m, int i, int what, float* out_dev, long long capacity, int dims[4], char* name,
                        int name_cap, void* stream);

/* Same call with HOST buffers: H2D of x, forward, D2H of bon/cor, synchronous.  This is what
 * inference.py:78-79 (`net(x.to(device))` + `.cpu()`) amounts to. */
int hn_model_forward_host(hn_model* m, const float* x_nchw_host, int batch, int in_channels,
                          float* bon_host, float* cor_host);

/* Pipelined form of the host call for streams of batches: hn_model_submit_host enqueues the H2D
 * copy of a batch (pinned memory recommended) on an internal copy stream into one of two input
 * slots, enqueues its forward behind it (two-stream schedule of hn_model_forward_async) and returns;
 * hn_model_collect_host waits for the OLDEST submitted batch, copies bon/cor back and synchronises
 * (a device-side failure of that batch is reported here).  Calling submit(i+1) before collect(i)
 * overlaps the upload and the encoder of the next batch with the forward / recurrence of the current
 * one (at most 2 batches in flight).  Results are identical to hn_model_forward_host. */
int hn_model_submit_host(hn_model* m, const float* x_nchw_host, int batch, int in_channels);
int hn_model_collect_host(hn_model* m, float* bon_host, float* cor_host);

/* Test-time-augmented inference on the device ("next" row f2; reference inference.py:32-62 augment /
 * augment_undo and inference.py:77-93).  x: ONE panorama [3][512][1024] fp32 on the device; views =
 * identity (+ horizontal flip if `flip`) + one np.roll per entry of shifts_host (pixels, as computed by
 * inference.py:40 `int(round(shift_p * W))`).  Outputs on the device: y_bon_pix [2][1024] = boundary rows in
 * pixels, mean over un-augmented views, clipped like inference.py:90-92; y_cor [1024] = mean of the
 * un-augmented sigmoid(cor).  Needs max_batch >= number of views. */
int hn_model_infer_tta(hn_model* m, const float* x_dev, int in_channels, int flip, const int* shifts_host,
                       int n_rotate, float* y_bon_pix_dev, float* y_cor_dev, void* stream);

/* Room layouts of B panoramas (reference inference.py:65-141, the whole inference() per panorama): x [B][3][512][1024]
 * fp32 on the device; the views of all panoramas (identity, + flip, + one np.roll per shift as in hn_model_infer_tta) run as
 * ONE forward of B * views panoramas, view-major like the reference's augment; the merge leaves y_bon_pix [B][2][1024] and
 * y_cor [B][1024] (device, caller-owned, the values hn_model_infer_tta gives per panorama) and hn_layout_postproc turns them
 * into corners with the remaining arguments.  Needs B * views <= max_batch and views <= 64. */
int hn_model_infer_layout(hn_model* m, const float* x_dev, int B, int in_channels, int flip, const int* shifts_host,
                          int n_rotate, int r_px, float min_v, int force_cuboid, int force_raw, int max_rows,
                          float* y_bon_pix_dev, float* y_cor_dev, float* cor_id_dev, int* n_rows_dev, float* z0_dev,
                          float* z1_dev, int* status_dev, void* stream);

/* Test hook: copies an intermediate result of the LAST forward, converted to the reference's
 * layout, into `out_dev` (fp32).  Stages: "stem" (conv1+bn1+relu, NCHW [B,64,256,512], model.py:73-75),
 * "layer1".."layer4" (NCHW [B,C,H,W], model.py:78-81),
 * "feature" ([B,c_last,256], c_last 1024 for resnet50 and 256 for resnet18; model.py:175-178), "rnn_out" ([256,B,1024], model.py:264; bi-LSTM model only),
 * "mlp_hidden" ([B,256,512], the post-ReLU, pre-dropout hidden layer = output of linear[1], model.py:272; MLP model
 * only).  dims receives the 4 (or 3, last = 0) extents. */
int hn_model_stage(hn_model* m, const char* stage, float* out_dev, long long capacity, int dims[4],
                   void* stream);

/* Options: "tensor_cores" = 1 routes every conv / projection GEMM the wgmma kernel supports
 * through the split-fp16 tensor-core path (default), 0 = exact fp32 CUDA-core kernels everywhere;
 * "fold_downsample" = 1 (default) runs the downsample of each layer's block 0 inside its conv3 in the eval forward on
 * the tensor cores (one GEMM over [t2 | x] with both BN scales folded into the weights, no identity tensor), 0 = a
 * launch of its own and conv3 with a residual;
 * "profile" = 1 turns on per-launch CUDA-event timing (see hn_model_profile_read). */
int hn_model_set_option(hn_model* m, const char* name, int value);

/* With option "profile" = 1 every forward records CUDA-event pairs (on the forward's stream)
 * around each launch; this call waits for them and returns, per op class
 * {0 stem, 1 maxpool, 2 encoder convs, 3 height-reduction convs, 4 upsample/concat tail,
 *  5 LSTM input-projection GEMMs, 6 LSTM recurrence, 7 linear head (with the MLP head: both of its layers, 5 and 6 stay 0)},
 * the accumulated device milliseconds, algorithmic FLOPs and launch counts (arrays of 8). */
int hn_model_profile_read(hn_model* m, double* ms, double* flops, long long* launches, int reset);

/* Synchronises the device and reports device-side failures recorded by earlier asynchronous
 * calls (the grid-barrier time-out of the training backward's cooperative LSTM BPTT kernel). */
int hn_model_check(hn_model* m);

void hn_model_destroy(hn_model* m);

/* ---- misc.panostretch.pano_stretch, image part (reference misc/panostretch.py:81-102) -------- */

/* n images [h][w][c] fp32 (HWC, c in 1..4) on the device, one (kx[i], ky[i]) pair per image
 * (host arrays of n doubles); order 0 (nearest) or 1 (bilinear); scipy legacy 'wrap' semantics. */
int hn_pano_stretch(const float* img_dev, float* out_dev, int n, int h, int w, int c,
                    const double* kx_host, const double* ky_host, int order, void* stream);
/* Same with host images (H2D + kernel + D2H inside), i.e. the numpy-in / numpy-out call of
 * dataset.py:82. */
int hn_pano_stretch_host(const float* img_host, float* out_host, int n, int h, int w, int c,
                         const double* kx_host, const double* ky_host, int order);

/* float64 images (the reference's own CLI feeds float64 0-255, misc/panostretch.py:171): taps, blend and result in double,
 * like scipy returns for a float64 input. */
int hn_pano_stretch_f64(const double* img_dev, double* out_dev, int n, int h, int w, int c,
                        const double* kx_host, const double* ky_host, int order, void* stream);
int hn_pano_stretch_host_f64(const double* img_host, double* out_host, int n, int h, int w, int c,
                             const double* kx_host, const double* ky_host, int order);

/* ---- layout post-processing (reference inference.py:95-141, misc/post_proc.py), one CTA per panorama ----------------
 *
 * y_bon_pix [B][2][1024] (ceiling / floor boundary rows in pixels, clipped) and y_cor [B][1024] (corner probability), fp32
 * on the device, as hn_model_infer_tta leaves them.  r_px = int(round(1024 * r / 2)) of inference.py:108 (Python rounding,
 * host side); min_v: the peak threshold (inference.py:106-107 picks 0 for cuboids, 0.05 otherwise).  force_raw exports the
 * 1024-column raw polygon.  Outputs (device): cor_id [B][max_rows][2] fp32 -- the first n_rows[b] rows are the reference's
 * cor_id (ceiling / floor pairs, normalised by W and H), the rest are zero; max_rows = 2048 holds every result, force_raw
 * included -- n_rows [B], z0 [B] (= 50), z1 [B] and status [B]:
 *   HN_LAYOUT_OK 0, HN_LAYOUT_FALLBACK 1 (the general layout was not a simple polygon; a cuboid replaced it, the
 *   reference's "Generate cuboid as fallback"), and where the reference raises: HN_LAYOUT_ERR_GROUPS 2 (gen_ww's
 *   AssertionError on the number of wall groups: a cuboid without 4 peaks, a general layout without any), HN_LAYOUT_ERR_VOTE
 *   3 (vote's AssertionError: the best run is one value), HN_LAYOUT_ERR_RING 4 (shapely's ValueError: fewer than 3 walls);
 *   HN_LAYOUT_ERR_OVERFLOW 5: the corners do not fit in max_rows rows (nothing is truncated).  n_rows is 0 unless the
 *   status is 0 or 1.  peaks [B][1024] / n_peaks [B] (NULL to skip): the peak columns of the fit that produced the result
 *   (the cuboid's after a fallback), -1 padded.  Top-4 ties in value go to the lower column. */
#define HN_LAYOUT_OK 0
#define HN_LAYOUT_FALLBACK 1
#define HN_LAYOUT_ERR_GROUPS 2
#define HN_LAYOUT_ERR_VOTE 3
#define HN_LAYOUT_ERR_RING 4
#define HN_LAYOUT_ERR_OVERFLOW 5
int hn_layout_postproc(const float* y_bon_pix_dev, const float* y_cor_dev, int B, int r_px, float min_v, int force_cuboid,
                       int force_raw, int max_rows, float* cor_id_dev, int* n_rows_dev, float* z0_dev, float* z1_dev,
                       int* status_dev, int* peaks_dev, int* n_peaks_dev, void* stream);

/* ---- layout evaluation (reference eval_general.py:14-122 test_general / layout_2_depth), on the device --------------
 *
 * B (dt, gt) corner-list pairs, each padded to max_rows (<= 2048) rows of [x, y] fp32 on the device: dt [B][max_rows][2]
 * normalised by W and H, as hn_layout_postproc leaves it (scaled by (1024, 512) in fp32 inside, eval_general.py:157-158),
 * with dt_rows [B]; gt [B][max_rows][2] in pixels, as the label_cor txt files hold them, with gt_rows [B].  dt_status [B]
 * (NULL to skip): the hn_layout_postproc status of each dt; a pair whose status is 2..5 is scored with train.py:309-313's
 * fallback box [k//2 * 1024, 256 - ((k%2)*2 - 1) * 120], k = 0..7, in int64 arithmetic like the reference.  Only 1024 x 512
 * panoramas: test_general hard-codes that size.  Outputs (device, fp64): iou2d, iou3d, rmse, delta_1 [B] and status [B]:
 *   HN_EVAL_OK 0; HN_EVAL_DT_INVALID 1 (the dt floor ring is not a simple polygon: iou2d = iou3d = 0, the reference's
 *   except branches); HN_EVAL_SKIP_GT_INVALID 2 (the gt floor ring is not a simple polygon: the reference skips the pair,
 *   all outputs NaN); and where the reference raises, all outputs NaN: HN_EVAL_ERR_GT_DEPTH 3 (layout_2_depth's assertions
 *   on the gt), HN_EVAL_ERR_COLUMNS 4 (an odd row count, or ceiling and floor columns that differ, eval_general.py:61-62),
 *   HN_EVAL_ERR_RING 5 (fewer than 3 floor corners, or a row count outside 0..max_rows).  layout_2_depth's assertions on the
 *   dt make its depth all zeros (rmse = RMS of the gt depth, delta_1 = 0), as the reference's except does.  Validity is
 *   layout.cu's simple-ring definition on the fp32 floor ring (DESIGN.md sections 8, 9).  depth_out [B][2][512][1024] fp32
 *   (NULL to skip) receives the dt (0) and gt (1) depth maps of every pair whose status is 0, 1 or 2; a dt map on which
 *   layout_2_depth asserts is all zeros. */
#define HN_EVAL_OK 0
#define HN_EVAL_DT_INVALID 1
#define HN_EVAL_SKIP_GT_INVALID 2
#define HN_EVAL_ERR_GT_DEPTH 3
#define HN_EVAL_ERR_COLUMNS 4
#define HN_EVAL_ERR_RING 5
int hn_layout_eval_general(const float* dt_dev, const int* dt_rows_dev, const int* dt_status_dev, const float* gt_dev,
                           const int* gt_rows_dev, int B, int max_rows, double* iou2d_dev, double* iou3d_dev,
                           double* rmse_dev, double* delta_1_dev, int* status_dev, float* depth_out_dev, void* stream);

/* The validation of train.py:301-318 for B panoramas: hn_model_infer_layout with force_raw = 1 and no augmentation, then
 * hn_layout_eval_general of its device outputs against gt [B][max_rows][2] (pixels) / gt_rows [B], a failed inference
 * scored as the fallback box.  Outputs as hn_layout_eval_general's.  Needs B <= max_batch. */
int hn_model_validate(hn_model* m, const float* x_dev, int B, int in_channels, const float* gt_dev, const int* gt_rows_dev,
                      int max_rows, double* iou2d_dev, double* iou3d_dev, double* rmse_dev, double* delta_1_dev,
                      int* status_dev, void* stream);

/* ---- cuboid evaluation (reference eval_cuboid.py:13-145 test / eval_3diou), on the device ---------------------------
 *
 * B (dt, gt) pairs of cuboid corner lists, each padded to max_rows (8..2048) rows of [x, y] fp32 on the device: dt
 * [B][max_rows][2] normalised by W and H, as hn_layout_postproc leaves it (scaled by (1024, 512) in fp32 inside,
 * eval_cuboid.py:192-194), with dt_rows [B]; gt [B][max_rows][2] in pixels, as the label_cor txt files hold them, with
 * gt_rows [B]; z0 [B], z1 [B] fp64 (the json floats of inference.py).  dt_status [B] (NULL to skip): the
 * hn_layout_postproc status of each dt.  Only 1024 x 512 panoramas: eval_3diou and pano_connect_points hard-code that
 * size.  Outputs (device, fp64): ce, pe (percent) and iou3d (percent) [B], and status [B]:
 *   HN_CUBOID_OK 0; where the reference raises, with all outputs NaN, the first exception in its order:
 *   HN_CUBOID_ERR_ROWS 1 (dt or gt is not 8 rows -- a deliberate restriction: with two equal row counts other than 8 the
 *   reference raises IndexError or scores the first 8 rows in PE, which is not a cuboid metric; with two different
 *   counts it raises ValueError), HN_CUBOID_ERR_INDEX 2 (a mark of the label surfaces rounds to a row >= 512 or
 *   < -512, or is NaN: IndexError; also a non-finite column or a boundary no wall samples), HN_CUBOID_ERR_COLUMNS 3
 *   (ceiling and floor columns differ: eval_3diou's AssertionError), HN_CUBOID_ERR_HULL 4 (qhull refuses: an unbounded
 *   or flat region, a NaN corner, a plane through the camera); HN_CUBOID_DT_FAILED 5: dt_status is 2..5, there is no
 *   cuboid to score.  The 3D IoU clips a box by the reference's oriented planes (DESIGN.md section 10). */
#define HN_CUBOID_OK 0
#define HN_CUBOID_ERR_ROWS 1
#define HN_CUBOID_ERR_INDEX 2
#define HN_CUBOID_ERR_COLUMNS 3
#define HN_CUBOID_ERR_HULL 4
#define HN_CUBOID_DT_FAILED 5
int hn_layout_eval_cuboid(const float* dt_dev, const int* dt_rows_dev, const int* dt_status_dev, const double* z0_dev,
                          const double* z1_dev, const float* gt_dev, const int* gt_rows_dev, int B, int max_rows,
                          double* ce_dev, double* pe_dev, double* iou3d_dev, int* status_dev, void* stream);

/* The README's cuboid protocol for B panoramas: hn_model_infer_layout with force_cuboid = 1 (flip / shifts_host /
 * n_rotate / r_px / min_v as there), then hn_layout_eval_cuboid of its device outputs against gt [B][max_rows][2]
 * (pixels) / gt_rows [B], z1 taken from the fp32 inference result.  A failed inference gives HN_CUBOID_DT_FAILED.
 * Outputs as hn_layout_eval_cuboid's.  Needs B * views <= max_batch. */
int hn_model_eval_cuboid(hn_model* m, const float* x_dev, int B, int in_channels, int flip, const int* shifts_host,
                         int n_rotate, int r_px, float min_v, const float* gt_dev, const int* gt_rows_dev, int max_rows,
                         double* ce_dev, double* pe_dev, double* iou3d_dev, int* status_dev, void* stream);

/* ---- dataset.PanoCorBonDataset.__getitem__, image path (reference dataset.py:53, 69-105, 124) ------
 *
 * One fused gather pass per image:  uint8 HWC / 255 -> pano_stretch(kx, ky) -> flip -> roll(dx) -> ** gamma -> CHW:
 * n uint8 images [h][w][3] on the device -> n float32 images [3][h][w] on the device (the network input layout,
 * dataset.py:124).  Host arrays of n entries: kx/ky (dataset.py:71-82; NULL or <= 0: no stretch for that image),
 * flip (dataset.py:88-91; NULL: none), dx (np.roll shift, dataset.py:95-98, 0 <= dx < w; NULL: 0),
 * gamma (exponent p of dataset.py:102-105; NULL or <= 0: none).  The random draws and the corner / boundary label
 * bookkeeping stay with the caller (horizonnet_b200/dataset.py mirrors them). */
int hn_augment(const unsigned char* img_u8_dev, float* out_chw_dev, int n, int h, int w,
               const double* kx_host, const double* ky_host, const int* flip_host, const int* dx_host,
               const float* gamma_host, void* stream);

/* ---- dataset.PanoCorBonDataset.__getitem__, label path (reference dataset.py:56-67, 84-120) -----------------------
 *
 * The training targets of N samples, on the device.  cor0 [N][max_rows][2] fp32: the corner lists as read (pixels,
 * rolled so the ceiling corner with the smallest x comes first, dataset.py:62); cor [N][max_rows][2] fp32: the same
 * corners after the stretch (cor0 itself without one); rows [N]; flip [N] (0 / 1); dx [N] (the np.roll shift,
 * 0 <= dx < 1024, or < 0 for no roll).  max_rows <= 2048, 0 < p_base < 1.  Only 1024 x 512 panoramas.  Outputs (device):
 * y_bon [N][2][1024] fp32 (cor_2_1d of cor, then flipped and rolled), y_cor [N][1][1024] fp32 (p_base ** the circular
 * distance to the nearest corner the camera sees), cor_out [N][max_rows][2] fp32 (cor flipped and rolled; NULL to skip)
 * and occlusion [N][max_rows] (find_occlusion of the ceiling corners of cor0, repeated to both rows of each corner; NULL
 * to skip) -- both written for every sample whose status is not ERR_ROWS or ERR_CORNERS -- and status [N]:
 *   HN_TARGETS_OK 0; where the reference raises, with y_bon and y_cor NaN, the first exception in its order:
 *   HN_TARGETS_ERR_ROWS 1 (an odd row count, or one outside 1..max_rows), HN_TARGETS_ERR_CORNERS 2 (fewer than 3 ceiling
 *   corners: shapely refuses the one-point polyline of the other corners), HN_TARGETS_ERR_BOUNDARY 3 (a boundary no wall
 *   samples: ys.max() of nothing), HN_TARGETS_ERR_OCCLUDED 4 (every corner occluded: dist.min(0) of nothing).
 * The occlusion test is exact on the fp32 floor-plane points (DESIGN.md section 11). */
#define HN_TARGETS_OK 0
#define HN_TARGETS_ERR_ROWS 1
#define HN_TARGETS_ERR_CORNERS 2
#define HN_TARGETS_ERR_BOUNDARY 3
#define HN_TARGETS_ERR_OCCLUDED 4
int hn_train_targets(const float* cor0_dev, const float* cor_dev, const int* rows_dev, const int* flip_dev,
                     const int* dx_dev, int N, int max_rows, double p_base, float* y_bon_dev, float* y_cor_dev,
                     float* cor_out_dev, int* occlusion_dev, int* status_dev, void* stream);

/* ---- misc.pano_lsd_align.rotatePanorama (reference misc/pano_lsd_align.py:125-171, warpImageFast :101-122) ----
 *
 * n images [h][w][c] on the device, float32 (in_is_f64 = 0) or float64 (1) -> n float64 images [h][w][c] rotated by
 * R; rinv_host = 9 doubles, row-major inverse of the reference's R (= vp.T when called with a vanishing-point
 * matrix, pano_lsd_align.py:143).  w must be even (the reference's padding rule, :160-163). */
int hn_rotate_panorama(const void* img_dev, int in_is_f64, double* out_dev, int n, int h, int w, int c,
                       const double* rinv_host, void* stream);

/* ---- kernel-level entry points (unit tests; halo-NHWC activations, see DESIGN.md) ------------ */

/* One convolution + folded BN/bias + optional residual + optional ReLU.
 * in:  [B][H][W + 2*in_halo][Cin]   out: [B][Ho][Wo + 2*out_halo][Cout]   (fp32, device)
 * w_packed: [kh*kw*Cin][Cout], k = (dy*kw + dx)*Cin + c;  scale/shift: [Cout];
 * ph = zero padding along H, pw = circular padding along W (<= in_halo).
 * impl: 0 = exact fp32 CUDA-core kernel, 1 = split-fp16 wgmma tensor-core kernel (split-plane output, merged to fp32),
 * 2 = the same kernel writing fp32 directly (the epilogue of the LSTM input projections, of the raw pass of a train-mode
 * convolution and of the data gradient; no residual), 3 = the narrow height-reduction kernel of resnet18 (conv_narrow.cu:
 * 3x3, stride (2, 1), pad (1, 1), halo 1, Cin -> Cout 32 -> 32, 32 -> 16 or 16 -> 8; split-plane operands made and merged
 * inside; no residual). */
int hn_conv2d(const float* in_dev, int B, int H, int W, int Cin, int in_halo,
              const float* w_packed_dev, const float* scale_dev, const float* shift_dev,
              const float* residual_dev, int Cout, int kh, int kw, int sh, int sw, int ph, int pw,
              int relu, float* out_dev, int out_halo, int impl, void* stream);
/* Backward building blocks of the training step, for unit tests against torch.autograd (train_step.cu):
 * weight + data gradient of one convolution (dz: halo-1 NHWC with circular halo columns; din may be NULL),
 * BatchNorm2d (+identity, ReLU) forward+backward (bn_scratch: 4*C floats, sums: 3*C doubles, C a multiple of 4), and one
 * bidirectional LSTM layer's gate gradients. */
int hn_conv2d_backward(const float* in, int B, int H, int W, int Cin, int in_halo, const float* w_oihw, const float* dz,
                       int Cout, int kh, int kw, int sh, int sw, int ph, int pw, float* din, float* dw_oihw, void* stream);
/* The weight gradient alone on the wgmma kernel (wgrad_tc.cu; in / dz: halo-1 NHWC fp32, Cin and Cout multiples of 64,
 * strides 1 or 2): the planes are made inside.  Returns -1 for a shape that kernel does not take. */
int hn_conv2d_wgrad_tc(const float* in, int B, int H, int W, int Cin, const float* dz, int Cout, int kh, int kw, int sh,
                       int sw, int ph, int pw, float* dw_oihw, void* stream);
/* Host-side plan of that kernel for one shape (no GPU work; sms = SM count to plan for): plan[10] = tile columns, rows per
 * tile, tiles per row, box rows, images per tile, pixel tiles (64 pixels each), tiles per slice, slices, work items per slice,
 * CTAs.  -1 for a shape the kernel does not take. */
int hn_wgrad_tc_plan(int B, int H, int W, int Cin, int Cout, int kh, int kw, int sh, int sw, int ph, int pw, int sms, int plan[10]);
/* Host-side plan of the fp32 CUDA-core weight gradient (hn_conv2d_backward; the training step's weight gradients the
 * tensor-core kernel does not take) for one shape (no GPU work; sms = SM count to plan for; dz has out_halo): plan[5] =
 * kernel (2: 128 x 128 tiles, 1: 64 x 64 with 16-byte input loads, 0: 64 x 64 scalar loads for Cin % 4 != 0), K tiles,
 * Cout tiles, pixel slices, pixels per slice.  -1 for a shape it does not take. */
int hn_wgrad_f32_plan(int B, int H, int W, int Cin, int in_halo, int Cout, int kh, int kw, int sh, int sw, int ph, int pw,
                      int out_halo, int sms, int plan[5]);
/* Returns 1: the training step runs the weight gradients on that kernel wherever option "tensor_cores" is on and the shape fits. */
int hn_wgrad_tc_enabled(void);
/* The data gradient on the tensor cores exactly as the training step computes it (zero-dilated dz for a strided conv,
 * power-of-two scaled planes of dz, flipped weights as planes, the transposed conv with fp32 output) and ADDED to din:
 * dz [B][Ho][Wo+2][Cout] and din [B][H][W+2][Cin], halo-1 NHWC fp32 with circular halo columns; w_oihw: the forward
 * weights [Cout][Cin][kh][kw].  Returns -1 for a shape the tensor-core kernel does not take. */
int hn_conv2d_dgrad_tc(int B, int H, int W, int Cin, const float* w_oihw, const float* dz, int Cout, int kh, int kw, int sh,
                       int sw, int ph, int pw, float* din, void* stream);
/* Host-side launch plan of the tensor-core convolution (no GPU work; sms = SM count to plan for) for the conv hn_conv2d
 * impl 1 (out_f32 = 0) or 2 (out_f32 = 1) would run, with or without a residual.  plan[18] = kernel (1 gemm_tc_kernel,
 * 0 conv_tc_kernel), BN, mode (0 GEMM rows, 1 conv rows), M (rows), tile columns, rows per tile, tiles per output row,
 * rowbox (1: conv-row tiles of several output rows, which one box per plane loads), box rows, box images, dx reuse,
 * parity (stride 2 along W), K chunks, chunks per accumulation segment, L2 prefetch distance, tiles along Cout, tiles,
 * CTAs.  -1 for a shape the kernel does not take. */
int hn_conv_tc_plan(int B, int H, int W, int Cin, int in_halo, int Cout, int kh, int kw, int sh, int sw, int ph, int pw,
                    int out_halo, int out_f32, int has_residual, int sms, int plan[18]);
/* Host-side tile plan of the fp32 CUDA-core convolution (hn_conv2d impl 0; no GPU work; sms = SM count to plan for):
 * plan[4] = output pixels per tile (BM), output channels per tile (BN), tiles along the pixels, tiles along Cout.
 * -1 for a shape that kernel does not take. */
int hn_conv_f32_plan(int B, int H, int W, int Cin, int in_halo, int Cout, int kh, int kw, int sh, int sw, int ph, int pw,
                     int out_halo, int sms, int plan[4]);
/* The same plan (same 18 fields) for the eval-mode conv3 of a bottleneck's block 0 with its downsample folded in:
 * relu([t2 | x at every stride-th pixel] . W + shift), x [B][H][W][Cin] (halo 1), t2 and the output [B][H/s][W/s][Cmid],
 * [Cout]; K chunks = (Cmid + Cin) / 64, the first Cmid / 64 over t2.  -1 for a shape the kernel does not take. */
int hn_conv_tc_fold_plan(int B, int H, int W, int Cin, int Cmid, int Cout, int stride, int sms, int plan[18]);
/* That convolution on the tensor cores with fp32 tensors (unit tests): t2 / x / out halo-1 NHWC fp32 with circular halo
 * columns in the geometry above, w the folded weights [Cout][Cmid + Cin], shift [Cout]. */
int hn_conv_tc_fold(const float* t2, const float* x, int B, int H, int W, int Cin, int Cmid, int Cout, int stride,
                    const float* w, const float* shift, float* out, void* stream);
/* The fused layer1 bottleneck kernel, conv2 + conv3 (unit tests): in = conv1 output [B][H][W][64], out [B][H][W][C3],
 * halo-1 NHWC fp32; w2 OIHW [64][64][3][3] with BN scale2 / shift2.  Exactly one of res and x is non-NULL:
 * res = the block's identity [B][H][W][C3] (layer1.1, 1.2), w3 the conv3 weights OIHW [C3][64][1][1] with BN scale3 /
 * shift3; or x = the block input [B][H][W][64] with the downsample folded in (layer1.0), w3 the folded conv3 weights
 * [C3][64 + 64] with shift3 (scale3 is not read). */
int hn_bott_tc(const float* in, const float* res, const float* x, int B, int H, int W, const float* w2, const float* scale2,
               const float* shift2, const float* w3, const float* scale3, const float* shift3, int C3, float* out,
               void* stream);
int hn_bn_forward_backward(const float* z, int B, int H, int W, int C, const float* gamma, const float* beta,
                           float* running_mean, float* running_var, double factor, int train, int relu, const float* res,
                           float* y, const float* dy, float* dz, float* dres, float* dgamma, float* dbeta, float* bn_scratch,
                           double* sums, void* stream);
/* One bidirectional LSTM layer's gate gradients from its saved forward tensors: xp [T][B][4096] (input projection + biases),
 * hout [T][B][1024], whf / whb: W_hh [2048][512] per direction, dout [T][B][1024] -> dgates [2][T][B][2048] (d xp).
 * persistent = 0: BPTT as one launch per time step; 1: the single cooperative launch the training step makes (staged dG in
 * shared memory for B <= 16), or -1 with "not supported" when the device cannot co-schedule its 128 CTAs (no fallback).
 * scratch, in 4-byte words, with R = T*B: hprev 2*R*512 | gates 2*R*2048 | cell 2*R*512 | dc carry 2*B*512 |
 * W_hh^T 2*512*2048 | ones 4096 | zeros 4096 | barrier counter (uint) | error flag (int; zeroed here before a persistent launch,
 * 1 after a grid-barrier time-out). */
int hn_lstm_layer_backward(const float* xp, const float* hout, const float* whf, const float* whb, const float* dout, int T,
                           int B, int persistent, float* dgates, float* scratch, void* stream);

/* One bidirectional LSTM layer recurrence: xproj [T][B][4096] (input projection + both biases,
 * column = dir*2048 + gate*512 + unit), w_hh_* [2048][512] (PyTorch layout), out [T][B][1024].
 * Asynchronous on `stream`, like hn_conv2d; fails with "not supported" on a device that cannot
 * co-schedule two of the recurrence's 16-CTA clusters. */
int hn_lstm_layer(const float* xproj_dev, const float* w_hh_fwd_dev, const float* w_hh_bwd_dev,
                  float* out_dev, int T, int B, void* stream);
/* Host-side launch layout of hn_lstm_layer for T steps of B columns on a device that co-schedules max_clusters of the
 * recurrence's 16-CTA clusters (max_clusters <= 0: the current device's count, the cached answer hn_lstm_layer uses; no GPU
 * work otherwise).  plan[7] = max_clusters used, 8-column groups, groups per cluster (1 or 2), clusters (both directions),
 * groups in the last cluster of a direction, columns in the last group, waves (ceil(clusters / max_clusters)).
 * -1 for T < 1, B < 1 or max_clusters < 2 (the device hn_lstm_layer refuses). */
int hn_lstm_plan(int T, int B, int max_clusters, int plan[7]);

/* Kernels at the two ends of the network, each through the library function the model calls (unit tests; asynchronous on
 * `stream`, scratch from cudaMallocAsync on it).  Halo-1 NHWC fp32 tensors unless said otherwise.
 * Stem: x [B][in_channels >= 3][512][1024] in [0, 1] (channels past 3 are not read), w OIHW [64][3][7][7], scale / shift
 * [64] -> out [B][256][514][64].  impl 0: stem_kernel (fp32; writes the wrap columns too); impl 1: stem_pack_kernel +
 * stem_tc_kernel (split-fp16 wgmma; interior columns only).  relu = 0 gives the raw conv * scale + shift of the training
 * step's statistics pass (with ones / zeros: the same weight planes and epilogue constants it runs with). */
int hn_stem(const float* x_nchw, int B, int in_channels, const float* w_oihw, const float* scale, const float* shift,
            int relu, int impl, float* out, void* stream);
/* MaxPool2d(3, 2, 1) with -inf padding: in [B][H][W+2][C] -> out [B][(H+1)/2][(W+1)/2+2][C], C a multiple of 4;
 * out_planes = 1 writes split planes (fp16 hi / lo of v * 2^-4, hi plane first) in the same bytes instead of fp32. */
int hn_maxpool(const float* in, int B, int H, int W, int C, int out_planes, float* out, void* stream);
/* Its backward: each output gradient dp is ADDED (atomically) to the first maximum of its window in scan order; dx has x's
 * geometry and its halo columns are not written. */
int hn_maxpool_backward(const float* x, const float* dp, int B, int H, int W, int C, float* dx, void* stream);
/* The feature sequence (model.py:152-155, 175-178, 263) of backbone "resnet50" (c_last 1024) or "resnet18" (256) from the
 * four height-reduction outputs ghc[s] [B][8 >> s][(256 >> s) + 2][C_s], C_s = the layer's channels / 8, into
 * seq [256][B][c_last]; planes = 1: inputs and output are split planes.  The backward ADDS the adjoint of d seq to the
 * interior columns of dghc (atomically). */
int hn_feature_sequence(const char* backbone, int B, const float* const ghc[4], int planes, float* seq, void* stream);
int hn_feature_sequence_backward(const char* backbone, int B, const float* dseq, float* const dghc[4], void* stream);
/* Linear(K -> 12) head, K = 1024 (bi-LSTM) or 512 (MLP), over rows t*B + b of rnn [T][B][K] with w [12][K], b [12]:
 * output o = 4s + k of row (t, b) goes to column 4t + k of cor [B][1][1024] (s = 0) or bon [B][2][1024] (s = 1, 2).  The
 * backward writes drnn [T][B][K], dw [12][K] and db [12]. */
int hn_linear_head(const float* rnn, const float* w, const float* b, float* bon, float* cor, int T, int B, int K,
                   void* stream);
int hn_linear_head_backward(const float* dbon, const float* dcor, const float* rnn, const float* w, float* drnn, float* dw,
                            float* db, int T, int B, int K, void* stream);
/* out[c] = sum over the rows of x [rows][cols] (the bias gradients of the LSTM and the MLP head). */
int hn_col_sum(const float* x, long long rows, int cols, float* out, void* stream);
/* The stem's weight-gradient operand: x as above -> the normalised input, halo-3 NHWC [B][512][1030][3]. */
int hn_stem_input(const float* x_nchw, int in_channels, int B, float* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* HORIZONNET_B200_H */
