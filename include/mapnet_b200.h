/* mapnet_b200.h -- C ABI of the H100-native MapNet/PoseNet training hot path.
 *
 * Drop-in boundary (SURVEY.md section 8b).  The reference (NVlabs/geomapnet) is pure
 * Python on PyTorch: it has NO native FFI for this path, so these entry points
 * are the contract a maintainer binds (ctypes stub in INTEGRATION.md) behind the
 * reference's own Python surface:
 *
 *   reference call site                               entry point that replaces it
 *   -----------------------------------------------   ------------------------------
 *   models/posenet.py:65-73  PoseNet.forward          mapnet_forward
 *   models/posenet.py:93-97  MapNet.forward           mapnet_forward (T folded into B)
 *   common/train.py:356      loss.backward() (trunk)  mapnet_backward
 *   common/criterion.py:42-52,76-109,137-184          mapnet_loss_fwd_bwd
 *   common/pose_utils.py:234-260 calc_vos*            mapnet_loss_fwd_bwd (folded in)
 *   common/optimizer.py:21-23 + train.py:357-359      mapnet_adam_step (+ mapnet_sqnorm)
 *   common/optimizer.py:16-27 (sgd, rmsprop)          mapnet_sgd_step_dev / mapnet_rmsprop_step_dev
 *   models/posenet.py:37-63  parameter layout         mapnet_param_count / mapnet_param_info
 *
 * Conventions: every pointer is a DEVICE pointer unless named host_*; all
 * tensors are contiguous fp32 in the reference's layouts (images NCHW
 * [B,3,H,W]; poses [..,6] = xyz + log-quaternion).  Functions enqueue work on
 * `stream` (a cudaStream_t passed as void*) and return 0 on success; non-zero
 * means failure and mapnet_last_error() (thread-local) describes it.  No
 * exception crosses this boundary; the library never frees caller memory.
 * Handles are not thread-safe (one Python thread drives one GPU, like nn.Module).
 * There is no CPU fallback: without a CUDA device every call fails.
 */
#ifndef MAPNET_B200_H_
#define MAPNET_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct mapnet_trunk mapnet_trunk_t;

/* precision of the conv engines / stored activations */
#define MAPNET_PREC_FP32 0      /* fp32 CUDA-core implicit GEMM: strict 1e-4 parity mode            */
#define MAPNET_PREC_BF16 1      /* wgmma tensor-core implicit GEMM, bf16 operands, fp32 accumulate */
#define MAPNET_PREC_BF16_SIMT 2 /* bf16 storage + CUDA-core fp32 math: cross-check of mode 1         */
#define MAPNET_PREC_TC_SPLIT 3  /* wgmma strict mode: fp32 conv outputs, conv operands as split fp16 hi/lo planes,\
                                   4 MMAs per product, fp32 accumulate -- meets the 1e-4 parity bar on tensor cores */
#define MAPNET_PREC_FP8 4       /* inference engine only (mapnet_infer_*): e4m3 conv operands, calibrated scales */

/* criterion modes (common/criterion.py) */
#define MAPNET_LOSS_POSENET 0    /* PoseNetCriterion      pred [N,6],    targ [N,6]        */
#define MAPNET_LOSS_MAPNET 1     /* MapNetCriterion       pred [N,T,6],  targ [N,T,6]      */
#define MAPNET_LOSS_ONLINE 2     /* MapNetOnlineCriterion pred [N,2T,6], targ [N,2T-1,6]   */
#define MAPNET_LOSS_ONLINE_GPS 3 /* ... gps_mode=True     pred [N,2T,6], targ [N,2T,6]     */

const char* mapnet_last_error(void);
int mapnet_abi_version(void);

/* ---- trunk handle: owns only scratch (activation arena, packed weights, BN partials).
 * max_B == 0 creates a spec-only handle (parameter table queries, no device needed). */
int mapnet_trunk_create(mapnet_trunk_t** out, int max_B, int H, int W, int feat_dim, int precision);
int mapnet_trunk_destroy(mapnet_trunk_t* h);

/* ---- parameter table (state_dict order of the reference PoseNet, 222 entries) */
/* kind: 0 = trainable fp32 in params_flat, 1 = fp32 buffer (BN running stats) in
 * bufs_flat, 2 = int64 num_batches_tracked (offset = index in a separate int64 vector) */
int mapnet_param_count(mapnet_trunk_t* h);
int mapnet_param_info(mapnet_trunk_t* h, int i, char* host_name, int name_cap, int* host_kind, int* host_ndim,
                      int64_t* host_shape4, int64_t* host_offset);
/* Element order of entry i inside its flat buffer.  0: torch's contiguous order of the entry's shape.  1: a conv weight
 * of shape [Co,Ci,KH,KW] stored as [Co][KH][KW][Ci] -- the K-major order the wgmma engines read (fprop operand) and
 * accumulate (wgrad), so neither direction needs a transposing pass per step.  To PyTorch that memory is the same
 * [Co,Ci,KH,KW] tensor in torch.channels_last strides: flat[off:off+n].view(Co,KH,KW,Ci).permute(0,3,1,2) -- logical
 * indexing, state_dict()/load_state_dict() and the reference's optimizer code are unaffected.  Every conv except the stem
 * (7x7, 3 input channels) has layout 1; -1 on a bad index.  (ABI version 2.) */
int mapnet_param_layout(mapnet_trunk_t* h, int i);
int64_t mapnet_params_numel(mapnet_trunk_t* h); /* floats in params_flat / grads_flat (padded) */
int64_t mapnet_bufs_numel(mapnet_trunk_t* h);   /* floats in bufs_flat                          */

/* ---- forward: x [B,3,H,W] -> pred [B,6].  training!=0: BN batch statistics + running-
 * stat update in bufs_flat; activations are kept for mapnet_backward.  droprate>0
 * applies dropout with a counter-based mask from (seed, step); step == UINT64_MAX uses and
 * advances a device-side counter owned by the handle (CUDA-graph capturable). */
int mapnet_forward(mapnet_trunk_t* h, const float* x, const float* params_flat, float* bufs_flat, int B,
                   int training, float droprate, uint64_t seed, uint64_t step, float* pred, void* stream);

/* ---- backward of the last training forward: dpred [B,6] -> every parameter gradient,
 * written (not accumulated) into grads_flat at the offsets of params_flat.
 * filter_nans: the NaN filter of the models/posenet.py:28-34 hook on fc_wpqr (NaN entries of that Linear's bias /
 * input / weight gradients become 0: a NaN in dpred[b,3+j] wipes row j of d W_wpqr and sample b's rotation
 * half of the gradient into the trunk). */
int mapnet_backward(mapnet_trunk_t* h, const float* dpred, const float* params_flat, float* grads_flat,
                    int filter_nans, void* stream);

/* The same backward pass in three parts, called in order 0, 1, 2 with the same arguments: after part k returns
 * (asynchronously, on `stream`) the gradients in grads_flat[lo_k, hi_k) (mapnet_grad_part_range) are final, so a
 * data-parallel caller can enqueue their allreduce on another stream while the next part computes.
 * Part 0 = head + layer4 (64 % of the parameters after ~20 % of the backward FLOPs), 1 = layer3, 2 = layer2, layer1, stem.
 * (The reference is single-GPU, common/train.py:193-196; this is the overlap hook of SURVEY.md section 8e.) */
int mapnet_backward_part(mapnet_trunk_t* h, int part, const float* dpred, const float* params_flat, float* grads_flat,
                         int filter_nans, void* stream);
int mapnet_grad_part_range(mapnet_trunk_t* h, int part, int64_t* host_lo, int64_t* host_hi);

/* Which trainable entries (kind 0 of the parameter table, in table order) need a gradient. n must equal the number
 * of kind-0 entries. Applies to every later mapnet_backward / mapnet_backward_part on this handle, until set again.
 * Default: all 1 (the full backward pass). Host-only, no launch: a CUDA graph captures the schedule of the mask in force.
 * The pass then skips the weight gradient of every frozen conv and head layer, and every input gradient below the
 * lowest layer that trains (torch's requires_grad_(False) semantics). The grads_flat entries of frozen parameters are 0.
 * A frozen BatchNorm still passes its input gradient through; its running statistics follow the forward as before.
 * (Added in ABI version 2, backward compatible.) */
int mapnet_trunk_set_trainable(mapnet_trunk_t* h, const uint8_t* host_mask, int n);

/* ---- fused criterion forward+backward.  s4 = device (sax,saq,srx,srq).
 * Outputs: loss[1], dpred (same shape as pred), ds4[4] = d loss / d s4. */
int mapnet_loss_fwd_bwd(int mode, const float* pred, const float* targ, int N, int T_pred, int T_targ,
                        const float* s4, float* loss, float* dpred, float* ds4, void* stream);

/* ---- every batch loss of a validation pass in one launch (csrc/loss.cu; geomapnet_b200.inference.validate).
 * Item i of the pass (loader order) is the window of rows pred_rows[i*T + t] of pred [n_pred][6] and targ_rows[i*T + t]
 * of targ [n_targ][6], t < T; batch b holds items [batch_items[b], batch_items[b+1]).  losses[b] is bit for bit the
 * loss mapnet_loss_fwd_bwd returns for batch b gathered into [N_b][T][6] (same per-pose core, thread mapping and
 * reduction tree, one block per batch, no atomics).  mode: posenet (0, T = 1) or mapnet (1).  pred, targ, s4 (device
 * sax, saq, srx, srq) and losses [n_batches] are device memory; pred_rows, targ_rows and batch_items [n_batches + 1]
 * are HOST int32 arrays, checked (bounds, batch_items[0] = 0 and strictly increasing) and copied before the call
 * returns.  Nothing is launched when a check fails. */
int mapnet_batch_losses(int mode, const float* pred, int n_pred, const float* targ, int n_targ, const int32_t* pred_rows,
                        const int32_t* targ_rows, int T, const int32_t* batch_items, int n_batches, const float* s4,
                        float* losses, void* stream);

/* ---- optimizer step on flat buffers (torch.optim.Adam semantics, L2 weight decay).
 * grad_scale multiplies the gradient first (1/world_size after a sum-allreduce).
 * sqnorm: device scalar holding the squared global grad norm (mapnet_sqnorm) to
 * apply clip_grad_norm_(max_norm), or NULL for no clipping. */
int mapnet_sqnorm(const float* g, int64_t n, float* scratch1024, float* out_sq, void* stream);
int mapnet_adam_step(float* p, const float* g, float* exp_avg, float* exp_avg_sq, int64_t n, float lr,
                     float beta1, float beta2, float eps, float weight_decay, int64_t step, float grad_scale,
                     const float* sqnorm, float max_norm, void* stream);

/* CUDA-graph capturable variant: the step count lives in device memory (*step_counter is
 * incremented, then used for the bias corrections), so a captured launch stays correct
 * on every replay. */
int mapnet_adam_step_dev(float* p, const float* g, float* exp_avg, float* exp_avg_sq, int64_t n, float lr,
                         float beta1, float beta2, float eps, float weight_decay, int32_t* step_counter,
                         float grad_scale, const float* sqnorm, float max_norm, void* stream);

/* torch.optim.SGD / torch.optim.RMSprop semantics (L2 weight decay, maximize=False) on flat buffers, CUDA-graph
 * capturable: the learning rate is read from the device float *lr_dev at run time (a schedule writes it between
 * replays), and *step_counter (device int32, may be NULL unless an SGD momentum buffer is given) is incremented
 * first -- SGD's step 1 sets momentum_buf = d instead of momentum*buf + (1-dampening)*d.  grad_scale, sqnorm and
 * max_norm as for mapnet_adam_step.  State buffers a configuration does not use are NULL: momentum_buf exactly when
 * momentum == 0, grad_avg unless RMSprop is centered.  (Added in ABI version 2, backward compatible.) */
int mapnet_sgd_step_dev(float* p, const float* g, float* momentum_buf, int64_t n, const float* lr_dev, float momentum,
                        double dampening, float weight_decay, int nesterov, int32_t* step_counter, float grad_scale,
                        const float* sqnorm, float max_norm, void* stream);
int mapnet_rmsprop_step_dev(float* p, const float* g, float* square_avg, float* grad_avg, float* momentum_buf,
                            int64_t n, const float* lr_dev, double alpha, float eps, float weight_decay, float momentum,
                            int32_t* step_counter, float grad_scale, const float* sqnorm, float max_norm, void* stream);

/* ---- GPU-side input pipeline (SURVEY.md section 8 row f2; geomapnet_b200/csrc/preprocess.cu).
 * Replaces the per-image CPU transform stack of /root/reference/scripts/train.py:119-128 (and eval.py:97-101):
 * transforms.Resize(size) [Pillow bilinear on 8-bit images, bit-exact] [-> ColorJitter, train.py:121-126, bit-exact]
 * -> ToTensor -> Normalize(mean, std), and the frame gather of the MF / MFOnline tuple datasets
 * (dataset_loaders/composite.py:60-97,117-126).
 * One plan per input size; frames are uint8 [n][Hin][Win][3] in device memory, the result float32 [n][3][Hout][Wout]
 * (what PoseNet.forward takes).  mean3 / std3 are HOST pointers to 3 floats (stats.txt row 0, sqrt of row 1). */
typedef struct mapnet_preprocess mapnet_preprocess_t;
int mapnet_preprocess_create(mapnet_preprocess_t** out, int Hin, int Win, int size, int max_images);
int mapnet_preprocess_output_size(const mapnet_preprocess_t* h, int* Hout, int* Wout);
int mapnet_preprocess_run(mapnet_preprocess_t* h, const void* img_nhwc_u8, int n, const float* mean3, const float* std3,
                          float* out_nchw, void* out_u8_or_null /* the resized uint8 image, tests */, void* stream);
/* frame_index_dev: NULL, or n int32 in DEVICE memory -- output image i is cut from frame frame_index[i] of the sequence
 * at img_nhwc_u8 (the tuple gather).  jitter_dev: NULL, or n records {int32 order[4]; float factor[4]} in DEVICE memory:
 * the adjustments (0 brightness, 1 contrast, 2 saturation, 3 hue -- torchvision's fn_idx) in the order they are applied
 * and their factors indexed by adjustment id, i.e. one ColorJitter.get_params() draw per image. */
int mapnet_preprocess_run_ex(mapnet_preprocess_t* h, const void* img_nhwc_u8, int n, const int32_t* frame_index_dev,
                             const void* jitter_dev, const float* mean3, const float* std3, float* out_nchw,
                             void* out_u8_or_null, void* stream);
int mapnet_preprocess_destroy(mapnet_preprocess_t* h);

/* ---- device-resident training set (geomapnet_b200/csrc/loader.cu; Python: geomapnet_b200.data.DeviceDataset).
 * Resize(size) is deterministic and comes before ColorJitter in the reference's transform stack, so its uint8 output is
 * computed once per frame and kept: a cache of n_frames frames [Hout][Wout][3] in device memory.
 * ingest: frames_nhwc_u8 (DEVICE memory, n <= chunk frames [Hin][Win][3]) are resized into cache slots [first, first + n).
 *   Chunks of one cache are ingested on one stream.
 * assemble: one training batch of n images, one kernel launch (two with ColorJitter: contrast needs the luma sum first):
 *   image i is cache frame frame_index[i], [ColorJitter record i applied,] ToTensor + Normalize -> out_nchw float32
 *   [n][3][Hout][Wout] (DEVICE memory, e.g. the static input of a captured training step).  The same launch writes n_targ
 *   target rows of 6 floats into targ_out (DEVICE): row k is poses_dev row targ_rows[2k] when targ_rows[2k+1] == -1,
 *   otherwise calc_vo_logq_safe(poses row targ_rows[2k], poses row targ_rows[2k+1]) (common/pose_utils.py:276-288; the
 *   VO targets of MFOnline).  poses_dev: [n_poses][6] float32 in DEVICE memory.
 *   frame_index, jitter (NULL, or n records as for mapnet_preprocess_run_ex) and targ_rows are HOST arrays, checked and
 *   copied before the call returns; mean3 / std3 are HOST pointers to 3 floats.  Nothing is launched when a check fails. */
typedef struct mapnet_frame_cache mapnet_frame_cache_t;
int mapnet_frame_cache_create(mapnet_frame_cache_t** out, int n_frames, int Hin, int Win, int size, int chunk,
                              int max_images, int max_targ);
int mapnet_frame_cache_ingest(mapnet_frame_cache_t* h, const void* frames_nhwc_u8, int first, int n, void* stream);
int mapnet_frame_cache_assemble(mapnet_frame_cache_t* h, int n, const int32_t* frame_index, const void* jitter,
                                const float* poses_dev, int n_poses, const int32_t* targ_rows, int n_targ,
                                const float* mean3, const float* std3, float* out_nchw, float* targ_out, void* stream);
int mapnet_frame_cache_destroy(mapnet_frame_cache_t* h);

/* ---- evaluation windows (csrc/loader.cu; geomapnet_b200.inference.evaluate_sequence): scripts/eval.py:163-170 for a
 * whole sequence whose frames went through the network once each.  For every window slot r < n_rows:
 *   pred7[r] = (t, qexp(log q)) of pred6[slot[r]],  targ7[r] = the same of poses[frame[r]]
 * and for every VO k < n_vo: vos7[k] = (t, qexp(log q)) of calc_vo_logq_safe(vo_poses[a], vo_poses[b]) with
 * (a, b) = vo_rows[2k], vo_rows[2k+1] (common/pose_utils.py:276-304; the same float32 arithmetic as the MFOnline VO
 * targets of mapnet_frame_cache_assemble).  qexp is mapnet_pose_post's, bit for bit; translations are not
 * un-normalised.  pred6 [n_pred][6], poses / vo_poses [n_poses][6] (float32) and the float64 outputs are device memory;
 * frame, slot and vo_rows are HOST int32 arrays, checked and copied before the call returns.  n_vo = 0: no VOs
 * (vo_poses, vo_rows, vos7 may be NULL).  Nothing is launched when a check fails. */
int mapnet_eval_windows(const float* pred6, int n_pred, const float* poses, const float* vo_poses, int n_poses,
                        const int32_t* frame, const int32_t* slot, int n_rows, const int32_t* vo_rows, int n_vo,
                        double* pred7, double* targ7, double* vos7, void* stream);

/* ---- batched inference post-processing + pose-graph optimisation (SURVEY.md section 8 row f3; csrc/pgo.cu).
 * mapnet_pose_post: scripts/eval.py:163-181 for n poses at once -- pred6 = (t, log q) float32 -> out7 = (t * pose_s +
 * pose_m, qexp(log q)) float64; pose_m3 / pose_s3 are HOST pointers (pose_stats.txt) or NULL (keep the translations).
 * mapnet_pgo_optimize: common/pose_utils.py:458-804 (PoseGraph / PoseGraphFC.optimize behind optimize_poses) for
 * n_windows windows of N <= 16 poses in one launch: poses [n_windows][N][7], vos [n_windows][E][7] (E = N-1, or N(N-1)/2
 * pairs i<j row-major when fc_vos), quaternions (w,x,y,z), fp64, device pointers; sax..srq are the covariances
 * eval.py passes; n_iters = 10 in the reference.  flags bit 0: 0 = the reference's linear solve taken literally
 * (pose_utils.py:605-608 calls solve_triangular(R.T, -b) with scipy's default lower=False, which reads only the diagonal
 * of R': x = R^-1 diag(R)^-1 (-b)), 1 = the Gauss-Newton step H^-1 (-b).  *status_dev (device int, may be NULL) is set
 * to 1 when a window's normal matrix is not positive definite (scipy's cholesky raises there). */
int mapnet_pose_post(const float* pred6, double* out7, int64_t n, const double* pose_m3, const double* pose_s3, void* stream);
int mapnet_pgo_optimize(const double* poses, const double* vos, double* out, int n_windows, int N, int fc_vos,
                        double sax, double saq, double srx, double srq, int n_iters, int flags, int* status_dev, void* stream);

/* ---- eval-mode inference engine (csrc/infer.cu): a frozen snapshot of a PoseNet / MapNet trunk for
 * scripts/eval.py-style prediction.  mapnet_infer_load copies the weights (packed fprop operands only), the eval-mode
 * BatchNorm scale / shift (computed from the running statistics exactly as mapnet_forward(training = 0) does) and the
 * head out of params_flat / bufs_flat; the engine never reads those buffers again.  mapnet_infer_forward then runs the
 * eval forward with every BatchNorm, residual add and ReLU fused into its conv's epilogue: one launch per conv plus the
 * stem operand, the pool and the head.  Dropout follows mapnet_forward (the reference's F.dropout is active at eval when
 * droprate > 0): the same mask for the same (seed, step); step == UINT64_MAX takes the engine's device step counter
 * (graph-capturable).  Precisions: MAPNET_PREC_BF16 and MAPNET_PREC_TC_SPLIT only.  Argument errors (precision, B >
 * max_B, a forward before a load) return non-zero before anything is allocated or launched.
 * MAPNET_PREC_FP8 (inference only): every conv but the stem runs on e4m3 operands -- weights with a power-of-two scale per
 * output channel (taken at load), activations with one power-of-two scale per tensor (the pool output, every block's h
 * and output: 33 at ResNet-34).  mapnet_infer_calibrate takes those scales from frames x [B,3,H,W] (B <= max_B),
 * progressively over the engine's own schedule; it is required after every load and before the next forward (a forward
 * without it fails before any launch) and rewrites the scales in place, so captured graphs stay valid.  It fails on
 * bf16 / tc_split handles.  mapnet_infer_act_scales copies the activation scales in schedule order to host memory and
 * returns 0 (cap: room in floats).
 * mapnet_infer_arena_bytes: host-only, the activation bytes a handle of these shapes allocates (< 0 on bad arguments);
 * fp8 adds the scale slots. */
typedef struct mapnet_infer mapnet_infer_t;
int mapnet_infer_create(mapnet_infer_t** out, int max_B, int H, int W, int feat_dim, int precision);
int mapnet_infer_load(mapnet_infer_t* h, const float* params_flat, const float* bufs_flat, void* stream);
int mapnet_infer_forward(mapnet_infer_t* h, const float* x, int B, float droprate, uint64_t seed, uint64_t step,
                         float* pred, void* stream);
int64_t mapnet_infer_arena_bytes(int max_B, int H, int W, int precision);
int mapnet_infer_destroy(mapnet_infer_t* h);
int mapnet_infer_calibrate(mapnet_infer_t* h, const float* x, int B, void* stream);
int mapnet_infer_act_scales(mapnet_infer_t* h, float* host_out, int cap);

/* ---- measurement support (bench.py): number of kernels this library has launched so
 * far in this process, and per-class conv timing with CUDA events on the launching
 * stream (class 0 fprop, 1 dgrad, 2 wgrad; algorithmic FLOPs of each launch summed). */
unsigned long long mapnet_launch_count(void);
int mapnet_profile(mapnet_trunk_t* h, int enable);
int mapnet_profile_read(mapnet_trunk_t* h, double* host_ms3, double* host_flops3, int* host_launches3);

/* ---- unit entry points used by the parity tests (tests/test_gpu_kernels.py) */
int mapnet_test_conv(int precision, int kind /*0 fprop 1 dgrad 2 wgrad*/, int B, int Hi, int Wi, int Ci, int Co,
                     int k, int stride, const void* in0, const void* in1, const void* wmat, void* out, void* stream);
/* mapnet_test_conv's tensor-core engines (precision bf16 or tc_split) plus, for dgrad, a residual added before the
 * store (out's type and shape; it may be `out` itself, as in the trunk's strict-mode downsampling blocks), and for
 * strict-mode dgrad / wgrad a gradient out-scale multiplied into the accumulators before they are stored (uploaded to
 * a device scalar; 0 = none).  Arguments are checked before the device is touched. */
int mapnet_test_conv_ex(int precision, int kind, int B, int Hi, int Wi, int Ci, int Co, int k, int stride,
                        const void* in0, const void* in1, const void* wmat, const void* residual, float out_scale,
                        void* out, void* stream);

/* host-only: the tile / parity-class / filter-tap plan of the tensor-core engines for one conv, as JSON
 * (tests/test_tc_plan.py replays it on the CPU against torch's convolutions; kind 0 fprop, 1 dgrad, 2 wgrad).
 * flags: bit 0 folds the downsample shortcut into a 3x3/s2 dgrad; bit 1 describes the strict-mode (tc_split) plan. */
int mapnet_test_plan_describe(int kind, int B, int Hi, int Wi, int Ci, int Co, int k, int stride, int flags,
                              char* buf, int cap);

/* the tensor-core dgrad of a downsampling BasicBlock's two input-side convs in ONE launch, as the trunk runs it:
 * dx = dgrad(conv1 3x3/s2/p1; dy1, w1_dg [Ci][3][3][Co]) + dgrad(downsample 1x1/s2; dy2, w2_dg [Ci][Co]), all bf16 NHWC
 * (torchvision BasicBlock.forward's two uses of the block input, /root/reference/models/posenet.py:66). */
int mapnet_test_dgrad_shortcut(int B, int Hi, int Wi, int Ci, int Co, const void* dy1, const void* dy2,
                               const void* w1_dg, const void* w2_dg, void* dx, void* stream);

/* one wgmma conv launch with the epilogue the training step fuses into it (bf16 mode; tensors bf16 NHWC):
 * kind 0 fprop -> out + the BatchNorm batch statistics (sum, sum of squares per output channel) of the stored values;
 * kind 1 dgrad -> out = the gradient gated by the consumer BatchNorm's ReLU (+ residual) and that BatchNorm's backward
 * reductions (sum g, sum g*y [, sum g*yd]).  host_sums: [3][C] doubles.  Replaces cuDNN BN forward-training statistics
 * and the reduction half of cuDNN BN backward behind torchvision BasicBlock (/root/reference/models/posenet.py:66). */
int mapnet_test_conv_epilogue(int kind, int B, int Hi, int Wi, int Ci, int Co, int k, int stride, const void* in0,
                              const void* wmat, const void* residual, const void* y, const void* zmask, const void* yd,
                              const float* mscale, const float* mshift, void* out, double* host_sums, void* stream);

/* one wgmma fprop launch with the inference epilogue: out = relu?(conv(in0, wmat) * scale[c] + shift[c] [+ residual]),
 * rounded once at the store.  flags: bit 0 ReLU; strict mode only: bit 1 the residual is stored as hi/lo planes (a block
 * input), bit 2 the output is (the next conv's operand).  k == 7 runs the stem as the engine does (in0 = fp32 NCHW
 * image, wmat = fp32 [64][3][7][7]).  Otherwise bf16 mode takes bf16 NHWC tensors and a bf16 [Co][k][k][Ci] matrix,
 * strict mode fp32 ones (cut into planes inside).  Only the variants the eval-mode schedule uses are built. */
int mapnet_test_conv_affine(int precision, int B, int Hi, int Wi, int Ci, int Co, int k, int stride, const void* in0,
                            const void* wmat, const float* scale, const float* shift, const void* residual, int flags,
                            void* out, void* stream);

/* one fp8 fprop launch of the inference engine: f = conv(in0, wmat) * scale[c] + shift[c] (+ residual) (ReLU), in0 e4m3
 * NHWC, wmat e4m3 [Co][k][k][Ci] (k = 1 or 3; Ci = 64 or a multiple of 128), scale / shift fp32 [Co].  flags: bit 0
 * ReLU; bit 1 the residual is e4m3 (times *res_scale), else bf16; bit 2 out is e4m3 (f * *out_inv, saturating), else
 * bf16; bit 3 the calibration pass: max |f| over the output into *amax (a float's bit pattern), nothing stored. */
int mapnet_test_conv_fp8(int B, int Hi, int Wi, int Ci, int Co, int k, int stride, const void* in0, const void* wmat,
                         const float* scale, const float* shift, const void* residual, const float* res_scale,
                         const float* out_inv, int flags, void* out, unsigned int* amax, void* stream);

/* ---- the element-wise kernels of the training step (bn.cu, head.cu) one launch sequence at a time, as the trunk
 * runs them, for the per-kernel tests (tests/test_gpu_bn_pool.py).  precision selects the storage types the trunk uses:
 * fp32 -> fp32 everywhere; bf16 / bf16_simt -> bf16; tc_split -> conv outputs and gradients w.r.t. block outputs fp32,
 * forward and backward conv operands (z, the identity residual, zmask, dy, dyd) fp16 hi/lo planes.  Tensors are NHWC
 * device memory; every call allocates its own accumulators and counter, synchronizes and frees them again.
 * BatchNorm state: host_params / host_out hold, per BatchNorm, 15 rows of C floats: gamma, beta, running_mean,
 * running_var, mean, invstd, scale, shift, mscale, mshift (ReLU gate recomputed from y), dgamma, dbeta and the three
 * dy = A*g + B*y + C coefficients.  host_params is uploaded before every pass, host_out receives the state after it.
 * Lazy sums (source 1): host_sums [nrep][3][C] doubles per BatchNorm, copied into nrep accumulator replicas that the
 * consuming kernel finalizes. */
/* z = relu?(scale*y + shift [+ res | + scale2*res + shift2]); res_mode 0 none, 1 identity (z's type), 2 downsample
 * branch (y's type, second BatchNorm).  source 0: batch statistics by the reducing kernel, run twice on the same
 * accumulators and counter (host_out: 2 passes); 1: lazy sums; 2: eval-mode scale / shift from the running statistics;
 * 3: scale / shift as given. */
int mapnet_test_bn_forward(int precision, int res_mode, int relu, int source, int64_t M, int C, const void* y,
                           const void* res, void* z, const float* host_params, const double* host_sums, int nrep,
                           float* host_out, void* stream);
/* dy = A*g + B*y + C [, dyd = Ad*g + Bd*yd + Cd] [, gout = g], g = dout gated by: gate 0 nothing, 1 zmask > 0, 2
 * mscale*y + mshift > 0.  yd / dyd: the downsample BatchNorm (second state block).  source 0: sums by the reducing
 * kernel, run twice (host_out: 2 passes); 1: lazy sums.  gscale > 0: dy / dyd are scaled by it (strict mode). */
int mapnet_test_bn_backward(int precision, int source, int gate, int64_t M, int C, const void* dout, const void* zmask,
                            const void* y, const void* yd, void* dy, void* dyd, void* gout, const float* host_params,
                            const double* host_sums, int nrep, float gscale, float* host_out, void* stream);
/* the stem's BatchNorm + ReLU + 3x3/s2/p1 max pool on y [B,Hc,Wc,64] -> z, argmax bytes -> amax (may be NULL), with
 * source as for mapnet_test_bn_forward (once).  precision MAPNET_PREC_FP8: bf16 y, e4m3 z, source 3 only.  dz != NULL:
 * then the backward from amax: g = pool / ReLU backward, the BatchNorm's sums (even Hc, Wc: fused into the pool backward,
 * finalized by k_bn_bwd_finalize_accum when bsource is 0, lazily over 32 replicas when 1; odd: a reducing pass), dy. */
int mapnet_test_stem_pool(int precision, int source, int bsource, int B, int Hc, int Wc, const void* y, void* z,
                          void* amax, const void* dz, void* g, void* dy, const float* host_params,
                          const double* host_sums, int nrep, float* host_out, void* stream);
/* feat [B,C] = mean over HW pixels of z [B,HW,C] (z's type); dz [B,HW,C] = dfeat / HW (gradient type) */
int mapnet_test_gap(int precision, int B, int HW, int C, const void* z, float* feat, const float* dfeat, void* dz,
                    void* stream);

/* the tensor-core stem (7x7/s2/p3, 3 -> 64) alone, as the trunk runs it: space-to-depth image, packed weights,
 * fprop into y_out (bf16 NHWC [B,Hc,Wc,64]) and, when dy / dw_oihw are given, the weight gradient in the
 * .grad layout [64,3,7,7].  Replaces torchvision ResNet.conv1 (/root/reference/models/posenet.py:66). */
int mapnet_test_stem(int B, int H, int W, const float* x_nchw, const float* w_oihw, void* y_out, const void* dy,
                     float* dw_oihw, void* stream);

/* micro-benchmark of one tensor-core conv configuration (tools/bench_conv.py): average ms per launch */
int mapnet_bench_conv(int kind, int B, int Hi, int Wi, int Ci, int Co, int k, int stride, const void* in0,
                      const void* in1, const void* wmat, void* out, int iters, float* host_ms);

#ifdef __cplusplus
}
#endif
#endif /* MAPNET_B200_H_ */
