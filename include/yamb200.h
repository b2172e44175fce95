/* yamb200 — C ABI of the H100-native inverted-residual training path.
 *
 * This is the drop-in boundary of the hot path of meijieru/yet_another_mobilenet_series
 * (SURVEY.md §8b).  The reference's boundary is a Python nn.Module registry
 * (models/mobilenet_base.py:484-489 `get_block`) plus two YAML plugin hooks
 * (common.py:129-130 `FLAGS.model`, utils/optim.py:277-279 `FLAGS.optimizer`); the Python package
 * `yet_another_mobilenet_series_b200` mirrors those and calls ONLY the entry points below
 * (through ctypes).  No torch types cross this boundary: plain device pointers, sizes and a
 * CUDA stream handle.
 *
 * Conventions
 *   - all pointers are DEVICE pointers unless the name ends in `_host`;
 *   - tensors are BORROWED: the library never allocates, frees or retains them past the call;
 *   - activations are NHWC bf16 (a [pixels, channels] row-major matrix, pixels = N*H*W,
 *     channels % 8 == 0 so every row is 16-byte aligned); parameters, statistics and
 *     gradients of parameters are fp32 in the reference's own layouts;
 *   - every call enqueues work on `stream` and returns without synchronising; it is
 *     CUDA-graph capturable (no allocation, no host sync);
 *   - return value: 0 on success, a negative YAMB_E* code otherwise; `yamb_last_error()` returns
 *     a thread-local message.  There is NO CPU fallback: without a CUDA device every compute
 *     entry point returns YAMB_ENODEV.
 */
#ifndef YAMB200_H_
#define YAMB200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define YAMB_OK 0
#define YAMB_EINVAL (-1)
#define YAMB_ENODEV (-2)
#define YAMB_ECUDA (-3)

/* activation codes; reference: models/mobilenet_base.py:461-469 get_active_fn,
 * :70-78 Swish, :81-88 HSwish */
#define YAMB_ACT_NONE 0
#define YAMB_ACT_RELU 1
#define YAMB_ACT_RELU6 2
#define YAMB_ACT_SWISH 3
#define YAMB_ACT_HSWISH 4

typedef void* yamb_stream_t; /* cudaStream_t */

/* ---- BatchNorm bookkeeping attached to a producer kernel ---------------------------------------
 * Forward (train mode), nn.BatchNorm2d semantics (reference: models/mobilenet_base.py:203,417;
 * momentum/eps from apps/mobilenet/mobilenet_v2_mnas.yml:10-11):
 *   scale = gamma*invstd, shift = beta - mean*scale  (what the consumer applies: z = scale*h+shift)
 *   running = (1-m)*running + m*batch  (running_var uses the UNBIASED batch variance)
 *   momentum < 0  => momentum=None in PyTorch: cumulative average with factor 1/num_batches_tracked
 *   (utils/common.py:175-187 bn_calibration). */
typedef struct yamb_bn_fwd {
  double* partials;             /* accumulator, >= 2*C doubles, ZERO on entry, returned to zero */
  uint32_t* counter;            /* one zero-initialised word, self-resetting */
  const float* gamma;           /* [C] or NULL (=1) */
  const float* beta;            /* [C] or NULL (=0) */
  float eps;
  float momentum;
  float* running_mean;          /* [C] or NULL */
  float* running_var;           /* [C] or NULL */
  int64_t* num_batches_tracked; /* scalar or NULL */
  float* scale;                 /* out [C] */
  float* shift;                 /* out [C] */
  float* mean;                  /* out [C] or NULL (saved for backward) */
  float* invstd;                /* out [C] or NULL (saved for backward) */
  int64_t count;                /* elements per channel (N*H*W) */
} yamb_bn_fwd;

/* Backward of the same BN: given sum(dz), sum(dz*xhat) produce dgamma, dbeta (ACCUMULATED into the
 * gradient buffers) and the affine form of the input gradient  dh = ca*dz + cb*h + cc. */
typedef struct yamb_bn_bwd {
  double* partials;
  uint32_t* counter;
  const float* gamma;  /* [C] or NULL */
  const float* mean;   /* [C] saved by forward */
  const float* invstd; /* [C] saved by forward */
  float* dgamma;       /* [C] += , or NULL */
  float* dbeta;        /* [C] += , or NULL */
  float* ca;           /* out [C] */
  float* cb;           /* out [C] */
  float* cc;           /* out [C] */
  int64_t count;
  int32_t use_batch_stats; /* 1: train-mode BN (batch statistics); 0: eval-mode BN => dh = ca*dz */
} yamb_bn_bwd;

/* ---- pointwise (1x1) convolution = GEMM on Hopper tensor cores (wgmma) ----------------------------------
 * Replaces nn.Conv2d(k=1) forward, dgrad and wgrad inside the block
 * (reference: models/mobilenet_base.py:391-395 expand, :413 project, :253-257/:284-285 fused).
 *
 *   D[M,N] = A'[M,K] * B'[N,K]^T        fp32 accumulation in registers
 *
 * a_mn_major = 0: A is a row-major [M][lda] array (K contiguous); 1: a row-major [K][lda] array
 * (M contiguous) — same for B with N.  With pixels on M this covers
 *   forward : A = activations [pix][Cin],  B = weight [Cout][Cin]           (0,0)
 *   dgrad   : A = dY [pix][Cout],          B = weight [Cout][Cin] as [K][N] (0,1)
 *   wgrad   : A = dY [pix][Cout] as [K][M],B = X [pix][Cin] as [K][N]       (1,1), split-K, epi=2
 * Operand transforms (applied to the tile in shared memory before the MMA):
 *   x' = act(scale[c]*x + shift[c])                     (xform = 1; BN-apply + activation)
 *   x' = scale[c]*x + shift2[c]*x2 + shift[c]           (xform = 2; BN-backward; x2 second tensor)
 * where c indexes the operand's contiguous (channel) dimension.
 * Epilogues:
 *   epi 0: D bf16 = acc (+ residual), optional per-column BN forward statistics (bn_fwd)
 *   epi 1: D bf16 = acc * act'(h_scale*H + h_shift), statistics sum(dz), sum(dz*xhat) (bn_bwd)
 *   epi 2: D fp32 += acc (split-K partial tiles added in slab order: deterministic) */
typedef struct yamb_gemm {
  int32_t M, N, K;
  int32_t a_mn_major, b_mn_major;
  const void* A; int64_t lda;
  const void* B; int64_t ldb;
  void* D; int64_t ldd;
  int32_t epi;
  int32_t a_xform; int32_t a_act;
  const float* a_scale; const float* a_shift; const float* a_scale2;
  const void* A2; int64_t lda2;
  int32_t b_xform; int32_t b_act;
  const float* b_scale; const float* b_shift; const float* b_scale2;
  const void* B2; int64_t ldb2;
  const void* residual; int64_t ldr;   /* epi 0: bf16 [M][ldr], or NULL */
  const yamb_bn_fwd* bn_fwd;           /* epi 0: or NULL */
  const void* H; int64_t ldh;          /* epi 1: bf16 [M][ldh] pre-BN activations */
  const float* h_scale; const float* h_shift; int32_t h_act;
  const yamb_bn_bwd* bn_bwd;           /* epi 1 */
  int32_t max_ctas;                    /* 0 = one CTA per SM */
  /* optional per-(sample, channel) gate applied after an xform=1 transform (SE: x * gate[n][c]);
   * the operand's rows must be pixels (A K-major, or A/B MN-major): n = pixel / rows_per_sample */
  const float* a_gate; const float* b_gate; int64_t gate_rows_per_sample;
} yamb_gemm;

int yamb_pointwise_gemm(const yamb_gemm* args, yamb_stream_t stream);

/* ---- depthwise k x k convolution (k in {3,5,7}, stride 1/2, pad (k-1)/2) -------------------------
 * Replaces nn.Conv2d(groups=C)+BatchNorm2d+activation of ConvBNReLU
 * (reference: models/mobilenet_base.py:405-411 unfused, :275-281 fused, :181-203 ConvBNReLU).
 * Operates on a channel SLICE [c0, c0+C) of NHWC tensors whose row pitch is ldc channels: all
 * pointers are pre-offset to the slice's first channel (multi-kernel-size branches of one hidden
 * tensor are one call per branch; reference :266 Narrow, :332-336 cat).
 *   forward : y = dwconv(act(in_scale*x + in_shift), w)   (in_scale NULL => y = dwconv(x, w))
 *             + BatchNorm statistics of y (bn, optional)
 *   backward: dh = ca*dz + cb*h + cc ;  da = dwconv^T(dh, w) ;  dw += sum dh * act(z) ;
 *             dx = da * act'(z) (+ residual),  z = in_scale*x + in_shift ;
 *             statistics sum(dx), sum(dx*xhat) for the preceding BatchNorm (bn, optional)
 * w / dw: fp32 [C][k][k] (the reference's [C,1,k,k] parameter layout). */
typedef struct yamb_dw_fwd {
  int32_t N, H, W, C, ldc, k, stride;
  const void* x;
  const float* in_scale; const float* in_shift; int32_t in_act;
  const float* w;
  void* y;
  const yamb_bn_fwd* bn;
} yamb_dw_fwd;

typedef struct yamb_dw_bwd {
  int32_t N, H, W, C, ldc, k, stride;
  const void* dz; const void* h;                     /* [N,Ho,Wo,ldc] */
  const float* ca; const float* cb; const float* cc; /* dh = ca*dz + cb*h + cc */
  const float* w; float* dw;
  const void* x;                                     /* [N,H,W,ldc] pre-BN input of the stage */
  const float* in_scale; const float* in_shift; int32_t in_act;
  void* dx;
  const void* residual;                              /* bf16 [N,H,W,ldc] added to dx, or NULL */
  const yamb_bn_bwd* bn;
} yamb_dw_bwd;

int yamb_depthwise_fwd(const yamb_dw_fwd* args, yamb_stream_t stream);
int yamb_depthwise_bwd(const yamb_dw_bwd* args, yamb_stream_t stream);

/* ---- per-channel elementwise / reduction on [M, C] bf16 matrices ---------------------------------
 * bn_apply : y = act(scale*h + shift) * gate[n][c] + residual     (pw_bn + skip connection,
 *            reference models/mobilenet_base.py:448-450, :340-341; SE gating :113)
 * bn_reduce: sum(dy), sum(dy*xhat) + BatchNorm-backward finalize  (autograd of :417 pw_bn) */
typedef struct yamb_bn_apply {
  int64_t M; int32_t C; int32_t ldh, ldr, ldy;
  const void* h; const float* scale; const float* shift; int32_t act;
  const void* residual; void* y;
  const float* gate; int64_t rows_per_sample;   /* optional [N][C] fp32 gate */
  const void* residual2; int32_t ldr2;          /* optional second bf16 addend (non-local block:
                                                 * bn(dw(f)) + l + x, models/mobilenet_base.py:173,
                                                 * :340-341) */
} yamb_bn_apply;

typedef struct yamb_bn_reduce {
  int64_t M; int32_t C; int32_t lddy, ldh;
  const void* dy; const void* h;
  const yamb_bn_bwd* bn;
  /* optional activation AFTER this BatchNorm (ConvBNReLU tail, models/mobilenet_base.py:181-203):
   * the statistics are those of dz = dy * act'(z_scale*h + z_shift); NULL = no activation */
  const float* z_scale; const float* z_shift; int32_t z_act;
} yamb_bn_reduce;

/* Stand-alone BatchNorm(+activation) of a convolution this library does not run itself (the stem
 * 3x3 and the 1x1 head ConvBNReLU, reference models/mobilenet_base.py:181-203 via :143-171 of
 * mobilenet_supernet.py): batch statistics of the raw conv output ... */
typedef struct yamb_bn_stats {
  int64_t M; int32_t C; int32_t ldh;
  const void* h;               /* [M][ldh] bf16 raw conv output */
  const yamb_bn_fwd* bn;       /* finalize: scale/shift/mean/invstd/running statistics */
} yamb_bn_stats;

/* ... and its input gradient dh = ca*dz + cb*h + cc with dz = dy * act'(z_scale*h + z_shift)
 * (ca/cb/cc from yamb_bn_reduce_bwd's finalize). */
typedef struct yamb_bn_bwd_apply {
  int64_t M; int32_t C; int32_t lddy, ldh, lddh;
  const void* dy; const void* h;
  const float* z_scale; const float* z_shift; int32_t z_act;   /* NULL scale = no activation */
  const float* ca; const float* cb; const float* cc;
  void* dh;
} yamb_bn_bwd_apply;

typedef struct yamb_se_pool {
  int32_t N, HW, C, ldh;
  const void* h; const float* scale; const float* shift; int32_t act;
  float* pooled;
} yamb_se_pool;

/* Squeeze-and-Excitation backward pieces (autograd of reference models/mobilenet_base.py:110-113,
 * y = x * gate, gate = sigmoid(W_e act(W_r mean_HW(x) + b_r) + b_e), x = act(scale*h+shift)):
 *   se_bwd_reduce: dgate[n][c] = sum_HW dY * x
 *   se_bwd_apply : dz = (dY*gate[n][c] + dpool[n][c]) * act'(scale*h+shift)  (+ BN-bwd statistics);
 *                  dpool = (d mean)/HW comes from the host-side tiny FC backward. */
typedef struct yamb_se_bwd_reduce {
  int32_t N, HW, C, ldd, ldh;
  const void* dy; const void* h; const float* scale; const float* shift; int32_t act;
  float* dgate;
} yamb_se_bwd_reduce;

typedef struct yamb_se_bwd_apply {
  int64_t M; int32_t C, ldd, ldh, ldz; int64_t rows_per_sample;
  const void* dy; const void* h; const float* scale; const float* shift; int32_t act;
  const float* gate; const float* dpool; int32_t ldg; /* row pitch of gate / dpool */
  void* dz;
  const yamb_bn_bwd* bn;
} yamb_se_bwd_apply;

/* The two fully connected layers of the SE branch on the pooled vectors (reference
 * models/mobilenet_base.py:110-113 se_reduce / active_fn / se_expand / sigmoid) and their backward,
 * fp32:  u = W_r s + b_r, v = act(u), gate = sigmoid(W_e v + b_e);
 * backward: dt = dgate*gate*(1-gate), du = (W_e^T dt)*act'(u), dpool = (W_r^T du)*inv_hw, and the
 * parameter gradients ACCUMULATED (+=) into g_* (sums over the N samples).  No float atomics: the
 * split-K products u, du and the bias-gradient column sums add per-CTA slabs in a fixed order, so
 * every call computes the same bits. */
typedef struct yamb_se_fc {
  int32_t N, C, R; int32_t act;
  const float* pooled;                     /* [N][C] */
  const float* w_r; const float* b_r;      /* [R][C], [R]  (se_reduce) */
  const float* w_e; const float* b_e;      /* [C][R], [C]  (se_expand) */
  float* u; float* v;                      /* out [N][R]: saved for backward */
  float* gate;                             /* out [N][C] */
} yamb_se_fc;

typedef struct yamb_se_fc_grad {
  int32_t N, C, R; int32_t act; float inv_hw;
  const float* dgate; const float* gate; const float* u; const float* v; const float* pooled;
  const float* w_r; const float* w_e;
  float* dpool;                            /* out [N][C] */
  float* dt; float* du;                    /* scratch [N][C], [N][R] */
  float* g_wr; float* g_br; float* g_we; float* g_be;
} yamb_se_fc_grad;

int yamb_se_fc_fwd(const yamb_se_fc* args, yamb_stream_t stream);
int yamb_se_fc_bwd(const yamb_se_fc_grad* args, yamb_stream_t stream);

int yamb_bn_apply_fwd(const yamb_bn_apply* args, yamb_stream_t stream);
int yamb_se_bwd_reduce_bwd(const yamb_se_bwd_reduce* args, yamb_stream_t stream);
int yamb_se_bwd_apply_bwd(const yamb_se_bwd_apply* args, yamb_stream_t stream);
int yamb_bn_reduce_bwd(const yamb_bn_reduce* args, yamb_stream_t stream);
int yamb_bn_stats_fwd(const yamb_bn_stats* args, yamb_stream_t stream);
int yamb_bn_bwd_apply_bwd(const yamb_bn_bwd_apply* args, yamb_stream_t stream);
int yamb_se_pool_fwd(const yamb_se_pool* args, yamb_stream_t stream);

/* ---- lightweight non-local block (AutoNL) -------------------------------------------------------
 * Replaces the two einsums of Nonlocal.forward (reference models/mobilenet_base.py:158-173) and
 * their autograd backward.  All tensors are NHWC bf16 [N][H*W][ld]; `sub` selects the row set:
 * every pixel (sub = 1) or the pixels of l[:, :, ::sub, ::sub] (:161).
 *   gram  : G[n][i][j] = alpha * sum_rows X[n,row,i] * Y[n,row,j]      i < I, j < J (fp32, overwritten)
 *           forward  F = phi^T g  (X = Y = l, I = int(nl_c*C), J = C, rows = subsampled)
 *           backward dF = (W/H) theta^T df  (X = l, Y = df, rows = all)
 *   rowmat: out[n,row,o] = {base[n,row,o] | out[n,row,o] | 0} + alpha * sum_k X[n,row,k] * Mat[n](k,o)
 *           with Mat[n](k,o) = Mat[n*mat_stride + k*sk + o*so], o < O; columns [O, O_copy) of
 *           `base` are copied through.  forward f = (W/H) theta F; backward dtheta, dphi, dg.
 * The reference's choice between (theta phi^T) g and theta (phi^T g) (:164-170) is a re-association
 * of the same sum; the channel matrix is always formed first here. */
typedef struct yamb_nl_gram {
  int32_t N, H, W, sub;
  const void* X; int64_t ldx; int32_t I;
  const void* Y; int64_t ldy; int32_t J;   /* J, ldy even */
  float alpha;
  float* G;                                /* [N][I][J]; the per-CTA row-chunk partial sums
                                            * are added in a fixed order (the same bits on
                                            * every run) */
} yamb_nl_gram;

typedef struct yamb_nl_rowmat {
  int32_t N, H, W, sub;
  const void* X; int64_t ldx; int32_t K;
  const float* Mat; int64_t mat_stride, sk, so; int32_t O;   /* O even */
  float alpha;
  const void* base; int64_t ldb; int32_t O_copy;             /* NULL, or bf16 addend + pass-through */
  int32_t accumulate;                                        /* 1: read-modify-write `out` */
  void* out; int64_t ldo;
} yamb_nl_rowmat;

int yamb_nl_gram_fwd(const yamb_nl_gram* args, yamb_stream_t stream);
int yamb_nl_rowmat_fwd(const yamb_nl_rowmat* args, yamb_stream_t stream);

/* ---- instance normalisation of the non-local block (nl_norm: nn.InstanceNorm) --------------------
 * nn.InstanceNorm2d(C, affine=True, track_running_stats=True) in training mode (reference
 * models/mobilenet_base.py:149-156, :472-481) on the raw depthwise output h of the non-local block:
 *   forward : per (n, c) mean mu and biased variance over the HW pixels of sample n,
 *             y = gamma*(h - mu)*invstd + beta (+ residual) (+ residual2)  (bf16);
 *             running = (1-m)*running + m*mean_n(batch), running_var from each instance's UNBIASED
 *             variance; momentum 0 (torch's momentum=None) or NULL running buffers: no update
 *   backward: per (n, c) sums of dy and dy*xhat,
 *             dh = gamma*invstd*(dy - sum(dy)/HW - xhat*sum(dy*xhat)/HW)  (bf16),
 *             dgamma += sum_n sum(dy*xhat), dbeta += sum_n sum(dy)
 * One CTA per (sample, 64-channel chunk) owns its statistics; the sums over n are added in sample
 * order by the last CTA (no float atomics: the same bits on every run).  HW >= 2; C, ld* multiples
 * of 8.  In eval mode the norm is a per-channel affine (yamb_bn_apply_fwd with folded
 * coefficients). */
typedef struct yamb_in_fwd {
  int32_t N, HW, C, ldh;
  const void* h;                              /* bf16 [N*HW][ldh] */
  const float* gamma; const float* beta;      /* [C] or NULL (=1 / =0) */
  float eps, momentum;
  float* running_mean; float* running_var;    /* [C] or NULL */
  float* mean; float* invstd;                 /* out [N][C], saved for backward */
  const void* residual; int32_t ldr;          /* bf16 [N*HW][ldr] addend, or NULL */
  const void* residual2; int32_t ldr2;        /* second bf16 addend, or NULL */
  void* y; int32_t ldy;                       /* out bf16 [N*HW][ldy] */
  uint32_t* counter;                          /* zero-initialised word, self-resetting */
} yamb_in_fwd;

typedef struct yamb_in_bwd {
  int32_t N, HW, C, ldh, lddy, lddh;
  const void* dy; const void* h;              /* bf16 [N*HW][lddy], [N*HW][ldh] */
  const float* gamma;                         /* [C] or NULL */
  const float* mean; const float* invstd;     /* [N][C] from the forward */
  float* dgamma; float* dbeta;                /* [C] +=, or NULL */
  void* dh;                                   /* out bf16 [N*HW][lddh] */
  uint32_t* counter;                          /* zero-initialised word, self-resetting */
} yamb_in_bwd;

int yamb_instance_norm_fwd(const yamb_in_fwd* args, yamb_stream_t stream);
int yamb_instance_norm_bwd(const yamb_in_bwd* args, yamb_stream_t stream);

/* ---- stem convolution -----------------------------------------------------------------------------
 * 3x3, stride 2, pad 1, 3 input channels -> Cout (multiple of 8, <= 64) on NHWC bf16: the first
 * layer of the network (reference models/mobilenet_supernet.py:124-130; its BatchNorm + activation
 * follow through yamb_bn_stats_fwd / yamb_bn_apply_fwd).  Weights fp32 in the parameter's own
 * [Cout][3][3][3] layout.  fwd writes y; wgrad ACCUMULATES dw += sum dh * x (no input gradient). */
typedef struct yamb_stem_conv {
  int32_t N, H, W, Cout;
  const void* x;        /* bf16 [N][H][W][3] */
  const float* w;       /* [Cout][3][3][3]            (fwd) */
  void* y;              /* bf16 [N][Ho][Wo][Cout]     (fwd) */
  const void* dh;       /* bf16 [N][Ho][Wo][Cout]     (wgrad) */
  float* dw;            /* [Cout][3][3][3] +=         (wgrad) */
} yamb_stem_conv;

int yamb_stem_conv_fwd(const yamb_stem_conv* args, yamb_stream_t stream);
int yamb_stem_conv_wgrad(const yamb_stem_conv* args, yamb_stream_t stream);

/* ---- label-smoothed softmax cross entropy + top-k -------------------------------------------------
 * Replaces CrossEntropyLabelSmooth(reduction='none') (reference utils/optim.py:150-158), the
 * top-1 / top-5 `correct_k` bookkeeping of forward_loss (common.py:73-79) and their backward.
 *   forward : loss[n] = sum_c -t[n][c] log_softmax(logits)[n][c], t = (1-eps) onehot + eps/C;
 *             correct1/5[n] in {0,1} (ties like torch.topk: lower index wins);
 *             G[n][c] = softmax - t (bf16), what the backward needs
 *   backward: dlogits[n][c] = G[n][c] * dloss[n];  dbias[c] += sum_n dlogits[n][c] (classifier
 *             bias gradient, optional) */
typedef struct yamb_softmax_ce {
  int32_t N, C; int64_t ld;
  const void* logits;          /* bf16 [N][ld] */
  const int64_t* target;       /* [N] */
  float smoothing;
  float* loss;                 /* [N] */
  float* correct1; float* correct5;   /* [N] or NULL */
  void* G; int64_t ldg;        /* bf16 [N][ldg] or NULL (no backward wanted) */
} yamb_softmax_ce;

typedef struct yamb_softmax_ce_grad {
  int32_t N, C;
  const void* G; int64_t ldg;
  const float* dloss;          /* [N] */
  void* dlogits; int64_t ldd;  /* bf16 [N][ldd] */
  float* dbias;                /* [C] += or NULL */
} yamb_softmax_ce_grad;

int yamb_softmax_ce_fwd(const yamb_softmax_ce* args, yamb_stream_t stream);
int yamb_softmax_ce_bwd(const yamb_softmax_ce_grad* args, yamb_stream_t stream);
/* out[c] += sum_rows X[row][c] over a bf16 [M][ld] matrix (bias gradient of the classifier,
 * reference models/mobilenet_supernet.py:163-167) */
int yamb_colsum_bf16(const void* X, int64_t M, int32_t C, int64_t ld, float* out,
                     yamb_stream_t stream);

/* ---- eval-mode inverted-residual block, ONE launch, no intermediate in HBM -----------------------
 * Replaces the forward of InvertedResidualChannels (reference models/mobilenet_base.py:446-451;
 * single branch, 3x3 depthwise, stride 1 or 2, with the 1x1 expansion or without it (:397-404,
 * hidden == input)) when every BatchNorm uses its running statistics (model.eval(): validation /
 * forward_loss under no_grad, common.py:67-80, train.py:273-309): x tile (TMA, halo zero-filled)
 * -> wgmma expand -> BN1+act -> 3x3 stencil -> BN2+act -> wgmma project (accumulated over
 * 64-channel slices of the hidden dimension) -> BN3 (+x) -> y.  The BatchNorm folding
 * scale = gamma*rsqrt(var+eps), shift = beta - mean*scale is done inside the kernel from the
 * module's buffers (csrc/block_eval.cu).  Shapes it does not cover return YAMB_EINVAL; the caller
 * then runs the four-launch sequence with folded coefficients.
 *
 * Squeeze-and-Excitation (InvertedResidualChannelsFused, reference :110-113, :336-339) takes three
 * calls: yamb_block_eval_pool_fwd writes pooled[n][c], the spatial mean of a2 = bf16(act(bn2(h2)))
 * (it recomputes expand -> BN1+act -> stencil -> BN2+act per tile and stops there: no project, no
 * hidden tensor in HBM; per-tile partial sums added in a fixed order, the same bits on every run;
 * bn3, w_project and y are not read); yamb_se_fc_fwd turns pooled into the gate; yamb_block_eval_fwd
 * with `gate` set feeds a2s = bf16(a2 * gate[n][c]) to the project MMAs. */
typedef struct yamb_bn_eval {
  const float* gamma;         /* [C] or NULL (=1) */
  const float* beta;          /* [C] or NULL (=0) */
  const float* running_mean;  /* [C] */
  const float* running_var;   /* [C] */
  float eps;
} yamb_bn_eval;

typedef struct yamb_block_eval {
  int32_t N, H, W;            /* input pixels (NHWC); output (H-1)/stride+1 x (W-1)/stride+1 */
  int32_t Cin, Chid, Cout;    /* multiples of 8; Cin <= 256, Cout <= 320 */
  int32_t kernel, stride;     /* 3, 5 or 7 (5 / 7: with expansion); 1 or 2 */
  int32_t act;                /* YAMB_ACT_* of the two inner activations */
  int32_t residual;           /* y += x (needs Cin == Cout, stride 1) */
  const void* x;              /* bf16 [N,H,W,Cin] */
  const void* w_expand;       /* bf16 [Chid][Cin], or NULL: no expansion (Chid == Cin, bn1 unused) */
  const float* w_dw;          /* fp32 [Chid][k][k] */
  const void* w_project;      /* bf16 [Cout][Chid] */
  yamb_bn_eval bn1, bn2, bn3; /* over Chid, Chid, Cout channels */
  void* y;                    /* bf16 [N,Ho,Wo,Cout] */
  const float* gate;          /* fp32 [N][Chid] SE gate applied to a2 before the project, or NULL */
  float* pooled;              /* pool pass: out fp32 [N][Chid] spatial mean of a2 */
} yamb_block_eval;

int yamb_block_eval_fwd(const yamb_block_eval* args, yamb_stream_t stream);
int yamb_block_eval_pool_fwd(const yamb_block_eval* args, yamb_stream_t stream);

/* ---- fused flat-arena RMSprop (+L2 decay, +DDP mean, +EMA, +bf16 repack) -------------------------
 * Replaces RMSprop.step (reference utils/rmsprop.py:67-129), the gradient of cal_l2_loss
 * (utils/optim.py:177-200; l2 * p added where bit 0 of wd_mask is set; bit 1 marks a parameter
 * that received no gradient this step, rmsprop.py:77-78: only its EMA moves), the division by world size of
 * _allreduce_coalesced (utils/distributed.py:136; grad_scale) and ExponentialMovingAverage.forward
 * (utils/optim.py:53-64; ema / ema_m) in ONE launch over flat fp32 arenas of n elements.
 * hyper: optional device array [lr, ema_m] read instead of the host scalars (CUDA-graph replay). */
typedef struct yamb_rmsprop {
  int64_t n;
  float* p; const float* g; float* sq; float* mom; float* grad_avg;
  float* ema; void* p_bf16; const uint8_t* wd_mask;
  const float* hyper;
  float lr, alpha, eps, momentum, weight_decay, l2, grad_scale, ema_m;
  int32_t eps_inside_sqrt, centered;
} yamb_rmsprop;

int yamb_rmsprop_step(const yamb_rmsprop* args, yamb_stream_t stream);

/* ---- fused flat-arena SGD (+L2 decay, +DDP mean, +EMA, +bf16 repack) -----------------------------
 * Replaces torch.optim.SGD.step with momentum / dampening / nesterov / weight_decay (the reference's
 * `optimizer: sgd`, utils/optim.py:262-267) over the same flat arenas and with the same services as
 * yamb_rmsprop: per element
 *   g = grad_scale*g (+ l2*p where bit 0 of wd_mask is set) (+ weight_decay*p)
 *   momentum > 0: buf = g on the parameter's first momentum step (bit 2 of wd_mask), else
 *                 buf = momentum*buf + (1-dampening)*g;  g = g + momentum*buf (nesterov) or buf
 *   p -= lr*g;  ema = ema_m*ema + (1-ema_m)*p;  p_bf16 = bf16(p)
 * Bit 1 of wd_mask: the parameter received no gradient this step; only its EMA moves.  `mom` is
 * required when momentum > 0; nesterov requires momentum > 0 and dampening == 0. */
typedef struct yamb_sgd {
  int64_t n;
  float* p; const float* g; float* mom;
  float* ema; void* p_bf16; const uint8_t* wd_mask;
  const float* hyper;         /* optional device [lr, ema_m] */
  float lr, momentum, dampening, weight_decay, l2, grad_scale, ema_m;
  int32_t nesterov;
} yamb_sgd;

int yamb_sgd_step(const yamb_sgd* args, yamb_stream_t stream);
/* shadow = m*shadow + (1-m)*x over n floats (BN running statistics; common.py:58-63) */
int yamb_ema_update(float* shadow, const float* x, int64_t n, const float* hyper, float m,
                    yamb_stream_t stream);
/* dst(bf16) = src(fp32) */
int yamb_cast_bf16(const float* src, void* dst, int64_t n, yamb_stream_t stream);

/* upper bound of CTAs any statistics-producing kernel launches; 4 x SM count; <= 0 without a
 * device */
int yamb_max_ctas(void);

/* sizeof() of the ABI structs (0 bn_fwd, 1 bn_bwd, 2 gemm, 3 dw_fwd, 4 dw_bwd, 5 bn_apply,
 * 6 bn_reduce, 7 se_pool, 8 rmsprop, 9 se_bwd_reduce, 10 se_bwd_apply, 11 bn_stats,
 * 12 bn_bwd_apply, 13 nl_gram, 14 nl_rowmat, 15 se_fc, 16 se_fc_grad, 17 softmax_ce,
 * 18 softmax_ce_grad, 19 stem_conv, 20 bn_eval, 21 block_eval, 22 in_fwd, 23 in_bwd, 24 sgd) so bindings
 * can self-check */
int yamb_struct_size(int which);

const char* yamb_last_error(void);
int yamb_version(void);

#ifdef __cplusplus
}
#endif
#endif /* YAMB200_H_ */
