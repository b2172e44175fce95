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

/* The launch plan yamb_pointwise_gemm makes for `args`, computed on the host without a launch:
 * the same argument checks (codes and messages) up to the shared-memory layout; pointers and their
 * alignment are not checked.  num_sms > 0 plans for that many SMs and needs no device; <= 0 uses
 * the current device (YAMB_ENODEV without one). */
typedef struct yamb_gemm_plan_info {
  int32_t xf, epi, block_n, a_mn, b_mn;  /* the gemm_tc_kernel instantiation */
  int32_t m_blocks, n_blocks, num_k_blocks, ksplit, kb_per_split, num_work, grid;
  int32_t a_tma, b_tma;                  /* transformed operand loaded by TMA (else registers) */
  int32_t wg2x;                          /* warps 8-11 load instead of running epilogues */
  int32_t lgroup;                        /* loader warps per pipeline stage */
  int32_t num_stages, out_bufs, smem_bytes;
  int32_t reg_stats;                     /* BatchNorm column sums held in registers to the end */
  int32_t simple_work;                   /* one work item = one m-block (ksplit 1, one n-block) */
} yamb_gemm_plan_info;

int yamb_gemm_plan(const yamb_gemm* args, int32_t num_sms, yamb_gemm_plan_info* out);

/* ---- expand-side backward in one pass (csrc/expand_bwd.cu) ------------------------------------
 * The two gradients of the expand 1x1 convolution, from one read of dz1 and h1:
 *   dh1 = ca[c]*dz1 + cb[c]*h1 + cc[c]      (BatchNorm-1 backward; the dgrad / wgrad GEMMs' xform 2)
 *   dx  = dh1 * W1 (+ residual)             bf16 [M][Cin]
 *   dW1 += dh1^T * x                        fp32 [Chid][Cin], one partial per slab of the split-K
 *                                           wgrad GEMM's plan, added in slab order: bitwise the
 *                                           values of the dgrad + wgrad GEMMs
 * Every tensor is dense: dz1, h1 [M][Chid]; W1 [Chid][Cin]; x, residual, dx [M][Cin].
 * Caps: 8 <= Cin <= 32, 64 <= Chid <= 192, both multiples of 8.  Other shapes, NULL or
 * misaligned (16-byte) pointers return YAMB_EINVAL before any device work.  Enqueues on `stream`,
 * never synchronises, CUDA-graph capturable. */
typedef struct yamb_expand_bwd_args {
  int32_t M, Cin, Chid;
  const void* dz1; const void* h1;
  const float* ca; const float* cb; const float* cc;
  const void* W1;                      /* bf16 */
  const void* x;                       /* bf16 */
  const void* residual;                /* bf16, or NULL */
  void* dx;                            /* bf16 */
  float* dW1;                          /* fp32, += */
} yamb_expand_bwd_args;

int yamb_expand_bwd(const yamb_expand_bwd_args* args, yamb_stream_t stream);

/* The launch plan of yamb_expand_bwd, computed on the host: the same shape checks (pointers are not
 * checked).  num_sms > 0 plans for that many SMs and needs no device; <= 0 uses the current
 * device (YAMB_ENODEV without one). */
typedef struct yamb_expand_bwd_plan_info {
  int32_t block_n;                     /* wgmma width: Cin padded to 16 or 32 */
  int32_t panels;                      /* 64-channel panels of Chid */
  int32_t slabs, slab_rows;            /* the split-K wgrad GEMM's slabs of pixels: one dW1 partial each */
  int32_t grid, num_stages, smem_bytes;
} yamb_expand_bwd_plan_info;

int yamb_expand_bwd_plan(const yamb_expand_bwd_args* args, int32_t num_sms,
                         yamb_expand_bwd_plan_info* out);

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

/* ---- the depthwise of up to three branches in one launch each way ---------------------------------
 * The branches of a multi-branch block (AtomNAS, the single-path supernet: one per kernel size) are
 * channel slices of one hidden tensor, each a yamb_depthwise_fwd / _bwd call of its own.  The grouped
 * launch's grid is the concatenation of those calls' grids: its CTA j finds its branch b from the
 * prefix sums of `grid` and runs what CTA j - (grid[0] + ... + grid[b-1]) of branch b's own launch
 * runs (same kernel instantiation, tile walk, pointers, statistics slice), so every output has the
 * bits of the per-branch calls.  Each branch with `bn` finalises its statistics in its own last CTA,
 * so each needs its own counter and partials.  The backward reduces each branch's weight-gradient
 * slabs in slab order after the kernel, as yamb_depthwise_bwd does.
 * grid[b] (and, backward with k == 7, grid_wgrad[b]: the CTAs of the taps-25..48 weight-gradient
 * kernel; 0 for k 3 / 5) must be what yamb_depthwise_fwd / _bwd launch for that branch on this
 * device: yamb_depthwise_grouped_grids fills them.  nbranch 1..3, one stride for all branches,
 * distinct statistics counters, every branch within the caps of yamb_depthwise_fwd / _bwd, positive
 * grids: otherwise YAMB_EINVAL before any device work (with or without a device); YAMB_ENODEV
 * without a device; YAMB_EINVAL also when a grid differs from the per-branch launch's. */
#define YAMB_DW_MAX_BRANCHES 3
typedef struct yamb_dw_fwd_grouped {
  int32_t nbranch;
  yamb_dw_fwd branch[YAMB_DW_MAX_BRANCHES];
  int32_t grid[YAMB_DW_MAX_BRANCHES];
} yamb_dw_fwd_grouped;

typedef struct yamb_dw_bwd_grouped {
  int32_t nbranch;
  yamb_dw_bwd branch[YAMB_DW_MAX_BRANCHES];
  int32_t grid[YAMB_DW_MAX_BRANCHES];
  int32_t grid_wgrad[YAMB_DW_MAX_BRANCHES];
} yamb_dw_bwd_grouped;

int yamb_depthwise_fwd_grouped(const yamb_dw_fwd_grouped* args, yamb_stream_t stream);
int yamb_depthwise_bwd_grouped(const yamb_dw_bwd_grouped* args, yamb_stream_t stream);
/* Fill grid (and grid_wgrad) of either struct (NULL: skipped) with the grids the per-branch calls
 * use on the current device, through the sizing those calls run; the other checks as above. */
int yamb_depthwise_grouped_grids(yamb_dw_fwd_grouped* fwd, yamb_dw_bwd_grouped* bwd);

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

/* ---- training-mode Squeeze-and-Excitation backward without a pass over the hidden tensor --------
 * The three calls below take the place of yamb_se_bwd_reduce_bwd, yamb_se_bwd_apply_bwd and
 * yamb_depthwise_bwd in the backward of a block with SE:
 *   yamb_se_bwd_stats -> yamb_se_fc_bwd -> yamb_se_bn_bwd_finalize (per BatchNorm-2 slice)
 *   -> yamb_depthwise_bwd_se (per branch)
 * so that dz2 = (dY*gate + dpool)*act'(z2) is never written: the depthwise backward forms it while
 * it stages dY.  z2 = scale*h + shift is BatchNorm-2's output, xhat2 = (h - mean)*invstd.
 *
 * se_bwd_stats reads dY and h once and writes
 *   dgate[n][c]: the bits of yamb_se_bwd_reduce_bwd on the same arguments (same pixel chunks,
 *                order and bf16 rounding of a2);
 *   sums [4][N][C] (double): A = sum_HW dY*act'(z2), B = sum_HW act'(z2),
 *                A' = sum_HW dY*act'(z2)*xhat2, B' = sum_HW act'(z2)*xhat2.
 *   Each thread sums in fp32 in a fixed order; its partials are added across threads and pixel
 *   chunks in double, in a fixed order.  No float atomics: the same bits on every call.
 * N <= 65535, C a multiple of 8, dy / h 16-byte aligned with pitches >= C and multiples of 8. */
typedef struct yamb_se_bwd_stats {
  int32_t N, HW, C, ldd, ldh;
  const void* dy; const void* h;            /* bf16 [N*HW][ldd], [N*HW][ldh] */
  const float* scale; const float* shift;   /* [C] BatchNorm-2 coefficients */
  int32_t act;                              /* YAMB_ACT_* after BatchNorm-2 */
  const float* mean; const float* invstd;   /* [C] BatchNorm-2 statistics of the forward */
  float* dgate;                             /* out [N][C] */
  double* sums;                             /* out [4][N][C]: A, B, A', B' */
} yamb_se_bwd_stats;

/* The BatchNorm-2 backward of one BatchNorm slice once dpool exists (yamb_se_fc_bwd):
 *   sum_HW dz2 = gate*A + dpool*B,  sum_HW dz2*xhat2 = gate*A' + dpool*B'  per (n, c), added over n
 *   in sample order in double, then bn's finalize (dgamma, dbeta +=; ca, cb, cc) as
 *   yamb_se_bwd_apply_bwd finalizes it.  bn->partials / bn->counter are not used.  sums, gate and
 *   dpool are pre-offset to the slice's first channel; lds, ldg >= C. */
typedef struct yamb_se_bn_bwd_finalize_args {
  int32_t N, C;
  const double* sums; int32_t lds;          /* [4][N][lds] from yamb_se_bwd_stats */
  const float* gate; const float* dpool; int32_t ldg;   /* [N][ldg] */
  const yamb_bn_bwd* bn;
} yamb_se_bn_bwd_finalize_args;

/* yamb_depthwise_bwd with dw.dz = dY = d(a2*gate), the project dgrad's output, instead of dz2: every
 * staged dY element becomes dz2 = bf16((dY*gate[n][c] + dpool[n][c]) * act'(scale*h + shift)), the
 * fp32 expression and rounding of yamb_se_bwd_apply_bwd, then dh = ca*dz2 + cb*h + cc as in
 * yamb_depthwise_bwd.  dx, dw and the statistics in dw.bn are bitwise those of
 * yamb_se_bwd_apply_bwd followed by yamb_depthwise_bwd with the same ca / cb / cc.  gate, dpool,
 * scale and shift are pre-offset to the slice and 16-byte aligned, ldg >= dw.C a multiple of 4. */
typedef struct yamb_dw_bwd_se {
  yamb_dw_bwd dw;
  const float* gate; const float* dpool; int32_t ldg;   /* [N][ldg] */
  const float* scale; const float* shift;               /* [C] BatchNorm-2 coefficients */
  int32_t act;                                          /* YAMB_ACT_* after BatchNorm-2 */
} yamb_dw_bwd_se;

int yamb_se_bwd_stats_bwd(const yamb_se_bwd_stats* args, yamb_stream_t stream);
int yamb_se_bn_bwd_finalize(const yamb_se_bn_bwd_finalize_args* args, yamb_stream_t stream);
int yamb_depthwise_bwd_se(const yamb_dw_bwd_se* args, yamb_stream_t stream);

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
 * 3x3, stride 2, pad 1, 3 input channels -> Cout on NHWC bf16: the first layer of the network
 * (reference models/mobilenet_supernet.py:124-130; its BatchNorm + activation follow through
 * yamb_bn_stats_fwd / yamb_bn_apply_fwd).  Weights fp32 in the parameter's own [Cout][3][3][3]
 * layout.  fwd writes y (16-byte aligned), Cout a multiple of 8, <= 64; wgrad ACCUMULATES
 * dw += sum dh * x (dh 16-byte aligned; no input gradient), Cout in {8, 16, 32, 64}.  Other
 * arguments return YAMB_EINVAL, with or without a device. */
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

/* Eval-mode stem ConvBNReLU in ONE launch: the forward kernel of yamb_stem_conv_fwd with the folded
 * BatchNorm and the activation applied before the store,
 *   y = bf16(act(scale[c] * bf16(conv) + shift[c]))
 * with exactly the expression of yamb_bn_apply_fwd, so y is bitwise equal to yamb_stem_conv_fwd
 * followed by yamb_bn_apply_fwd with the same scale / shift.  Shapes as yamb_stem_conv_fwd
 * (conv.dh / conv.dw unused). */
typedef struct yamb_stem_conv_eval {
  yamb_stem_conv conv;
  const float* scale;   /* [Cout] gamma * rsqrt(running_var + eps) */
  const float* shift;   /* [Cout] beta - running_mean * scale */
  int32_t act;          /* YAMB_ACT_* */
} yamb_stem_conv_eval;

int yamb_stem_conv_eval_fwd(const yamb_stem_conv_eval* args, yamb_stream_t stream);

/* The three stem entry points on uint8 images: x is uint8 [N][H][W][3] (HWC bytes, as a decoded
 * RGB image), normalised while the kernel stages it, with the fp32 operations and rounding of
 * torchvision's ToTensor() + Normalize(mean, std) followed by the bf16 rounding:
 *   x_staged = bf16(((float)u / 255 - mean[c]) / std[c])   inside the image, 0 in the padding.
 * Each entry computes the bits its bf16 twin computes on that normalised image.  Shapes, y, dh, dw
 * and ev.scale / ev.shift / ev.act (eval entry only) as the bf16 entries; a non-finite mean, or a
 * std that is zero or not finite, returns YAMB_EINVAL. */
typedef struct yamb_stem_conv_u8 {
  yamb_stem_conv_eval ev;    /* ev.conv.x: uint8 [N][H][W][3]; ev.scale/shift/act: eval entry only */
  float mean[3], std[3];     /* staged x = bf16(((float)u / 255 - mean[c]) / std[c]), 0 outside */
} yamb_stem_conv_u8;

int yamb_stem_conv_u8_fwd(const yamb_stem_conv_u8* args, yamb_stream_t stream);
int yamb_stem_conv_u8_wgrad(const yamb_stem_conv_u8* args, yamb_stream_t stream);
int yamb_stem_conv_u8_eval_fwd(const yamb_stem_conv_u8* args, yamb_stream_t stream);

/* ---- training-mode stem: BatchNorm statistics in the convolution, BatchNorm backward on load ------
 * For a stem ConvBNReLU whose only consumer applies the stem's BatchNorm + activation on load and
 * returns dz = da * act'(z) with the BatchNorm-backward statistics (yamb_dw_fwd in_scale /
 * in_shift, yamb_dw_bwd dx / bn: the depthwise of a first block without expansion), so neither the
 * activation nor its gradient nor dh reaches HBM:
 *   fwd  : y = the bits of yamb_stem_conv_fwd, plus the batch statistics of y finalised through
 *          `bn` (scale / shift, saved mean / invstd, running statistics, num_batches_tracked) as
 *          yamb_bn_stats_fwd does; per-thread fp32 sums in a fixed order, double across warps
 *          and CTAs
 *   wgrad: dw += sum dh * x with dh = bf16(fmaf(ca, dz, fmaf(cb, h, cc))) formed on load (the
 *          expression of yamb_bn_bwd_apply_bwd, 0 outside the image), the partial slabs and their
 *          order those of yamb_stem_conv_wgrad: dw is bitwise yamb_bn_bwd_apply_bwd followed by
 *          yamb_stem_conv_wgrad, the same on every run
 * x_u8 = 1: x is uint8 [N][H][W][3] normalised while staged, as yamb_stem_conv_u8 with mean / std.
 * Cout in {8, 16, 32, 64}; y, dz, h 16-byte aligned; bn.count = N*Ho*Wo.  Other arguments return
 * YAMB_EINVAL before any device work, with or without a device; YAMB_ENODEV without one. */
typedef struct yamb_stem_conv_train {
  int32_t N, H, W, Cout;
  const void* x;          /* bf16, or uint8 with x_u8 = 1: [N][H][W][3] */
  int32_t x_u8;
  float mean[3], std[3];  /* x_u8 = 1: staged x = bf16(((float)u / 255 - mean[c]) / std[c]) */
  const float* w;         /* [Cout][3][3][3] */
  void* y;                /* out bf16 [N][Ho][Wo][Cout], the raw convolution output h */
  const yamb_bn_fwd* bn;  /* the BatchNorm of y (batch statistics) */
} yamb_stem_conv_train;

typedef struct yamb_stem_conv_train_grad {
  int32_t N, H, W, Cout;
  const void* x;          /* as in the forward */
  int32_t x_u8;
  float mean[3], std[3];
  const void* dz;         /* bf16 [N][Ho][Wo][Cout]: gradient of the BatchNorm's output z */
  const void* h;          /* bf16 [N][Ho][Wo][Cout]: the forward's y */
  const float* ca; const float* cb; const float* cc;   /* [Cout] BatchNorm-backward coefficients */
  float* dw;              /* [Cout][3][3][3] += */
} yamb_stem_conv_train_grad;

int yamb_stem_conv_train_fwd(const yamb_stem_conv_train* args, yamb_stream_t stream);
int yamb_stem_conv_train_wgrad(const yamb_stem_conv_train_grad* args, yamb_stream_t stream);

/* ---- eval-mode head: 1x1 ConvBNReLU + full-extent average pool, ONE launch ------------------------
 * Replaces, in eval mode, the head ConvBNReLU (reference models/mobilenet_supernet.py:152-158) and
 * the AvgPool2d over the whole final feature map (:159):
 *   pooled[n][c] = bf16((1/HW) * sum_p bf16(act(scale[c] * bf16(x[n,p,:] . w[c,:]) + shift[c])))
 * The per-element rounding points are those of yamb_pointwise_gemm -> yamb_bn_apply_fwd; the sum
 * over p is fp32 in a fixed order (the same bits on every run).  The conv output and the activation
 * never reach HBM; `pooled` is the bf16 [N][Cout] operand of the classifier GEMM.  wgmma tensor
 * cores; Cin, Cout multiples of 8, Cin <= 512, any HW >= 1.  Other shapes return YAMB_EINVAL. */
typedef struct yamb_head_pool_eval {
  int32_t N, HW, Cin, Cout;
  const void* x;        /* bf16 [N][HW][Cin] (NHWC), 16-byte aligned */
  const void* w;        /* bf16 [Cout][Cin], 16-byte aligned */
  const float* scale;   /* [Cout] */
  const float* shift;   /* [Cout] */
  int32_t act;          /* YAMB_ACT_* */
  void* pooled;         /* out bf16 [N][Cout] */
} yamb_head_pool_eval;

int yamb_head_pool_eval_fwd(const yamb_head_pool_eval* args, yamb_stream_t stream);

/* ---- training-mode head: BatchNorm (batch statistics) + activation + full-extent average pool ----
 * Follows yamb_pointwise_gemm of the head 1x1 convolution run with `bn_fwd`, whose epilogue took
 * the batch statistics of its output h and wrote scale / shift, mean / invstd and the running
 * statistics.  Replaces yamb_bn_apply_fwd -> torch's mean over the pixels, and in backward the
 * broadcast of the pooled gradient -> yamb_bn_reduce_bwd -> yamb_bn_bwd_apply_bwd:
 *   forward : pooled[n][c] = bf16((1/HW) * sum_p bf16(act(scale[c] * h[n,p,c] + shift[c])))
 *             (the activation a is never written; the sum is fp32 in a fixed order: per-thread
 *             pixel lanes, lanes in order, then pixel-chunk slabs in order; no atomics)
 *   backward: dz = act'(scale*h + shift) * (dpooled[n][c] * (1/HW)), formed from h on the fly;
 *             pass 1: sum(dz), sum(dz * xhat) per channel -> bn (dgamma, dbeta +=; ca, cb, cc),
 *             the BatchNorm-backward finalize of yamb_bn_reduce_bwd (double across CTAs);
 *             pass 2: dh = bf16(ca*dz + cb*h + cc), skipped when dh is NULL.
 * C a multiple of 8, N * HW < 2^31, bf16 operands 16-byte aligned; bn.count must be N * HW.
 * Other arguments return YAMB_EINVAL, with or without a device.  The forward takes a
 * stream-ordered scratch of its own when it splits the pixels of an image over several CTAs. */
typedef struct yamb_head_pool_train {
  int32_t N, HW, C;
  const void* h;          /* bf16 [N][HW][C] (NHWC), the head convolution's raw output */
  const float* scale;     /* [C] */
  const float* shift;     /* [C] */
  int32_t act;            /* YAMB_ACT_* */
  void* pooled;           /* out bf16 [N][C] */
} yamb_head_pool_train;

typedef struct yamb_head_pool_train_grad {
  int32_t N, HW, C;
  const void* h;          /* bf16 [N][HW][C], as in the forward */
  const float* scale;     /* [C] the forward's coefficients (z = scale*h + shift) */
  const float* shift;     /* [C] */
  int32_t act;            /* YAMB_ACT_* */
  const void* dpooled;    /* bf16 [N][C], gradient of pooled */
  yamb_bn_bwd bn;         /* the forward's mean / invstd; dgamma, dbeta +=; ca, cb, cc out */
  void* dh;               /* out bf16 [N][HW][C], or NULL */
} yamb_head_pool_train_grad;

int yamb_head_pool_train_fwd(const yamb_head_pool_train* args, yamb_stream_t stream);
int yamb_head_pool_train_bwd(const yamb_head_pool_train_grad* args, yamb_stream_t stream);

/* ---- label-smoothed softmax cross entropy + top-k -------------------------------------------------
 * Replaces CrossEntropyLabelSmooth(reduction='none') (reference utils/optim.py:150-158), the
 * top-1 / top-5 `correct_k` bookkeeping of forward_loss (common.py:73-79) and their backward.
 *   forward : loss[n] = sum_c -t[n][c] log_softmax(logits)[n][c], t = (1-eps) onehot + eps/C;
 *             correct1/5[n] in {0,1} (ties like torch.topk: lower index wins);
 *             G[n][c] = softmax - t (bf16), what the backward needs
 *   backward: dlogits[n][c] = G[n][c] * dloss[n];  dbias[c] += sum_n dlogits[n][c] (classifier
 *             bias gradient, optional)
 * forward: C <= 4096, ld >= C, ldg >= C; backward: C, ldg, ldd even and >= C, G / dlogits 4-byte
 * aligned.  Other arguments return YAMB_EINVAL, with or without a device. */
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
 * reference models/mobilenet_supernet.py:163-167); C and ld >= C even, X 4-byte aligned */
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

/* The same two calls with the 64-channel slices of the hidden dimension of every output tile split
 * over the `cluster` CTAs (2, 4 or 8) of a thread-block cluster: rank r runs the slices
 * [r*NC/cluster, (r+1)*NC/cluster) of NC = ceil(Chid/64) and the ranks add their fp32 project
 * partials in rank order over distributed shared memory before BN3 (+x).  For small batches, whose
 * tiles leave most SMs idle.  The same function as yamb_block_eval_fwd, with the fp32 sum over the
 * slices associated differently (a fixed order: the same bits on every run); the pool pass writes
 * the same values as yamb_block_eval_pool_fwd.  YAMB_EINVAL for another cluster size, for a shape
 * yamb_block_eval_fwd does not cover, and when the tile plan with the partials does not fit a CTA's
 * shared memory (nothing enqueued). */
int yamb_block_eval_cluster_fwd(const yamb_block_eval* args, int32_t cluster, yamb_stream_t stream);
int yamb_block_eval_cluster_pool_fwd(const yamb_block_eval* args, int32_t cluster,
                                     yamb_stream_t stream);

/* ---- eval-mode multi-branch block (several depthwise kernels: AtomNAS), ONE launch ---------------
 * In eval mode a block of several branches (reference models/mobilenet_base.py:330-342 and
 * :446-451) is one single-branch block over the concatenated hidden dimension whose depthwise kernel
 * varies by channel: the project sums over the hidden channels, so their order is free.
 * yamb_block_eval_mb_pack lays the branches out as groups of decreasing k (each branch padded to a
 * multiple of 8 channels: zero W1 rows and W3 columns, BatchNorm gamma = beta = mean = 0, var = 1,
 * so a padded channel's a1 and a2 are exactly 0), with every tap table zero-embedded in the centre
 * of K_MAX x K_MAX.  yamb_block_eval_mb_fwd / _pool_fwd then run the yamb_block_eval_fwd / _pool_fwd
 * tile walk over the packed tensors, every 64-channel slice with the stencil of the group of its
 * first channel (the largest k among its channels; the smaller-k channels of a boundary slice add
 * products with zero taps, which leaves the fp32 sums unchanged).
 *
 * Pack: one branch's fp32 tensors as the modules hold them.  `w_project` and `se_reduce` point at
 * the branch's first column of row-major matrices with row stride `ld`. */
typedef struct yamb_mb_branch {
  int32_t k;                  /* 3, 5 or 7 */
  int32_t C;                  /* hidden channels of the branch */
  int32_t ld;                 /* row stride of w_project / se_reduce (>= C) */
  const float* w_expand;      /* [C][Cin] */
  yamb_bn_eval bn1, bn2;      /* over the branch's C channels (eps: that of the block call) */
  const float* w_dw;          /* [C][k][k] */
  const float* w_project;     /* [Cout][ld], the branch's columns */
  const float* se_reduce;     /* [R][ld], the branch's columns; NULL without Squeeze-and-Excitation */
  const float* se_expand;     /* [C][R] */
  const float* se_expand_bias;/* [C] */
} yamb_mb_branch;

typedef struct yamb_block_eval_mb_pack_args {
  int32_t Cin, Cout, R;       /* R: SE reduced width (0 without SE) */
  int32_t nbranch;            /* 1..3 */
  yamb_mb_branch branch[3];
  int32_t Chid, kmax;         /* packed hidden width (multiple of 8); largest k of the branches */
  const int32_t* map;         /* device [Chid]: (branch << 16) | channel, or -1 for a padded channel */
  void* w_expand;             /* out bf16 [Chid][Cin] */
  void* w_project;            /* out bf16 [Cout][Chid] */
  float* w_dw;                /* out [Chid][kmax][kmax] */
  float* bn1; float* bn2;     /* out [4][Chid]: gamma, beta, running mean, running var */
  float* se_reduce;           /* out [R][Chid] (with SE) */
  float* se_expand;           /* out [Chid][R] */
  float* se_expand_bias;      /* out [Chid] */
} yamb_block_eval_mb_pack_args;

/* base: the yamb_block_eval of the packed block (kernel = kmax in {5, 7}, with expansion, Chid the
 * packed width, w_expand / w_dw / w_project / bn1 / bn2 the packed tensors, gate / pooled over Chid).
 * Hidden channels [group_c0[i], group_c0[i+1]) (the last group up to Chid) have kernel group_k[i];
 * group_k strictly decreasing from group_k[0] = kmax, group_c0 increasing multiples of 8 from 0.
 * No cluster split (see yamb_block_eval_mb_cluster_fwd below).  YAMB_EINVAL for what
 * yamb_block_eval_fwd does not cover or bad groups (nothing enqueued), YAMB_ENODEV without a
 * device. */
typedef struct yamb_block_eval_mb {
  yamb_block_eval base;
  int32_t ngroups;            /* 1..3 */
  int32_t group_k[3];
  int32_t group_c0[3];
} yamb_block_eval_mb;

int yamb_block_eval_mb_pack(const yamb_block_eval_mb_pack_args* args, yamb_stream_t stream);
int yamb_block_eval_mb_fwd(const yamb_block_eval_mb* args, yamb_stream_t stream);
int yamb_block_eval_mb_pool_fwd(const yamb_block_eval_mb* args, yamb_stream_t stream);

/* The same two calls with the 64-channel slices of the packed hidden dimension of every output tile
 * split over the `cluster` CTAs (2, 4 or 8) of a thread-block cluster, as yamb_block_eval_cluster_fwd
 * splits a single-branch block: every slice runs the stencil of its own group whatever rank holds
 * it, and the ranks add their fp32 project partials in rank order before BN3 (+x).  For small
 * batches (AtomNAS at batch 1).  The same function as yamb_block_eval_mb_fwd with the sum over the
 * slices associated differently (the same bits on every run); the pool pass writes the same values
 * as yamb_block_eval_mb_pool_fwd.  YAMB_EINVAL for another cluster size, bad groups, a shape
 * yamb_block_eval_mb_fwd does not cover, and a tile plan whose partials do not fit a CTA's shared
 * memory (nothing enqueued: the caller runs the unsplit call); YAMB_ENODEV without a device. */
int yamb_block_eval_mb_cluster_fwd(const yamb_block_eval_mb* args, int32_t cluster, yamb_stream_t stream);
int yamb_block_eval_mb_cluster_pool_fwd(const yamb_block_eval_mb* args, int32_t cluster,
                                        yamb_stream_t stream);

/* ---- training-mode expand + depthwise forward, the expanded tile recomputed from x ---------------
 * Step 2 of a single-branch training block with expansion (reference models/mobilenet_base.py:
 * 391-411) without reading h1 back: once the expand GEMM (yamb_pointwise_gemm with bn_fwd) has
 * stored h1 = W1 x and finalised BatchNorm 1's batch coefficients, every depthwise output tile is a
 * function of an x tile with its halo.  Per tile: x (+halo, TMA) -> wgmma with the GEMM's bf16 W1
 * -> bf16 (the bits the GEMM stored) -> act(bn1_scale*h1 + bn1_shift) with yamb_depthwise_fwd's
 * on-load expression, 0 outside the image -> k x k stencil with yamb_depthwise_fwd's tap order ->
 * raw bf16 z2 -> h2, plus BatchNorm 2's batch statistics of the fp32 z2 into `bn` (last CTA
 * finalises; count = N*Ho*Wo).  h2 has the bits yamb_depthwise_fwd writes from the GEMM's h1; the
 * statistics agree with its to double rounding of the partial-sum order.
 * Covers k in {3,5,7}, stride 1 / 2, 8 <= Cin <= 256, any Chid (multiples of 8).  YAMB_EINVAL for
 * other shapes or bad pointers before any device work (with or without a device), and when the tile
 * plan does not fit the device's shared memory (nothing enqueued); YAMB_ENODEV without a device. */
typedef struct yamb_expand_dw_train {
  int32_t N, H, W;            /* input pixels (NHWC); output (H-1)/stride+1 x (W-1)/stride+1 */
  int32_t Cin, Chid;          /* multiples of 8; Cin <= 256 */
  int32_t kernel, stride;     /* 3, 5 or 7; 1 or 2 */
  int32_t act;                /* YAMB_ACT_* after BatchNorm 1 */
  int32_t ldh;                /* row pitch of h2 in channels (>= Chid, multiple of 8) */
  const void* x;              /* bf16 [N,H,W,Cin] */
  const void* w_expand;       /* bf16 [Chid][Cin] (the expand GEMM's operand) */
  const float* bn1_scale;     /* [Chid] BatchNorm-1 coefficients of the batch */
  const float* bn1_shift;     /* [Chid] */
  const float* w_dw;          /* fp32 [Chid][k][k] */
  void* h2;                   /* out bf16 [N,Ho,Wo] rows of ldh channels, channels [0, Chid) */
  const yamb_bn_fwd* bn;      /* BatchNorm-2 statistics of h2 */
} yamb_expand_dw_train;

int yamb_expand_dw_train_fwd(const yamb_expand_dw_train* args, yamb_stream_t stream);

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
 * 18 softmax_ce_grad, 19 stem_conv, 20 bn_eval, 21 block_eval, 22 in_fwd, 23 in_bwd, 24 sgd,
 * 25 stem_conv_eval, 26 head_pool_eval, 27 gemm_plan_info, 28 stem_conv_u8, 29 expand_bwd_args,
 * 30 expand_bwd_plan_info, 31 head_pool_train, 32 head_pool_train_grad, 33 stem_conv_train,
 * 34 stem_conv_train_grad, 35 block_eval_mb_pack_args, 36 block_eval_mb, 37 se_bwd_stats,
 * 38 se_bn_bwd_finalize_args, 39 dw_bwd_se, 40 expand_dw_train, 41 dw_fwd_grouped,
 * 42 dw_bwd_grouped) so bindings can self-check */
int yamb_struct_size(int which);

const char* yamb_last_error(void);
int yamb_version(void);

#ifdef __cplusplus
}
#endif
#endif /* YAMB200_H_ */
