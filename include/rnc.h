/* rnc.h — C ABI of librnc.so: the H100 (sm_90a) kernels behind RAFT-NCUP's per-iteration hot path.
 *
 * The reference (abdo-eldesokey/RAFT-NCUP @ 51ac387) has NO native layer: every op below is a chain of
 * PyTorch eager calls.  Each entry point therefore cites the reference *Python* interface it replaces
 * (file:line under /root/reference).  INTEGRATION.md shows the ctypes stub a maintainer of the reference
 * would add at each call site.
 *
 * Conventions
 *   - every function returns 0 (RNC_OK) or a negative rnc_status; nothing throws across the boundary
 *   - all pointers are DEVICE pointers to caller-owned buffers (e.g. torch tensor.data_ptr()); no hidden
 *     allocation, no global mutable state, re-entrant; work is enqueued on `stream` (a cudaStream_t passed
 *     as void*) and the call returns immediately
 *   - "NCHW" tensors are the reference's own layout; "CL" = channel-last [B][H][W][C] fp32, the resident
 *     layout of the 1/8-resolution activations inside the iteration loop
 */
#ifndef RNC_H_
#define RNC_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  RNC_OK = 0,
  RNC_ERR_BAD_SHAPE = -1,     /* dimension <= 0, unsupported radius/levels/channel count */
  RNC_ERR_BAD_POINTER = -2,   /* null or misaligned (16 B) pointer */
  RNC_ERR_UNSUPPORTED = -3,   /* valid request this build does not implement */
  RNC_ERR_CUDA = -4,          /* launch failed; see rnc_last_cuda_error() */
  RNC_ERR_WORKSPACE = -5      /* workspace too small */
} rnc_status;

/* Library identity / diagnostics. */
int rnc_abi_version(void);                 /* bumps on any signature change (now 18) */
const char* rnc_build_info(void);          /* e.g. "sm_90a nvcc 12.9" */
const char* rnc_status_string(int status);
int rnc_last_cuda_error(void);             /* cudaError_t of the last failed launch on this thread */
/* Number of kernels launched by this library on the calling thread since the last reset (bench.py's
 * `gpu_launches` claim is read from here). */
long long rnc_launch_count(void);
void rnc_launch_count_reset(void);

/* ------------------------------------------------------------------------------------------------
 * A1  CorrBlock.__init__  (core/corr.py:7-21, 47-55)
 * Replaces the all-pairs matmul + avg_pool2d pyramid.  Nothing quadratic is built: fmap1 is transposed to
 * CL and fmap2 is transposed + average-pooled (floor mode, 2x2) into a `levels`-deep CL pyramid; pooling
 * commutes with the dot product so lookups against it equal lookups into the reference's 4-D pyramid.
 *   fmap1, fmap2 : [B][D][H][W] fp32 NCHW
 *   f1_cl        : [B][H*W][D]
 *   f2_pyr       : level l at element offset rnc_pyramid_offset(B,D,H,W,l), shape [B][H>>l][W>>l][D]
 */
size_t rnc_pyramid_offset(int B, int D, int H, int W, int level);   /* in elements; level==levels -> total */
int rnc_fmap_prepare(const float* fmap1, const float* fmap2, int B, int D, int H, int W, int levels,
                     float* f1_cl, float* f2_pyr, void* stream);

/* ------------------------------------------------------------------------------------------------
 * A2/A3  CorrBlock.__call__ + bilinear_sampler  (core/corr.py:23-44, core/utils/utils.py:59-73)
 * Fused multi-scale lookup straight from the feature maps.
 *   coords : [B][2][H][W] fp32 NCHW (channel 0 = x, 1 = y), level-0 pixel units
 *   out    : layout 0 -> [B][L*(2r+1)^2][H][W]   (the reference's return value, corr.py:44)
 *            layout 1 -> CL [B][H][W][ldo], channels [0, L*(2r+1)^2) written, ldo >= that
 *   channel k = l*(2r+1)^2 + i*(2r+1) + j  samples level l at (cx/2^l + i - r, cy/2^l + j - r): the slow
 *   window index offsets x (corr.py:31-37).  Bilinear, zero outside, scaled by 1/sqrt(D).
 * Supported: D % 32 == 0, radius == 4 (the only value the reference's models use, raft_nc_dbl.py:41), 1 <= levels <= 4.
 */
int rnc_corr_lookup_fwd(const float* f1_cl, const float* f2_pyr, const float* coords,
                        int B, int D, int H, int W, int levels, int radius,
                        float* out, int layout, int ldo, void* stream);

/* Same lookup, written as exact fp16 hi/lo split planes (CL [B][H][W][ldo] halves each; value = hi + lo): the operand
 * format of rnc_conv2d_umma_fwd, so the 1x1 convc1 (update.py:82,90) consumes it without a conversion pass. */
int rnc_corr_lookup_split_fwd(const float* f1_cl, const float* f2_pyr, const float* coords,
                              int B, int D, int H, int W, int levels, int radius,
                              void* out_hi, void* out_lo, int ldo, int lvl_stride, void* stream);
/* lvl_stride: channels reserved per pyramid level in the output row (>= 81; level l starts at l*lvl_stride, the
 * channels [81, lvl_stride) of each level are written as zeros).  The tensor-core path uses 88 so that every 8-channel
 * group is one aligned 16-byte store and convc1's K stays 6 blocks of 64.
 * Channel order of the split planes inside a level ("resident order"; only convc1 consumes them, with its weight rows
 * permuted to match): tap (i, j) -> j*8 + i for i < 8, tap (8, j) -> 72 + j  — a pixel's 8 values of one window row are
 * one aligned 16-byte group.  The reference order k = i*9 + j is what rnc_corr_lookup_fwd returns. */

/* Tensor-core version of the lookup (wgmma + TMA; same reference code, corr.py:7-55 + utils.py:59-73).
 *   f1h_cl / f2h_pyr : the CL feature map / pyramid of rnc_fmap_prepare rounded once to halves (rnc_f32_to_f16), same
 *                      element offsets (rnc_pyramid_offset)
 *   f1_cl / f2_pyr   : the fp32 originals, used by the exact CUDA-core kernel for tiles whose lookup windows do not
 *                      fit the fixed per-level boxes (incoherent flow) — results never depend on a coherence assumption
 *   out_hi / out_lo  : CL split halves planes [B][H][W][ldo] (value = hi + lo)
 *   workspace        : rnc_corr_lookup_umma_workspace_bytes(B,H,W) bytes of device memory (per-tile fallback flags)
 * Supported: D == 256, levels == 4, radius == 4.
 */
size_t rnc_corr_lookup_umma_workspace_bytes(int B, int H, int W);
int rnc_corr_lookup_umma_fwd(const void* f1h_cl, const void* f2h_pyr, const float* f1_cl, const float* f2_pyr,
                             const float* coords, int B, int D, int H, int W, int levels, int radius,
                             void* out_hi, void* out_lo, int ldo, int lvl_stride, void* workspace, size_t workspace_bytes,
                             void* stream);   /* lvl_stride must be 88; resident channel order (above); out_hi/out_lo
                                                 16-byte aligned, ldo % 8 == 0: the tiles leave through TMA stores */
/* fp32 -> fp16 (round to nearest), n % 4 == 0. */
int rnc_f32_to_f16(const float* src, void* dst, size_t n, void* stream);

/* ------------------------------------------------------------------------------------------------
 * A5..A8  update block convolutions  (core/update.py:6-14, 33-60, 79-97, 114-141)
 * One generic channel-last convolution with the update block's fusions expressed as epilogues.
 * The input is the virtual concatenation of up to two CL segments (replaces torch.cat, update.py:46,49,95,132).
 * weight is pre-packed [KH*KW][Cin][CoutPad] fp32 (CoutPad = Cout rounded up to 64), bias [CoutPad].
 */
typedef enum {
  RNC_EPI_LINEAR = 0,   /* out = acc + bias                                                     */
  RNC_EPI_RELU = 1,     /* out = relu(acc + bias)                       update.py:90-96, 14     */
  RNC_EPI_SIGMOID = 2,  /* out = sigmoid(acc + bias)                                            */
  RNC_EPI_GRU_ZR = 3,   /* Cout = 2*C: ch<C: aux0[p][ch] = z = sigmoid(.)                       */
                        /*             ch>=C: out[p][ch-C] = sigmoid(.) * h[p][ch-C]   update.py:47-49 */
  RNC_EPI_GRU_Q = 4,    /* q = tanh(.); h[p][ch] = (1-z)*h + z*q with z = aux0       update.py:49-50 */
  RNC_EPI_RELU_FLOW = 5,/* RELU, and channels [Cout, Cout+2) of out receive flow = coords1-coords0 (update.py:97);
                           aux0 = coords1 NCHW [B][2][H][W]                                     */
  RNC_EPI_RELU_ADD_RELU = 6, /* relu(res + relu(acc + bias)): residual block tail, extractor.py:48-55 (umma only) */
  RNC_EPI_TANH_RELU = 7,     /* ch < Cout/2: tanh (-> out_f32 and split), else relu (-> split): raft_nc_dbl.py:138-140 (umma only) */
  RNC_EPI_FLOW_DELTA = 8     /* Cout = 2 (FlowHead.conv2, update.py:10,14): aux0 = coords1 NCHW [B][2][H][W] += (acc + bias)
                                (raft_nc_dbl.py:157); out_f32, if given, receives delta_flow NCHW (umma only) */
} rnc_epilogue;

/* rnc_conv_umma_desc.flags */
#define RNC_CONV_NO_HALO 1          /* force one A tile per filter tap (disable the row/column halo sharing) */
#define RNC_CONV_AUX_BLOCKED 16     /* aux0 (z gate) and add are tile-blocked: element (tile, channel c, row r) at ((tile*ld + c)*128 + r) */
#define RNC_CONV_OUT_BLOCKED 32     /* RNC_EPI_LINEAR: out_f32 in the same tile-blocked layout (produces an `add` operand)          */
#define RNC_CONV_WINDOW 128        /* in0 is a sliding-window view of a padded plane, see rnc_conv_umma_desc.win_pitch */
#define RNC_CONV_TF32 64            /* operands are fp32 hi/lo planes consumed as TF32 (wgmma .tf32, K = 8): value = hi + lo with
                                     * hi = tf32(value), 3 MMAs per K step as in the fp16 form but with fp32's exponent range — the
                                     * training path's layers (output gradients underflow the fp16 split).  The in / w pointers address float
                                     * planes, ld / ktot count floats, K blocks hold 32 channels, only out_f32 is written. */

typedef struct {
  const float* in0; int c0; int ld0;   /* segment 0: channels [0,c0), pixel stride ld0 floats   */
  const float* in1; int c1; int ld1;   /* segment 1 (optional, c1 = 0 if absent)                */
  const float* weight; const float* bias;
  float* out; int ldo;                 /* CL output, pixel stride ldo                           */
  float* h; int ldh;                   /* GRU hidden state (read; written by GRU_Q)             */
  float* aux0; int ldaux;              /* z buffer (GRU) or coords1 (RELU_FLOW)                 */
  int B, H, W;
  int cout;                            /* logical Cout (<= CoutPad)                             */
  int kh, kw;                          /* odd; zero padding kh/2, kw/2 (all reference convs)    */
  int epilogue;                        /* rnc_epilogue                                          */
} rnc_conv_desc;

int rnc_conv2d_cl_fwd(const rnc_conv_desc* desc, void* stream);
/* rnc_conv2d_cl_fwd with filter dilation dil (1..8): tap (ky, kx) reads input (y + (ky - kh/2)*dil, x + (kx - kw/2)*dil), zero
 * outside, i.e. nn.Conv2d(dilation=dil, padding=(k/2)*dil).  dil > 1 takes the LINEAR / RELU / SIGMOID epilogues. */
int rnc_conv2d_cl_dil_fwd(const rnc_conv_desc* desc, int dil, void* stream);

/* Tensor-core version of rnc_conv2d_cl_fwd (same reference code, same epilogues): wgmma on fp16 hi/lo split
 * operands with fp32 accumulation in registers (3 MMAs per K step: hi*hi + hi*lo + lo*hi), TMA-staged tiles.
 * Activations live as two CL planes of halves (value = hi + lo); weights are pre-split and pre-scaled by a power of two:
 *   w_hi/w_lo : [coutpad][ktot] halves, ktot = kh*kw * nblocks * 64, K index = (tap * nblocks + block) * 64 + c,
 *               blocks enumerate 64-channel slices of segment 0 then segment 1, zero rows for channels beyond Cin
 *   unscale   : 1 / (weight scale); out = act(acc * unscale + bias)
 * Outputs: out_f32 (CL fp32) and/or out_hi/out_lo (CL split halves); either may be NULL.
 *   GRU_ZR : z -> aux0 (fp32), r*h -> out_hi/out_lo;   GRU_Q : h (fp32, in place) and its split copy -> out_hi/out_lo
 *   RELU_FLOW: split output, flow appended at channels [cout, cout+2); aux0 = coords1 NCHW
 */
typedef struct {
  const void* in0_hi; const void* in0_lo; int c0; int ld0;
  const void* in1_hi; const void* in1_lo; int c1; int ld1;
  const void* w_hi; const void* w_lo; int ktot; int coutpad;
  const float* bias; float unscale;
  float* out_f32; int ldo_f32;
  void* out_hi; void* out_lo; int ldo_split;
  float* h; int ldh;
  float* aux0; int ldaux;
  int B, H, W;
  int cout;
  int kh, kw;
  int epilogue;
  int stride;                          /* 1 (or 0) | 2: output pixel (y,x) reads input (stride*y + ky - kh/2, ...) */
  int hin, win;                        /* input height/width (0 -> same as H, W)                                    */
  const float* res; int ldres;         /* residual (fp32 CL at output resolution) for RELU_ADD_RELU                 */
  int flags;                           /* RNC_CONV_*                                                                 */
  double* stats;                       /* optional (RNC_EPI_LINEAR + out_f32 only): [B][cout][2] sum / sum of squares of the
                                        * outputs, every term added in fp64, ACCUMULATED (caller keeps it zeroed:
                                        * rnc_instnorm_finalize re-zeroes) */
  const float* add; int ldadd;         /* optional: fp32 [B*H*W][ldadd] added to the pre-activation (after bias), e.g. the
                                        * hoisted contribution of input channels that do not change between calls */
  int win_pitch;                       /* RNC_CONV_WINDOW (kw = 1, stride 2, c1 = 0): position x of input row y exposes the c0
                                        * consecutive halves that start at element y*win_pitch + x*ld0 of in0 (ld0 < c0: the
                                        * windows overlap; the TMA unit builds the im2col rows); win = positions per row (one
                                        * per output column), hin = rows, the stride applies to rows only. Used by the encoders'
                                        * 7x7/2 stem: a [hin][win_pitch/4][4] zero-padded pixel plane, 16-pixel windows, ld0 = 8 */
  int dil;                             /* filter dilation 0..8 (0 or 1: none): tap (ky, kx) reads input (y + (ky - kh/2)*dil,
                                        * x + (kx - kw/2)*dil), zero outside (padding (k/2)*dil, nn.Conv2d(dilation=dil)).  dil > 1:
                                        * stride 1, LINEAR / RELU / SIGMOID, no stats / add / blocked / window operands; fp16 and TF32.
                                        * Runs as dil^2 launches, one per output phase (y % dil, x % dil), each the undilated
                                        * convolution of that phase's input and output sub-images (strided tensor maps). */
} rnc_conv_umma_desc;

/* Pixel tiles (128 output pixels each) a layer of this shape is cut into: a tile-blocked tensor with ld channels has
 * rnc_conv_umma_tiles(...) * ld * 128 floats; the tiling depends on (kh, kw, stride, H, W, flags & RNC_CONV_NO_HALO) only. */
long long rnc_conv_umma_tiles(int kh, int kw, int stride, int B, int H, int W, int flags);
int rnc_conv2d_umma_fwd(const rnc_conv_umma_desc* desc, void* stream);

/* fp32 CL [M][lds] channels [0,C) -> split halves planes [M][ldd] at channel offset ch_off, by the convolution epilogues'
 * rule: hi = rn_satfinite(value), lo = rn_satfinite(value - hi); hi + lo reproduces |value| <= 65504 to 22 bits, carries
 * 11 bits of the excess up to 131008 and saturates there. */
int rnc_f32_to_split(const float* src, int lds, int C, long long M, void* dst_hi, void* dst_lo, int ldd, int ch_off,
                     void* stream);

/* fp32 CL [M][lds] channels [0,C) -> TF32 hi/lo planes of floats [M][ldd] at channel offset ch_off: hi = value rounded to TF32
 * (cvt.rna), lo = value - hi (operands of RNC_CONV_TF32 layers; hi + lo reproduces the value to ~2^-21). */
int rnc_f32_to_tf32_split(const float* src, int lds, int C, long long M, float* dst_hi, float* dst_lo, int ldd, int ch_off,
                          void* stream);

/* convf1: Conv2d(2,128,7,padding=3)+ReLU on flow = coords1 - coords0 (update.py:83,92).
 * coords1 NCHW [B][2][H][W]; weight packed [49][2][Cout]; out CL. */
int rnc_conv_flow7x7_fwd(const float* coords1, const float* weight, const float* bias, int B, int H, int W,
                         int cout, float* out, int ldo, void* stream);

/* ------------------------------------------------------------------------------------------------
 * C6  BasicEncoder pieces (core/extractor.py:118-192) that are not wide convolutions; the 3x3/1x1 layers run on
 * rnc_conv2d_umma_fwd (stride 1/2, RELU / RELU_ADD_RELU / TANH_RELU epilogues).
 */
/* Image normalisation 2*(x/255)-1 (raft_nc_dbl.py:118-119) + conv1 = Conv2d(3,64,7,stride=2,padding=3) (extractor.py:135,171).
 * img NCHW [N][3][Hin][Win] raw 0..255; weight [147 = (c*7+ky)*7+kx][64]; bias [64]; out CL [N][ceil(Hin/2)][ceil(Win/2)][64]
 * as fp32 and/or split halves; relu != 0 applies ReLU (norm folded into the weights). */
int rnc_stem_conv7x7s2_fwd(const float* img, const float* weight, const float* bias, int N, int Hin, int Win, int relu,
                           float* out_f32, void* out_hi, void* out_lo, void* stream);
/* The same layer on the tensor cores: this call normalises the image and repacks it as a zero-padded pixel plane of split
 * halves [N][Hin][pitch_px][4] (pixel p = image column p - 3, channel 3 = 0; pitch_px even, >= Win + 6; the caller keeps
 * >= 16 zero pixels after the last row); rnc_conv2d_umma_fwd then reads it as a sliding-window view (RNC_CONV_WINDOW:
 * c0 = 64 = 16 pixels x 4, ld0 = 8, win_pitch = 4*pitch_px, kh = 7, kw = 1, stride 2) with the 7x7x3 filter laid out as
 * [64][7 rows][16 px x 4 ch] (zeros for px >= 7 and channel 3): the TMA unit builds the im2col rows, no copy. */
int rnc_stem_window_prep(const float* img, int N, int Hin, int Win, int pitch_px, void* out_hi, void* out_lo, void* stream);
/* nn.InstanceNorm2d (no affine, biased variance; extractor.py:28-33,128-129) statistics of x CL fp32 [N][P][C], C <= 128:
 * stats = fp64 scratch [N][C][2]; mean_rstd = [N][C][2] floats (mean, 1/sqrt(var+eps)).  Every route (this one,
 * rnc_instnorm_stats_det, and rnc_conv_umma_desc.stats + rnc_instnorm_finalize) adds x and x^2 in fp64 from the first term
 * and takes var = sum(x^2)/P - mean^2 in fp64, so at fnet's sizes (P up to 1.2e5 positions per image)
 * rstd stays within 1e-6 relative up to |mean|/std = 1e4. */
int rnc_instnorm_stats(const float* x, int N, int P, int C, float eps, double* stats, float* mean_rstd, void* stream);
/* Second half of rnc_instnorm_stats when the sums were accumulated elsewhere (rnc_conv_umma_desc.stats): stats [N][C][2]
 * fp64 sums over P positions -> mean_rstd, then stats is zeroed for the next producer. */
int rnc_instnorm_finalize(double* stats, int N, int P, int C, float eps, float* mean_rstd, void* stream);
/* Deterministic rnc_instnorm_stats (torch.use_deterministic_algorithms): each CTA of 512 positions writes its fp64 sums to
 * workspace (rnc_instnorm_stats_det_workspace_bytes(N, P, C) bytes, 16-byte aligned, no zeroing needed), and a second kernel
 * adds them in ascending CTA order; identical inputs give bit-identical mean_rstd.  Returns 0 bytes for a bad shape. */
size_t rnc_instnorm_stats_det_workspace_bytes(int N, int P, int C);
int rnc_instnorm_stats_det(const float* x, int N, int P, int C, float eps, void* workspace, size_t workspace_bytes,
                           float* mean_rstd, void* stream);
/* apply: mode 0: norm(x) -> out_f32;  1: relu(norm(x));  2: relu(res + relu(norm(x)))  (ResidualBlock.forward,
 * extractor.py:48-56); outputs fp32 and/or split halves, all CL [N][P][C]. */
int rnc_instnorm_apply(const float* x, const float* mean_rstd, const float* res, int N, int P, int C, int mode,
                       float* out_f32, void* out_hi, void* out_lo, void* stream);
/* Pooling half of rnc_fmap_prepare for feature maps that are already CL: fills levels 1..levels-1 of f2_pyr from level 0. */
int rnc_fmap_pyramid(float* f2_pyr, int B, int D, int H, int W, int levels, void* stream);

/* FlowHead.conv2 (update.py:10,14) fused with `coords1 = coords1 + delta_flow` (raft_nc_dbl.py:157):
 * in CL [B][H][W][cin]; weight packed [9][cin][2]; delta (optional, may be NULL) and coords1 NCHW [B][2][H][W]. */
int rnc_flow_head2_fwd(const float* in, int cin, int ldi, const float* weight, const float* bias,
                       int B, int H, int W, float* delta, float* coords1, void* stream);

/* convf1 = Conv2d(2,128,7,padding=3) on flow = coords1 - grid (update.py:83,93-94), first half of the tensor-core
 * formulation: writes, for every pixel, its zero-padded 7x7x2 flow neighbourhood as 98 (+30 zero) split halves,
 * column k = 2*(7*ky+kx)+c, rows of ld >= 128 halves; a 1x1 rnc_conv2d_umma_fwd with the [128][98] weight finishes it. */
int rnc_flow_im2col7_split_fwd(const float* coords1, int B, int H, int W, void* out_hi, void* out_lo, int ld, void* stream);

/* FlowHead.conv2 (update.py:10,14), second half of the tensor-core formulation: `taps` [B*H*W][ldt] fp32 holds, for every
 * pixel q, the 18 values W[o][:, ky, kx] . in[q] at column 2*(3*ky+kx)+o (a 1x1 convolution by rnc_conv2d_umma_fwd, K =
 * cin instead of 9*cin); this sums the in-image 3x3 neighbours (zero padding), adds bias[2] (device), writes delta
 * (optional, NCHW [B][2][H][W]) and does `coords1 = coords1 + delta_flow` (raft_nc_dbl.py:157). */
int rnc_flow_tap_gather_fwd(const float* taps, int ldt, const float* bias, int B, int H, int W, float* delta, float* coords1,
                            void* stream);

/* coords_grid / initialize_flow (core/utils/utils.py:76-79, raft_nc_dbl.py:83-90) (+ optional flow_init, :144-145).
 * coords1 = grid (+ flow_init);  flow_init may be NULL. */
int rnc_coords_init(float* coords1, const float* flow_init, int B, int H, int W, void* stream);
/* flow = coords1 - grid  -> NCHW [B][2][H][W]  (raft_nc_dbl.py:152,170). */
int rnc_coords_to_flow(const float* coords1, float* flow, int B, int H, int W, void* stream);

/* Warm start: forward_interpolate (core/utils/utils.py:28-56; evaluate.py:38-40): push every pixel along its flow,
 * keep samples landing strictly inside the image, give each grid point the flow of its nearest kept sample
 * (scipy griddata 'nearest', fill 0).  flow, out: NCHW [B][2][H][W]. */
int rnc_forward_interpolate_fwd(const float* flow, int B, int H, int W, float* out, void* stream);
/* Both warm starts of a bidirectional sequence step in one launch.  flow, out: NCHW [2B][2][H][W]; rows [0, B) are
 * forward flows and get rnc_forward_interpolate_fwd's result; rows [B, 2B) are backward flows b, whose samples move to
 * x - b(x) carrying b(x) (the constant-velocity warm start of the next backward pair), i.e. -forward_interpolate(-b). */
int rnc_forward_interpolate_bidir_fwd(const float* flow, int B, int H, int W, float* out, void* stream);

/* Layout plumbing between the reference's NCHW tensors and the resident CL buffers. */
int rnc_nchw_to_cl(const float* src, int B, int C, int H, int W, float* dst, int ldd, int ch_off, void* stream);
int rnc_cl_to_nchw(const float* src, int lds, int ch_off, int B, int C, int H, int W, float* dst, void* stream);

/* ------------------------------------------------------------------------------------------------
 * U1  RAFT.upsample_flow, convex combination  (core/raft.py:73-84)
 *   flow NCHW [B][2][H8][W8]; mask CL [B][H8][W8][ldm] with 576 logits (c = k*64 + sy*8 + sx, k = ky*3+kx),
 *   already scaled by 0.25 (update.py:140); out NCHW [B][2][8*H8][8*W8].
 */
int rnc_convex_upsample_fwd(const float* flow, const float* mask, int ldm, int B, int H8, int W8,
                            float* out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * U2  RAFT.upsample_flow prologue (raft_nc_dbl.py:110): x4 = nearest-x2 of flow_lr = coords1 - grid.
 *   coords1 NCHW [B][2][H8][W8] -> x4 NCHW [B][2][2*H8][2*W8]
 */
int rnc_flow_x2_fwd(const float* coords1, int B, int H8, int W8, float* x4, void* stream);

/* U3 (input staging)  upsampler.py:150,155 — builds the weights-net input at 1/4 resolution, CL [B][2*H8][2*W8][ldo]:
 *   channels 0,1 = x_lowres (NCHW [B][2][2*H8][2*W8]); channels 2..2+C = guidance (net, CL [B][H8][W8][ldg]) resized
 *   'area' H8 -> 2*H8, which for an integer x2 upscale is replication; channels >= 2+C are zero-filled.
 */
int rnc_ncup_guidance_fwd(const float* x_lowres, const float* net, int ldg, int C, int B, int H8, int W8,
                          float* out, int ldo, void* stream);

/* The same staging written directly as split halves planes [B][2*H8][2*W8][ldo] (ldo % 8 == 0, channels >= 2+C zero): the
 * operand of the tensor-core weights net, without the fp32 intermediate. */
int rnc_ncup_guidance_split_fwd(const float* x_lowres, const float* net, int ldg, int C, int B, int H8, int W8,
                                void* out_hi, void* out_lo, int ldo, void* stream);

/* U4 tail: Simple.out (1x1 conv 32->2) + sigmoid (interp_weights_est.py:37,47; upsampler.py:44-46):
 *   in CL [B][H4][W4][cin] -> conf NCHW [B][2][H4][W4]. weight packed [cin][2]. */
int rnc_conf_head_fwd(const float* in, int cin, int ldi, const float* weight, const float* bias,
                      int B, int H4, int W4, float* conf, void* stream);

/* ------------------------------------------------------------------------------------------------
 * U3/U5/U6  NConvUpsampler.forward + NConvUNet.forward (live path) + NConv2d.forward
 *           (core/upsampler.py:143-177,179-210; core/nconv_modules.py:106-136,164-199)
 * Fused zero-stuff (scale 4, offset 2) + 4 normalized convolutions + the x8 of raft_nc_dbl.py:161.
 *   x_lowres: NCHW [B][2][H4][W4]   low-resolution data (in RAFT: nearest-x2 flow at 1/4 resolution)
 *   conf    : NCHW [B][2][H4][W4]   sigmoid output of the weights net
 *   wts_host: HOST pointer to 224 floats = softplus_{beta=10}(weight_p) of nconv_in[2,1,5,5], nconv_x2.0[2,2,5,5],
 *             decoder.0[2,4,3,3], nconv_out[1,2,1,1] in that order (nconv_modules.py:250-264).  They are copied
 *             into the kernel's parameter bank at launch (read before the call returns), so the call stays
 *             re-entrant with no device-side global state.
 *   out     : NCHW [B][2][4*H4][4*W4] = out_scale * NConvUNet output  (out_scale = 8 in RAFT, raft_nc_dbl.py:161)
 *   conf_out: NCHW [B][2][4*H4][4*W4] or NULL: the chain's output confidence, the cout of NConvUNet.forward that
 *             upsampler.py:168 discards, i.e. nconv_out's den4 / (W4[0] + W4[1]) with den4 = W4[0]*c3[0] + W4[1]*c3[1] (c3: the
 *             decoder's output confidence).  It lies in [0, 1] and is not multiplied by out_scale.  NULL skips it.
 * out does not depend on whether conf_out is requested: it is bit-identical either way.
 * Returns RNC_ERR_UNSUPPORTED, before any launch, when 2*B or the rows of 30x30 output tiles exceed 65535.
 *
 * Training form of the same chain (fine-tuning the upsampler on a frozen trunk).
 * rnc_ncup_train_fwd: rnc_ncup_fwd with the 224 positive weights read from DEVICE memory (weights_dev, same order), so a
 *   trainable upsampler needs no device-to-host copy per call; out and conf_out (may be NULL, as above) are bit-identical to
 *   rnc_ncup_fwd's on the same weights.
 * rnc_ncup_bwd: gradients of L = sum(g_out * out) + sum(g_conf_out * conf_out) for (out, conf_out) = rnc_ncup_train_fwd(...):
 *   g_out      : NCHW [B][2][4*H4][4*W4] (may be NULL when g_conf_out is given)
 *   g_conf_out : NCHW [B][2][4*H4][4*W4] (may be NULL: no confidence term; at least one of g_out and g_conf_out is required)
 *   g_x_lowres : NCHW [B][2][H4][W4] (may be NULL)        g_conf : NCHW [B][2][H4][W4] (may be NULL)
 *   g_weights  : [224] w.r.t. the UNFOLDED positive weights (may be NULL): decoder.0's folded gradient goes to both halves
 *                W[:, :2] and W[:, 2:], and every layer's 1/sum(W) normalisation contributes to all of that layer's weights
 *   workspace  : rnc_ncup_bwd_workspace_bytes(B,H4,W4) bytes, 16-byte aligned, needed only with g_weights (no zeroing needed)
 * The kernel recomputes the forward per tile with the forward's own code and differentiates the (y*c, c) pairs it carries,
 * so gradients stay finite where the confidence is zero.  The confidence's adjoint enters at the last layer, dL/dc3[k] +=
 * g * W4[k] / S4 and dL/dW4[k] += g * (c3[k] / S4 - den4 / S4^2) with S4 = W4[0] + W4[1], and flows through the chain like
 * the flow's.  With g_conf_out NULL the call differentiates sum(g_out * out) alone: the gradients do not depend on whether
 * the forward wrote conf_out.  Deterministic: every input gradient is written by one CTA, the weight gradient is a fixed-order fp64 reduction of per-CTA
 * partials; identical inputs give bit-identical gradients.  Returns RNC_ERR_UNSUPPORTED, before any launch, when 2*B or the
 * rows of 32x32 output tiles exceed 65535 (rnc_ncup_bwd_workspace_bytes returns 0 then). */
int rnc_ncup_fwd(const float* x_lowres, const float* conf, const float* wts_host, int B, int H4, int W4,
                 float out_scale, float* out, float* conf_out, void* stream);
int rnc_ncup_train_fwd(const float* x_lowres, const float* conf, const float* weights_dev, int B, int H4, int W4,
                       float out_scale, float* out, float* conf_out, void* stream);
size_t rnc_ncup_bwd_workspace_bytes(int B, int H4, int W4);
int rnc_ncup_bwd(const float* x_lowres, const float* conf, const float* weights_dev, int B, int H4, int W4, float out_scale,
                 const float* g_out, const float* g_conf_out, float* g_x_lowres, float* g_conf, float* g_weights,
                 void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * A3  bilinear_sampler  (core/utils/utils.py:59-73) as a standalone operator: grid_sample(align_corners=True, bilinear,
 * zero padding) with the grid in pixel coordinates.  img NCHW [N][C][H][W]; coords [N][h][w][2] = (x, y); out NCHW
 * [N][C][h][w]; mask (optional, may be NULL) [N][h][w][1] as utils.py:69-71.  H, W >= 2 (the reference divides by W-1).
 */
int rnc_bilinear_sample_fwd(const float* img, const float* coords, int N, int C, int H, int W, int h, int w,
                            float* out, float* mask, void* stream);

/* ------------------------------------------------------------------------------------------------
 * U6  NConv2d.forward  (core/nconv_modules.py:164-199) — ONE normalized-convolution layer, the operator seam
 *     `NConv2d((data, conf)) -> (y, conf_out)`, the per-layer form the training path differentiates through, and the
 *     per-level chain of every NConvUNet configuration other than the shipped one (which runs the fused rnc_ncup_fwd).
 *   The input is the channel concatenation [up, full]: Cup channels of up_data/up_conf NCHW [N][Cup][Hup][Wup], read at
 *   full resolution through F.interpolate(mode='nearest', size=(H, W))'s index map min(floor(dst * (in/out)), in-1)
 *   (the decoder's `cat(F.interpolate(x_prev), skip)`, nconv_modules.py:129-131; Cup = 0 -> no up source, pointers
 *   ignored), then Cin channels of data/conf NCHW [N][Cin][H][W].
 *   weight: [Cout][Cup+Cin][kh][kw] fp32 = softplus_{beta=10}(weight_p) (nconv_modules.py:250-264; the caller applies it),
 *   zero padding k/2, stride 1;  bias: [Cout] or NULL
 *   y = (conv(data*conf, W) / (conv(conf, W) + eps) + bias) * y_scale,   conf_out = conv(conf, W) / sum_{i,ky,kx} W[o]
 *   (y_scale folds a caller's output scale into the last layer; 1 elsewhere.)
 * Supported: Cup + Cin <= 8, Cout <= 4, odd kh, kw <= 7.
 */
int rnc_nconv2d_fwd(const float* data, const float* conf, const float* weight, const float* bias, int N, int Cin, int Cout,
                    int H, int W, int kh, int kw, float eps, const float* up_data, const float* up_conf, int Cup, int Hup,
                    int Wup, float y_scale, float* y, float* conf_out, void* stream);
/* Backward of rnc_nconv2d_fwd at y_scale = 1 (autograd of nconv_modules.py:169-194: quotient rule through num/(den+eps),
 * bias, confidence propagation incl. its dependence on sum(W)).  y, conf_out: the forward's outputs (same bias).
 * g_y / g_conf_out: upstream gradients (either may be NULL = zero); g_data, g_conf ([N][Cin][H][W]), g_up_data, g_up_conf
 * ([N][Cup][Hup][Wup]: each coarse pixel sums the full-resolution pixels that read it), g_weight ([Cout][Cup+Cin][kh][kw],
 * w.r.t. the POSITIVE kernel; the caller chains softplus'), g_bias ([Cout], needs g_weight): outputs, each may be NULL.
 * With a bias, the quotient num/(den+eps) is recovered as y - bias from the forward's rounded output (an error of an ulp
 * of y, against autograd's exact quotient); den is recovered as conf_out * sum(W), as without a bias.
 * workspace: rnc_nconv2d_bwd_workspace_bytes(...) bytes, 16-byte aligned, no zeroing needed.  Every reduction runs in a
 * fixed order: identical inputs give bit-identical gradients. */
size_t rnc_nconv2d_bwd_workspace_bytes(int N, int Cin, int Cup, int Cout, int H, int W, int kh);
int rnc_nconv2d_bwd(const float* data, const float* conf, const float* weight, const float* bias, const float* y,
                    const float* conf_out, const float* g_y, const float* g_conf_out, int N, int Cin, int Cout, int H, int W,
                    int kh, int kw, float eps, const float* up_data, const float* up_conf, int Cup, int Hup, int Wup,
                    float* g_data, float* g_conf, float* g_up_data, float* g_up_conf, float* g_weight, float* g_bias,
                    void* workspace, size_t workspace_bytes, void* stream);

/* U6  NConvUNet.downsample_data_conf (core/nconv_modules.py:94-104), ds_factor 2:
 *   conf_out = max_pool2d(conf, 2, 2) / 4 (floor mode; the first maximum in row-major window order wins, as F.max_pool2d);
 *   data_out = data at the confidence argmax (max_pool_data = 0, 'conf_based') or max_pool2d(data, 2, 2) (1, 'max_pooling').
 *   data, conf NCHW [N][C][H][W], H, W >= 2;  data_out, conf_out [N][C][H/2][W/2];
 *   idx: int32 [2][N][C][H/2][W/2], written: the in-plane flat index (y*W + x) of the confidence argmax, then of the data's.
 * rnc_nconv_pool2_bwd routes g_conf_out / 4 and g_data_out (either may be NULL = zero) to those argmaxes; g_data, g_conf
 * [N][C][H][W] (either may be NULL) are fully written (zero elsewhere). */
int rnc_nconv_pool2_fwd(const float* data, const float* conf, int N, int C, int H, int W, int max_pool_data, float* data_out,
                        float* conf_out, int* idx, void* stream);
int rnc_nconv_pool2_bwd(const int* idx, const float* g_data_out, const float* g_conf_out, int N, int C, int H, int W,
                        float* g_data, float* g_conf, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Training path (train.py:203-227; SURVEY.md §8f-3, Appendix G): backward kernels, exact fp32.
 *
 * Gradient of CorrBlock.__call__ (core/corr.py:23-44; the reference back-propagates through the stored 4-D pyramid) w.r.t.
 * the feature maps.  coords are detached (raft_nc_dbl.py:149): no gradient flows to them.
 *   g_out    : CL [B][H][W][ldg], channels [0, 324) in the reference order k = l*81 + i*9 + j
 *   g_f1     : CL [B][H*W][D], written
 *   g_f2_pyr : pyramid layout of rnc_fmap_prepare, ACCUMULATED with atomics — the caller zero-fills it; finish with
 *              rnc_pyramid_pool_bwd, which folds levels 3..1 into level 0 (adjoint of the 2x2 average pooling,
 *              core/corr.py:18-21 applied to features) so that level 0 holds d loss / d fmap2 (CL)
 */
int rnc_corr_lookup_bwd(const float* f1_cl, const float* f2_pyr, const float* coords, const float* g_out, int ldg,
                        int B, int D, int H, int W, int levels, int radius, float* g_f1, float* g_f2_pyr, void* stream);
int rnc_pyramid_pool_bwd(float* g_f2_pyr, int B, int D, int H, int W, int levels, void* stream);
/* Deterministic rnc_corr_lookup_bwd: the same g_f1; d fmap2 without atomics, and g_f2_pyr is WRITTEN (every position of every
 * level; no zero-fill needed).  Each pixel stages its 100 window gradients per level and its window-origin cell; a stable
 * radix sort groups the pixels by cell; then every pyramid position sums gv * f1[p] over the 10x10 cells whose window
 * covers it, cells in a fixed order and pixels in ascending index.  Each product is rounded as the atomic kernel rounds it,
 * so the result is one of the sums the atomic kernel can produce.  workspace: rnc_corr_lookup_bwd_workspace_bytes(B, H, W,
 * levels) bytes, 16-byte aligned (0 for a bad shape). */
size_t rnc_corr_lookup_bwd_workspace_bytes(int B, int H, int W, int levels);
int rnc_corr_lookup_bwd_det(const float* f1_cl, const float* f2_pyr, const float* coords, const float* g_out, int ldg,
                            int B, int D, int H, int W, int levels, int radius, float* g_f1, float* g_f2_pyr,
                            void* workspace, size_t workspace_bytes, void* stream);

/* Weight and bias gradient of a channel-last convolution y = conv(x, w) + b (stride 1 or 2, zero padding k/2):
 *   x  : CL [B][Hin][Win][ldx], cin % 4 == 0;   gy : CL [B][ceil(Hin/s)][ceil(Win/s)][ldg] = d loss / d y
 *   gw : [kh*kw][cin][ldw] fp32 (the packing of rnc_conv2d_cl_fwd's weight), WRITTEN (no zero-fill needed)
 *   gb : [cout], written, may be NULL
 * Deterministic: 64x64 (ci, co) tiles per tap, the pixels split over blocks by a count chosen from the shape alone; every
 * block writes its fp32 partial sums to workspace, and a second kernel adds them in ascending block order, from 0, in fp32.
 * Identical inputs give bit-identical gradients.  workspace: rnc_conv2d_cl_wgrad_workspace_bytes(...) bytes, at most 52 MB
 * (0 for a bad shape).
 * The data gradient is rnc_conv2d_cl_fwd on gy (zero-dilated for stride 2) with the flipped, transposed weights. */
size_t rnc_conv2d_cl_wgrad_workspace_bytes(int cin, int cout, int B, int Hin, int Win, int kh, int kw, int stride);
int rnc_conv2d_cl_wgrad_det(const float* x, int ldx, int cin, const float* gy, int ldg, int cout, int B, int Hin, int Win,
                            int kh, int kw, int stride, float* gw, int ldw, float* gb, void* workspace, size_t workspace_bytes,
                            void* stream);
/* The same weight / bias gradient for a stride-1 convolution with dilation dil (1..8; rnc_conv2d_cl_dil_fwd): tap (ky, kx) pairs
 * gy at (y, x) with x at (y + (ky - kh/2)*dil, x + (kx - kw/2)*dil).  Same tiles, K split, fixed-order sum and workspace size as
 * the undilated layer (0 bytes for a bad shape or dil).  Its data gradient is rnc_conv2d_cl_dil_fwd on gy with the flipped,
 * transposed weights and the same dil. */
size_t rnc_conv2d_cl_wgrad_dil_workspace_bytes(int cin, int cout, int B, int Hin, int Win, int kh, int kw, int dil);
int rnc_conv2d_cl_wgrad_dil_det(const float* x, int ldx, int cin, const float* gy, int ldg, int cout, int B, int Hin, int Win,
                                int kh, int kw, int dil, float* gw, int ldw, float* gb, void* workspace, size_t workspace_bytes,
                                void* stream);

/* ------------------------------------------------------------------------------------------------
 * T1  FlowAugmentor / SparseFlowAugmentor.__call__ (core/utils/augmentor.py) and the tensor conversion after it in
 * FlowDataset.__getitem__ (core/datasets.py:75-90), for a batch of samples of any source sizes.  rnc/augment.py draws
 * every random parameter on the host in the reference's order; these kernels apply them with Pillow's and cv2's
 * rounding, so that the outputs equal the reference's for the same draws (images and valid bit for bit).
 *
 * One descriptor per sample.  Offsets are in bytes into `src`:
 *   img1, img2 : uint8 [3][H][W] planar RGB       flow : fp32 [2][H][W]       valid : fp32 [H][W] (sparse only)
 * rh, rw       : size after the resize (cv2's rint(W * fx), rint(H * fy)); H, W when resized == 0
 * y0, x0       : crop origin in the resized, flipped image; 0 <= y0 <= rh - crop_h, 0 <= x0 <= rw - crop_w
 * asym         : 1 = img1 is jittered with perm[0]/factor[0]/hue[0] and img2 with the [1] entries; 0 = both with [0],
 *                the contrast mean taken over the stacked pair
 * perm         : ColorJitter's op order (torch.randperm(4)): 0 brightness, 1 contrast, 2 saturation, 3 hue
 * factor       : brightness, contrast, saturation factors;  hue: uint8 added to Pillow's H band (np.int32(h * 255))
 * erase        : n_erase rectangles {x0, y0, dx, dy} of img2 in source pixels, painted with its jittered mean colour
 * fx, fy       : the resize factors;  ifx, ify: 1.0 / fx, 1.0 / fy (cv2's source-coordinate step)
 */
typedef struct {
  long long img1, img2, flow, valid;
  int H, W, rh, rw;
  int resized, hflip, vflip, y0, x0, asym;
  int perm[2][4];
  float factor[2][3];
  int hue[2];
  int n_erase;
  int erase[2][4];
  int pad;
  double fx, fy, ifx, ify;
} rnc_aug_desc;

/* Workspace of rnc_augment: per-sample integer statistics, plus the crop-sized winner map when sparse (0 for a bad shape). */
size_t rnc_augment_workspace_bytes(int B, int crop_h, int crop_w, int sparse);
/* desc_host and desc_dev hold the same B descriptors; the host copy is checked (RNC_ERR_BAD_SHAPE for sizes, crops, offsets
 * or draws out of range, RNC_ERR_BAD_POINTER for null or misaligned pointers), the device copy is read by the kernels.
 * sparse = 0: FlowAugmentor semantics (valid = |u| < 1000 & |v| < 1000); 1: SparseFlowAugmentor (no vflip, no asym).
 * Outputs: img1, img2 fp32 [B][3][crop_h][crop_w] with integer values, flow fp32 [B][2][crop_h][crop_w], valid fp32
 * [B][crop_h][crop_w].  workspace: 16-byte aligned, zeroed by the call.  Integer reductions only: outputs repeat bit for bit. */
int rnc_augment(const rnc_aug_desc* desc_host, const rnc_aug_desc* desc_dev, int B, const void* src, size_t src_bytes,
                int crop_h, int crop_w, int sparse, float* img1, float* img2, float* flow, float* valid, void* workspace,
                size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * V1  flow_to_image (core/utils/flow_viz.py:240-275, with compute_color :196-237) for a batch of float32 flows, as evaluate.py
 * and demo.py call it before cv2.imwrite, with numpy 2.x's float32 / float64 promotion.
 *   flow      : fp32, element (b, c, y, x) at flow[b*sb + c*sc + y*sy + x*sx] (c = 0 is u, 1 is v); 4-byte aligned
 *   out       : uint8 [B][H][W][3] contiguous, the reference's channel order (RGB, handed unchanged to cv2.imwrite)
 *   workspace : rnc_flow_to_image_workspace_bytes(B) bytes, 4-byte aligned, zeroed by the call (per-image maximum radius)
 * Two launches, no host synchronisation.  Every output bit repeats from run to run.  Radius and maximum are float32, the rest
 * float64 (np.finfo(float).eps is a float64 scalar), every step rounded as numpy rounds it.  The arc tangent is CUDA's float64
 * atan2 (within 2 ulp) where the reference's is numpy's, so a channel could differ by one level where the two land on either
 * side of a level boundary. */
size_t rnc_flow_to_image_workspace_bytes(int B);   /* 0 for B <= 0 */
int rnc_flow_to_image(const float* flow, long long sb, long long sc, long long sy, long long sx, int B, int H, int W,
                      unsigned char* out, void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * V2  validation metrics (evaluate.py:88-182 validate_chairs / validate_sintel / validate_kitti) for a batch of float32 flows.
 *   flow, gt  : fp32, element (b, c, y, x) at flow[b*fb + c*fc + y*fy + x*fx] (gt likewise; c = 0 is u, 1 is v); 4-byte aligned
 *   valid     : fp32, pixel (b, y, x) at valid[b*vb + y*vy + x*vx], valid where >= 0.5; NULL: every pixel is valid
 *   counts    : int64 [B][5], per image the valid pixels, of them epe < 1, < 3, < 5, and KITTI outliers
 *               (epe > 3 and epe / |gt| > 0.05); 8-byte aligned
 *   epe_sum   : fp64 [B], per image the sum of the valid pixels' epe; 8-byte aligned
 *   workspace : rnc_flow_metrics_workspace_bytes(B, H, W) bytes, 16-byte aligned, no zeroing needed (per-CTA partials)
 * Each pixel is rounded as torch's float32 formulas round it (no FMA; IEEE division, so x/0 = inf and 0/0 = NaN).  Two launches,
 * no host synchronisation; the sums are added in a fixed order that depends only on H*W, so an image's results are bit for
 * bit the same whatever B, its position in the batch or the GPU.  Bad arguments return before any launch. */
size_t rnc_flow_metrics_workspace_bytes(int B, int H, int W);   /* 0 for a bad shape */
int rnc_flow_metrics(const float* flow, long long fb, long long fc, long long fy, long long fx, const float* gt, long long gb,
                     long long gc, long long gy, long long gx, const float* valid, long long vb, long long vy, long long vx,
                     int B, int H, int W, long long* counts, double* epe_sum, void* workspace, size_t workspace_bytes,
                     void* stream);

/* ------------------------------------------------------------------------------------------------
 * V3  sparsification curves of a confidence score (AUSE) for a batch of float32 flows, over the fractions f_k = k/100, k < 100.
 *   flow, gt, valid : as rnc_flow_metrics (epe rounded as it rounds it; valid where >= 0.5, NULL: every pixel is valid)
 *   score           : fp32, pixel (b, y, x) at score[b*sb + y*sy + x*sx], higher is more confident; 4-byte aligned
 *   count           : int64 [B][100], N - m_k, with N the image's valid pixels and m_k = floor(k*N/100); 8-byte aligned
 *   kept_epe        : fp64 [B][100], the sum of the epe of the valid pixels left once the m_k of lowest score are removed
 *                     (ties: lower row-major index first; a NaN score ranks below -inf); 8-byte aligned
 *   ideal_epe       : fp64 [B][100], the same once the m_k of largest epe are removed (a NaN epe ranks largest); 8-byte aligned
 *   workspace       : rnc_sparsification_workspace_bytes(B, H, W) bytes, 16-byte aligned, no zeroing needed (sort buffers)
 * One device-wide radix sort per order with the image index in the key's high bits, then fixed-order fp64 range sums and
 * suffix sums: no atomics and no host synchronisation, so an image's results are bit for bit the same whatever B, its position
 * in the batch or the GPU.  An image without a valid pixel gives zeros.  RNC_ERR_BAD_SHAPE when B*H*W >= 2^31 (the sort's
 * index range) or B > 65535.  Bad arguments return before any launch. */
size_t rnc_sparsification_workspace_bytes(int B, int H, int W);   /* 0 for a bad shape */
int rnc_sparsification(const float* flow, long long fb, long long fc, long long fy, long long fx, const float* gt, long long gb,
                       long long gc, long long gy, long long gx, const float* valid, long long vb, long long vy, long long vx,
                       const float* score, long long sb, long long sy, long long sx, int B, int H, int W, long long* count,
                       double* kept_epe, double* ideal_epe, void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * V4  forward-backward consistency of B flow pairs, both directions in one launch.
 *   flow_fw, flow_bw : fp32 [B,2,H,W] through element strides (fb..fx, gb..gx), component c of pixel (b, y, x) at
 *                      flow[b*fb + c*fc + y*fy + x*fx]; 4-byte aligned
 *   occ_fw, occ_bw   : uint8 [B][H][W] contiguous.  For pixel x of direction F -> G (G -> F for the _bw outputs), p = x + F(x)
 *                      and G^(p) bilinear with zero padding on align_corners=True pixel coordinates: bit 0 when
 *                      |F + G^|^2 > alpha1 (|F|^2 + |G^|^2) + alpha2 or that sum is not finite; bit 1 when p lies outside
 *                      [0, W-1] x [0, H-1] (a NaN target is outside, and gets bit 0 too)
 *   err_fw, err_bw   : fp32 [B][H][W] contiguous, |F(x) + G^(p)|; +inf where p is outside or the sum is not finite
 * Every operation rounded once in float32 (no FMA).  No atomics, no host synchronisation: a pixel's outputs depend only on its
 * own image.  RNC_ERR_BAD_SHAPE for B > 65535 or H*W >= 2^31. */
int rnc_fb_consistency(const float* flow_fw, long long fb, long long fc, long long fy, long long fx, const float* flow_bw,
                       long long gb, long long gc, long long gy, long long gx, int B, int H, int W, float alpha1,
                       float alpha2, unsigned char* occ_fw, unsigned char* occ_bw, float* err_fw, float* err_bw,
                       void* stream);

/* ------------------------------------------------------------------------------------------------
 * V5  per-region validation metrics: Sintel's matched / unmatched, boundary-distance and speed regions, KITTI 2015's
 * background / foreground over all and non-occluded pixels (definitions: rnc/metrics.py, DESIGN §3.14).
 *
 * rnc_boundary_dist2: the exact squared Euclidean distance, in pixels, of every pixel to the nearest occlusion-boundary pixel
 * of its image.  A boundary pixel has a 4-neighbour inside the image whose label (occluded where occ >= 0.5) differs from its
 * own; pixels on both sides of the boundary count.
 *   occ : fp32, pixel (b, y, x) at occ[b*ob + y*oy + x*ox]; 4-byte aligned
 *   d2  : int32 [B][H][W] contiguous; RNC_DIST2_NONE in an image without a boundary pixel
 * A column pass, then the lower envelope of parabolas along each row, in integers only (intersections compared by
 * cross-multiplying in int64): the result is exact.  Two launches, no atomics, no host synchronisation.  RNC_ERR_BAD_SHAPE
 * unless 1 <= H, W <= 4096 and 1 <= B <= 65535.  Bad arguments return before any launch.
 *
 * rnc_region_metrics: per image and per cell, the five counts and the fp64 EPE sum of rnc_flow_metrics (each pixel rounded
 * as it rounds it, valid where valid >= 0.5, NULL: every pixel is valid).  A cell is one joint label of a pixel:
 *   RNC_REGIONS_SINTEL (32 cells): 16*occluded + 4*d + s, occluded where mask (occ) >= 0.5; d from d2 (rnc_boundary_dist2's
 *     output, int32 [B][H][W] contiguous): 0 for d2 < 100, 1 for < 3600, 2 for < 19600, else 3; s from mag = |gt|: 0 for
 *     mag < 10, 1 for < 40, 2 for >= 40, 3 for NaN.  fg must be NULL.
 *   RNC_REGIONS_KITTI (4 cells): 2*(mask (noc) < 0.5) + (fg >= 0.5); fg NULL: every pixel is background.  d2 must be NULL.
 *   mask, fg   : fp32 through element strides (mb..mx, qb..qx), as valid; 4-byte aligned
 *   counts     : int64 [B][cells][5] (valid, epe < 1, < 3, < 5, KITTI outliers); 8-byte aligned
 *   epe_sum    : fp64 [B][cells]; 8-byte aligned
 *   workspace  : rnc_region_metrics_workspace_bytes(kind, B, H, W) bytes, 16-byte aligned, no zeroing needed
 * Two launches, no host synchronisation, no floating-point atomics; the sums are added in a fixed order that depends only on
 * H*W and the cell count, so an image's results are bit for bit the same whatever B, its position in the batch or the GPU.
 * RNC_ERR_UNSUPPORTED for an unknown kind.  Bad arguments return before any launch. */
#define RNC_DIST2_NONE 2147483647
#define RNC_REGIONS_SINTEL 0
#define RNC_REGIONS_KITTI 1
#define RNC_REGION_CELLS_SINTEL 32
#define RNC_REGION_CELLS_KITTI 4
int rnc_boundary_dist2(const float* occ, long long ob, long long oy, long long ox, int B, int H, int W, int* d2,
                       void* stream);
size_t rnc_region_metrics_workspace_bytes(int kind, int B, int H, int W);   /* 0 for a bad kind or shape */
int rnc_region_metrics(int kind, const float* flow, long long fb, long long fc, long long fy, long long fx, const float* gt,
                       long long gb, long long gc, long long gy, long long gx, const float* valid, long long vb, long long vy,
                       long long vx, const float* mask, long long mb, long long my, long long mx, const int* d2,
                       const float* fg, long long qb, long long qy, long long qx, int B, int H, int W, long long* counts,
                       double* epe_sum, void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * V6  frame interpolation from both flows and the occlusion masks, and the interpolation error (definition: rnc/interp.py,
 * DESIGN §3.15).
 *
 * rnc_interpolate: for each pair b and each time t_k, the frame between frame0 and frame1 at t_k.
 *   frame0, frame1 : fp32 [B,3,H,W] (0..255) through element strides (ab..ax, bb..bx); 4-byte aligned
 *   flow, flow_bw  : fp32 [B,2,H,W] through element strides, F (frame 0 -> 1) and G (1 -> 0); 4-byte aligned
 *   occ0, occ1     : uint8 [B][H][W] contiguous, rnc_fb_consistency's occ_fw / occ_bw of F and G; a pixel is visible where 0
 *   times          : T host floats, each 0 < t < 1; 1 <= T <= RNC_INTERP_MAX_TIMES
 *   out            : fp32 [B][T][3][H][W] contiguous; 4-byte aligned
 *   workspace      : rnc_interpolate_workspace_bytes(B, T, H, W) bytes, 16-byte aligned, no zeroing needed: the uint64 splat
 *                    map [B][T][H][W], then the int32 nearest-site map [B][T][H][W]
 * 1. Splat: a pixel x of frame 0 with occ0 == 0 and a finite F(x) proposes u = F(x) at q = rint(x + t F(x)) (half to even)
 *    when q is in the frame, keyed by e = sum_c |I1^_c(x + F(x)) - I0_c(x)| (channels in order); a pixel y of frame 1 likewise
 *    proposes u = -G(y) at rint(y + (1 - t) G(y)) with occ1 and e = sum_c |I0^_c(y + G(y)) - I1_c(y)|.  I^ is bilinear with
 *    the coordinates clamped to the frame.  Each pixel keeps the smallest (e, source index), frame 0's sources 0..HW-1 and
 *    frame 1's HW..2HW-1: an integer atomicMin of (float bits of e) << 32 | index.
 * 2. Fill: a pixel without a proposal takes the u of the nearest pixel with one (exact squared distance, ties to the smallest
 *    column, then row); u = 0 in an image without a proposal.
 * 3. Composite: x0 = x - t u, x1 = x + (1 - t) u; v0 when x0 is in the frame and occ0(rint(x0)) == 0, v1 likewise; the output
 *    is (1 - t) I0^(x0) + t I1^(x1) when v0 == v1, else the visible sample.
 * Every operation rounded once in float32 (no FMA).  A memset and four launches, no host synchronisation, no floating-point
 * atomics: an output depends only on its own pair and time.  RNC_ERR_BAD_SHAPE for a time outside (0, 1), H or W above 4096,
 * or B*T above 65535.  Bad arguments return before any launch.
 *
 * rnc_interp_error: per image n, sq_sum[n] = the fp64 sum over its pixels of sum_c (pred - gt)^2 (each difference and square in
 * fp64) and count[n] = H*W.
 *   pred, gt  : fp32 [N,3,H,W] through element strides; 4-byte aligned
 *   sq_sum    : fp64 [N], 8-byte aligned; count: int64 [N], 8-byte aligned
 *   workspace : rnc_interp_error_workspace_bytes(N, H, W) bytes, 16-byte aligned, no zeroing needed (per-CTA partials)
 * Two launches, no host synchronisation; the sums are added in a fixed order that depends only on H*W, so an image's result is
 * bit for bit the same whatever N, its position in the batch or the GPU.  Bad arguments return before any launch. */
#define RNC_INTERP_MAX_TIMES 64
size_t rnc_interpolate_workspace_bytes(int B, int T, int H, int W);   /* 0 for a bad shape */
int rnc_interpolate(const float* frame0, long long ab, long long ac, long long ay, long long ax, const float* frame1,
                    long long bb, long long bc, long long by, long long bx, const float* flow, long long fb, long long fc,
                    long long fy, long long fx, const float* flow_bw, long long gb, long long gc, long long gy, long long gx,
                    const unsigned char* occ0, const unsigned char* occ1, const float* times, int T, int B, int H, int W,
                    float* out, void* workspace, size_t workspace_bytes, void* stream);
size_t rnc_interp_error_workspace_bytes(int N, int H, int W);   /* 0 for a bad shape */
int rnc_interp_error(const float* pred, long long pb, long long pc, long long py, long long px, const float* gt, long long gb,
                     long long gc, long long gy, long long gx, int N, int H, int W, double* sq_sum, long long* count,
                     void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * V7  unsupervised losses of N rows (source image I1, target image I2, flow F), forward and backward (definition:
 * rnc/unsupervised.py, DESIGN §3.16).  Shapes: 1 <= N <= 65535, H, W >= 8, H*W < 2^30; RNC_ERR_BAD_SHAPE otherwise.  Bad
 * arguments return before any launch.  No atomics: every output is a fixed-order sum, bit-identical from run to run, and a
 * row's results are the same bits whatever N or its position in the batch.
 *
 * rnc_census_loss_fwd: per row r, S_r = sum_p v l (fp64) and M_r = sum_p v, where g(I) = 0.2989 R + 0.5870 G + 0.1140 B,
 * W^ = g(I2) sampled bilinearly at p + F(p) (align_corners pixel coordinates, taps outside the frame 0), c_d(A)(p) =
 * delta / sqrt(0.81 + delta^2) with delta = A(p+d) - A(p) over the 7x7 offsets d (A = 0 outside the frame), h = sum_d e^2 /
 * (0.1 + e^2) with e = c_d(g(I1)) - c_d(W^), l = (h + 0.01)^0.4, and v = mask(p) for 3 <= x <= W-4, 3 <= y <= H-4, else 0.
 *   image1, image2 : fp32 [N,3,H,W] (0..255) through element strides (ab..ax, bb..bx); 4-byte aligned
 *   flow           : fp32 [N,2,H,W] through element strides; 4-byte aligned
 *   mask           : uint8 [N][H][W] contiguous, weight where != 0; NULL: all ones
 *   loss_sum       : fp64 [N] S_r; count: int64 [N] M_r; total: fp64 [2] = (sum_r S_r, sum_r M_r), rows added in row order
 *   state          : 28 N H W bytes, 8-byte aligned: the fp64 planes g(I1) and W^ ([N][H][W] each), then the fp32 planes
 *                    dW^/dpx, dW^/dpy (the floor convention at integer positions) and v dl/dh; what rnc_census_loss_bwd reads
 *   workspace      : rnc_census_loss_workspace_bytes(N, H, W) bytes, 16-byte aligned, no zeroing needed
 * Five launches, no host synchronisation.
 *
 * rnc_census_loss_bwd: grad_flow (fp32 [N][2][H][W] contiguous) = *scale (a device fp32 scalar: the upstream gradient over
 * sum_r M_r + 1e-6) times the gradient of sum_r S_r with respect to F, gathered per pixel over its 7x7 window from state.  One
 * launch.
 *
 * rnc_smoothness_fwd: per row, sum_x[r] = sum over 1 <= x <= W-2, all y, and both flow channels of
 * rho(F(x+1,y) - 2F(x,y) + F(x-1,y)) exp(-edge_constant mean_c |I_c(x,y) - I_c(x-1,y)| / 255), rho(d) = sqrt(d^2 + 1e-6),
 * and sum_y[r] the same along y (fp64); total: fp64 [2] = (sum_r sum_x, sum_r sum_y) in row order.
 *   image          : fp32 [N,3,H,W] through element strides; flow: fp32 [N,2,H,W] through element strides; 4-byte aligned
 *   workspace      : rnc_smoothness_workspace_bytes(N, H, W) bytes, 16-byte aligned, no zeroing needed
 * Three launches, no host synchronisation.
 *
 * rnc_smoothness_bwd: grad_flow (fp32 [N][2][H][W] contiguous) = scale[0] d(sum_x)/dF + scale[1] d(sum_y)/dF, scale a
 * device fp32 [2]; per pixel a gather of the three x- and three y-terms that hold it.  One launch. */
size_t rnc_census_loss_workspace_bytes(int N, int H, int W);   /* 0 for a bad shape */
int rnc_census_loss_fwd(const float* image1, long long ab, long long ac, long long ay, long long ax, const float* image2,
                        long long bb, long long bc, long long by, long long bx, const float* flow, long long fb, long long fc,
                        long long fy, long long fx, const unsigned char* mask, int N, int H, int W, double* loss_sum,
                        long long* count, double* total, void* state, void* workspace, size_t workspace_bytes,
                        void* stream);
int rnc_census_loss_bwd(const void* state, int N, int H, int W, const float* scale, float* grad_flow, void* stream);
size_t rnc_smoothness_workspace_bytes(int N, int H, int W);    /* 0 for a bad shape */
int rnc_smoothness_fwd(const float* image, long long ib, long long ic, long long iy, long long ix, const float* flow,
                       long long fb, long long fc, long long fy, long long fx, int N, int H, int W, float edge_constant,
                       double* sum_x, double* sum_y, double* total, void* workspace, size_t workspace_bytes, void* stream);
int rnc_smoothness_bwd(const float* image, long long ib, long long ic, long long iy, long long ix, const float* flow,
                       long long fb, long long fc, long long fy, long long fx, int N, int H, int W, float edge_constant,
                       const float* scale, float* grad_flow, void* stream);

/* ------------------------------------------------------------------------------------------------
 * V8  point tracking through video by chaining the bidirectional flows, and the TAP-Vid metrics of the tracks (definition:
 * rnc/track.py, DESIGN §3.17).  Shapes: 1 <= V <= 65535 videos, N >= 1 points, T >= 2 frames, N*T < 2^30, 1 <= H, W <= 2^24;
 * RNC_ERR_BAD_SHAPE otherwise.  Bad arguments return before any launch.
 *
 * rnc_track: for each query (t, x, y) of video v, its position and visible flag in every frame.
 *   flow, flow_bw : fp32 [V][T-1][2][H][W] through element strides (fv, fk, fc, fy, fx), F_k (frame k -> k+1) and G_k
 *                   (frame k+1 -> k); 4-byte aligned
 *   occ, occ_bw   : uint8 [V][T-1][H][W] through element strides, occ_k on frame k (of F_k) and occ_bw_k on frame k+1 (of G_k);
 *                   a pixel is visible where 0
 *   queries       : fp32 [V][N][3] contiguous, (t, x, y) with t an integer in [0, T-1] and (x, y) in [0, W-1] x [0, H-1]
 *   tracks        : fp32 [V][N][T][2] contiguous (x, y), 8-byte aligned; visible: uint8 [V][N][T] contiguous
 * At frame t the position is the query, visible.  Forward, for k = t .. T-2 from p at frame k: u = F_k^(p) (bilinear, the
 * coordinates clamped to the frame); p' = p + u when both components are finite, else p; the point is lost at k+1 (and
 * after) when it was lost at k, u is not finite, occ_k(rint(p)) != 0 (half to even) or p' is outside the frame; positions
 * advance while lost.  Backward, for k = t-1 .. 0, the same with G_k and occ_bw_k from frame k+1 to frame k.  Every
 * operation rounded once in float32 (no FMA).  One launch, a thread per query, no atomics, no host synchronisation.  A
 * query outside the bounds above gets NaN positions and visible 0 in every frame.
 *
 * rnc_track_metrics: per video v, counts[v][RNC_TRACK_COUNTS] over the (point, frame) pairs except each point's query frame,
 * with positions scaled to 256x256 (x * 256 / W, y * 256 / H, rounded once) and within_d = dx^2 + dy^2 < d^2 for
 * d = 1, 2, 4, 8, 16: [0] pairs evaluated, [1] occlusion agreements (pred visible == gt visible), [2] gt visible,
 * [3 + j] within_dj & gt visible, [8 + j] within_dj & gt visible & pred visible (true positives),
 * [13 + j] pred visible & (!gt visible | !within_dj) (false positives).
 *   tracks, gt_tracks   : fp32 [V][N][T][2] contiguous, 8-byte aligned; visible, gt_visible: uint8 [V][N][T] contiguous
 *   queries             : fp32 [V][N][3] contiguous, as rnc_track's
 *   counts              : int64 [V][RNC_TRACK_COUNTS], 8-byte aligned
 *   workspace           : rnc_track_metrics_workspace_bytes(V, N, T) bytes, 16-byte aligned, no zeroing needed
 * Two launches, no atomics, no host synchronisation: the counts are exact, whatever V or the video's position. */
#define RNC_TRACK_THRESHOLDS 5
#define RNC_TRACK_COUNTS 18
int rnc_track(const float* flow, long long fv, long long fk, long long fc, long long fy, long long fx, const float* flow_bw,
              long long gv, long long gk, long long gc, long long gy, long long gx, const unsigned char* occ, long long ov,
              long long ok, long long oy, long long ox, const unsigned char* occ_bw, long long pv, long long pk, long long py,
              long long px, const float* queries, int V, int N, int T, int H, int W, float* tracks, unsigned char* visible,
              void* stream);
size_t rnc_track_metrics_workspace_bytes(int V, int N, int T);   /* 0 for a bad shape */
int rnc_track_metrics(const float* tracks, const unsigned char* visible, const float* gt_tracks,
                      const unsigned char* gt_visible, const float* queries, int V, int N, int T, int H, int W,
                      long long* counts, void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * V9  video object segmentation: first-frame labels propagated along the backward flows, and the DAVIS semi-supervised
 * metrics J and F as exact counts (definition: rnc/segment.py, DESIGN §3.18).  Bad arguments return before any launch.
 *
 * rnc_propagate_labels: one step k -> k+1 of V videos, L_{k+1} from L_k, G_k and occ_bw_k.
 *   labels    : uint8 [V][H][W] through element strides (lv, ly, lx), L_k; 0 background, 1..254 objects (255 is not a label)
 *   flow_bw   : fp32 [V][2][H][W] through element strides (gv, gc, gy, gx), G_k (frame k+1 -> k); 4-byte aligned
 *   occ_bw    : uint8 [V][H][W] through element strides, on frame k+1; a pixel is visible where 0
 *   out       : uint8 [V][H][W] through element strides (qv, qy, qx), L_{k+1}; must not overlap labels
 *   workspace : rnc_propagate_labels_workspace_bytes(V, H, W) bytes, 16-byte aligned, no zeroing needed (an int32 map)
 * A pixel p of frame k+1 is matched when u = G_k(p) has both components finite, occ_bw_k(p) == 0 and p' = p + u lies in
 * [0, W-1] x [0, H-1]; it takes the bilinear vote of L_k at p': taps (y0,x0), (y0,x1), (y1,x0), (y1,x1) (x1 = min(x0+1, W-1),
 * y1 likewise) weighted bx*by, ax*by, bx*ay, ax*ay, each label's weights added in tap order, the largest sum winning and a
 * tie going to the smaller label.  An unmatched pixel takes the label of the nearest matched pixel of frame k+1 (exact squared
 * distance, ties to the smallest column, then row); 0 in a frame without a matched pixel.  Every operation rounded once in
 * float32 (no FMA).  Three launches, no atomics, no host synchronisation.  RNC_ERR_BAD_SHAPE unless 1 <= V <= 65535 and
 * 1 <= H, W <= 4096.
 *
 * rnc_segmentation_counts: per frame n and object o = 1..K, counts[n][o-1][RNC_SEGMENT_COUNTS] with void = gt == 255,
 * M = pred == o & !void, G = gt == o, and bM, bG their boundary maps (the DAVIS toolkit's seg2bmap at full resolution:
 * s differs from its right, lower or lower-right neighbour; on the last row from its right one, on the last column from its
 * lower one; never the bottom-right pixel): [0] |M & G|, [1] |M | G|, [2] |bM|, [3] |bG|, [4] bM pixels with a bG pixel at
 * squared distance <= r^2, [5] bG pixels with a bM pixel at squared distance <= r^2, r = ceil(0.008 sqrt(H^2 + W^2)) in fp64.
 *   pred, gt  : uint8 [N][H][W] through element strides (pn, py, px), (gn, gy, gx)
 *   counts    : int64 [N][K][RNC_SEGMENT_COUNTS], 8-byte aligned
 *   workspace : rnc_segmentation_counts_workspace_bytes(N, K, H, W) bytes, 16-byte aligned, no zeroing needed: the int32
 *               distance maps [2][N][K][H][W], then the per-CTA partials
 * Four launches, no atomics, no host synchronisation: the counts are exact, whatever N or the frame's position.
 * RNC_ERR_BAD_SHAPE unless N, K >= 1, K <= 254, 2 N K <= 65535 and 1 <= H, W <= 4096. */
#define RNC_SEGMENT_COUNTS 6
size_t rnc_propagate_labels_workspace_bytes(int V, int H, int W);   /* 0 for a bad shape */
int rnc_propagate_labels(const unsigned char* labels, long long lv, long long ly, long long lx, const float* flow_bw,
                         long long gv, long long gc, long long gy, long long gx, const unsigned char* occ_bw, long long ov,
                         long long oy, long long ox, int V, int H, int W, unsigned char* out, long long qv, long long qy,
                         long long qx, void* workspace, size_t workspace_bytes, void* stream);
size_t rnc_segmentation_counts_workspace_bytes(int N, int K, int H, int W);   /* 0 for a bad shape */
int rnc_segmentation_counts(const unsigned char* pred, long long pn, long long py, long long px, const unsigned char* gt,
                            long long gn, long long gy, long long gx, int N, int K, int H, int W, long long* counts,
                            void* workspace, size_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* RNC_H_ */
