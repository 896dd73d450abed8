/*
 * latex_ocr_b200 — C ABI of the H100-native (sm_90a) im2latex hot path.
 *
 * The reference (LinXueyuanStdio/LaTeX_OCR) has no FFI: its boundary is the Python class surface
 * (SURVEY.md §8-b).  Each entry point below replaces the library call(s) the reference makes at the
 * cited lines; the Python mirror in latex_ocr_b200/ (EncoderCNN, Attention, DecoderWithAttention,
 * Img2SeqModel) reaches them through ctypes.  Conventions:
 *   - plain pointers and sizes only; every pointer is a DEVICE pointer unless the name ends in _host;
 *   - stream-ordered on `stream` (a cudaStream_t passed as void*); no allocation, no synchronisation,
 *     no host-visible global state -> every call is CUDA-graph capturable;
 *   - programmatic dependent launch: most kernels are launched so that they may become resident while the preceding
 *     launch of the stream drains, and read their PARAMETER operands (weights, biases, projection tables — never
 *     activations) before they wait for it.  A parameter must therefore not be produced by the launch enqueued
 *     immediately before the call that consumes it (an optimiser step followed by anything else is fine: every
 *     entry point enqueues more than one launch or waits first).  The stand-alone attention entry points
 *     (lo_attention_forward / _forward_mask / _backward), whose early reads include activations (att1, enc; alpha,
 *     ctx, gate of the forward pass), are launched WITHOUT that overlap unless lo_set_option("att_abi_pdl", 1) says the
 *     caller guarantees those tensors are older than the preceding launch; lo_set_option("pdl", 0) turns the overlap
 *     off everywhere;
 *   - return 0 on success, negative LO_E* otherwise (never throws); lo_last_error() gives the text;
 *   - dtype arguments are LO_F32 or LO_BF16 and name the STORAGE type of the "big" tensors
 *     (feature maps, conv/linear weight shadows, encoder_out, att1).  Small per-step state is fp32.
 *     Accumulation is always fp32.
 */
#ifndef LATEX_OCR_B200_H
#define LATEX_OCR_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LO_F32 0
#define LO_BF16 1

#define LO_OK 0
#define LO_EINVAL (-1)   /* bad argument / unsupported shape */
#define LO_ECUDA (-2)    /* a CUDA runtime call or launch failed */
#define LO_ENOTSUP (-3)  /* path not available on this device (needs sm_90) */

#define LO_IMPL_SIMT 0   /* CUDA-core kernels (fp32 or bf16 storage) — the tight-parity path */
#define LO_IMPL_TC 1     /* wgmma + TMA kernels (bf16 storage only) */

int lo_version(void);
const char* lo_last_error(void);
/* number of kernels launched through this library since load (bench.py's gpu_launches) */
int64_t lo_launch_count(void);
/* Run-time options.  lo_set_option sets one by name and accepts any int value (an unknown name is refused with LO_EINVAL);
 * lo_get_option reads it back (-1: unknown name); lo_option_name(i) is the i-th name, NULL past the last.  From Python,
 * LO_OPTS=name=value,... in the environment sets them when the library is loaded.  [p]: parity-tested, tests/test_gpu_tc.py,
 * tests/test_gpu_parity.py, tests/test_gpu_attention_grid.py or tests/test_gpu_l2_keep.py runs the other value against the default and requires the same
 * results (measured A/B: DESIGN.md §8).
 *
 *   name             default  meaning
 *   att_pipe         1 [p]    attention step kernels: 1 TMA bulk-copy -> shared-memory ring, 0 register-streaming
 *   pdl              1        programmatic dependent launch (above); 0 turns it off everywhere
 *   att_abi_pdl      0        1: the stand-alone attention entry points use it too (the caller vouches for their inputs, above)
 *   att_l2_keep_mb   24 [p]   MiB of the loop-invariant att1 / enc rows that each forward pipe / tensor-core backward attention launch
 *                             keeps in L2 (evict_normal) from one time step to the next; every other row streams evict_first.  Clamped
 *                             to the device's L2 size; 0 keeps nothing.  Same results for every value
 *   att_nsplit       0        splits of one batch row in the attention kernels; 0: automatic
 *   att_cluster      1 [p]    how the splits of a batch row meet.  Forward kernel and 512-wide tensor-core backward: 1 launches them
 *                             without a cluster (the last CTA of a row combines the partials in split order) when that grid is one
 *                             resident wave, else as a thread-block cluster combining through distributed shared memory; 2 always
 *                             as a cluster; 0 never.  The other attention kernels: cluster unless 0.  Same results for 1 and 2
 *   att_maskbits     1 [p]    1: the forward attention kernel stores the ReLU mask bits, the backward streams them instead of att1
 *   att_bwd_mma      1 [p]    1: the 512-wide bf16 attention backward runs both contractions on mma.sync
 *   skinny_mma       1 [p]    decoder per-step GEMMs (M <= 64) on mma.sync; 0: on wgmma
 *   skinny_tma       1 [p]    1: their operands by cp.async.bulk, one copy per row; 0: 16-byte cp.async
 *   skinny8          1        1: 8-stage (198 KB shared memory) wgmma config for GEMMs with M <= 128
 *   conv_mc          1        1: cluster-of-2 multicast of the A tile in the wgmma GEMM
 *   wgrad256         0 [p]    1: the TN weight-gradient GEMMs also run 128 x 256 tiles when N % 256 == 0 (the conv weight gradient
 *                             always does when Cin % 256 == 0); off: slower on two of the decoder backward's four such GEMMs
 *   deterministic    0        1: cross-CTA sums of the train step add in a fixed order, bit-reproducible but slower; 0: fp32 atomics
 *   dbg_skip         0        timing aid, results garbage: skips bwd hoisted part (1), loop attention (2), loop GEMM/LSTM (4), fwd hoisted (8)
 *   l2_persist_mb    0        an action: sets the persisting-L2 set-aside to value MiB (0: driver default); reads back the last value set
 */
int lo_set_option(const char* name, int value);
int lo_get_option(const char* name);
const char* lo_option_name(int i);
/* L2 persistence: access-policy window of `stream` over [base, base+bytes) (hits persist, misses stream) with the
 * persisting carve-out sized to fit; bytes = 0 resets.  It applies to loads without an explicit cache hint; the attention
 * kernels' bulk copies carry one (att_l2_keep_mb). */
int lo_set_l2_window(const void* base, int64_t bytes, float hit_ratio, void* stream);
/* development aid: device buffer (>= 16 int64) that CTA (0,0,0) of the wgmma NT GEMM stamps with clock64 at its
 * pipeline milestones; NULL disables */
int lo_debug_buffer(void* p);
/* 1 if the wgmma/TMA kernels are built in and the current device is sm_90 */
int lo_tc_available(void);

/* ------------------------------------------------------------------------------------------------
 * Generic strided (batched) GEMM:  C[b][m][n] (+)= sum_k A[b][m*sam + k*sak] * B[b][k*sbk + n*sbn] (+ bias[n]) (ReLU)
 * Replaces nn.Linear / torch.mm call sites: seq2seq_torch.py:172-176, :223-227 and their autograd.
 * dtA/dtB/dtC in {LO_F32, LO_BF16}; supported combos: (f,f,f) (f,bf,f) (bf,bf,bf) (bf,bf,f).
 * impl=LO_IMPL_TC requires bf16 A and B, sak==1, sbk==1 (both K-major), K%64==0, 16B-aligned rows.
 */
int lo_gemm(const void* A, int dtA, const void* B, int dtB, void* C, int dtC,
            int M, int N, int K,
            int64_t sam, int64_t sak, int64_t sbk, int64_t sbn, int64_t ldc,
            int batch, int64_t sA, int64_t sB, int64_t sC,
            const float* bias, int accumulate, int relu, int impl, void* stream);

/* column sums: out[n] (+)= sum_m X[m*ld + n]  (bias gradients) ; X fp32 or bf16 */
int lo_colsum(const void* X, int dt, float* out, int M, int N, int64_t ld, int accumulate, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Encoder.  Feature maps are NHWC; conv weights are [Cout][3][3][Cin] ("KRSC", K-major for the
 * implicit GEMM); replaces nn.Conv2d/nn.ReLU/nn.MaxPool2d at seq2seq_torch.py:35-56 and
 * convolution_backward (autograd of img2seq_torch.py:165).
 */
/* conv1 (Cin=1) + bias + ReLU + 2x2/2 max-pool fused; img fp32 [N][H][W] raw 0..255
 * (img2seq_torch.py:115-117); out [N][H/2][W/2][64] */
int lo_conv1_pool_forward(const float* img, const float* w, const float* bias, void* out, int dt,
                          int N, int H, int W, void* stream);
/* same with the image as uint8 pixels [N][H][W] (what pad_batch_images produces, model/utils/image.py:27-64): 4x less
 * host->device traffic; pixel values 0..255 are exact in fp32, so results are identical */
int lo_conv1_pool_forward_u8(const uint8_t* img, const float* w, const float* bias, void* out, int dt,
                             int N, int H, int W, void* stream);
int lo_conv1_pool_wgrad_u8(const uint8_t* img, const float* w, const float* bias, const void* dpool, int dt,
                           float* dw, float* db, int N, int H, int W, void* stream);
/* conv1 weight/bias gradient from the POOLED output gradient; recomputes conv1 to find the
 * ReLU mask and pool argmax (first maximum in window scan order, as PyTorch).  All conv1 weight-gradient entry points write dw / db
 * (no accumulation).  With lo_set_option("deterministic", 1) their per-block partial sums go through a device buffer of the
 * library (summed in block order), so two of them must not then run concurrently on the same device. */
int lo_conv1_pool_wgrad(const float* img, const float* w, const float* bias, const void* dpool, int dt,
                        float* dw, float* db, int N, int H, int W, void* stream);
/* the same two kernels with the pixel normalisation x' = x * scale + offset applied to in-bounds pixels (zero padding stays
 * zero in the normalised space): the TF flavour feeds (img - 128) / 128 (model/encoder.py:26-27) -> scale 1/128, offset -1.
 * img: fp32 or uint8 [N][H][W] (img_is_u8). */
int lo_conv1_pool_forward_norm(const void* img, int img_is_u8, float scale, float offset, const float* w,
                               const float* bias, void* out, int dt, int N, int H, int W, void* stream);
int lo_conv1_pool_wgrad_norm(const void* img, int img_is_u8, float scale, float offset, const float* w,
                             const float* bias, const void* dpool, int dt, float* dw, float* db, int N, int H, int W,
                             void* stream);
/* Training variant: the forward additionally stores one byte per pooled output and channel, [N][H/2][W/2][64] — bits 0-1 the
 * window index (py*2+px) of the pool arg-max (first maximum in scan order, as nn.MaxPool2d), bit 2 the ReLU bit — and the
 * weight gradient reads the codes instead of recomputing conv1.  img fp32 or uint8 (img_is_u8); scale/offset as above (1, 0 for
 * the torch flavour). */
int lo_conv1_pool_forward_code(const void* img, int img_is_u8, float scale, float offset, const float* w, const float* bias,
                               void* out, uint8_t* code, int dt, int N, int H, int W, void* stream);
int lo_conv1_pool_wgrad_code(const void* img, int img_is_u8, float scale, float offset, const uint8_t* code, const void* dpool,
                             int dt, float* dw, float* db, int N, int H, int W, void* stream);
/* conv1 data gradient (d image) through the ReLU and the 2x2 max-pool, from those codes and dpool [N][H/2][W/2][64] (dt):
 * dpre[n,oy,ox,c] = dpool[n,oy/2,ox/2,c] where the code has its ReLU bit set and window index (oy&1)*2+(ox&1), else 0 (an odd
 * H / W's last conv row / column, which the pool drops, gets none); dimg[n,y,x] = scale * sum_{r,q<3} sum_c w[c][r][q] *
 * dpre[n,y+1-r,x+1-q,c] over in-bounds conv positions.  w: the fp32 conv1 weights [64][9]; scale: the pixel scale of the
 * forward (1, or 1/128 for the TF flavour; the offset does not enter).  dimg fp32 [N][H][W] is written, not accumulated.  Each
 * pixel is summed by one thread in a fixed order (no atomics), so the result is bit-reproducible without "deterministic".
 * Null pointers, dt other than LO_F32 / LO_BF16, N < 1, H < 2 or W < 2 are refused before any GPU work. */
int lo_conv1_pool_dgrad_code(const uint8_t* code, const void* dpool, int dt, const float* w, float scale, float* dimg,
                             int N, int H, int W, void* stream);
/* General strided convolution = im2col + lo_gemm: the 'cnn' encoder variant's Conv2d(512,512,(2,4),stride=2,padding=1)
 * (seq2seq_torch.py:80).  col [N*Ho*Wo][R*S*C], taps-major, C % 8 == 0; forward y = relu(col W^T + b) with W [Cout][R][S][C];
 * weight gradient dW = dy^T col; data gradient dcol = dy W then lo_col2im (a gather over the windows covering each input
 * pixel, optional ReLU mask of the producing layer). */
int lo_im2col(const void* x, void* col, int dt, int N, int H, int W, int C, int R, int S, int stride, int pad,
              void* stream);
int lo_col2im(const void* dcol, const void* mask, void* dx, int dt, int N, int H, int W, int C, int R, int S,
              int stride, int pad, void* stream);
/* out[n][k] = in[k][n] for k < K, n < N */
int lo_transpose(const void* in, int64_t ld_in, void* out, int64_t ld_out, int dt, int K, int N, void* stream);
/* y = [relu](conv3x3(x, w, pad) + bias) [* (mask > 0)] ; x [N][H][W][Cin], y [N][H+2pad-2][W+2pad-2][Cout];
 * pad in {0,1,2}.  mask (optional, same shape/dtype as y) implements the ReLU backward when this
 * call computes a data gradient.  bias may be NULL. */
int lo_conv3x3(const void* x, const void* w, const float* bias, const void* mask, void* y, int dt,
               int N, int H, int W, int Cin, int Cout, int pad, int relu, int impl, void* stream);
/* dw[Cout][3][3][Cin] = sum x (*) dy ; db[Cout] = sum dy ; x [N][H][W][Cin], dy [N][Ho][Wo][Cout] */
int lo_conv3x3_wgrad(const void* x, const void* dy, float* dw, float* db, int dt,
                     int N, int H, int W, int Cin, int Cout, int pad, int impl, void* stream);
/* wt[Cin][3][3][Cout] = w[Cout][2-r][2-s][Cin]  (weights of the data-gradient convolution) */
int lo_conv_weight_flip(const void* w, void* wt, int dt, int Cin, int Cout, void* stream);
/* floor-mode max-pool kh x kw, stride = kernel (nn.MaxPool2d seq2seq_torch.py:37,42,49,52) */
int lo_maxpool_forward(const void* x, void* y, int dt, int N, int H, int W, int C, int kh, int kw, void* stream);
/* dx = route dy to the first maximum of each window, times (x > 0) (x is a ReLU output) */
int lo_maxpool_backward(const void* x, const void* y, const void* dy, void* dx, int dt,
                        int N, int H, int W, int C, int kh, int kw, void* stream);
/* out = y + timing_signal (seq2seq_torch.py:115-157); table fp32 [H][W][C] built once by the host */
int lo_add_table(const void* y, const float* table, void* out, int dt, int N, int64_t HWC, void* stream);
/* dY6 = denc (fp32) * (y6 > 0), cast to dt */
int lo_relu_mask_cast(const float* g, const void* y, void* out, int dt, int64_t n, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Attention (single step): Attention.forward seq2seq_torch.py:178-192 with att1 hoisted.
 * att1,enc [B][R][A|C] (dt) ; att2 [B][A] fp32 (= decoder_att(h)) ; wf [A] fp32 (full_att.weight; its bias
 * cancels in the softmax) ; alpha out fp32 [B][alpha_stride>=R] ; ctx out fp32 [B][C].
 * gate_pre (optional) [B][gate_stride]: if given, gate = sigmoid(gate_pre) is written back in place and
 * gctx [B][C] = gate*ctx (seq2seq_torch.py:311-312).  work: lo_attention_workspace_bytes(B, C) bytes.
 * Layout of one attention workspace of B rows: B int32 ticket counters at offset 0 (zero when given; every launch leaves them
 * zero), then the split partials [B][16][C + 2] fp32 at offset P = 4096 for B <= 1024, P = 4 * B rounded up to 256 above
 * (decoding has no row cap).  Size: P + B * 16 * (C + 2) * 4 bytes.
 */
int64_t lo_attention_workspace_bytes(int B, int C);
int64_t lo_decoder_workspace_bytes(int B, int C);   /* `work` of lo_decoder_args: two attention regions (time loop; ragged decode's CTA map) */
int lo_attention_forward(const void* att1, const void* enc, int dt, const float* att2, int64_t att2_stride,
                         const float* wf, float* alpha, int64_t alpha_stride, float* ctx,
                         float* gate_pre, int64_t gate_stride, float* gctx,
                         int B, int R, int A, int C, void* work, void* stream);
/* the same, additionally storing the ReLU mask bits for lo_attention_backward(relu_mask = ...): relu_mask_out is
 * [B][Rp][A/8] bytes with Rp = R rounded up to an even count; bit 7 - a % 8 of the byte of (r, a / 8) = att1 + att2 > 0, and that
 * byte lives at (r / 2) * 2 * (A/8) + (a / 8) * 2 + (r & 1) within image b (the bytes of an even/odd row pair are adjacent).
 * The buffer is opaque to callers: only its size matters. */
int lo_attention_forward_mask(const void* att1, const void* enc, int dt, const float* att2, int64_t att2_stride,
                              const float* wf, float* alpha, int64_t alpha_stride, float* ctx,
                              float* gate_pre, int64_t gate_stride, float* gctx, uint8_t* relu_mask_out,
                              int B, int R, int A, int C, void* work, void* stream);

/* Backward of one attention step (autograd of seq2seq_torch.py:186-190 + the gate of :311-312), reading att1 and enc ONCE:
 *   dctx = dgctx * gate ; dgp = dgctx * ctx * gate (1 - gate) ; s = <dctx, ctx> + sreg[b]
 *   dalpha_r = <dctx, enc_r> + dreg[b][r] ; de_r = alpha_r (dalpha_r - s) ; datt2_a = wf_a sum_r de_r [att1_ra + att2_a > 0]
 * att2 / gate [B][o1_stride] fp32 as the forward left them (gate after the sigmoid; NULL = ungated context) ; alpha / de
 * [B][alpha_stride] ; ctx / dctx_out [B][C] ; dgctx [B][dg_stride] ; dreg [B][dreg_stride] and sreg [B][sreg_stride] may be NULL ;
 * datt2 / dgp [B][dcat_stride] ; dwf_part (optional) [B][A] += sum_r de_r relu(att1_r + att2) (full_att.weight gradient).
 * d att1 and d enc are NOT produced here: they are hoisted out of the time loop (see lo_decoder_backward).
 * relu_mask (optional): the bits lo_attention_forward_mask stored; att1 is then NOT read, and dwf_part (optional) receives only the
 * att2 term of the full_att.weight gradient, sum_r de_r [on] att2_a — the term that needs att1 itself, sum_r de_r [on] att1_ra, is
 * added by lo_decoder_backward's single sweep over att1 after the time loop. */
int lo_attention_backward(const void* att1, const void* enc, int dt, const float* att2, const float* gate, int64_t o1_stride,
                          const float* wf, const float* alpha, int64_t alpha_stride, const float* ctx, const float* dgctx,
                          int64_t dg_stride, const float* dreg, int64_t dreg_stride, const float* sreg, int64_t sreg_stride,
                          float* de, float* datt2, float* dgp, int64_t dcat_stride, float* dctx_out, float* dwf_part,
                          const uint8_t* relu_mask, int B, int R, int A, int C, void* work, void* stream);

/* Whole backward of ONE stand-alone Attention.forward call (autograd of seq2seq_torch.py:185-190: encoder_att, decoder_att,
 * full_att, softmax and the context sum), where lo_decoder_backward hoists d att1 and d enc out of its time loop:
 *   s = <dctx, ctx> + sum_r alpha_r dalpha_r ; de_r = alpha_r (<dctx, enc_r> + dalpha_r - s) ; on_ra = att1_ra + att2_a > 0
 *   datt1_ra = wf_a de_r on_ra ; datt2_a = wf_a sum_r de_r on_ra ; g_w_full_a = sum_b sum_r de_r relu(att1_ra + att2_a) ; g_b_full = 0
 *   denc = alpha (x) dctx + datt1 W_enc ; g_w_enc = datt1^T enc ; g_b_enc = colsum(datt1)
 *   dh = datt2 W_dec ; g_w_dec = datt2^T h ; g_b_dec = colsum(datt2)
 * One pass of the TMA-ring backward kernel reads att1 and enc once and writes de, datt2, the per-row g_w_full partials and datt1.
 * Inputs (required): enc / att1 [B][R][C|A] (dt) and h [B][D] fp32 as the forward used them, att2 [B][A] fp32 (= h W_dec^T + b_dec),
 * w_enc [A][C] and w_dec [A][D] (dt: the weights the forward read), wf [A] fp32, alpha [B][R] and ctx [B][C] fp32 (forward results),
 * dctx [B][C] fp32; dalpha [B][R] fp32 may be NULL (zero).  Outputs, all fp32 except datt1 (dt), all written (never accumulated),
 * each optional — NULL means not needed and skips the work only it needs: denc [B][R][C], dh [B][D], g_w_enc [A][C], g_b_enc [A],
 * g_w_dec [A][D], g_b_dec [A], g_w_full [A], g_b_full [1], de [B][R], datt2 [B][A], datt1 [B][R][A].  Without denc, g_w_enc,
 * g_b_enc and datt1, d att1 is not written and neither of its GEMMs runs.  impl = LO_IMPL_TC with dt = LO_BF16: the two
 * [B*R, A] x [A, C] products run on the wgmma GEMMs (fp32 storage ignores it).  work: lo_attention_step_workspace_bytes(B, R, A, C,
 * dt) bytes, zero-initialised once by the caller.  With lo_set_option("deterministic", 1) every cross-CTA sum adds in a fixed
 * order, so two identical calls give identical bits.  Launched stream-ordered unless "att_abi_pdl" (above).  Null inputs, a bad
 * dt or impl, A != C, C not in {256, 512, 1024}, B outside 1..512, R < 1, D < 1 and enc, att1 or datt1 not 16-byte aligned are
 * refused (LO_EINVAL) before any GPU work. */
int64_t lo_attention_step_workspace_bytes(int B, int R, int A, int C, int dt);
int lo_attention_step_backward(const void* enc, const void* att1, int dt, const float* h, const float* att2, const void* w_enc,
                               const void* w_dec, const float* wf, const float* alpha, const float* ctx, const float* dctx,
                               const float* dalpha, float* denc, float* dh, float* g_w_enc, float* g_b_enc, float* g_w_dec,
                               float* g_b_dec, float* g_w_full, float* g_b_full, float* de, float* datt2, void* datt1,
                               int B, int R, int A, int C, int D, int impl, void* work, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Whole teacher-forced decoder: DecoderWithAttention.forward seq2seq_torch.py:267-320 (+ the loss of
 * img2seq_torch.py:147-159) and its hand-derived backward.  One struct carries every buffer; the
 * Python side (latex_ocr_b200/decoder.py) parses THIS header to build the ctypes mirror.
 * Shapes: B rows (already sorted by length), T steps, R regions, C=enc dim, A=att dim, D=decoder dim,
 * E=embed dim, V=vocab.  "f32" fields are float*, "big" fields are `dt` storage.
 */
typedef struct lo_decoder_args {
  int32_t B, T, R, C, A, D, E, V;
  int32_t dt;              /* storage of enc/att1/weight shadows */
  int32_t impl;            /* LO_IMPL_SIMT | LO_IMPL_TC for the hoisted GEMMs */
  int32_t has_dropout;     /* 0: eval ; 1: multiply h by dropout_mask before fc (injected mask: parity tests) ;
                              2: draw the inverted-dropout mask inside the LSTM kernels (Philox4x32-10 keyed by dropout_state,
                                 regenerated in the backward; nothing is stored) */
  int32_t ldl;             /* row stride of logits/dlogits (>= V; a multiple of 64 enables the wgmma fc GEMMs); 0 -> V */
  float alpha_c;           /* doubly-stochastic regulariser weight (img2seq_torch.py:157) */
  int32_t rows_per_img;    /* decode only: consecutive rows that share one image (beam size); 0/1 for training.  Images of
                              different sizes: reg_off / reg_off_host below */
  int32_t phase;           /* 0: whole call (default).  EXTENSION (a second decoder layer between the cell and fc): 1 = time loop
                              only — lo_decoder_forward stops after writing hd, lo_decoder_backward starts from the dhd the caller
                              put there; 2 = head only — logits + loss from whatever the caller left in hd, backward of fc -> dhd.
                              A split backward runs phase 2, then the caller's layer (dhd in place), then phase 1; phase 1
                              bumps the dropout call counter, phase 2 does not.  Generic mode across phases: dpred_ext is the
                              mode flag and must be set in BOTH calls — phase 2 reads it (dpred_kernel -> dlogits, fc backward
                              -> dhd, g_w_fc, g_b_fc), phase 1 does not read it but takes d alpha from dalpha_ext (NULL: zero)
                              instead of the regulariser's dreg, which a with_loss = 0 forward never wrote.  dalpha_ext in a
                              phase-2 call and a phase outside 0..2 are refused (LO_EINVAL) before any GPU work. */
  const int32_t* bt_host;  /* HOST int[T]: rows active at step t (seq2seq_torch.py:308); non-increasing */
  const int64_t* caps;     /* [B][caps_stride] token ids (sorted rows) */
  int64_t caps_stride;
  /* scheduled sampling (Bengio et al. 2015).  ss_prob != NULL selects the mode; it must then be set in BOTH the forward and the
   * backward call, as dpred_ext is.  Step t >= 1 of an active row b feeds
   *     fed[b][t] = argmax_v logits[b][t-1][v]  if u[b][t] < p   (lowest index wins ties, as torch.argmax)
   *               = caps[b][t]                  otherwise ;       fed[b][0] = caps[b][0]
   * where logits[b][t-1] is the returned prediction row (fc(dropout(h)) with the dropout of this call), p = *ss_prob.  The choice
   * is not differentiated: given fed, forward and backward are teacher forcing on the input sequence fed (the embedding and
   * weight_ih[:, :E] gradients go to the rows of the tokens fed); ce_kernel's targets stay caps[b][t+1].  In this mode the head
   * fc(hd_t) runs inside the time loop (one GEMM per step, writing only the rows active at step t) instead of once after it.
   * Refused (LO_EINVAL) before any GPU work: ss_prob without fed, without ss_u and dropout_state, with phase != 0, with
   * rows_per_img > 1, and on the greedy / beam entry points. */
  int64_t* fed;            /* [B][T] tokens fed at each step: written by the forward (positions past a row's decode length get
                              caps[b][t]), read by the backward */
  const float* ss_prob;    /* DEVICE scalar p, read inside the kernels (a captured graph stays valid when p changes); NULL: off */
  const float* ss_u;       /* optional injected uniforms [B][T] (parity tests); NULL: u = (x >> 8) * 2^-24 with x the first word
                              of Philox4x32-10(counter = (0xFFFFFFFF, t, b, call), key = seed) of dropout_state {seed, call} — a
                              counter the dropout stream (j >> 2, t, b, call) never uses.  lo_decoder_backward advances the
                              call counter in this mode as it does for has_dropout = 2 */
  const float* ss_temp;    /* optional DEVICE scalar tau > 0 (self-critical training, lo_scst_*): a step that samples (u < p) feeds a
                              draw from softmax(logits[b][t-1] / tau) instead of the argmax,
                                  fed[b][t] = argmax_v (logits[b][t-1][v] / tau + g_v),  g_v = -log(-log u_v)   (Gumbel-max),
                              lowest index on ties.  NULL: the argmax above.  A separate pointwise kernel runs the draw */
  const float* ss_gu;      /* optional injected uniforms [B][T][V] in (0, 1) (parity tests); NULL: u_v = ((x >> 8) + 0.5) * 2^-24 with
                              x word (v & 3) of Philox4x32-10(counter = (0x80000000 | v >> 2, t, b, call), key = seed) of
                              dropout_state — a first counter word neither the dropout stream nor the coin uses.  ss_temp or
                              ss_gu without ss_prob, and ss_gu without ss_temp, are refused (LO_EINVAL) before any GPU work */
  /* inputs */
  const void* enc;         /* big [B][R][C] */
  /* parameters: weight shadows in `dt`, biases fp32.  Wcat1 = [decoder_att; f_beta; weight_hh] rows
   * (contiguous [A+C+4D][D]), bcat1 likewise.  w_ih is [4D][E+C]. */
  const void* w_enc_att; const float* b_enc_att;   /* [A][C] */
  const void* wcat1; const float* bcat1;           /* [A+C+4D][D] */
  const float* w_full;                             /* [A] fp32 */
  const void* emb;                                 /* [V][E] */
  const void* w_ih; const float* b_ih;             /* [4D][E+C] */
  const void* w_init; const float* b_init;         /* [2D][C]: init_h rows then init_c rows */
  const void* w_fc; const float* b_fc;             /* [V][D] */
  /* transposed shadows for the backward per-step GEMMs (built by lo_decoder_pack_bwd_weights) */
  void* wbwd1;             /* [C+D][4D]: rows 0..C-1 = w_ih[:,E+j]^T, rows C.. = w_hh[:,j]^T */
  void* wbwd2;             /* [D][A+C]: [n][k] = k<A ? w_dec_att[k][n] : w_f_beta[k-A][n] */
  /* forward state (f32 unless noted) */
  void* att1;              /* big [B][R][A] */
  float* ptab;             /* [V][4D] = emb @ w_ih[:, :E]^T + b_ih */
  float* mean;             /* [B][C] */
  float* hall;             /* [T+1][B][D] */
  float* call;             /* [T+1][B][D] */
  float* out1;             /* [T][B][A+C+4D]: att2 | gate (sigmoid applied) | h@w_hh^T+b_hh */
  float* alphas;           /* [B][T][R] */
  uint8_t* att_mask;       /* optional, training only: [T][B][Rp][A/8], Rp = R rounded up to even (layout: lo_attention_forward_mask) — bit = (att1[b][r][a] + att2_t[b][a] > 0),
                              written by the forward attention kernel; the backward then streams enc + these 64 bytes per region
                              instead of enc + att1 (60.5 MB instead of 114 MB per step at cfg #2).  NULL: att1 is re-read. */
  float* ctx;              /* [T][B][C] */
  float* gctx;             /* [T][B][C] */
  float* gates;            /* [T][B][4D] post-activation i,f,g,o */
  float* gtmp;             /* [B][4D] scratch */
  const float* dropout_mask; /* [B][T][D] multipliers or NULL */
  const uint64_t* dropout_state; /* has_dropout=2: device {seed, call counter}; lo_decoder_backward increments the counter */
  float dropout_p;         /* has_dropout=2: drop probability (seq2seq_torch.py:216 nn.Dropout(p)) */
  float* hd;               /* [B][T][D] h after dropout */
  float* logits;           /* [B][T][ldl]  (== predictions in the first V columns) */
  /* loss */
  float* row_loss;         /* [B*T + B*R]: per-position CE, then the B*R regulariser partials (1 - sum_t alpha)^2 */
  float* loss;             /* [4]: total, ce, reg, n_valid */
  /* backward state */
  float* dlogits;          /* [B][T][ldl] */
  float* dhd;              /* [B][T][D] */
  float* dreg;             /* [B][R] gradient of the regulariser w.r.t. alpha (same for every t) */
  const float* dalpha_ext; /* optional external d loss/d alphas [B][T][R] (generic mode, below); overrides dreg */
  const float* dpred_ext;  /* generic mode: upstream gradient of predictions, fp32 rows (b, t) in sorted-row order.  Non-NULL
                              selects the generic mode, also in a phase-1 call, which does not read it (see phase) */
  int64_t dpred_stride;    /* elements between consecutive (b, t) rows of dpred_ext (>= V) */
  float* sreg;             /* [B][T] */
  float* dcat;             /* [T][B][A+C+4D]: datt2 | dgate_pre | dgates_pre */
  float* dxh;              /* [B][C+D] scratch: dgctx | dh_prev */
  float* dc;               /* [2][B][D] ping-pong dc */
  float* dctx;             /* [T][B][C] */
  float* de;               /* [B][T][R] */
  float* dptab;            /* [V][4D] */
  void* datt1;             /* big [B][R][A] */
  float* denc;             /* f32 [B][R][C]  (output: gradient w.r.t. encoder_out) */
  float* dinit;            /* [B][2D] = dh0 | dc0 */
  float* dmean;            /* [B][max(A,C)]: d mean_r(enc); doubles as the [B][A] d full_att.weight scratch of the time loop */
  /* parameter gradients (fp32, reference layouts) */
  float* g_w_enc_att; float* g_b_enc_att;
  float* g_wcat1; float* g_bcat1;
  float* g_w_full; float* g_b_full;
  float* g_emb;
  float* g_w_ih; float* g_b_ih;
  float* g_w_init; float* g_b_init;
  float* g_w_fc; float* g_b_fc;
  /* decode of images of different sizes (lo_decoder_greedy[_hist] and lo_decoder_beam[_div] only): prefix offsets of the images'
   * regions, [B / rows_per_img + 1] each, the same values on the device and on the host.  Image i owns regions [reg_off[i],
   * reg_off[i+1]) of a PACKED enc [reg_off[n]][C] and att1 [reg_off[n]][A] (n = B / rows_per_img; beam rows share their image's
   * regions).  R is then the largest count: the row stride of alphas [B][T][R], whose entries past an image's own count are left
   * untouched.  Every image attends over its own regions only, so its tokens are those it gets when decoded alone.  Both NULL:
   * every image has R regions ([n][R][.]).  Refused (LO_EINVAL) before any GPU work: one set without the other, either on
   * lo_decoder_forward / lo_decoder_backward, reg_off_host[0] != 0, a count below 1 or above R, and att_pipe = 0. */
  const int32_t* reg_off;
  const int32_t* reg_off_host;
  void* work;              /* lo_decoder_workspace_bytes(B, max(A,C)), zero-initialised once */
  void* bfwork;            /* optional (impl=TC, dt=bf16): bf16 staging for the hoisted wgmma GEMMs,
                              lo_decoder_bfwork_bytes(args) bytes */
} lo_decoder_args;

int64_t lo_decoder_bfwork_bytes(const lo_decoder_args* a);
/* sizeof(lo_decoder_args) as compiled into the library (the ctypes mirror checks it) */
int64_t lo_sizeof_decoder_args(void);
/* forward through all T steps + logits ; if with_loss, also CE + regulariser into loss[] */
int lo_decoder_forward(const lo_decoder_args* a, int with_loss, void* stream);
/* backward of loss[0]; fills every g_* and denc.  Requires lo_decoder_forward(with_loss=1) state.
 * Generic mode (dpred_ext != NULL): the backward of an arbitrary loss of predictions and alphas (the autograd path of
 * DecoderWithAttention).  Contract:
 *   - the forward ran with with_loss = 0 and the backward buffers (dlogits, dhd, dreg, ..., g_*) allocated;
 *   - dpred_ext holds d loss / d predictions [B][T] rows of V (dpred_stride >= V apart) and dalpha_ext d loss / d alphas
 *     [B][T][R] (NULL: zero).  The first launch copies dpred_ext into dlogits (and its bf16 mirror when the wgmma fc backward
 *     runs), writing zeros for rows t >= the row's decode length and for the padding columns [V, ldl): the forward zeroes those
 *     predictions, so their gradient reaches neither g_w_fc, g_b_fc nor dhd;
 *   - dreg and loss are not touched;
 *   - the attention backward reads its d alpha rows before it waits on the preceding launch (programmatic dependent launch):
 *     dalpha_ext must be complete before the call, which stream order gives for anything enqueued before it.
 * Without dpred_ext, dalpha_ext only replaces the regulariser's d alpha of a with_loss = 1 forward (dlogits from its loss). */
int lo_decoder_backward(const lo_decoder_args* a, void* stream);
int lo_decoder_pack_bwd_weights(const lo_decoder_args* a, void* stream);

/* greedy decode on the same step kernels (decode loop semantics of dynamic_decode.py:17-74 +
 * greedy_decoder_cell.py:46-66): tokens out [B][max_steps] int64, first input token = start_id */
int lo_decoder_greedy(const lo_decoder_args* a, int64_t start_id, int64_t end_id, int max_steps,
                      int64_t* tokens, int32_t* finished, void* stream);
/* greedy: tokens [B][max_steps]; fin_hist (optional) [B][max_steps] int32 = finished flag after each step */
int lo_decoder_greedy_hist(const lo_decoder_args* a, int64_t start_id, int64_t end_id, int max_steps,
                           int64_t* tokens, int32_t* finished, int32_t* fin_hist, void* stream);

/* Sampling decode (lo_decoder_sample, lo_tfdec_sample, lo_decoder2_sample): the greedy loop of the flavour with every step's token
 * drawn instead of taken as the argmax, rows_per_img = n consecutive rows (n samples) sharing one image.  Row b of step t, with
 * logits x [V]:
 *   q = softmax(x / tau); the tokens in the order (q descending, index ascending)
 *   top_k >= 1 keeps the first top_k tokens of that order (0: off); top_p < 1 keeps token v iff the mass of the tokens before v
 *   is < top_p (1: off), so the most probable token is always kept; with both set a token must pass both
 *   token = argmax over the kept v of (x_v / tau + g_v), g_v = -log(-log u_v), the lowest index among equals: one draw from q
 *   renormalised over the kept set (Gumbel-max).  u_v: u[t][b][v] when u is given, else ((w >> 8) + 0.5) * 2^-24, w word
 *   (v & 3) of Philox4x32-10(counter = (0x80000000 | v >> 2, t, b, call), key = seed) of the device state {seed, call} — the
 *   stream of lo_decoder_args.ss_gu's Philox uniforms (host mirror: philox.gumbel_uniforms).
 * The token goes to tokens[b][t] and is fed to step t + 1; a row is finished after its first end_id, and from then on emits end_id
 * and adds nothing.  logp[b] = the sum over the row's tokens through its first end_id of log_softmax(x)[token] at temperature 1,
 * unfiltered: the model's log-likelihood of the sample, comparable with beam search's logp.  fin_hist, finished, images of
 * different sizes (reg_off) and the outputs are those of the flavour's greedy entry point.  With `state`, the call adds 1 to
 * state[1] after its last step, so the next call draws new uniforms.
 *   tau      temperature, finite and > 0
 *   top_k    0..V
 *   top_p    (0, 1]
 *   u        optional device fp32 [max_steps][B][V] in (0, 1) (tests); NULL: Philox from state
 *   state    device {seed, call} (needed without u)
 *   logp     device fp32 out [B]
 * Refused (LO_EINVAL) before any GPU work: a null struct, tau not finite or <= 0, top_k outside 0..V, top_p outside (0, 1], neither
 * u nor state, a null logp, rows_per_img outside 1..16, V above 2048 (the shared-memory sort of a row, 12 bytes per entry), any
 * ss_* field of the args, and every refusal of the flavour's greedy entry point. */
typedef struct lo_sample_args {
  float tau;
  int32_t top_k;
  float top_p;
  const float* u;
  uint64_t* state;
  float* logp;
} lo_sample_args;
int64_t lo_sizeof_sample_args(void);
int lo_decoder_sample(const lo_decoder_args* a, const lo_sample_args* s, int64_t start_id, int64_t end_id, int max_steps,
                      int64_t* tokens, int32_t* finished, int32_t* fin_hist, void* stream);

/* beam search on the same step kernels: beam_search_decoder_cell.py:98-187 (log-softmax, finished mask with
 * dtype.min, only beam 0 at time 0, top-k over beam*V with the lower index winning ties, state gather by parents;
 * no length normalisation (lo_decoder_beam_pen adds it), diversity penalty off as in configs/model.json:15-16).  a->B = n_img*beam rows,
 * a->rows_per_img = beam, a->enc holds n_img images.  ids/parents out [n_img][max_steps][beam] int64,
 * fin_hist [n_img][max_steps][beam] int32 (finished flags after each step), logp [n_img][beam] final scores.  beam above 16 or
 * above V (time 0 ranks beam 0's V tokens alone) is refused (LO_EINVAL) before any GPU work, in every flavour's beam search. */
int lo_decoder_beam(const lo_decoder_args* a, int64_t start_id, int64_t end_id, int max_steps, int64_t* ids,
                    int64_t* parents, int32_t* fin_hist, float* logp, void* stream);
/* the same with the diversity penalty of beam_search_decoder_cell.py:258-287 (Li et al. 2016; configs/model.json:15-16
 * div_gamma / div_prob): every candidate's accumulated log-prob gets log(div_gamma) * (its rank inside its beam row, 0 = best)
 * where div_prob > u, u ~ U[0,1) per (image, beam, token).  Off when div_gamma == 1 or div_prob == 0 (:270-273).
 * div_u (optional) injects the uniforms [max_steps][B][V] (parity tests); otherwise they are drawn in the kernel from
 * Philox4x32-10 keyed by div_state = device {seed, call counter}. */
int lo_decoder_beam_div(const lo_decoder_args* a, int64_t start_id, int64_t end_id, int max_steps, int64_t* ids,
                        int64_t* parents, int32_t* fin_hist, float* logp, float div_gamma, float div_prob,
                        const float* div_u, const uint64_t* div_state, void* stream);

/* Length and coverage penalties of beam search (lo_decoder_beam_pen, lo_tfdec_beam_pen): the penalties of GNMT (Wu et al. 2016,
 * eq. 14) in the form of TF's BeamSearchDecoder(length_penalty_weight=alpha).  Every rule of the beam step above stays; per row k
 * the search also keeps len[k], the tokens other than END its hypothesis has emitted (grows only while the row is unfinished),
 * and cov[k][r], the sum over the unfinished steps of the row's attention weights, following the hypothesis's lineage, over the
 * image's own regions r.  Candidate (k, v) at step t, with carried = logp[k] + log-softmax (+ diversity penalty) as today:
 *   new_len = len[k] + (finished[k] || v == END ? 0 : 1)
 *   cov'    = finished[k] ? cov[k] : cov[k] + alpha_t[k]             (alpha_t[k]: the attention row step t wrote for row k)
 *   score   = carried / len_pen[new_len] + beta * sum_r ln(min(max(cov'_r, 1e-30), 1))
 * A finished row's non-END candidates keep dtype.min as their score.  The top-k ranks by score; each winner carries its raw
 * `carried` as the new logp (logp keeps its meaning), its new_len and cov' follow it to its slot.  With alpha = beta = 0 the call
 * is lo_*_beam_div bit for bit (and scores == logp).
 *   alpha, beta  weights, finite and >= 0; alpha = 0: no length penalty, beta = 0: no coverage penalty
 *   len_pen      device fp32 [max_steps + 1], len_pen[l] = ((5 + l) / 6)^alpha computed by the caller (needed when alpha != 0)
 *   cov          device fp32 scratch of 2 * B * R + B floats: the coverage [2][B][R] (read and written alternately, step by step)
 *                then the coverage term of every row [B] (needed when beta > 0; R: the args' region capacity)
 *   len          device int32 scratch [2][B] (always needed)
 *   scores       optional device fp32 out [n_img][beam]: the winners' score after the last step
 * Refused (LO_EINVAL) before any GPU work: a null struct, a negative or non-finite alpha or beta, alpha != 0 without len_pen,
 * beta > 0 without cov, a null len, and beam * V * 8 bytes (the totals and the scores) above 200 kB when a penalty is on. */
typedef struct lo_beam_penalty {
  float alpha;
  float beta;
  const float* len_pen;
  float* cov;
  int32_t* len;
  float* scores;
} lo_beam_penalty;
int64_t lo_sizeof_beam_penalty(void);
/* lo_decoder_beam_div with the penalties of *pen */
int lo_decoder_beam_pen(const lo_decoder_args* a, int64_t start_id, int64_t end_id, int max_steps, int64_t* ids,
                        int64_t* parents, int32_t* fin_hist, float* logp, float div_gamma, float div_prob,
                        const float* div_u, const uint64_t* div_state, const lo_beam_penalty* pen, void* stream);

/* The hypotheses of a finished beam search of either flavour (lo_decoder_beam[_div], lo_tfdec_beam[_div]) and the attention weights
 * under which their tokens were chosen.  ids / parents: that call's outputs, [n_img][ids_stride_steps][beam] int64 (ids_stride_steps =
 * its max_steps), of which the first n steps are read.  alphas: the attention rows the decode wrote, row b = i*beam + s (slot s of
 * image i), step t at alphas + b * alpha_row_stride + t * R (lo_decoder_args.alphas / lo_tfdec_args.alphas: alpha_row_stride = T * R).
 * For every image i and slot s it writes ids_out [n_img][beam][n] int64 and att_out [n_img][beam][n][R] fp32:
 *   mode LO_BEAM_SLOTS (the reference's identity finalize): ids_out[i][s][t] = ids[i][t][s], att_out[i][s][t] = alphas row i*beam + s
 *     at step t — the rows the reference collects in attention_mechanism.ctx_vector;
 *   mode LO_BEAM_LINEAGE (lineage-consistent hypotheses): cur = s at t = n-1, then for t = n-1 down to 0: ids_out[i][s][t] =
 *     ids[i][t][cur], p = parents[i][t][cur], att_out[i][s][t] = alphas row i*beam + p at step t, cur = p.  Each att_out row is the
 *     attention of the step that chose that token, what a teacher-forced pass over the hypothesis computes.
 * A parent outside [0, beam) is read as 0, so foreign data cannot make the walk read out of bounds.  reg_off / reg_off_host (both or
 * neither; as in lo_decoder_args): images of different sizes, image i has reg_off[i+1] - reg_off[i] regions; att_out entries past
 * an image's count are written as 0 and the alphas past it are not read.  alphas and att_out NULL together: the ids only.
 * Refused (LO_EINVAL) before any GPU work: null ids / parents / ids_out, one of alphas / att_out without the other, n_img < 1, beam
 * outside 1..16, n < 1 or n > ids_stride_steps, a mode other than the two below, n * (beam + 2) * 4 bytes above 48 kB, and with
 * att_out: R < 1, alpha_row_stride < n * R, one of reg_off / reg_off_host without the other, a count outside 1..R. */
#define LO_BEAM_SLOTS 0
#define LO_BEAM_LINEAGE 1
int lo_beam_backtrack(const int64_t* ids, const int64_t* parents, int64_t ids_stride_steps, int n_img, int beam, int n,
                      const float* alphas, int64_t alpha_row_stride, int R, const int32_t* reg_off, const int32_t* reg_off_host,
                      int mode, int64_t* ids_out, float* att_out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Self-critical sequence training (SCST, Rennie et al. 2017) of the decoder above: a sample pass (lo_decoder_forward with ss_prob
 * = 1 and ss_temp), a greedy rollout (ss_prob = 1, no ss_temp) as the baseline, the reward of both against the reference
 * (lo_scst_edit_reward), the policy gradient of the sample (lo_scst_pg_grad) into dpred_ext, and lo_decoder_backward in its
 * generic mode with ss_prob set (teacher forcing on the sampled fed).
 */
/* Edit-distance reward of B rows.  h = a row's tokens truncated at the first end_id (metrics.truncate_end), the reference likewise;
 * r(h) = 1 - lev(h, ref) / max(|h|, |ref|) (unit-cost Levenshtein), 1 when both are empty.  hyp [B][hyp_stride] (Lh tokens per row),
 * greedy [B][greedy_stride] (Lg tokens; optional), ref [B][ref_stride] (Lr tokens), all int64.  Writes r_sample [B] and, with greedy,
 * r_greedy [B] and adv [B] = r_sample - r_greedy (each output but r_sample optional); n_len (optional) int32 [B] = the first t >= 1
 * with hyp[b][t] == end_id, else Lh - 1 (the steps lo_scst_pg_grad differentiates).  Distances are integers: the result is exact
 * and deterministic.  Null hyp / ref / r_sample, B < 1 and a length outside 1..512 are refused (LO_EINVAL) before any GPU work. */
int lo_scst_edit_reward(const int64_t* hyp, int64_t hyp_stride, int Lh, const int64_t* greedy, int64_t greedy_stride, int Lg,
                        const int64_t* ref, int64_t ref_stride, int Lr, int B, int64_t end_id, float* r_sample, float* r_greedy,
                        float* adv, int32_t* n_len, void* stream);
/* Policy gradient of L = -(1/B) sum_b adv[b] sum_{t=1..n_len[b]} log softmax(preds[b][t-1] / tau)[fed[b][t]], tau = *temp (a device
 * scalar): writes dpred[b][t-1][v] = -adv[b] / (B tau) (1[v = fed[b][t]] - softmax(preds[b][t-1] / tau)_v) for 1 <= t <= n_len[b] and
 * 0 in every other row (b, s) of [B][T] — V columns, dpred_stride apart: the layout of lo_decoder_args.dpred_ext — and
 * stats[4] = {L, mean r_sample, mean r_greedy, mean n_len} (r_sample / r_greedy may be NULL: 0).  preds [B][T] rows of V fp32,
 * pred_stride apart; fed [B][fed_stride] int64 (fed_stride >= T); n_len int32 [B] in 0..T-1; partial [B][T] fp32 scratch.  The
 * per-row partials are summed in a fixed order without atomics, so the result is bit-reproducible.  Null inputs, B, T < 1, V < 2
 * and strides below V are refused (LO_EINVAL) before any GPU work. */
int lo_scst_pg_grad(const float* preds, int64_t pred_stride, const int64_t* fed, int64_t fed_stride, const float* adv,
                    const int32_t* n_len, const float* temp, const float* r_sample, const float* r_greedy, int B, int T, int V,
                    float* dpred, int64_t dpred_stride, float* partial, float* stats, void* stream);
/* The two calls above in the layout of the TensorFlow-flavour decoder (lo_tfdec_args.ss_prob, below), where every step predicts
 * and nothing is given: the sample is hyp[b][0..Lh) = fed[b][0..T) and every token of it was drawn.
 * lo_scst_edit_reward_tf: lo_scst_edit_reward with n_len[b] = min(e + 1, Lh), e the first t >= 0 with hyp[b][t] == end_id, else
 * Lh (so n_len = 1 when the sample starts with END, Lh when it has none).  Same arguments, refusals and exactness.
 * lo_scst_pg_grad_tf: lo_scst_pg_grad for L = -(1/B) sum_b adv[b] sum_{t=0..n_len[b]-1} log softmax(logits[t][b] / tau)[fed[b][t]]
 * over the time-major logits [T][B] of lo_tfdec_args.logits (rows of V fp32, ldl apart: row (t, b) at (t B + b) ldl).  dpred is
 * batch-major, the layout of lo_tfdec_args.dlogits_ext: dpred[b][t][v] = -adv[b] / (B tau) (1[v = fed[b][t]] - softmax(logits[t][b]
 * / tau)_v) for t < n_len[b], 0 in every other row (b, t); n_len in 0..T.  stats, partial and the refusals as lo_scst_pg_grad,
 * with ldl in place of pred_stride. */
int lo_scst_edit_reward_tf(const int64_t* hyp, int64_t hyp_stride, int Lh, const int64_t* greedy, int64_t greedy_stride, int Lg,
                           const int64_t* ref, int64_t ref_stride, int Lr, int B, int64_t end_id, float* r_sample, float* r_greedy,
                           float* adv, int32_t* n_len, void* stream);
int lo_scst_pg_grad_tf(const float* logits, int64_t ldl, const int64_t* fed, int64_t fed_stride, const float* adv,
                       const int32_t* n_len, const float* temp, const float* r_sample, const float* r_greedy, int B, int T, int V,
                       float* dpred, int64_t dpred_stride, float* partial, float* stats, void* stream);

/* ------------------------------------------------------------------------------------------------
 * TensorFlow-flavour decoder (SURVEY.md §8-a row a7): the Genthial attention cell of
 * model/components/attention_cell.py:58-89 + attention_mechanism.py:43-94,145-153, driven like
 * model/decoder.py:24-72 (teacher forcing = tf.nn.dynamic_rnn over [start_token ; E[formula[:, :-1]]]),
 * masked cross-entropy of model/img2seq.py:68-71, hand-derived backward, greedy / beam decode.
 *   per step:  [i j f o] = [emb_{t-1}; o_{t-1}; h_{t-1}] K + b        (TF LSTMCell, forget_bias 1)
 *              e_r = beta . tanh(att_img_r + h_t W_h) ; alpha = softmax ; ctx = sum alpha_r img_r
 *              o_t = tanh(h_t o_W_h + ctx o_W_c) ; logits_t = o_t y_W_o
 * Parameter storage is [out][in] (K-major for the forward GEMMs; the Python side exposes TF-shaped
 * [in][out] views of the same memory).  Shapes: B rows, T steps (buffer capacity), R regions, C channels,
 * A=dim_e ((A, C) equal or (256, 512): the instantiated widths of the attention kernels), D=num_units, O=dim_o,
 * E=dim_embeddings, V=vocab.
 */
typedef struct lo_tfdec_args {
  int32_t B, T, R, C, A, D, O, E, V;
  int32_t dt;              /* storage of enc / att_img / weight shadows */
  int32_t impl;            /* LO_IMPL_SIMT | LO_IMPL_TC */
  int32_t ldl;             /* row stride of logits / dlogits (>= V, multiple of 8) */
  int32_t rows_per_img;    /* decode only: beam size (consecutive rows share one image); 0/1 otherwise */
  float inv_n_words;       /* 1 / sum(lengths): the loss is the mean over valid tokens */
  const void* enc;         /* big [B/rows_per_img][R][C] (packed [reg_off[n]][C] with reg_off, below) */
  const int64_t* formula;  /* [B][formula_stride] target ids; step t consumes formula[:, t-1], predicts formula[:, t] */
  int64_t formula_stride;
  const int32_t* lengths;  /* device [B]: valid tokens per row incl. END (sequence_mask, img2seq.py:69) */
  const float* keep_h;     /* optional [T][B][D] dropout multipliers for new_h (attention_cell.py:72), pre-scaled by 1/keep */
  const float* keep_o;     /* optional [T][B][O] for new_o (:83) */
  /* parameters: weight shadows in `dt`, biases / beta fp32 */
  const void* w_img;       /* [A][C]          att_img.kernel^T */
  const void* w_cat2;      /* [A+O][D]        att_h.kernel^T rows, then o_W_h^T rows */
  const float* beta;       /* [A]             att_beta */
  const void* w_lstm;      /* [4D][E+O+D]     lstm.kernel^T (gate rows i, j, f, o) */
  const float* b_lstm;     /* [4D] */
  const void* w_oc;        /* [O][C]          o_W_c^T */
  const void* w_y;         /* [V][O]          y_W_o^T */
  const void* w_init;      /* [2D+O][C]       W_c_0^T, W_h_0^T, W_o_0^T */
  const float* b_init;     /* [2D+O] */
  const void* emb;         /* [V+1][E]        embedding_table rows, then start_token */
  /* parameter gradients, fp32, same layouts */
  float* g_w_img; float* g_w_cat2; float* g_beta; float* g_w_lstm; float* g_b_lstm; float* g_w_oc; float* g_w_y;
  float* g_w_init; float* g_b_init; float* g_emb;
  /* results */
  float* logits;           /* [T][B][ldl] time-major */
  float* alphas;           /* [B][T][R] */
  uint8_t* att_mask;       /* optional, training only: [T][B][Rp][A/8], Rp = R rounded up to even (layout: lo_attention_forward_mask) — bit = (att1[b][r][a] + att2_t[b][a] > 0),
                              written by the forward attention kernel; the backward then streams enc + these 64 bytes per region
                              instead of enc + att1 (60.5 MB instead of 114 MB per step at cfg #2).  NULL: att1 is re-read. */
  float* loss;             /* [4]: mean CE over valid tokens (x2), 0, n_words — ce_words (img2seq.py:74) = loss[0] * loss[3] */
  float* denc;             /* f32 [B][R][C] gradient w.r.t. the encoder output */
  /* scheduled sampling (Bengio et al. 2015) and self-critical training (lo_scst_*_tf), as lo_decoder_args.ss_prob in the TF layout:
   * every step predicts and step t consumes token t-1 (the start token at t = 0).  ss_prob != NULL selects the mode; it must then
   * be set in BOTH the forward and the backward call.  The forward writes, for t = 0 .. T-1,
   *     fed[b][t] = choice(logits[t][b])   if u[b][t] < p
   *               = formula[b][t]          otherwise ;       step t+1 consumes fed[b][t]
   * where logits[t][b] is the returned row (o_t y_W_o with this call's keep_o), p = *ss_prob and choice the lowest-index argmax
   * (argmax_kernel's rule) or, with ss_temp, the Gumbel-max draw below.  fed[b][T-1] is recorded but consumed by no step.  The
   * choice is not differentiated: given fed, forward and backward are teacher forcing on fed (the backward scatters the gradient of
   * the embedding rows and of lstm.kernel's embedding part by fed, not formula); the CE targets stay formula[b][t].  In this mode
   * the head runs inside the time loop (one GEMM of B rows per step) instead of once after it.  Refused (LO_EINVAL) before any GPU
   * work: ss_prob without fed, without ss_u and ss_state, with rows_per_img > 1; ss_temp or ss_gu without ss_prob; ss_gu without
   * ss_temp; any of these six fields on lo_tfdec_greedy / lo_tfdec_beam[_div]. */
  int64_t* fed;            /* [B][T] tokens chosen at each step (layout of formula, stride T): written by the forward, read by the
                              backward */
  const float* ss_prob;    /* DEVICE scalar p, read inside the kernels; NULL: teacher forcing */
  const float* ss_u;       /* optional injected coins [B][T] (parity tests); NULL: u = (x >> 8) * 2^-24 with x the first word of
                              Philox4x32-10(counter = (0xFFFFFFFF, t, b, call), key = seed) of ss_state {seed, call} — the coin
                              stream of lo_decoder_args.ss_u */
  const float* ss_temp;    /* optional DEVICE scalar tau > 0: a step that samples feeds argmax_v (logits[t][b][v] / tau + g_v),
                              g_v = -log(-log u_v) (Gumbel-max: one draw from softmax(logits / tau)), lowest index on ties */
  const float* ss_gu;      /* optional injected uniforms [B][T][V] in (0, 1) (parity tests); NULL: u_v = ((x >> 8) + 0.5) * 2^-24 with
                              x word (v & 3) of Philox4x32-10(counter = (0x80000000 | v >> 2, t, b, call), key = seed) of ss_state */
  const uint64_t* ss_state; /* DEVICE {seed, call} keying the Philox coins and Gumbel uniforms (the TF flavour has no in-kernel
                              dropout state to borrow).  Read only: the caller advances call between sampling forwards */
  /* decode of images of different sizes (lo_tfdec_greedy and lo_tfdec_beam[_div] only), as lo_decoder_args.reg_off: prefix offsets
   * of the images' regions, [B / rows_per_img + 1] each, the same values on the device and on the host.  Image i owns regions
   * [reg_off[i], reg_off[i+1]) of a PACKED enc [reg_off[n]][C] (n = B / rows_per_img; beam rows share their image's regions).  R is
   * then the largest count: the row stride of alphas [B][T][R], whose entries past an image's own count are left untouched.  Every
   * image attends over its own regions only, so its tokens are those it gets when decoded alone.  Both NULL: every image has R
   * regions.  Refused (LO_EINVAL) before any GPU work, with the messages of lo_decoder_args: one set without the other, either on
   * lo_tfdec_forward / lo_tfdec_backward, reg_off_host[0] != 0, a count below 1 or above R, and att_pipe = 0. */
  const int32_t* reg_off;
  const int32_t* reg_off_host;
  void* ws;                /* lo_tfdec_workspace_bytes(args) bytes, zero-initialised once by the caller */
  const float* dlogits_ext; /* generic backward (below): d loss / d logits, fp32 rows (b, t) batch-major, dlogits_stride apart */
  int64_t dlogits_stride;  /* elements between consecutive (b, t) rows of dlogits_ext (>= V) */
  const float* dalpha_ext; /* generic backward, optional: d loss / d alphas [B][T][R] (NULL: zero) */
} lo_tfdec_args;

int64_t lo_sizeof_tfdec_args(void);
int64_t lo_tfdec_workspace_bytes(const lo_tfdec_args* a);
/* all T steps + logits; with_loss: masked CE into loss[] (and d logits kept for the backward).  With ss_prob: the tokens consumed
 * are chosen in the loop and recorded in fed (lo_tfdec_args, above) */
int lo_tfdec_forward(const lo_tfdec_args* a, int with_loss, void* stream);
/* backward of loss[0]: fills every g_* and denc (requires lo_tfdec_forward(with_loss=1) state in ws).
 * Generic mode (dlogits_ext != NULL): the backward of an arbitrary loss of the train logits and the alphas (the autograd path of
 * tf_decoder.Decoder).  Contract:
 *   - the forward ran with with_loss = 0 or 1 on the same args (lengths, inv_n_words and the CE's d logits are not used);
 *   - dlogits_ext holds d loss / d logits, batch-major [B][T] rows of V floats (dlogits_stride >= V apart); every one of the T
 *     positions carries its gradient (the forward computes logits for all of them, no row is masked).  The first launch copies it
 *     into the workspace's time-major d logits (and their bf16 mirror when the wgmma GEMMs read it), zeros in columns [V, ldl);
 *   - dalpha_ext holds d loss / d alphas [B][T][R] (NULL: zero).  The attention backward reads its d alpha rows before it waits on
 *     the preceding launch (programmatic dependent launch): dalpha_ext must be complete before the call, which stream order gives
 *     for anything enqueued before it;
 *   - loss is not touched.
 * With ss_prob set (both modes) the backward is teacher forcing on fed: the token-table gradient is scattered by fed, not formula.
 * dalpha_ext without dlogits_ext and dlogits_stride < V are refused (LO_EINVAL) before any GPU work. */
int lo_tfdec_backward(const lo_tfdec_args* a, void* stream);
/* greedy decode (greedy_decoder_cell.py:38-66 + dynamic_decode.py:38-61): tokens [B][max_steps], fin_hist (optional)
 * [B][max_steps] finished flags after each step; max_steps <= T */
int lo_tfdec_greedy(const lo_tfdec_args* a, int64_t end_id, int max_steps, int64_t* tokens, int32_t* fin_hist, void* stream);
/* sampling decode (see lo_sample_args): tokens [B][max_steps], fin_hist (optional) as lo_tfdec_greedy */
int lo_tfdec_sample(const lo_tfdec_args* a, const lo_sample_args* s, int64_t end_id, int max_steps, int64_t* tokens, int32_t* fin_hist,
                    void* stream);
/* beam search (beam_search_decoder_cell.py:98-187): B = n_img*beam rows, rows_per_img = beam; ids/parents/fin_hist
 * [n_img][max_steps][beam], logp [n_img][beam] */
int lo_tfdec_beam(const lo_tfdec_args* a, int64_t end_id, int max_steps, int64_t* ids, int64_t* parents, int32_t* fin_hist,
                  float* logp, void* stream);
/* with the diversity penalty (see lo_decoder_beam_div) */
int lo_tfdec_beam_div(const lo_tfdec_args* a, int64_t end_id, int max_steps, int64_t* ids, int64_t* parents, int32_t* fin_hist,
                      float* logp, float div_gamma, float div_prob, const float* div_u, const uint64_t* div_state, void* stream);
/* with the diversity penalty and the length and coverage penalties of *pen (see lo_beam_penalty) */
int lo_tfdec_beam_pen(const lo_tfdec_args* a, int64_t end_id, int max_steps, int64_t* ids, int64_t* parents, int32_t* fin_hist,
                      float* logp, float div_gamma, float div_prob, const float* div_u, const uint64_t* div_state,
                      const lo_beam_penalty* pen, void* stream);

/* ------------------------------------------------------------------------------------------------
 * EXTENSION (not in the reference; BASELINE.json configs[3]): generic sequence LSTM with nn.LSTM semantics (gate order i,f,g,o,
 * two bias vectors), forward over S steps for M independent sequences + hand-derived backward.  Used for the row-encoder biLSTM
 * over the CNN feature rows (two calls, `reverse` = 0 / 1, writing the two halves of the output channels) and for a second decoder
 * layer.  Element (t, m) of x / dx lives at m * row + t * step (+ channel); of hs / hs_st / dhs at m * hs_row + t * hs_step.
 * x and dx are read and written 16 bytes at a time: x must be 16-byte aligned with x_row, x_step multiples of 8 elements, and a
 * dx given to the backward 16-byte aligned with dx_row, dx_step multiples of 4; otherwise both calls return LO_EINVAL before any
 * GPU work.
 */
typedef struct lo_lstm_seq_args {
  int32_t S, M, I, H;      /* steps, sequences, input width, hidden width (I, H multiples of 8) */
  int32_t dt;              /* storage of x / hs_st / the weight shadows: LO_F32 | LO_BF16 */
  int32_t impl;            /* LO_IMPL_SIMT | LO_IMPL_TC (bf16 only) */
  int32_t reverse;         /* 1: process t = S-1 .. 0 */
  int32_t dx_accumulate;   /* backward: add onto dx instead of overwriting (second direction of a bidirectional layer) */
  const void* x;           /* dt */
  int64_t x_row, x_step;
  const void* w_ih;        /* dt [4H][I] */
  const void* w_hh;        /* dt [4H][H] */
  const float* b_ih; const float* b_hh;   /* fp32 [4H] */
  const float* h0; const float* c0;       /* optional fp32 [M][H] (NULL = zeros) */
  float* hs;               /* optional out fp32 */
  void* hs_st;             /* optional out, storage dtype */
  int64_t hs_row, hs_step;
  const float* dhs;        /* backward in: d loss / d hs (fp32, hs strides); NULL = zeros */
  float* dx;               /* optional backward out fp32 */
  int64_t dx_row, dx_step;
  float* g_w_ih; float* g_w_hh; float* g_b_ih; float* g_b_hh;   /* backward out, fp32, overwritten */
  float* dh0; float* dc0;  /* optional backward out fp32 [M][H] */
  void* ws;                /* lo_lstm_seq_workspace_bytes(args) bytes; forward state is kept there for the backward */
} lo_lstm_seq_args;
int64_t lo_sizeof_lstm_seq_args(void);
int64_t lo_lstm_seq_workspace_bytes(const lo_lstm_seq_args* a);
int lo_lstm_seq_forward(const lo_lstm_seq_args* a, void* stream);
int lo_lstm_seq_backward(const lo_lstm_seq_args* a, void* stream);

/* EXTENSION: greedy and beam decode of the two-layer decoder (oracle/ref_ext.py decoder2_forward, no dropout at decode time).
 * Layer 1 is the attention LSTM of lo_decoder_args, started from init_hidden_state of enc; layer 2 is nn.LSTMCell(D, D) over
 * h1_t from a zero state (h2 = c2 = 0); logits_t = fc(h2_t).  The token and finish rules, the outputs, images of different sizes
 * (reg_off / reg_off_host), the diversity penalty and the penalties of lo_beam_penalty are those of lo_decoder_greedy_hist and
 * lo_decoder_beam_pen; lo_beam_backtrack reads the results unchanged (attention rows in a->alphas).  Layer 2 runs per step as
 * two GEMMs on the step-GEMM dispatcher of layer 1 (one K slice each: a bf16 decode repeats its bits), one cell launch and the
 * head on h2.  Its state lives in `scratch` (two slots of h2 / c2, their bf16 mirror, the gate pre-activations).
 *   w_ih, w_hh   [4D][D] in the args' storage dtype `dt` (gate order i, f, g, o)
 *   b_ih, b_hh   fp32 [4D]
 *   scratch      device, lo_decoder2_scratch_bytes(a) bytes (depends on a->B and a->D only)
 * Refused (LO_EINVAL) before any GPU work: a null layer, a null weight, bias or scratch, phase != 0, ss_prob, and every refusal
 * of lo_decoder_greedy_hist / lo_decoder_beam_pen (pen NULL: no penalty, as lo_decoder_beam_div). */
typedef struct lo_decoder2_layer {
  const void* w_ih;
  const void* w_hh;
  const float* b_ih;
  const float* b_hh;
  void* scratch;
} lo_decoder2_layer;
int64_t lo_sizeof_decoder2_layer(void);
int64_t lo_decoder2_scratch_bytes(const lo_decoder_args* a);
int lo_decoder2_greedy(const lo_decoder_args* a, const lo_decoder2_layer* l2, int64_t start_id, int64_t end_id, int max_steps,
                       int64_t* tokens, int32_t* finished, int32_t* fin_hist, void* stream);
/* sampling decode of the two-layer decoder (see lo_sample_args), with the refusals of lo_decoder2_greedy */
int lo_decoder2_sample(const lo_decoder_args* a, const lo_decoder2_layer* l2, const lo_sample_args* s, int64_t start_id, int64_t end_id,
                       int max_steps, int64_t* tokens, int32_t* finished, int32_t* fin_hist, void* stream);
int lo_decoder2_beam(const lo_decoder_args* a, const lo_decoder2_layer* l2, int64_t start_id, int64_t end_id, int max_steps,
                     int64_t* ids, int64_t* parents, int32_t* fin_hist, float* logp, float div_gamma, float div_prob,
                     const float* div_u, const uint64_t* div_state, const lo_beam_penalty* pen, void* stream);

/* EXTENSION: balanced brackets in greedy, beam and sampling decode of every flavour (the *_brackets entry points).  A rule gives
 * every token a role: 0 neutral, +k opens kind k, -k closes kind k (1 <= k <= n_kinds).  Every decode row keeps a stack of kinds.
 * At step t of a call of max_steps steps, with d the row's depth and r = max_steps - 1 - t the steps left after this one, the row
 * may take token v only if
 *   close of kind k:   d > 0 and kind k on top of the stack
 *   open:              d < max_depth and d + 1 <= r
 *   neutral, not END:  d <= r
 *   END:               d == 0
 * so d <= r + 1 holds at every step, the close of the top kind is always allowed and a row never runs out of tokens.  The excluded
 * tokens get logit -inf before the token choice: greedy takes the argmax over the allowed tokens, beam search's log-softmax runs
 * over them alone (the finished mask, diversity rank and lo_beam_penalty act on those totals unchanged, logp sums restricted
 * log-probs), and sampling filters and draws from the restricted distribution (its logp at temperature 1 is the restricted one).
 * The chosen token then pushes or pops the row's stack; finished rows keep theirs; in beam search the stacks follow the hypotheses
 * by parent, as the coverage of lo_beam_penalty does.  Every greedy and sampled row, and every beam hypothesis followed by
 * lineage (lo_beam_backtrack LO_BEAM_LINEAGE), cut at its first END or ending at max_steps, nests properly and leaves no bracket
 * open; slot-wise hypotheses (LO_BEAM_SLOTS) are not lineages and carry no such guarantee.  One launch per step (one warp per
 * row, the role table in shared memory), between the flavour's head and the token choice; the other launches are those of the
 * entry point without the rule.
 *   role       device int32 [V]; a precondition the kernel does not check: every |role| <= n_kinds, end_id neutral, every kind
 *              with an opening and a closing token (the kernel reads role[0..V) and nothing else, whatever the contents)
 *   n_kinds    1..255
 *   max_depth  1..32
 *   state      device scratch of lo_bracket_state_bytes(B, max_depth) bytes: [2][B] int32 depths, then [2][B][max_depth] uint8
 *              kinds (read and written alternately, step by step; zeroed by the call)
 * Refused (LO_EINVAL) before any GPU work: a null rule, role or state, n_kinds outside 1..255, max_depth outside 1..32, V above
 * 24576 (the role table as int16 in shared memory), and every refusal of the entry point without the rule.  Beam search ranks
 * beam distinct tokens at step 0: the caller makes sure at least beam tokens are allowed at depth 0. */
typedef struct lo_bracket_rule {
  const int32_t* role;
  int n_kinds;
  int max_depth;
  void* state;
} lo_bracket_rule;
int64_t lo_sizeof_bracket_rule(void);
/* bytes of lo_bracket_rule.state for B rows (0 for B < 1 or max_depth outside 1..32) */
int64_t lo_bracket_state_bytes(int B, int max_depth);
/* lo_decoder_greedy_hist, lo_decoder_sample and lo_decoder_beam_pen (pen NULL: no penalty) under the rule *br */
int lo_decoder_greedy_brackets(const lo_decoder_args* a, int64_t start_id, int64_t end_id, int max_steps, int64_t* tokens,
                               int32_t* finished, int32_t* fin_hist, const lo_bracket_rule* br, void* stream);
int lo_decoder_sample_brackets(const lo_decoder_args* a, const lo_sample_args* s, int64_t start_id, int64_t end_id, int max_steps,
                               int64_t* tokens, int32_t* finished, int32_t* fin_hist, const lo_bracket_rule* br, void* stream);
int lo_decoder_beam_brackets(const lo_decoder_args* a, int64_t start_id, int64_t end_id, int max_steps, int64_t* ids, int64_t* parents,
                             int32_t* fin_hist, float* logp, float div_gamma, float div_prob, const float* div_u,
                             const uint64_t* div_state, const lo_beam_penalty* pen, const lo_bracket_rule* br, void* stream);
/* lo_tfdec_greedy, lo_tfdec_sample and lo_tfdec_beam_pen (pen NULL: no penalty) under the rule *br */
int lo_tfdec_greedy_brackets(const lo_tfdec_args* a, int64_t end_id, int max_steps, int64_t* tokens, int32_t* fin_hist,
                             const lo_bracket_rule* br, void* stream);
int lo_tfdec_sample_brackets(const lo_tfdec_args* a, const lo_sample_args* s, int64_t end_id, int max_steps, int64_t* tokens,
                             int32_t* fin_hist, const lo_bracket_rule* br, void* stream);
int lo_tfdec_beam_brackets(const lo_tfdec_args* a, int64_t end_id, int max_steps, int64_t* ids, int64_t* parents, int32_t* fin_hist,
                           float* logp, float div_gamma, float div_prob, const float* div_u, const uint64_t* div_state,
                           const lo_beam_penalty* pen, const lo_bracket_rule* br, void* stream);
/* lo_decoder2_greedy, lo_decoder2_sample and lo_decoder2_beam under the rule *br */
int lo_decoder2_greedy_brackets(const lo_decoder_args* a, const lo_decoder2_layer* l2, int64_t start_id, int64_t end_id, int max_steps,
                                int64_t* tokens, int32_t* finished, int32_t* fin_hist, const lo_bracket_rule* br, void* stream);
int lo_decoder2_sample_brackets(const lo_decoder_args* a, const lo_decoder2_layer* l2, const lo_sample_args* s, int64_t start_id,
                                int64_t end_id, int max_steps, int64_t* tokens, int32_t* finished, int32_t* fin_hist,
                                const lo_bracket_rule* br, void* stream);
int lo_decoder2_beam_brackets(const lo_decoder_args* a, const lo_decoder2_layer* l2, int64_t start_id, int64_t end_id, int max_steps,
                              int64_t* ids, int64_t* parents, int32_t* fin_hist, float* logp, float div_gamma, float div_prob,
                              const float* div_u, const uint64_t* div_state, const lo_beam_penalty* pen, const lo_bracket_rule* br,
                              void* stream);

/* ------------------------------------------------------------------------------------------------
 * Optimiser: torch.optim.Adam defaults (img2seq_torch.py:86-87, :168-170) on one flat buffer.
 * state_dev: float[2] = {step (as float), lr}; step is incremented on the device so the call is
 * graph-replayable.  shadow (optional) receives the bf16 copy of the updated parameters.
 */
int lo_adam_step(float* p, const float* g, float* m, float* v, void* shadow_bf16, int64_t n,
                 float* state_dev, float beta1, float beta2, float eps, float grad_scale, void* stream);
/* Same update restricted to n_ranges element ranges {offset, count} (host array of 2*n_ranges int64) of the flat buffers:
 * parameters outside the ranges are frozen (requires_grad=False after fine_tune(), seq2seq_torch.py:102-113, :246-253 —
 * torch.optim.Adam skips them: no moment decay, no update).  One step-counter increment for the whole call. */
int lo_adam_step_ranges(float* p, const float* g, float* m, float* v, void* shadow_bf16, const int64_t* ranges,
                        int n_ranges, float* state_dev, float beta1, float beta2, float eps, float grad_scale,
                        void* stream);
/* The optimisers of the TF trainer (model/img2seq.py:98-111) with TensorFlow 1.12's update rules, on one flat buffer:
 * kind 1 AdamOptimizer (epsilon outside the bias correction: lr_t = lr sqrt(1-b2^t)/(1-b1^t), p -= lr_t m/(sqrt(v)+eps)),
 * 2 GradientDescentOptimizer, 3 AdagradOptimizer (s1 = accumulator, initial value 0.1), 4 RMSPropOptimizer (s1 = rms slot,
 * initial value 1; beta2 = decay 0.9, eps 1e-10, momentum 0).  state_dev as in lo_adam_step. */
int lo_tf_optim_step(int kind, float* p, const float* g, float* s1, float* s2, void* shadow_bf16, int64_t n,
                     float* state_dev, float beta1, float beta2, float eps, float grad_scale, void* stream);
int lo_cast(const void* src, int dt_src, void* dst, int dt_dst, int64_t n, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* LATEX_OCR_B200_H */
