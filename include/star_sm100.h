/* star_sm100.h -- C ABI of libstar_sm100.so (star_b200/csrc), the sm_90a (H100) kernel library
 * behind star_b200's drop-in for the STAR denoising hot path.
 *
 * The reference (NJU-PCALab/STAR) has no FFI: every kernel it runs is dispatched by
 * PyTorch (cuDNN / cuBLAS / xformers).  Each entry point below replaces the library call
 * made at the cited reference line(s); a maintainer binds them with ctypes (see
 * INTEGRATION.md) from the module that currently makes that call.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer (tensor.data_ptr()); fp16 unless stated
 *   - activations are channels-last token matrices X[rows, C], rows ordered (b, t, h, w)
 *   - ld* arguments are leading dimensions in ELEMENTS
 *   - `stream` is a cudaStream_t; all calls are asynchronous on it, allocate nothing and
 *     keep no state besides the per-process driver entry point resolved by star_init
 *   - return 0 on success, non-zero on error; star_last_error() gives the message
 */
#ifndef STAR_SM100_H
#define STAR_SM100_H
#ifdef __cplusplus
extern "C" {
#endif

#define STAR_FLAG_GEGLU 1     /* W has 2N rows (value|gate): out = value * gelu_erf(gate)  (unet_v2v.py:496-504) */
#define STAR_FLAG_GELU_ERF 4  /* out = gelu_erf(acc) (nn.GELU of the OpenCLIP text tower's MLP, video_to_video/modules/embedder.py:27)    */
#define STAR_FLAG_GELU_TANH 8 /* out = gelu_tanh(acc) (sat MLP activation, cogvideox-based/transformer.py:202-312)  */
#define STAR_FLAG_SILU_OUT 2  /* out = silu(acc)                                            (unet_v2v.py:1340-1342) */

int star_version(void);
const char* star_last_error(void);
/* number of kernels this library has launched since it was loaded (all streams) */
long long star_launch_count(void);
/* Resolve cuTensorMapEncodeTiled, opt kernels into >48 KB shared memory.  Fails on non-sm_90 devices. */
int star_init(int device);

/* nn.Linear / Conv2d 1x1 / Conv1d k=1: out[r, n] = sum_k A[r,k] W[n,k] (+bias[n]) (+rowvec[r/rowvec_div, n])
 * (+residual[r,n]); replaces F.linear / conv at unet_v2v.py:159-162,:195 (attention projections), :503,:526 (GEGLU
 * feed-forward), :309,:313 (SpatialTransformer proj), :1046,:1084 (TemporalTransformer Conv1d), :648 (skip 1x1),
 * :2132 (zero convs), :1341-1342,:628 (time embedding). */
int star_linear(const void* A, long long lda, const void* W, const void* bias, const void* rowvec,
                long long rowvec_div, const void* residual, long long ldres, void* out, long long ldo,
                long long rows, int K, int N, int flags, void* stream);

/* star_linear with a per-output-column scale applied before the residual add:
 * out = residual + colscale[n] * (acc + bias[n])  -- the adaLN gates of the CogVideoX DiT layer
 * (cogvideox-based/sat/dit_video_concat.py:543-544,:560-561).  flags may also carry STAR_FLAG_GELU_TANH.
 * a_block_cols > 0: A is head-blocked, row r of A being K / a_block_cols blocks of a_block_cols columns side by side, block
 * b of row r at A + b * a_block_pitch + r * lda (the attention output a token-sharded DiT rank gets back from its head
 * all-to-all, star_b200/cogvideox/parallel.py); a_block_cols a multiple of 64 dividing K, at most 27 blocks, no GEGLU.  The
 * result is the unblocked call's on the concatenated rows, bit for bit.  a_block_cols = 0: A is [rows, lda]. */
int star_linear_ex(const void* A, long long lda, const void* W, const void* bias, const void* rowvec,
                   long long rowvec_div, const void* colscale, const void* residual, long long ldres, void* out,
                   long long ldo, long long rows, int K, int N, int flags, int a_block_cols, long long a_block_pitch,
                   void* stream);

/* Conv2d 3x3 stride 1 pad 1 on X[BT,H,W,Cin]; W9 = weight permuted to [Cout][3][3][Cin]; rowvec = per-clip time
 * embedding added before the next GroupNorm; replaces cuDNN at unet_v2v.py:612,:639,:553-554,:1552.  Only output rows
 * [row0, row0 + H_out) are computed, out = [BT, H_out, W, Cout]: a band of X whose halo rows come from X itself (the temporal
 * VAE upsamples and convolves a large frame band by band).  row0 = 0, H_out = H is the whole frame. */
int star_conv2d_3x3(const void* X, const void* W9, const void* bias, const void* rowvec, long long rowvec_div, long long ldrowvec,
                    const void* residual, long long ldres, void* out, long long ldo, int BT, int H, int W, int Cin,
                    int Cout, int row0, int H_out, void* stream);
/* Downsample: Conv2d 3x3 stride 2 padding (2,1) (unet_v2v.py:709-729).  Ho = (H+1)/2 + 1, Wo = (W-1)/2 + 1.
 * planes_ws: scratch of star_conv2d_s2_workspace_bytes(). */
long long star_conv2d_s2_workspace_bytes(int BT, int H, int W, int Cin);
int star_conv2d_3x3_s2(const void* X, const void* W9, const void* bias, void* out, long long ldo, void* planes_ws,
                       int BT, int H, int W, int Cin, int Cout, void* stream);
/* Same with explicit zero padding (top, bottom, left, right): the temporal VAE's encoder downsamples with
 * F.pad(x, (0,1,0,1)) + Conv2d(stride 2, padding 0) (diffusers 0.30.0 Downsample2D, reached from
 * video_to_video_model.py:158 vae.encode).  Ho = (H+pad_t+pad_b-3)/2 + 1, Wo likewise. */
long long star_conv2d_s2p_workspace_bytes(int BT, int H, int W, int Cin, int pad_t, int pad_b, int pad_l, int pad_r);
int star_conv2d_3x3_s2p(const void* X, const void* W9, const void* bias, void* out, long long ldo, void* planes_ws,
                        int BT, int H, int W, int Cin, int Cout, int pad_t, int pad_b, int pad_l, int pad_r,
                        void* stream);
/* Conv3d (3,1,1) pad (1,0,0) over frames on X[B,T,HW,Cin]; W3 = weight permuted to [Cout][3][Cin]
 * (unet_v2v.py:1209-1220).  Runs over pixels [p0, p0 + band) of every frame: X holds that band compactly ([B, T, band, Cin]),
 * residual and out are the full [B, T, HW] row space of which only the band's rows are read / written (the temporal VAE
 * decodes large frames band by band).  p0 = 0, band = HW is the whole clip. */
int star_conv_t3(const void* X, const void* W3, const void* bias, const void* residual, long long ldres, void* out,
                 long long ldo, int B, int T, long long HW, long long p0, long long band, int Cin, int Cout, void* stream);
/* Stem convs with Cin = 4 (unet_v2v.py:1353 input conv, :2128 input_hint_block); W9 as above.  Runs as im2col
 * (K = 36 padded to 64) + tensor-core GEMM; ws = scratch of star_conv2d_c4_workspace_bytes(). */
long long star_conv2d_c4_workspace_bytes(int BT, int H, int W, int Cout);
int star_conv2d_3x3_c4(const void* X, const void* W9, const void* bias, const void* residual, void* out, void* ws,
                       int BT, int H, int W, int Cout, void* stream);

/* softmax(Q K^T * scale) V, head_dim 64, heads side by side along the row (column offset h*64); batch b uses rows
 * [b*Nq,(b+1)*Nq) of Q/O and rows [(b/kv_batch_div)*Nk, ...) of K/V.  Replaces
 * xformers.ops.memory_efficient_attention at unet_v2v.py:179,:184 for spatial self- and text cross-attention. */
int star_attention(const void* Q, long long ldq, const void* K, long long ldk, const void* V, long long ldv, void* O,
                   long long ldo, int batch, int heads, int Nq, int Nk, int kv_batch_div, float scale, void* stream);
/* Causal self-attention, head_dim 64: query i attends keys 0..i.  Replaces nn.MultiheadAttention with the text tower's
 * attn_mask inside the OpenCLIP ViT-H-14 residual blocks FrozenOpenCLIPEmbedder.text_transformer_forward iterates
 * (video_to_video/modules/embedder.py:56-71; mask = open_clip's build_attention_mask, -inf above the diagonal). */
int star_attention_causal(const void* Q, long long ldq, const void* K, long long ldk, const void* V, long long ldv, void* O,
                          long long ldo, int batch, int heads, int N, float scale, void* stream);

/* Temporal self-attention over T frames per pixel; QKV [B*T*HW, ld] with q|k|v at column 0|Ci|2Ci
 * (unet_v2v.py:483-489 through :158-195).  Any T >= 1: T <= 64 runs the mma.sync kernel (tattn2.cuh), T > 64 the
 * wgmma kernel (tattn_long.cuh; needs heads*64 <= Ci <= ld/3, B*HW*heads < 2^31 and T*HW*ld*2 bytes < 2^40). */
int star_temporal_attention(const void* QKV, long long ld, void* O, long long ldo, int B, int T, long long HW,
                            int heads, int Ci, float scale, void* stream);

/* GroupNorm(32) (+SiLU): nsamples blocks of rows_per_sample rows share statistics -- one frame for the 4-D norms
 * (unet_v2v.py:268,:610,:635,:1551), the whole clip for the 5-D norms (:1002,:1210-1219). fp32 statistics. */
/* Causal Conv3d 3x3x3 of the CogVideoX 3-D VAE: replaces ContextParallelCausalConv3d.forward
 * (cogvideox-based/sat/vae_modules/cp_enc_dec.py:384-430, the F.pad + Conv3d at :426-428).  X holds T + 2 frames of H x W x Cin
 * tokens: the two leading frames are the temporal context the reference concatenates (:265-268 -- copies of frame 0, or the
 * cache kept from the previous latent chunk), the spatial zero padding is implicit.  W27 [Cout, 3, 3, 3, Cin] (t, h, w). */
int star_conv3d_causal(const void* X, const void* W27, const void* bias, const void* residual, long long ldres, void* out,
                       long long ldo, int T, int H, int W, int Cin, int Cout, void* stream);

/* phases: STAR_GN_STATS computes the statistics into the workspace (star_groupnorm_workspace_bytes(nsamples, C)),
 * STAR_GN_APPLY normalises with the workspace's statistics: each sample is viewed as frames of frame_rows rows, and rows
 * [p0, p0 + band) of every frame are written compactly to out ([frames * band, C]), so clip statistics can be applied a pixel
 * band at a time.  Both phases over whole samples (frame_rows = band = rows_per_sample, p0 = 0) is one GroupNorm; out may
 * then alias X.  Split phases and bands need C <= 2048. */
#define STAR_GN_STATS 1
#define STAR_GN_APPLY 2
long long star_groupnorm_workspace_bytes(int nsamples, int C);
int star_groupnorm(const void* X, const void* gamma, const void* beta, void* out, int nsamples, long long rows_per_sample, int C,
                   float eps, int silu, long long frame_rows, long long p0, long long band, int phases, void* workspace,
                   void* stream);
/* SpatialNorm3D.forward of the CogVideoX 3-D VAE decoder (cp_enc_dec.py:491-510): out = GroupNorm32(X) * Ymod[src] + Bmod[src]
 * (+ SiLU, the `nonlinearity` that always follows, :673,:687,:977) over one clip of T x H x W rows.  Ymod / Bmod are conv_y(zq) /
 * conv_b(zq) evaluated at the latent's resolution (Tl, Hl, Wl): 1x1x1 convolutions commute with the nearest-neighbour
 * interpolation of zq (:492-500, incl. its first-frame split for odd T); ldmod = their row pitch.  workspace: star_groupnorm_workspace_bytes(1, C). */
int star_groupnorm_mod(const void* X, const void* gamma, const void* beta, const void* Ymod, const void* Bmod, long long ldmod,
                       void* out, int T, int H, int W, int Tl, int Hl, int Wl, int C, float eps, int silu, void* workspace, void* stream);

/* LayerNorm over C (unet_v2v.py:448-450) with fused LIEM gate: gate_mode 0 none, 1 per-row gate[] (spatial LIEM),
 * 2 temporal LIEM sigmoid(w0*max + w1*mean) (unet_v2v.py:396-411). */
int star_layernorm(const void* X, const void* gamma, const void* beta, void* out, long long rows, int C, float eps,
                   int gate_mode, const void* gate, float w0, float w1, void* stream);
/* Spatial LIEM gate: channel max/mean -> 7x7 conv (2->1) -> sigmoid (unet_v2v.py:380-394).  w98 = conv1.weight
 * flattened [2][7][7]; mm_ws = the clip's channel max/mean map [BT*H*W][2] fp16.  Runs over tokens [r0, r0 + n) of the clip
 * (r0 = 0, n = BT*H*W: the whole clip): X (NULL: skipped) holds those tokens' rows [n, C], and their max/mean go to
 * mm_ws rows [r0, r0 + n); gate (NULL: skipped) receives their n gates, from mm_ws over the whole clip.  A token-sharded
 * DiT rank reduces its own tokens, all-gathers the map and gates its own tokens. */
int star_liem_spatial_gate(const void* X, const void* w98, void* mm_ws, void* gate, int BT, int H, int W, int C,
                           long long r0, long long n, void* stream);

/* CogVideoX DiT layer helpers (cogvideox-based/sat/dit_video_concat.py).
 * star_row_gate: out = X * g(row); mode 1: g = gate[row] (spatial LIEM, :523-527, gate from star_liem_spatial_gate);
 * mode 2: g = sigmoid(w0*max_c + w1*mean_c) (temporal LIEM, :529-531).
 * star_qk_ln_rope: in-place per-head LayerNorm(64) of q (column 0) and k (column koff) of QKV[rows, ld] (:583-587)
 * followed by the 3-D rotary embedding of the image tokens (rows with (row % seq) >= text_len; :306-333);
 * cos/sin are fp32 [seq - text_len, 64]. */
int star_row_gate(const void* X, void* out, long long rows, int C, int mode, const void* gate, float w0, float w1,
                  void* stream);
int star_qk_ln_rope(void* QKV, long long ld, long long rows, int heads, int koff, const void* qg, const void* qb,
                    const void* kg, const void* kb, const void* cos_f32, const void* sin_f32, int seq, int text_len,
                    float eps, void* stream);

/* out[rows, Ca+Cb] = [a | b (+c)]  (torch.cat + control residual, unet_v2v.py:1792); c may be NULL */
int star_concat_add(const void* a, int Ca, const void* b, const void* c, int Cb, void* out, long long rows,
                    void* stream);
int star_add(const void* a, const void* b, void* out, long long n, void* stream);
/* nearest x2 + crop first/last row (unet_v2v.py:563-564): out [BT, 2H-2, 2W, C] */
int star_upsample2x_crop(const void* X, void* out, int BT, int H, int W, int C, void* stream);
/* Temporal half of DownSample3D.forward in the CogVideoX 3-D VAE encoder (cogvideox-based/sat/vae_modules/cp_enc_dec.py:581-596):
 * avg_pool1d(kernel 2, stride 2) over the frames of a [(T HW), C] clip; odd T keeps the first frame and pools the other T - 1.
 * out has ceil(T / 2) frames. */
int star_time_avgpool2(const void* X, void* out, int T, long long HW, int C, void* stream);

/* nearest x2, crop_rows = 1 as above, 0 = plain F.interpolate(scale_factor=2) of the VAE decoder's Upsample2D
 * (video_to_video_model.py:142 vae.decode): out [BT, 2H - 2*crop_rows, 2W, C] */
int star_upsample2x(const void* X, void* out, int BT, int H, int W, int C, int crop_rows, void* stream);

/* ---- temporal VAE (video_to_video_model.py:141-161 -> diffusers AutoencoderKLTemporalDecoder) ----------------
 * The single-head (d = 512) mid-block attention runs as S = Q K^T (star_linear, N = tokens), star_softmax_rows,
 * O = S V (star_linear against V^T).  star_softmax_rows: in place over the first `cols` entries of each
 * 16-byte-aligned row of the fp16 matrix S[rows, ld] (logits already scaled), columns cols..ld-1 zeroed.  Each row is
 * split over a cluster of ctas_per_row (1..8) CTAs that each stage at most 102 400 columns in shared memory, so
 * cols <= ctas_per_row * 102400; the caller picks ctas_per_row from the row length.  ctas_per_row = 1 is one CTA per row. */
int star_softmax_rows(void* S, long long ld, long long rows, int cols, int ctas_per_row, void* stream);
/* decoder tail: time_conv_out = Conv3d(3,3,(3,1,1),padding (1,0,0)) over X[(b t hw), ldx] (3 valid channels) fused with
 * the tokens -> (b t, 3, h, w) layout change; W27 = weight [3][3][3] (co, ci, dt) fp16, bias3 fp16, out fp16. */
int star_vae_head(const void* X, long long ldx, const void* W27, const void* bias3, void* out, int B, int T,
                  long long HW, void* stream);
/* (b,c,f,h,w) fp32 -> tokens fp16 [(b f h w), c]  and back (fp16 -> fp16)  (unet_v2v.py:1772,:1808) */
int star_nchw5_to_tokens(const void* x_f32, void* out, int B, int C, int F, long long HW, void* stream);
int star_tokens_to_nchw5(const void* x, long long ldx, void* out, int B, int C, int F, long long HW, void* stream);
/* ---- pipeline glue on the GPU ---------------------------------------------------------------------------------
 * F.interpolate(x, [H, W], mode='bilinear') + F.pad(x, (pad_l, pad_r, pad_t, pad_b), 'constant', pad_value)
 * (video_to_video_model.py:81,:86-87): x fp32 (NC, h, w) -> out fp32 (NC, H + pad_t + pad_b, W + pad_l + pad_r). */
int star_bilinear_pad(const void* x_f32, void* out_f32, long long NC, int h, int w, int H, int W, int pad_l, int pad_r,
                      int pad_t, int pad_b, float pad_value, void* stream);
/* tensor2vid + adain_color_fix (inference_utils.py:16-23, video_super_resolution/color_fix.py:15-29,47-74): per frame and channel
 * t = clamp((video + 1) / 2, 0, 1) is re-normalised to the mean / std (unbiased var + 1e-5) of s = (source + 1) / 2, clamped to [0, 1]
 * and written * 255 as (F, H*W, C).  video fp32 (C, F, HW) = test()'s (1, C, F, H, W); source fp32 (F, C, src_hw) = the LR clip.
 * Exactly one of out_f32 / out_u8 (rounded) is written.  workspace: star_adain_workspace_bytes(C, F). */
long long star_adain_workspace_bytes(int C, int F);
int star_adain_color_fix(const void* video_f32, const void* source_f32, void* out_f32, void* out_u8, int C, int F, long long HW,
                         long long src_hw, void* workspace, void* stream);
/* Classifier-free guidance + std-ratio rescale + v -> x0 (diffusion_sdedit.py:89-99) in two launches:
 *   out = u + g (y - u)   (fp16, each op rounded like the reference's fp16 tensor arithmetic)
 *   out *= r * std(y) / (std(out) + 1e-12) + (1 - r)      per sample over `per_sample` elements; r < 0: no rescale
 *   x0 = alpha[sample] * xt - sigma[sample] * out          fp32
 * y_out / u_out fp16 [samples, per_sample]; xt / x0 fp32; guided_out (fp16, may be NULL) receives `out`;
 * alpha / sigma fp32 [samples] on the device; workspace: star_cfg_x0_workspace_bytes(samples). */
long long star_cfg_x0_workspace_bytes(int samples);
int star_cfg_x0(const void* y_out, const void* u_out, const void* xt_f32, void* x0_f32, void* guided_out,
                float guide_scale, float guide_rescale, const void* alpha_f32, const void* sigma_f32, int samples,
                long long per_sample, void* workspace, void* stream);
/* star_cfg_x0 for one (temporal chunk, spatial tile) model call of tiled sampling, accumulated into the clip's x0:
 *   acc[s, c, f0 + f, r0 + i, c0 + j] += wy[i] * wx[j] * x0[s, c, f, i, j]      for lo <= f < hi
 * y_out / u_out fp16 [samples, C, Ft, th, tw] contiguous (the tile's outputs; the std-ratio statistics span all Ft frames);
 * xt_f32 / acc_f32 fp32 [samples, C, F, H, W] contiguous (the clip, read / updated in place at the window); wy [th], wx [tw]
 * fp32 blend weights on the device.  A unit weight into a zeroed acc gives star_cfg_x0's x0 bit for bit.  Each tile sample
 * must have fewer than 2^31 elements.  workspace: star_cfg_x0_workspace_bytes(samples). */
int star_cfg_x0_blend(const void* y_out, const void* u_out, const void* xt_f32, void* acc_f32, float guide_scale,
                      float guide_rescale, const void* alpha_f32, const void* sigma_f32, const void* wy_f32, const void* wx_f32,
                      int samples, int C, int Ft, int th, int tw, int F, int H, int W, int f0, int lo, int hi, int r0, int c0,
                      void* workspace, void* stream);
/* sinusoidal timestep embedding (unet_v2v.py:96-108); t = int64 [B]; out fp16 [B, dim] */
int star_sinusoidal(const void* t_i64, void* out, int B, int dim, void* stream);
int star_silu(const void* x, void* out, long long n, void* stream);

#ifdef __cplusplus
}
#endif
#endif
