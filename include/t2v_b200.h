/*
 * t2v_b200 - C ABI of the H100-native text-to-video finetune hot path.
 *
 * The reference (ExponentialML/Text-To-Video-Finetuning) has no FFI of its own: its hot path is the chain
 *   train.py:339-347 (tensor_to_vae_latent) -> train.py:720-836 (finetune_unet) ->
 *   models/unet_3d_condition.py:325-500 (UNet3DConditionModel.forward) -> models/unet_3d_blocks.py ->
 *   diffusers leaf modules -> ATen -> cuDNN/cuBLAS/SDPA.
 * Each entry point below replaces one class of ATen/library call reached from those leaves; the reference call
 * site each one stands in for is cited on the declaration.  The Python host code in
 * text-to-video-finetuning_b200/ binds these with ctypes (INTEGRATION.md shows the stub).
 *
 * Conventions
 *   - All pointers are raw CUDA device pointers owned by the caller (PyTorch's allocator); nothing is allocated
 *     or freed inside, nothing synchronises the device.  `stream` is a cudaStream_t passed as void*.
 *   - Activations are bf16, channels-last: a (N, C, H, W) tensor is stored [N][H][W][C]; a clip (B, C, F, H, W)
 *     is stored [B][F][H][W][C] (== frames-major [B*F][H][W][C]).
 *   - Convolution weights are bf16 [Cout][KH][KW][Cin] (torch.channels_last of the diffusers (Cout,Cin,KH,KW)
 *     parameter); linear weights are [out][in].  Weight gradients are fp32, same layout, ACCUMULATED (+=).
 *   - Channel counts must be multiples of 8 (16-byte TMA rows); 3/4-channel tensors are padded to 8 by the host.
 *   - Return value: 0 on success, negative on error; t2v_last_error() returns a thread-local message.
 *     Functions are re-entrant and hold no thread-local state besides that message (autograd calls backward
 *     entry points from worker threads).
 */
#ifndef T2V_B200_H_
#define T2V_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

int t2v_version(void);
const char* t2v_last_error(void);
/* Number of kernels this library has launched since load (bench.py reports it as gpu_launches). */
int64_t t2v_launch_count(void);
/* Identifier of the CUDA-graph capture `stream` is currently part of, 0 when it is not capturing.  The host layer uses it to
 * keep zero-initialised scratch (GroupNorm statistics) from crossing a capture boundary: memory zeroed by a memset node of
 * one graph is not zero for launches outside that graph.                                                            */
int64_t t2v_stream_capture_id(void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Fused epilogue shared by the tensor-core entry points:  y = alpha * acc + bias[c] + rowbias[n][c] + residual
 */
typedef struct {
    const float* bias;      /* [Cout] fp32 or NULL                                                       */
    const float* rowbias;   /* [N][Cout] fp32 or NULL (ResnetBlock2D time_emb_proj broadcast over H, W)   */
    const void* residual;   /* bf16, same shape/layout as the output, or NULL                             */
    float alpha;
    int32_t out_fp32;       /* 0: bf16 output, 1: fp32 output                                             */
    int32_t rowbias_div;    /* rowbias row = n / rowbias_div (frames per clip: one time-embedding row per
                               clip instead of the reference's repeat_interleave, unet_3d_condition.py:400) */
    void* workspace;        /* optional scratch of t2v_conv_workspace_bytes(...) bytes: lets conv_fwd / conv_dgrad
                               split the reduction over SMs when the output has few tiles (deep, small maps)   */
    int64_t workspace_bytes;
    /* GroupNorm input statistics of the OUTPUT, produced by the epilogue (conv_fwd only; NULL: none): for output row r (rows
     * flattened in [N][Ho][Wo] order) and column c
     *     stats[((r / stats_rows) * stats_ld + c) * 2 + {0, 1}] += {y, y*y}          (fp32, red.add; zero the buffer first)
     * i.e. one (sum, sum of squares) pair per frame and channel; stats_rows = output rows per frame.  The consumer GroupNorm
     * (t2v_groupnorm_fwd) finalises them per frame or per clip, so its statistics pass over the tensor disappears.       */
    float* stats;
    int64_t stats_ld;
    int32_t stats_rows;
    int32_t pad_;
} T2VEpilogue;

/* Implicit-GEMM convolution forward on wgmma tensor cores (TMA-fed, zero padding by TMA OOB fill).
 * Replaces nn.Conv2d / nn.Conv3d(3,1,1) / nn.Linear forward as reached from
 *   ResnetBlock2D.conv1/conv2/conv_shortcut, Downsample2D.conv, Upsample2D.conv  (unet_3d_blocks.py:295-306,457-469,506-513,741-744)
 *   TemporalConvLayer.conv1..4  (unet_3d_blocks.py:308-314; tensor viewed as W=H*W, H=F, N=B, KH=3, KW=1)
 *   conv_in / conv_out          (unet_3d_condition.py:132,249)
 *   every nn.Linear             (viewed as W=rows, H=N=1, 1x1)
 * x [N][H][W][Cin], w [Cout][KH][KW][Cin], y [N][Ho][Wo][Cout];  Ho = (H + pad_h0 + pad_h1 - KH)/stride + 1.  */
int t2v_conv_fwd(const void* x, const void* w, void* y, int32_t N, int32_t H, int32_t W, int32_t Cin, int32_t Cout,
                 int32_t KH, int32_t KW, int32_t stride, int32_t pad_h0, int32_t pad_h1, int32_t pad_w0,
                 int32_t pad_w1, const T2VEpilogue* epi, void* stream);

/* Data gradient of the same convolution: dx [N][H][W][Cin] = conv_transpose(dy [N][Ho][Wo][Cout], w).
 * epi->residual (bf16, shape of dx) is added, which lets the caller sum gradient branches for free.
 * (autograd of the call sites above; train.py:861 accelerator.backward)                                */
int t2v_conv_dgrad(const void* dy, const void* w, void* dx, int32_t N, int32_t H, int32_t W, int32_t Cin, int32_t Cout,
                   int32_t KH, int32_t KW, int32_t stride, int32_t pad_h0, int32_t pad_h1, int32_t pad_w0,
                   int32_t pad_w1, const T2VEpilogue* epi, void* stream);

/* Scratch bytes t2v_conv_fwd (dgrad = 0) / t2v_conv_dgrad (dgrad = 1) would like for this problem (0: none).
 * Without the scratch the same result is computed unsplit (slower on the 4x4 .. 16x16 levels of the UNet).   */
int64_t t2v_conv_workspace_bytes(int32_t dgrad, int32_t N, int32_t H, int32_t W, int32_t Cin, int32_t Cout, int32_t KH, int32_t KW,
                                 int32_t stride, int32_t pad_h0, int32_t pad_h1, int32_t pad_w0, int32_t pad_w1);

/* Weight gradient: dw [Cout][KH][KW][Cin] (fp32) += dy^T * shifted(x).  Split over pixels to fill the GPU;
 * partial products are reduced with red.global.add.f32 directly into the fp32 gradient buffer.              */
int t2v_conv_wgrad(const void* x, const void* dy, float* dw, int32_t N, int32_t H, int32_t W, int32_t Cin, int32_t Cout,
                   int32_t KH, int32_t KW, int32_t stride, int32_t pad_h0, int32_t pad_h1, int32_t pad_w0,
                   int32_t pad_w1, void* stream);
/* The same plus the bias gradient of the layer: dbias [Cout] (fp32) += sum over output pixels of dy - what autograd's
 * conv / linear backward returns as grad_bias (reference: every biased Conv2d / Conv3d / Linear of models/unet_3d_*.py).
 * The sums come out of the same launch (an extra 16-column MMA of the dy tile against a tile of ones, added from the
 * epilogue with red.global.add.f32) unless the chosen tiling has no spare accumulator columns; then a column-sum pass
 * over dy follows.  dbias == NULL is t2v_conv_wgrad.                                                               */
int t2v_conv_wgrad_bias(const void* x, const void* dy, float* dw, float* dbias, int32_t N, int32_t H, int32_t W, int32_t Cin,
                        int32_t Cout, int32_t KH, int32_t KW, int32_t stride, int32_t pad_h0, int32_t pad_h1, int32_t pad_w0,
                        int32_t pad_w1, void* stream);

/* Strided-batched GEMM on the same kernel:  C[z1][z2] = alpha * opA(A[z1][z2]) * opB(B[z1][z2])^T  (+= if accumulate)
 *   a_kmajor=1: A is [M][K] rows (K contiguous);  a_kmajor=0: A is stored [K][M] (M contiguous)
 *   b_kmajor=1: B is [N][K] rows (K contiguous);  b_kmajor=0: B is stored [K][N] (N contiguous)
 * Used for the attention products QK^T, PV and their gradients (Attention in Transformer2DModel /
 * AutoencoderKL mid-block; diffusers AttnProcessor2_0 -> SDPA in the reference, train.py:138-152), and for
 * nn.Linear weight gradients.  out_mode: 0 bf16, 1 fp32, 2 fp32 accumulate (split-K allowed).              */
typedef struct {
    const void* ptr;
    int64_t ld;         /* elements between consecutive rows of the stored matrix */
    int64_t stride_z1;  /* elements */
    int64_t stride_z2;
    int32_t kmajor;
} T2VMat;
int t2v_bgemm(const T2VMat* A, const T2VMat* B, void* C, int64_t ldc, int64_t c_stride_z1, int64_t c_stride_z2,
              int32_t M, int32_t N, int32_t K, int32_t Z1, int32_t Z2, float alpha, int32_t out_mode, void* stream);

/* The GEMM launches the four entry points above would make for a problem on a device with `sm_count` SMs, computed on the
 * host without touching a device: the tiling, split-K, pipeline and epilogue decisions of the planner, one record per
 * launch (t2v_conv_dgrad with stride 2 makes one launch per output parity class).  The planner overrides T2V_FORCE_BN,
 * T2V_FORCE_SPLITS, T2V_FORCE_FWD_SPLITS, T2V_FORCE_STAGES, T2V_NO_SPLIT and T2V_NO_ROWSUM_FUSE are read from the environment
 * on every call, as the entry points do.  Pointers are assumed 16-byte aligned.  Writes min(result, max_out) records and
 * returns the number of launches, or a negative error for a problem the entry point would reject.                   */
enum { T2V_GEMM_CONV_FWD = 0, T2V_GEMM_CONV_DGRAD = 1, T2V_GEMM_CONV_WGRAD = 2, T2V_GEMM_BGEMM = 3 };
enum { T2V_FOLLOW_NONE = 0, T2V_FOLLOW_SPLITK_FINISH = 1, T2V_FOLLOW_CHANNEL_STATS = 2, T2V_FOLLOW_COLSUM = 3 };
typedef struct {
    int32_t kind;          /* T2V_GEMM_*                                                                           */
    int32_t N, H, W, Cin, Cout, KH, KW, stride, pad_h0, pad_h1, pad_w0, pad_w1;   /* convolutions, as in t2v_conv_*   */
    int32_t workspace;     /* fwd / dgrad: the caller passes split-K scratch (T2VEpilogue.workspace != NULL)          */
    int32_t stats_rows;    /* fwd: GroupNorm statistics requested, T2VEpilogue.stats_rows (0: not requested)          */
    int32_t dbias;         /* wgrad: t2v_conv_wgrad_bias rather than t2v_conv_wgrad                                 */
    int32_t gemm_m, gemm_n, gemm_k, z1, z2, b_kmajor, out_mode;   /* bgemm: M, N, K, Z1, Z2, B->kmajor, out_mode      */
} T2VGemmProblem;
typedef struct {
    int32_t block_n, num_stages;   /* wgmma N, pipeline stages                                                       */
    int32_t splits, kb_per_split;  /* split-K factor (1: none) and k-blocks per split (0 when not split)              */
    int32_t ksplit_var;            /* tile variable that selects the k-range (-1: none)                              */
    int32_t num_tiles, grid;       /* work tiles, persistent CTAs = min(num_tiles, sm_count)                         */
    int32_t box[3];                /* pixel box (w, h, n) of a tile's 128 rows                                       */
    int32_t tdim[6], kdim[3];      /* tile grid (t[0] = N tiles) and k-block grid                                    */
    int32_t flags;                 /* epilogue work chosen by the planner: 16 GroupNorm statistics, 32 bias gradient */
    int32_t st[5];                 /* statistics row -> sample map (cw, ch, cn, div, seg) when flags has 16          */
    int32_t follow;                /* T2V_FOLLOW_*: the pass that completes this launch                               */
} T2VGemmPlan;
int t2v_gemm_plan(const T2VGemmProblem* problem, int32_t sm_count, T2VGemmPlan* out, int32_t max_out);

/* Fused attention (head_dim 64): O = softmax(Q K^T / 8) V per (batch, head) without materialising the score matrix,
 * plus its backward; replaces the t2v_bgemm / t2v_softmax composition for Transformer2DModel's self- and cross-attention
 * (diffusers AttnProcessor2_0 -> F.scaled_dot_product_attention in the reference, train.py:138-152).
 * Operands are [Nb][L][heads*64] with arbitrary row pitch (*_ld) and batch stride (*_bs) in elements, so q / k / v and
 * dq / dk / dv may be column slices of fused QKV / K|V projections.  o and dout are [Nb][Lq][heads*64] (o_ld, o_bs).
 * lse: fp32 [Nb][heads][Lq] (natural-log sum-exp of the scaled scores), written by fwd, read by bwd.
 * delta_ws: fp32 scratch [Nb][heads][Lq].  dkv_ws: fp32 scratch [2][Nb][Lk][heads*64], ZERO on entry, required only when
 * t2v_flash_attn_bwd_splits(...) > 1 (few keys, many queries: cross-attention); dK / dV are then left in dkv_ws (fp32)
 * for the caller to cast, and dk / dv are not written.                                                               */
int t2v_flash_attn_fwd(const void* q, const void* k, const void* v, void* o, float* lse, int32_t Nb, int32_t heads, int32_t Lq,
                       int32_t Lk, int32_t head_dim, int64_t q_ld, int64_t q_bs, int64_t k_ld, int64_t k_bs, int64_t v_ld,
                       int64_t v_bs, int64_t o_ld, int64_t o_bs, void* stream);
int32_t t2v_flash_attn_bwd_splits(int32_t Nb, int32_t heads, int32_t Lq, int32_t Lk);
int t2v_flash_attn_bwd(const void* q, const void* k, const void* v, const void* o, const void* dout, const float* lse, void* dq,
                       void* dk, void* dv, float* delta_ws, float* dkv_ws, int32_t Nb, int32_t heads, int32_t Lq, int32_t Lk,
                       int32_t head_dim, int64_t q_ld, int64_t q_bs, int64_t k_ld, int64_t k_bs, int64_t v_ld, int64_t v_bs,
                       int64_t o_ld, int64_t o_bs, int64_t dq_ld, int64_t dq_bs, int64_t dk_ld, int64_t dk_bs, int64_t dv_ld,
                       int64_t dv_bs, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * HBM-bound kernels (128-bit accesses, fp32 statistics, warp-shuffle reductions).
 */

/* GroupNorm (+ fused SiLU) over x [S][P][C] bf16: S normalisation samples of P pixels; replaces nn.GroupNorm + SiLU in
 * ResnetBlock2D.norm1/norm2 (per frame: S = B*F), Transformer2DModel.norm (eps 1e-6), TemporalConvLayer /
 * TransformerTemporalModel.norm (per clip: S = B, P = F*H*W) and conv_norm_out (unet_3d_condition.py:239-243,488-490).
 * stat [S][G][2] = (mean, rstd), ab [S][C][2] = per-channel affine with y = act(a x + b) (both saved for backward).
 * Two kernels per direction: per-channel sums (red.add into zeroed fp32 scratch) and a finalise + apply pass.  The forward
 * sums are skipped when the producer of x already emitted them (T2VEpilogue.stats): stats0 / stats1 then hold the per-frame
 * (sum, sum of squares) of channels [0, C0) and [C0, C) - two sources for a channel concatenation - with `fps` frames per
 * normalisation sample (1: per-frame norm, F: per-clip norm) and row pitches ld0 / ld1 in channels.
 * workspace: t2v_groupnorm_workspace_bytes(S, P, C) bytes, ZERO on entry, garbage afterwards (forward needs it only when
 * stats0 is NULL).                                                                                                  */
int64_t t2v_groupnorm_workspace_bytes(int32_t S, int64_t P, int32_t C);
int t2v_groupnorm_fwd(const void* x, const float* gamma, const float* beta, void* y, float* stat, float* ab, const float* stats0,
                      int32_t C0, int64_t ld0, const float* stats1, int64_t ld1, int32_t fps, void* workspace, int32_t S, int64_t P,
                      int32_t C, int32_t G, float eps, int32_t silu, void* stream);
/* dx = d/dx [act(GN(x))]^T dy (+ add); dgamma / dbeta (fp32) are accumulated (+=) and may be NULL.               */
int t2v_groupnorm_bwd(const void* dy, const void* x, const float* gamma, const float* stat, const float* ab, const void* add,
                      void* dx, float* dgamma, float* dbeta, void* workspace, int32_t S, int64_t P, int32_t C, int32_t G,
                      int32_t silu, void* stream);
/* stats[(s * ld + c) * 2 + {0,1}] += sum over the P pixels of sample s of {x, x*x}: the statistics pass on its own (what
 * T2VEpilogue.stats produces inside a GEMM epilogue), for GroupNorm inputs that do not come out of a GEMM.            */
int t2v_channel_stats(const void* x, float* stats, int32_t S, int64_t P, int32_t C, int64_t ld, void* stream);

/* LayerNorm over rows of x [rows][C] (BasicTransformerBlock.norm1/2/3, eps 1e-5); stat [rows][2] = (mean, rstd).  */
int t2v_layernorm_fwd(const void* x, const float* gamma, const float* beta, void* y, float* stat, int64_t rows, int32_t C,
                      float eps, void* stream);
int t2v_layernorm_bwd(const void* dy, const void* x, const float* gamma, const float* stat, const void* add, void* dx,
                      float* dgamma, float* dbeta, int64_t rows, int32_t C, void* stream);

/* Latent boundary.  (B, C<=8, F, H, W) fp32 -> [B*F][H*W][8] bf16 with zero-padded channels; when `noise` is given this
 * is DDPMScheduler.add_noise fused in: x_t = sqrt(abar[t_b]) x0 + sqrt(1 - abar[t_b]) eps  (train.py:751-760) and the
 * permute/reshape of unet_3d_condition.py:404.  nhwc8_to_latents is the inverse (unet_3d_condition.py:495).        */
int t2v_latents_to_nhwc8(const float* x0, const float* noise, const float* alphas_cumprod, const int64_t* timesteps, void* out,
                         int32_t B, int32_t C, int32_t F, int32_t HW, void* stream);
int t2v_nhwc8_to_latents(const void* in, float* out, int32_t B, int32_t C, int32_t F, int32_t HW, void* stream);
/* F.mse_loss(pred.float(), target.float()) (train.py:827) straight from the channels-last prediction.
 * loss != NULL: *loss = mean((pred - target)^2).  dpred != NULL: dpred = *gout * 2 (pred - target) / numel.         */
int t2v_mse_loss(const void* pred, const float* target, float* loss, const float* gout, void* dpred, int32_t B, int32_t C,
                 int32_t F, int32_t HW, void* stream);
/* The same loss for a v-prediction model (train.py:792-800): the target is DDPMScheduler.get_velocity(x0, noise, t),
 * sqrt(abar[t_b]) noise - sqrt(1 - abar[t_b]) x0, formed per element from the (B, C<=8, F, H, W) fp32 x0 and noise; it is
 * never stored.  abar (fp32 [T]) and timesteps (int64 [B]) are read on the device.  loss / gout / dpred as t2v_mse_loss. */
int t2v_velocity_mse_loss(const void* pred, const float* x0, const float* noise, const float* alphas_cumprod, const int64_t* timesteps,
                          float* loss, const float* gout, void* dpred, int32_t B, int32_t C, int32_t F, int32_t HW, void* stream);
/* Weighted and robust diffusion objectives (diffusers' --snr_gamma, --loss_type, --huber_schedule, --huber_c).  Per sample b,
 * with a_b = abar[t_b], target y (noise, or the velocity above when prediction is T2V_PRED_V) and d = pred - y:
 *   psi(d)  T2V_LOSS_L2: d^2   T2V_LOSS_HUBER: 2c_b (sqrt(d^2 + c_b^2) - c_b)   T2V_LOSS_SMOOTH_L1: 2 (sqrt(d^2 + c_b^2) - c_b)
 *   c_b     T2V_HUBER_CONSTANT: huber_c   T2V_HUBER_EXPONENTIAL: huber_c^(t_b / T)
 *           T2V_HUBER_SNR: (1 - huber_c) / (1 + sigma_b)^2 + huber_c, sigma_b = sqrt((1 - a_b) / a_b)   (huber_c at a_b = 0)
 *   w_b     snr_gamma <= 0: 1.  Otherwise, snr_b = a_b / (1 - a_b): min(snr_b, gamma) / snr_b for T2V_PRED_EPSILON (1 at
 *           a_b = 0), min(snr_b, gamma) / (snr_b + 1) for T2V_PRED_V (0 at a_b = 0)  (Hang et al. 2023, Min-SNR-gamma).
 * loss != NULL: *loss = sum_e w_b(e) psi(d_e) / numel.  dpred != NULL: dpred = *gout * w_b psi'(d) / numel.  With
 * T2V_LOSS_L2 and snr_gamma <= 0 this is t2v_mse_loss / t2v_velocity_mse_loss.  x0 is read only for T2V_PRED_V.        */
enum { T2V_PRED_EPSILON = 0, T2V_PRED_V = 1 };
enum { T2V_LOSS_L2 = 0, T2V_LOSS_HUBER = 1, T2V_LOSS_SMOOTH_L1 = 2 };
enum { T2V_HUBER_CONSTANT = 0, T2V_HUBER_EXPONENTIAL = 1, T2V_HUBER_SNR = 2 };
typedef struct {
    int32_t prediction;      /* T2V_PRED_*                                                   */
    int32_t loss;            /* T2V_LOSS_*                                                   */
    int32_t huber_schedule;  /* T2V_HUBER_*, ignored under T2V_LOSS_L2                       */
    int32_t num_timesteps;   /* T, the length of alphas_cumprod                              */
    float huber_c;           /* > 0; <= 1 with T2V_HUBER_EXPONENTIAL                          */
    float snr_gamma;         /* > 0: Min-SNR-gamma weighting; <= 0: none                      */
} T2VLossParams;
int t2v_diffusion_loss(const void* pred, const float* noise, const float* x0, const float* alphas_cumprod, const int64_t* timesteps,
                       const T2VLossParams* params, float* loss, const float* gout, void* dpred, int32_t B, int32_t C, int32_t F,
                       int32_t HW, void* stream);

/* AutoencoderKL latent_dist.sample() + rearrange + * scale (train.py:343-345): moments [B*F][HW][8] bf16 (mean | logvar),
 * eps (B,4,F,HW) fp32 -> out (B,4,F,HW) fp32 = (mean + exp(0.5 clamp(logvar,-30,20)) eps) * scale.                    */
int t2v_vae_sample(const void* moments, const float* eps, float* out, int32_t B, int32_t F, int32_t HW, float scale, void* stream);

/* GEGLU (diffusers FeedForward.net[0]): proj [M][2I] -> out [M][I] = h * gelu_erf(gate).                           */
int t2v_geglu_fwd(const void* proj, void* out, int64_t M, int32_t I, void* stream);
int t2v_geglu_bwd(const void* proj, const void* dout, void* dproj, int64_t M, int32_t I, void* stream);

/* SiLU on the (tiny) time-embedding path, casts, scaled copies and gradient fan-in adds.                           */
int t2v_silu_f32_to_bf16(const float* x, void* y, int64_t n, int32_t apply_silu, void* stream);
int t2v_silu_bwd_f32(const float* x, const float* dy, float* dx, int64_t n, int32_t accumulate, void* stream);
int t2v_silu_bf16(const void* x, void* y, int64_t n, void* stream);
int t2v_silu_bf16_bwd(const void* x, const void* dy, void* dx, int64_t n, void* stream);
int t2v_add_bf16(const void* a, const void* b, const void* c, void* out, int64_t n, void* stream);
int t2v_scale_bf16(const void* a, void* out, int64_t n, float alpha, void* stream);
int t2v_add_f32(const float* a, const float* b, float* out, int64_t n, void* stream);
int t2v_cast_f32_bf16(const float* src, void* dst, int64_t n, void* stream);
/* Frozen CLIP text encoder (train.py:784-790 `text_encoder(token_ids)[0]`; SURVEY 8(f) row 2) - the two ops it needs beyond
 * the shared GEMM / LayerNorm / softmax kernels: token + position embedding lookup (fp32 tables -> bf16 [rows][C], rows =
 * B * L) and the MLP activation (quick = 0: exact GELU as in the OpenCLIP ViT-H text tower of ms-1.7b; 1: quick_gelu).
 * t2v_softmax_fwd's causal_period > 0 applies the encoder's causal mask (row r sees columns <= r % causal_period).         */
int t2v_embed_tokens(const int64_t* ids, const float* tok_emb, const float* pos_emb, void* out, int64_t rows, int32_t L, int32_t C,
                     int32_t vocab, void* stream);
/* Backward of t2v_embed_tokens for text-encoder training: dy bf16 [rows][C] (rows = B * L) is accumulated (+=) into the fp32
 * gradients dtok [vocab][C] (dtok[id] += sum of the rows with that id, the id clamped to [0, vocab) as the forward clamps it)
 * and dpos [>= L][C] (dpos[l] += sum over b of row b*L + l).  Either may be null (that table is frozen).  No atomics: each
 * output row is summed by one block in row order, so two launches on the same inputs give the same bits.               */
int t2v_embed_tokens_bwd(const int64_t* ids, const void* dy, float* dtok, float* dpos, int64_t rows, int32_t L, int32_t C,
                         int32_t vocab, void* stream);
int t2v_gelu_bf16(const void* x, void* y, int64_t n, int32_t quick, void* stream);
/* Backward of t2v_gelu_bf16 for text-encoder LoRA training: dx = dy * gelu'(x), x the saved input, same `quick` switch;
 * n a multiple of 8.                                                                                                     */
int t2v_gelu_bwd_bf16(const void* x, const void* dy, void* dx, int64_t n, int32_t quick, void* stream);
/* Data pipeline front end (reference utils/dataset.py:22-41 normalize_input after the video reader's resize): decoded RGB
 * frames uint8 [F][H0][W0][3] -> bilinear resize to h x w (half-pixel centres) -> x / 127.5 - 1 -> bf16 channels-last
 * [F][h][w][8] (channels 3..7 zero), the layout AutoencoderKL.encode consumes.                                          */
int t2v_frames_u8_to_nhwc8(const uint8_t* src, void* dst, int32_t F, int32_t H0, int32_t W0, int32_t h, int32_t w, void* stream);
/* The same for a ragged batch (train_batch_size > 1 on clips of different native sizes), in one launch: `src` packs every
 * clip's uint8 [F_k][H0_k][W0_k][3] frames back to back; `table` (device, int64 [n_clips][4]) holds per clip its byte offset
 * in `src`, F_k, H0_k and W0_k; total_frames = sum of F_k.  dst = bf16 [total_frames][h][w][8], clip after clip, each
 * clip's slice bitwise equal to t2v_frames_u8_to_nhwc8 on that clip alone.  1 <= n_clips <= 256; the table's rows are
 * trusted (prims.frames_u8_to_nhwc8_ragged checks them against the buffer size before the launch).                     */
int t2v_frames_u8_to_nhwc8_ragged(const uint8_t* src, const int64_t* table, int32_t n_clips, int64_t total_frames, void* dst, int32_t h,
                                  int32_t w, void* stream);
/* Gradient compression around the data-parallel all-reduce (the reference reduces through accelerate/DDP, train.py:661,861):
 * dst (bf16) = alpha * src (fp32), alpha = 1 / world so that a SUM all-reduce averages; and the widening inverse.          */
int t2v_scale_cast_f32_bf16(const float* src, void* dst, int64_t n, float alpha, void* stream);
int t2v_cast_bf16_f32(const void* src, float* dst, int64_t n, void* stream);

/* nn.Dropout fused with the LoRA branch / TemporalConvLayer stage: out = base + scale * x * mask / (1 - p), mask drawn
 * from a stateless counter-based generator keyed by (seed, element index); calling it again with the same seed on dy
 * (base NULL) is the backward.  (reference utils/lora.py:57-62 dropout after lora_up; TemporalConvLayer Dropout(0.1))    */
int t2v_dropout_scale_add(const void* x, const void* base, void* out, int64_t n, float p, float scale, uint64_t seed, const int64_t* epoch,
                          void* stream);
/* *counter += value on the device (the per-step dropout epoch: `epoch` above may be NULL or point at such a counter, whose
 * value is mixed into the seed when the kernel RUNS, so a replayed CUDA graph draws new masks every step).              */
int t2v_counter_add(int64_t* counter, int64_t value, void* stream);

/* Upsample2D's F.interpolate(mode="nearest") on [N][H][W][C] and its gradient (any size ratio).                      */
int t2v_upsample_nearest_fwd(const void* x, void* y, int32_t N, int32_t H, int32_t W, int32_t Ho, int32_t Wo, int32_t C, void* stream);
int t2v_upsample_nearest_bwd(const void* dy, void* dx, int32_t N, int32_t H, int32_t W, int32_t Ho, int32_t Wo, int32_t C, void* stream);
/* Channel-range copy between row-major bf16 matrices: the skip-connection torch.cat / its split in backward
 * (unet_3d_blocks.py:764,861).                                                                                     */
int t2v_copy_cols(const void* src, void* dst, int64_t M, int32_t C, int32_t src_ld, int32_t src_off, int32_t dst_ld, int32_t dst_off,
                  void* stream);
/* out [S][C] (fp32) += sum_p x [S][P][C]: bias gradients and the per-clip time-embedding gradient.                 */
int t2v_colsum(const void* x, float* out, int32_t S, int64_t P, int32_t C, void* stream);
int t2v_colsum_f32(const float* x, float* out, int32_t S, int32_t C, void* stream);
/* Row softmax between the two attention GEMMs: fp32 scores [rows][ld_in] -> bf16 probabilities [rows][ld_out]
 * (columns >= n_valid written as 0), and dS = P * (dP - rowsum(P dP)) * scale.                                     */
int t2v_softmax_fwd(const float* s, void* p, int64_t rows, int32_t n_valid, int32_t ld_in, int32_t ld_out, int32_t causal_period,
                    void* stream);
int t2v_softmax_bwd(const void* p, const float* dp, void* ds, int64_t rows, int32_t n_valid, int32_t ld_p, int32_t ld_dp, float scale,
                    void* stream);
/* Timesteps(dim, flip_sin_to_cos=True, shift 0) (unet_3d_condition.py:138,392): int64 [B] -> bf16 [B][dim] = [cos | sin]. */
int t2v_timestep_embedding(const int64_t* t, void* out, int32_t B, int32_t dim, void* stream);

/* Self-attention over short sequences (L <= 32, head_dim 32 or 64) addressed by strides: the frame-axis attention of
 * TransformerTemporalModel (unet_3d_condition.py:147-152; unet_3d_blocks.py:331-340) without its permutes.
 * Token t of sequence z lives in ROW (z / inner) * outer_rows + (z % inner) * inner_rows + t * seq_rows of a token matrix;
 * q/k/v (and dq/dk/dv) have row pitch ld_in (so they may be column slices of one fused [rows][3C] QKV projection),
 * o / dout have row pitch ld_out; head h occupies columns h*D .. h*D+D-1 of each pointer.                                 */
int t2v_attn_small_fwd(const void* q, const void* k, const void* v, void* o, int64_t nseq, int32_t inner, int64_t outer_rows,
                       int64_t inner_rows, int64_t seq_rows, int64_t ld_in, int64_t ld_out, int32_t heads, int32_t L, int32_t D,
                       void* stream);
int t2v_attn_small_bwd(const void* q, const void* k, const void* v, const void* dout, void* dq, void* dk, void* dv, int64_t nseq,
                       int32_t inner, int64_t outer_rows, int64_t inner_rows, int64_t seq_rows, int64_t ld_in, int64_t ld_out,
                       int32_t heads, int32_t L, int32_t D, void* stream);
/* The same attention for 1 <= L <= 256 (clips longer than 32 frames), one CTA per (sequence, head), same addressing and
 * head_dim.  The forward also writes lse: fp32 [nseq][heads][L], the natural-log logsumexp of each row of scaled scores.
 * The backward reads lse and the forward's o (delta = rowsum(dout * o)); it is one pass without atomics and deterministic.  */
int t2v_attn_long_fwd(const void* q, const void* k, const void* v, void* o, float* lse, int64_t nseq, int32_t inner, int64_t outer_rows,
                      int64_t inner_rows, int64_t seq_rows, int64_t ld_in, int64_t ld_out, int32_t heads, int32_t L, int32_t D,
                      void* stream);
int t2v_attn_long_bwd(const void* q, const void* k, const void* v, const void* o, const void* dout, const float* lse, void* dq, void* dk,
                      void* dv, int64_t nseq, int32_t inner, int64_t outer_rows, int64_t inner_rows, int64_t seq_rows, int64_t ld_in,
                      int64_t ld_out, int32_t heads, int32_t L, int32_t D, void* stream);

/* Fused AdamW + global-norm clipping on the flat arena (torch.optim.AdamW semantics; reference train.py:616-623, clipping
 * :868-876).  The trainable set is a chunk table of int64 (offset, length) pairs into the flat fp32 buffers (multiples of 64
 * elements).  All step-dependent scalars live in device memory so the three launches can be captured in a CUDA graph:
 *   t2v_sqnorm_chunks   *out += sum g^2 over the chunks (fp64)
 *   t2v_adamw_prepare   state[0] (int64 step count) += 1; for each of n_sets hyper-parameter rows hp_in[s] = (lr, beta1, beta2,
 *                       eps, weight_decay) writes hp[s] = (.., bias_c1, sqrt(bias_c2), clip factor); the clip factor is
 *                       min(1, max_norm / (sqrt(sq[0]) + 1e-6)) (1 when max_norm <= 0); sq[1] = norm, sq[0] = 0
 *   t2v_adamw_chunks    updates p, m, v from g * clip, writes the bf16 compute copy of p for offsets < n_shadow (shadow may be
 *                       NULL) and zeroes g when zero_grad != 0.  hp points at ONE 8-float row.
 * g_bf16 (sqnorm, adamw_chunks; may be NULL): flat bf16 buffer with the same offsets as g - when given, the gradient VALUES are
 * read from it (the all-reduced, averaged gradient of a data-parallel step) and the fp32 buffer g is only zeroed.        */
int t2v_sqnorm_chunks(const float* g, const void* g_bf16, const int64_t* chunks, int32_t n_chunks, double* out, void* stream);
int t2v_adamw_prepare(const float* hp_in, float* hp, int32_t n_sets, int64_t* state, double* sq, float max_norm, void* stream);
int t2v_adamw_chunks(float* p, float* g, const void* g_bf16, float* m, float* v, void* shadow_bf16, int64_t n_shadow, const int64_t* chunks,
                     int32_t n_chunks, const float* hp, int32_t zero_grad, void* stream);

/* Blockwise 8-bit AdamW (optim.AdamW8bit): the same update, with the moments of large tensors kept as uint8 codes into two
 * 256-entry maps (qmaps[0..255] signed for m, qmaps[256..511] unsigned for v) times one fp32 absmax per 256-element block.
 * chunks: n_chunks int64 rows (arena offset, length, state offset, bits), each inside one tensor and at most 64 K elements.
 *   bits 32: m32 / v32 (fp32) at the state offset, exactly t2v_adamw_chunks' update.
 *   bits 8:  code_m / code_v (uint8) at the state offset (a multiple of 256), absmax_m / absmax_v at state offset / 256; the
 *            length is a multiple of 256 except in a tensor's last row (a multiple of 64).  Per element: dequantise
 *            (map[code] * absmax), update as t2v_adamw_chunks with the fp32 moments, then per block absmax = max |moment| and
 *            code = the smallest i with moment / absmax <= 0.5f * (map[i] + map[i+1]); a block whose absmax is 0 stores the
 *            code of 0.0.
 * hp, g_bf16, shadow_bf16, n_shadow and zero_grad as for t2v_adamw_chunks.                                                */
int t2v_adamw8bit_chunks(float* p, float* g, const void* g_bf16, void* shadow_bf16, int64_t n_shadow, const int64_t* chunks, int32_t n_chunks,
                         const float* hp, const float* qmaps, float* m32, float* v32, void* code_m, void* code_v, float* absmax_m,
                         float* absmax_v, int32_t zero_grad, void* stream);

/* Exponential moving average of the trained weights (`use_ema`; diffusers' EMAModel with its default arguments), updated in
 * the same pass as the weights.  k = *step, the step count after t2v_adamw_prepare's increment, read on the device so that a
 * replayed CUDA graph uses each step's decay: d = 0 for k = 1, else min(ema_decay, k / (9 + k)) (fp64); then per element
 * ema -= (1 - d) * (ema - p_new), with 1 - d rounded to fp32 and each operation rounded on its own.  ema (fp32, 16-byte
 * aligned) is compact: the EMA offset column of each row says where its elements start.  ema_decay must lie in [0, 1].
 *   t2v_adamw_ema_chunks      t2v_adamw_chunks with rows (arena offset, length, EMA offset)
 *   t2v_adamw8bit_ema_chunks  t2v_adamw8bit_chunks with rows (arena offset, length, state offset, bits, EMA offset); both the
 *                             32-bit and the 8-bit rows update the fp32 EMA
 *   t2v_ema_swap_chunks       exchanges p and ema over n_rows rows (arena offset, length, EMA offset) and rewrites the bf16
 *                             copy of p for offsets < n_shadow as the update kernels round it; a second call restores all
 *                             three bit for bit                                                                          */
int t2v_adamw_ema_chunks(float* p, float* g, const void* g_bf16, float* m, float* v, void* shadow_bf16, int64_t n_shadow, const int64_t* chunks,
                         int32_t n_chunks, const float* hp, int32_t zero_grad, float* ema, const int64_t* step, float ema_decay, void* stream);
int t2v_adamw8bit_ema_chunks(float* p, float* g, const void* g_bf16, void* shadow_bf16, int64_t n_shadow, const int64_t* chunks, int32_t n_chunks,
                             const float* hp, const float* qmaps, float* m32, float* v32, void* code_m, void* code_v, float* absmax_m,
                             float* absmax_v, int32_t zero_grad, float* ema, const int64_t* step, float ema_decay, void* stream);
int t2v_ema_swap_chunks(float* p, float* ema, void* shadow_bf16, int64_t n_shadow, const int64_t* rows, int32_t n_rows, void* stream);

/* Stable (loralib-style) LoRA on a convolution: W_eff = W + scaling * view(B @ A), A [r*k][Cin*k], B [Cout*k][r*k] fp32
 * row-major (stable_lora/lora.py Conv2d / Conv3d forward).  With f = ((o*Cin + c)*k + kh)*k + kw the logical (o, c, kh, kw)
 * element of the Conv2d view is BA[f / (Cin*k)][f % (Cin*k)]; the Conv3d (3,1,1) view (k = 3) is the mean of the three
 * consecutive BA columns f = ((o*Cin + c)*3 + t)*3 + 0..2.  Weights are in the physical layout [Cout][KH][KW][Cin] ([Cout][3][1][Cin]).
 *   t2v_lora_delta_merge  out_bf16 = bf16(base + scaling * view(B @ A)): the fp32 base is added before the single rounding.
 *   t2v_lora_delta_grad   dBA = scaling * view^T(dw) (Conv3d: dw / 3 on each averaged column), then dB += dBA A^T and
 *                         dA += B^T dBA (fp32, red.add, so not bitwise reproducible); dw is read once.
 * k must be 1 or 3 (Conv2d) or 3 (conv3d != 0); 1 <= r <= 256.                                                             */
int t2v_lora_delta_merge(const float* base, const float* A, const float* B, float scaling, int32_t k, int32_t conv3d, int32_t cout,
                         int32_t cin, int32_t r, void* out_bf16, void* stream);
int t2v_lora_delta_grad(const float* dw, const float* A, const float* B, float scaling, int32_t k, int32_t conv3d, int32_t cout,
                        int32_t cin, int32_t r, float* dA, float* dB, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* T2V_B200_H_ */
