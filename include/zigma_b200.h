/*
 * zigma_b200 -- C-ABI of the H100 (sm_90a) kernels for the ZigMa denoiser hot path.
 *
 * This header is the drop-in boundary.  Every entry point replaces one native interface of the
 * reference (CompVis/zigma, paths relative to /root/reference):
 *
 *   zg_selective_scan_fwd   <- selective_scan_cuda.fwd   dis_mamba/csrc/selective_scan/selective_scan.cpp:226-336
 *   zg_selective_scan_bwd   <- selective_scan_cuda.bwd   dis_mamba/csrc/selective_scan/selective_scan.cpp:338-492
 *   zg_causal_conv1d_fwd    <- causal_conv1d_cuda.causal_conv1d_fwd   dis_causal_conv1d/csrc/causal_conv1d.cpp:130-189
 *   zg_causal_conv1d_bwd    <- causal_conv1d_cuda.causal_conv1d_bwd   dis_causal_conv1d/csrc/causal_conv1d.cpp:191-268
 *   zg_add_norm_fwd         <- Triton _layer_norm_fwd_1pass_kernel    dis_mamba/mamba_ssm/ops/triton/layernorm.py:64-177
 *   zg_add_norm_bwd         <- Triton _layer_norm_bwd_kernel          dis_mamba/mamba_ssm/ops/triton/layernorm.py:195-377
 *   zg_block_tail_fwd       <- the unfused elementwise tail of Block.forward + next block's fused add+norm
 *                              model_zigma.py:416-445 (gate * mixer + x, residual add, RMSNorm, modulate)
 *                              and backward_permutation  mamba_simple.py:59-61,388-394
 *   zg_gemm_bf16_tn         <- the cuBLAS calls behind in_proj / x_proj / dt_proj / out_proj
 *                              mamba_simple.py:290-294, selective_scan_interface.py:322-323,365
 *
 * Conventions
 *   - plain pointers and sizes only; all pointers are DEVICE pointers unless stated otherwise;
 *   - the caller allocates every output (the reference allocates inside the op with the caller's
 *     allocator, selective_scan.cpp:304-313 -- here Python/torch allocates, the kernels fill);
 *   - strides are in ELEMENTS;
 *   - all launches are asynchronous on `stream` (a cudaStream_t passed as void*); no allocation,
 *     no synchronisation inside -> CUDA-graph capturable;
 *   - return value 0 = success; non-zero = error, message via zg_last_error() (thread local).
 *     The Python wrapper turns that into RuntimeError like TORCH_CHECK does in the reference.
 */
#ifndef ZIGMA_B200_H
#define ZIGMA_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum { ZG_F32 = 0, ZG_F16 = 1, ZG_BF16 = 2 };

/* flags for zg_scan_params.flags */
enum {
    ZG_SCAN_DELTA_SOFTPLUS = 1,  /* delta' = softplus(delta + bias), identity above 20 */
    ZG_SCAN_VARIABLE_B = 2,      /* B is (batch, groups, dstate, seqlen) in act dtype; else (dim, dstate) fp32 */
    ZG_SCAN_VARIABLE_C = 4,
    /* output placement of the hot-path kernel (dim-contiguous 16-bit activations, dstate 16, seqlen % 8 == 0, dim % 64 == 0;
     * other calls return an error): the two sweeps of scan_type "v2" (mamba_simple.py:304-339: y = y_fwd + y_bwd.flip(-1))
     * without materialising the flipped tensor or a separate add --
     *   OUT_REVERSE     step l is written to sequence position seqlen - 1 - l;
     *   OUT_ACCUMULATE  out = round(out + round(y)) in the I/O dtype, i.e. the eager `a + b` of two 16-bit tensors. */
    ZG_SCAN_OUT_REVERSE = 8,
    ZG_SCAN_OUT_ACCUMULATE = 16
};

int zg_abi_version(void);
const char *zg_last_error(void);
/* number of kernels launched through this library since load (bench `gpu_launches` evidence) */
uint64_t zg_launch_count(void);
/* name of the kernel the most recent zg_selective_scan_fwd call launched ("" before the first call): bench / profile labels */
const char *zg_last_scan_kernel(void);
/* The shape rule behind that choice (host arithmetic only, no GPU needed): which hot-path forward kernel runs a call of
 * units16 = batch * dim / 16 sixteen-channel units on a device with `sms` SMs -- 0 the CTA-wide kernel, 3 the 32-channel-per-warp
 * pipeline, 5 CTAs of *nd wide + *ns narrow warps.  All kernels produce identical bits (DESIGN.md section 4.1). */
int zg_scan_kernel_choice(int64_t units16, int32_t sms, int32_t training_forward, int32_t *nd, int32_t *ns);

/* ---------------------------------------------------------------------------------------------
 * Selective scan (S6).  Logical shapes: u, delta, z, out (batch, dim, seqlen); any of the two
 * layouts is accepted through the strides, but ONE of {seq stride, dim stride} must be 1 for all
 * four tensors alike:
 *     seq-contiguous ("channel first", the reference layout, selective_scan.cpp:252-253)  *_sl == 1
 *     dim-contiguous ("token major", what the fused model path uses)                      *_sd == 1
 * B/C variable: (batch, groups, dstate, seqlen) with the SAME contiguity class (seq stride 1 for
 * seq-contiguous activations, dstate stride 1 for dim-contiguous activations).
 * A (dim, dstate) fp32 contiguous, real only (complex64 A of the reference is not supported: ZigMa
 * never uses it).  D, delta_bias (dim) fp32 or NULL.  z NULL -> out = y, else out = y * silu(z).
 * z_rowmap (int32[seqlen], NULL = identity): step l reads z at sequence position z_rowmap[l]
 *   (fuses forward_permutation of the z half, mamba_simple.py:55-56,365-370; dim-contiguous only).
 * last_state (batch, dim, dstate) fp32 or NULL.
 * ckpt (batch, n_ckpt, dim, dstate) fp32 or NULL: state after every ckpt_every steps
 *   (n_ckpt = ceil(seqlen / ckpt_every); ckpt_every must be a multiple of 8; the backward needs 8) -- the recompute
 *   seeds of the backward pass; plays the role of the reference's `x` (selective_scan.cpp:313).
 * dstate <= 64.
 *
 * Fused dt_proj prologue (optional; replaces the separate `delta = dt_proj.weight @ x_dbl[:, :R].t()` GEMM of
 * selective_scan_interface.py:323 / mamba_simple.py:372-380 and the (batch, dim, seqlen) delta round trip through HBM):
 * with dt_w != NULL, `delta` is ignored (may be NULL) and the kernel computes, per step,
 *     delta[b, :, l] = round_to_io_dtype( dt_w (dim, dt_rank) . dt_x[b, l, 0:dt_rank] )      (fp32 accumulate, tensor cores)
 * before adding delta_bias / softplus, i.e. with the rounding point of the reference's 16-bit GEMM output.
 * Requirements (else an error is returned): dim-contiguous layout, 16-bit I/O, variable B and C with dstate 16 that live in
 * the SAME rows as the dt input (B == dt_x + dt_rank, C == dt_x + dt_rank + 16, i.e. the x_dbl rows of x_proj), dt_rank in
 * {8, 16, ..., 64}, seqlen % 8 == 0, (dim / groups) % 64 == 0, 16-byte aligned rows.  dt_w is in the I/O dtype, row stride
 * dt_w_ld elements.
 */
typedef struct {
    const void *u, *delta, *z, *B, *C;
    const float *A, *D, *delta_bias;
    const int32_t *z_rowmap;
    void *out;
    float *last_state, *ckpt;
    int64_t u_sb, u_sd, u_sl;
    int64_t delta_sb, delta_sd, delta_sl;
    int64_t z_sb, z_sd, z_sl;
    int64_t out_sb, out_sd, out_sl;
    int64_t B_sb, B_sg, B_sn, B_sl;
    int64_t C_sb, C_sg, C_sn, C_sl;
    int32_t batch, dim, seqlen, dstate, ngroups;
    int32_t dtype, flags, ckpt_every;
    const void *dt_w, *dt_x;          /* fused dt_proj prologue: weight (dim, dt_rank), input rows (batch, seqlen, >= dt_rank) */
    int64_t dt_w_ld, dt_x_sb, dt_x_sl;
    int32_t dt_rank;
    /* two-level batch for z (hot-path kernel with z_rowmap only): z_batch_inner = K > 0 addresses batch element b of the call
     * at  z + (b / K) z_sb + (b % K) z_sbi  -- the (b k) t sequences of the temporal video scan read their gate rows out of the
     * (b, t k) token-major xz tensor (z_sl = K rows) without a permuted copy. */
    int32_t z_batch_inner;
    int64_t z_sbi;
} zg_scan_params;

int zg_selective_scan_fwd(const zg_scan_params *p, void *stream);

/* Backward of the above.  Extra inputs: dout (like out), ckpt from the forward.  Outputs: du,
 * ddelta (like u), dz (like z, NULL if no z), dA (dim, dstate), dD, ddelta_bias (dim) fp32
 * ACCUMULATED with atomics -> caller zero-fills (reference: selective_scan.cpp:460-466),
 * dB, dC (batch, groups, dstate, seqlen) fp32 accumulated likewise.  Both layouts (like the forward); z_rowmap redirects
 * the z reads and the dz writes.  The fused dt_proj fields of `fwd` must be NULL/0 (the backward takes delta explicitly).
 */
typedef struct {
    zg_scan_params fwd;
    const void *dout;
    int64_t dout_sb, dout_sd, dout_sl;
    void *du, *ddelta, *dz;
    int64_t du_sb, du_sd, du_sl;
    int64_t ddelta_sb, ddelta_sd, ddelta_sl;
    int64_t dz_sb, dz_sd, dz_sl;
    float *dA, *dD, *ddelta_bias, *dB, *dC;
} zg_scan_bwd_params;

int zg_selective_scan_bwd(const zg_scan_bwd_params *p, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Depthwise causal conv1d (+bias, +SiLU).  x, out logical (batch, dim, seqlen), either layout (the
 * reference's channel-first and channel-last kernels, causal_conv1d_fwd.cu:39-158,193-330).
 * weight (dim, width) and bias (dim) in weight dtype `wdtype`; 2 <= width <= 4 (causal_conv1d.cpp:157).
 * x_rowmap (int32[seqlen] or NULL; dim-contiguous only): output position l convolves the input
 *   positions x_rowmap[l-w], i.e. the conv runs over the PERMUTED sequence without materialising
 *   it (fuses forward_permutation of the x half, mamba_simple.py:365-370).
 */
typedef struct {
    const void *x, *weight, *bias;
    const int32_t *x_rowmap;
    void *out;
    int64_t x_sb, x_sd, x_sl;
    int64_t out_sb, out_sd, out_sl;
    int32_t batch, dim, seqlen, width;
    int32_t dtype, wdtype, silu;
    /* seg_len > 0 (forward, 16-bit dim-contiguous fast path only; a multiple of 8 dividing seqlen): the sequence is a
     * concatenation of independent segments of that length -- the taps never reach across a segment start.  With x_rowmap
     * this convolves the (b k) t sequences of the factorised temporal video scan (mamba_simple.py:416-442) straight out of
     * the (b, t k) token-major activations: x_rowmap[k T + t] = perm[t] K + k, seg_len = T. */
    int32_t seg_len;
} zg_conv_params;

int zg_causal_conv1d_fwd(const zg_conv_params *p, void *stream);

/* Backward: dx (like x, written), dweight (dim, width) / dbias (dim) fp32 accumulated with atomics
 * (caller zero-fills; reference causal_conv1d.cpp:247-249, causal_conv1d_bwd.cu:225-239). */
typedef struct {
    zg_conv_params fwd;
    const void *dout;
    int64_t dout_sb, dout_sd, dout_sl;
    void *dx;
    int64_t dx_sb, dx_sd, dx_sl;
    float *dweight, *dbias;
} zg_conv_bwd_params;

int zg_causal_conv1d_bwd(const zg_conv_bwd_params *p, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Fused residual-add + RMSNorm / LayerNorm over rows of length ncols (rows contiguous in the last
 * dim, row strides in elements).   r = x (+ residual) in fp32;  residual_out = r  (dtype
 * res_dtype, NULL to skip);  y = norm(r) * weight (+ bias)  in dtype `dtype`;  rstd (and mean for
 * LayerNorm) saved when non-NULL.  weight/bias have dtype wdtype (NULL weight = 1).
 */
typedef struct {
    const void *x, *residual, *weight, *bias;
    void *y, *residual_out;
    float *mean, *rstd;
    int64_t x_rs, res_rs, y_rs, resout_rs;
    int32_t nrows, ncols;
    int32_t dtype, res_dtype, wdtype, is_rms;
    float eps;
} zg_norm_params;

int zg_add_norm_fwd(const zg_norm_params *p, void *stream);

typedef struct {
    const void *dy, *dresidual;   /* dresidual: grad wrt residual_out (res dtype) or NULL */
    const void *x;                /* the saved residual_out = r (res dtype)               */
    const void *weight;
    const float *mean, *rstd;
    void *dx, *dresidual_in;      /* dx in dtype; dresidual_in (res dtype) or NULL        */
    float *dweight, *dbias;       /* (ncols) fp32 accumulated with atomics, caller zero-fills */
    int64_t dy_rs, dres_rs, x_rs, dx_rs, dresin_rs;
    int32_t nrows, ncols;
    int32_t dtype, res_dtype, wdtype, is_rms;
} zg_norm_bwd_params;

int zg_add_norm_bwd(const zg_norm_bwd_params *p, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Block tail (inference fast path), token-major (batch, seqlen, dim) contiguous tensors:
 *     hidden   = x + gate[b,:] * mix[b, rowmap[l], :]          (rowmap = perm_rev or NULL)
 *     r        = residual + hidden              (fp32, written to residual_out)
 *     normed   = r * rsqrt(mean(r^2) + eps) * norm_w            (dtype; the next block's x)
 *     modded   = normed * (1 + scale[b,:]) + shift[b,:]         (dtype; the next in_proj input)
 * gate/shift/scale are (batch, dim) with row stride mod_rs (views into adaLN's (batch, 3*dim)).
 * Alignment (here and in the backward): row tensors 16 bytes; gate/shift/scale/norm_w 4 elements (8 bytes for 16-bit
 * dtypes, 16 for fp32) with mod_rs % 4 == 0.
 * With final != 0 the last two lines become the model tail (model_zigma.py:971-984,335):
 *     normed = LayerNorm_noaffine(normed, eps=1e-6) and modded is not written.
 * Intermediate roundings replicate the reference's unfused bf16 path: hidden and normed are
 * rounded to `dtype` where the reference materialises them.
 */
typedef struct {
    const void *x, *mix, *gate, *shift, *scale, *norm_w;
    const float *residual;
    const int32_t *rowmap;
    float *residual_out;
    void *normed, *modded;
    int64_t mod_rs;
    int32_t batch, seqlen, dim;
    int32_t dtype, final_layer;
    float eps;
    float *rstd;                  /* (batch * seqlen) fp32 or NULL: 1 / sqrt(mean(r^2) + eps), saved for the backward */
} zg_block_tail_params;

int zg_block_tail_fwd(const zg_block_tail_params *p, void *stream);

/* The FIRST tail of a forward with the positional embedding folded in: `mix` is ONE (seqlen, dim) table shared by every
 * batch element, gate / rowmap / residual are NULL:
 *     hidden = round_to_dtype(x + mix[l, :])        -- the reference's `x = x + self.pos_embed` (model_zigma.py:941)
 * then r = hidden, normed, modded as above.  Saves the elementwise pass over (batch, seqlen, dim) that the add costs as a
 * kernel of its own.  dim <= 2048. */
int zg_block_tail_fwd_pe(const zg_block_tail_params *p, void *stream);

/* Backward of the block tail (training).  With the forward's
 *     hidden = x + gate * mix[rowmap];  r = residual + hidden;  normed = r * rstd * norm_w;  modded = normed * (1 + scale) + shift
 * and incoming gradients d_residual_out (fp32), d_normed, d_modded (dtype; any of them may be NULL = zero):
 *     dy      = d_normed + d_modded * (1 + scale)          dshift[b] += sum_l d_modded      dscale[b] += sum_l d_modded * normed
 *     dr      = rmsnorm_bwd(dy; r, rstd, norm_w) + d_residual_out                           d_norm_w  += sum dy * r * rstd
 *     d_residual_in = dr (fp32);   dh = round_to_dtype(dr);   d_x = dh
 *     d_mix[rowmap[l]] = gate * dh[l]                       dgate[b] += sum_l dh[l] * mix[rowmap[l]]
 * r = the forward's residual_out, rstd its rstd.  dgate / dshift / dscale are (batch, dim) fp32 accumulated with atomics
 * (caller zero-fills).  d_norm_w is a PARTIALS buffer (nparts, dim) fp32: the kernel runs nparts persistent CTAs and CTA i
 * stores its column sums in row i (no atomics; the caller adds the rows up; nparts ~ 3 per SM is a good choice).  mix / gate / d_mix / dgate NULL together for the first block;
 * d_residual_in NULL when the forward had no residual input.  Replaces, in the reference's training graph, the backward
 * of _layer_norm_fwd/_bwd (layernorm.py:195-290) plus the autograd nodes of modulate and the gated residual add
 * (model_zigma.py:416-445). */
typedef struct {
    const float *d_residual_out;
    const void *d_normed, *d_modded;
    const float *r, *rstd;
    const void *mix, *gate, *scale, *norm_w;
    const int32_t *rowmap;
    void *d_x, *d_mix;
    float *d_residual_in, *dgate, *dshift, *dscale, *d_norm_w;
    int64_t mod_rs;
    int32_t batch, seqlen, dim, dtype, nparts;
} zg_block_tail_bwd_params;

int zg_block_tail_bwd(const zg_block_tail_bwd_params *p, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Deterministic backward (bitwise-identical outputs for bitwise-identical inputs on the same device and build, whatever
 * order the CTAs run in; the Python layer calls these while torch.are_deterministic_algorithms_enabled()).
 * Same params struct, outputs and zero-fill contract as the atomic twin above; the kernels are the same code compiled
 * with every fp32 atomicAdd of a gradient reduction turned into a plain store into the value's own row of a partials
 * workspace (the row follows from the static grid mapping: channel tile, warp, batch row or chunk index), and one
 * reduction kernel then adds the rows into the outputs in row order (DESIGN.md section 4.6).
 *   workspace:  device memory of at least zg_*_bwd_det_workspace_bytes(p) bytes, 16-byte aligned, no initial contents
 *               needed; it must stay untouched until the call's work on `stream` is done.  A smaller workspace returns an
 *               error (nothing is launched).
 *   *_workspace_bytes: host arithmetic only (no GPU needed, no CUDA call), evaluated on the SAME params as the call: it
 *               follows the kernel dispatch (dstate-16 vs generic scan kernel, token-major vs channel-first conv,
 *               vectorised vs scalar norm, ...) and counts only the outputs that are not NULL.
 * No allocation and no synchronisation inside: CUDA-graph capturable like the rest of the ABI.  The partial rows of
 * zg_add_norm_bwd_det (one per CTA or warp, at most 528 CTAs) do not depend on the device; those of
 * zg_block_tail_bwd_det follow p->nparts, so equal bits across devices need equal nparts.
 * zg_block_tail_bwd_det additionally needs 4 * nparts >= batch (each warp stays inside one batch element). */
int64_t zg_selective_scan_bwd_det_workspace_bytes(const zg_scan_bwd_params *p);
int zg_selective_scan_bwd_det(const zg_scan_bwd_params *p, void *workspace, int64_t workspace_bytes, void *stream);
int64_t zg_causal_conv1d_bwd_det_workspace_bytes(const zg_conv_bwd_params *p);
int zg_causal_conv1d_bwd_det(const zg_conv_bwd_params *p, void *workspace, int64_t workspace_bytes, void *stream);
int64_t zg_add_norm_bwd_det_workspace_bytes(const zg_norm_bwd_params *p);
int zg_add_norm_bwd_det(const zg_norm_bwd_params *p, void *workspace, int64_t workspace_bytes, void *stream);
int64_t zg_block_tail_bwd_det_workspace_bytes(const zg_block_tail_bwd_params *p);
int zg_block_tail_bwd_det(const zg_block_tail_bwd_params *p, void *workspace, int64_t workspace_bytes, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Block tail with stochastic depth (training with drop_path_rate > 0; model_zigma.py:138-160,416-438).  The reference's
 * Block applies its DropPath to the previous block's hidden before the fused add+norm: with s[b] the multiplier it drew
 * for batch element b (0 or round_to_dtype(1 / keep), a tensor value, never recomputed here):
 *     hidden   = round(x + round(gate * mix[rowmap]))           (as zg_block_tail_fwd)
 *     kept     = round(hidden * s[b])                           (new: the eager `x * mask`, rounded before the add)
 *     r        = residual + kept            (fp32, residual_out)
 *     normed, modded, rstd                                      (as zg_block_tail_fwd)
 * and in the backward, with dr = rmsnorm_bwd(...) + d_residual_out as in zg_block_tail_bwd:
 *     d_residual_in = dr                                        (the multiplier is not on the residual path)
 *     dh = round(round(dr) * s[b]);   d_x = dh;   d_mix[rowmap[l]] = round(gate * dh[l]);   dgate[b] += sum_l dh[l] * mix[rowmap[l]]
 *     dshift, dscale, d_norm_w                                  (as zg_block_tail_bwd: they do not see the multiplier)
 * With s == 1 the results equal the plain entry points' bit for bit; with s[b] == 0 the d_x, d_mix rows and the dgate row
 * of b are zero.
 *   path_scale: (batch) in `dtype`, aligned to its element size, read once per token row.
 * Everything the plain entry points take and check applies, plus: path_scale, residual (forward) and mix non-NULL (the first
 * block has no residual and so no drop path), final_layer == 0 and dim <= 1024.  The forward runs the four-warps-per-row
 * kernel; the backward has the plain one's grid, nparts contract and, for the _det twin, the same workspace
 * (zg_block_tail_bwd_dp_det_workspace_bytes returns what zg_block_tail_bwd_det_workspace_bytes returns for `base`). */
typedef struct {
    zg_block_tail_params base;
    const void *path_scale;
} zg_block_tail_dp_params;

typedef struct {
    zg_block_tail_bwd_params base;
    const void *path_scale;
} zg_block_tail_bwd_dp_params;

int zg_block_tail_fwd_dp(const zg_block_tail_dp_params *p, void *stream);

/* Block tail whose x is the previous tail's normed output, rebuilt instead of read: with r_prev = this call's residual (the previous
 * tail's residual_out), rstd_prev and w_prev the previous tail's rstd and norm_w,
 *     x = round_to_dtype(r_prev * rstd_prev[row] * w_prev)      -- the previous tail's normed, bit for bit
 * then everything as zg_block_tail_fwd.  So a chain of tails needs no normed tensor between them: each passes its rstd on, and
 * writes normed only where something else reads it.  Saves a (batch, seqlen, dim) write and read per tail.
 *   base.x: NULL.  base.residual: required.  base.normed: may be NULL unless final_layer.  dim <= 1024.
 *   x_rstd: (batch * seqlen) fp32, 4-byte aligned.  x_norm_w: (dim) in dtype, aligned to 4 elements. */
typedef struct {
    zg_block_tail_params base;
    const float *x_rstd;
    const void *x_norm_w;
} zg_block_tail_rebuild_params;

int zg_block_tail_fwd_rebuild(const zg_block_tail_rebuild_params *p, void *stream);
int zg_block_tail_bwd_dp(const zg_block_tail_bwd_dp_params *p, void *stream);
int64_t zg_block_tail_bwd_dp_det_workspace_bytes(const zg_block_tail_bwd_dp_params *p);
int zg_block_tail_bwd_dp_det(const zg_block_tail_bwd_dp_params *p, void *workspace, int64_t workspace_bytes, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Text cross-attention of has_text blocks (model_zigma.py:95-135; DESIGN.md section 4.7), per (batch, head):
 *     O = softmax(Q K^T * 0.125) V          head dimension 64, no mask, no dropout
 * Q, O (batch, L, dim) and K, V (batch, Lk, dim) token-major, dim = heads * 64, head h in columns [64 h, 64 h + 64) of
 * every row; columns contiguous, rows and batches at the given strides (elements).  1 <= Lk <= 256; any heads >= 1;
 * dtype fp32, fp16 or bf16 for all four.  lse (batch, heads, L) fp32 contiguous, or NULL: the natural-log log-sum-exp
 * log(sum_j exp(0.125 q.k_j)) of each row, written by the forward, read by the backward.
 * Alignment: q, k, v, o (and dout, dq, dk, dv of the backward) 16-byte aligned, with batch and row strides whole multiples
 * of 16 bytes (8 elements for 16-bit dtypes, 4 for fp32): column slices of a fused (rows, 3 dim) buffer qualify.
 * Errors (nothing launched): Lk outside [1, 256], dim not a multiple of 64 or != 64 heads, a misaligned pointer or stride,
 * a workspace too small.  batch == 0 or L == 0 passes the checks and launches nothing.
 * Roundings: 16-bit -- S = Q K^T and O = P V accumulate in fp32 on the tensor cores, P is rounded to the I/O dtype as the
 * A operand of P V, O divided by the fp32 row sum once and rounded once at the store; fp32 -- CUDA cores, same formula.
 */
typedef struct {
    const void *q, *k, *v;
    void *o;
    float *lse;
    int64_t q_sb, q_rs, k_sb, k_rs, v_sb, v_rs, o_sb, o_rs;
    int32_t batch, L, Lk, heads, dim, dtype;
} zg_xattn_params;

int zg_cross_attn_fwd(const zg_xattn_params *p, void *stream);

/* Backward: inputs dout (like o), fwd.q / k / v, fwd.o (the forward's output) and fwd.lse; outputs dq (like q), dk, dv
 * (like k, v), all written (no zero-fill needed).  P is recomputed from lse, D_i = sum dout_i o_i, dS = P (dout V^T - D),
 * dq = 0.125 dS K, dk = 0.125 dS^T Q, dv = P^T dout, in fp32, rounded once at the store.  No floating-point atomics: the
 * dk / dv sums over the L query rows are taken per segment of whole 64-row query tiles into the workspace, then added in
 * segment order, so the result is bitwise reproducible whatever the CTA order (and whatever torch's deterministic flag).
 * sms (>= 1) is the SM count of the device; it fixes the segment count:
 *     tiles = ceil(L / 64),  ctas = batch * heads * ceil(Lk / 32),  n = min(tiles, ceil(8 sms / ctas)),
 *     per = ceil(tiles / n),  nseg = ceil(tiles / per)          (segments of per * 64 query rows)
 * workspace: at least zg_cross_attn_bwd_workspace_bytes(p) bytes, 16-byte aligned, no initial contents needed:
 *     roundup16(4 batch heads L) + 2 * 4 * nseg * batch * heads * Lk * 64        (0 when batch, L or heads is 0)
 * (D per row, then the fp32 dk and dv partials per segment).  Equal bits across devices need equal sms.
 * zg_cross_attn_bwd_workspace_bytes is host arithmetic only.  batch * heads <= 65535. */
typedef struct {
    zg_xattn_params fwd;
    const void *dout;
    void *dq, *dk, *dv;
    int64_t dout_sb, dout_rs, dq_sb, dq_rs, dk_sb, dk_rs, dv_sb, dv_rs;
    int32_t sms;
} zg_xattn_bwd_params;

int64_t zg_cross_attn_bwd_workspace_bytes(const zg_xattn_bwd_params *p);
int zg_cross_attn_bwd(const zg_xattn_bwd_params *p, void *workspace, int64_t workspace_bytes, void *stream);

/* ---------------------------------------------------------------------------------------------
 * bf16 GEMM on the Hopper tensor cores (wgmma):  C[M,N] = A[M,K] * B[N,K]^T (+ bias[N]), fp32 accumulate in
 * registers, bf16 output.  A, B row-major with leading dims lda/ldb (elements, multiples of 8);
 * C row-major ldc.  out_rowmap (int32[rows_per_batch] or NULL): output row m of batch
 * m / rows_per_batch is stored at row out_rowmap[m % rows_per_batch] of that batch (scatter of
 * the out_proj result back to raster order, mamba_simple.py:388-394).
 * Any M, N, K >= 1 with lda/ldb/ldc multiples of 8 (remainders come from TMA zero fill / clipped stores); nothing of C outside
 * its M x N window is written, so C may be a window of a wider matrix.  The CUtensorMaps are built on the host per call and passed to the
 * kernel by value (__grid_constant__), so nothing has to outlive the call.
 */
typedef struct {
    const void *A, *B, *bias;
    void *C;
    const int32_t *out_rowmap;
    int64_t lda, ldb, ldc;
    int32_t M, N, K, rows_per_batch;
} zg_gemm_params;

int zg_gemm_bf16_tn(const zg_gemm_params *p, void *stream);
/* The kernel zg_gemm_bf16_tn launches for an M x N output (host arithmetic only, no GPU needed): tile width *bn (64, 80, 128, 160,
 * 256) and cluster size *cl (1, 2, 4), after the ZG_GEMM_BN / ZG_GEMM_CLUSTER overrides (read on every call) and the halving of
 * the cluster.  Returns 0, or nonzero for M or N < 1. */
int zg_gemm_kernel_choice(int32_t M, int32_t N, int32_t *bn, int32_t *cl);


/* ---------------------------------------------------------------------------------------------
 * Fused AdamW + EMA step over flat fp32 buffers of n elements (the optimiser / EMA part of the training
 * step around the path: train_acc.py:213-215,442-448, utils/train_utils.py:104-115 of the reference):
 *     g  = grad * grad_scale (* *grad_scale_ptr when given: a device scalar, e.g. a clip coefficient)
 *     p *= 1 - lr * weight_decay;   m = beta1 m + (1-beta1) g;   v = beta2 v + (1-beta2) g^2
 *     p -= lr / bias_correction1 * m / (sqrt(v) / sqrt(bias_correction2) + eps)
 *     ema = ema_decay * ema + (1 - ema_decay) * p            (ema may be NULL)
 * bias_correction{1,2} = 1 - beta{1,2}^step are computed by the caller.  grad is not modified.
 */
typedef struct {
    float *param, *exp_avg, *exp_avg_sq, *ema;
    const float *grad, *grad_scale_ptr;
    int64_t n;
    float lr, beta1, beta2, eps, weight_decay, bias_correction1, bias_correction2, ema_decay, grad_scale;
} zg_adamw_params;

int zg_adamw_ema_step(const zg_adamw_params *p, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Text prologue of a has_text block (model_zigma.py:206-208): what lies between the mixer and the cross-attention,
 *     hidden = x + gate * mixer_out;   q_in = modulate(norm_msa(hidden), shift_msa, scale_msa)
 * in one pass.  Token-major (batch, seqlen, dim) contiguous rows; round() = round to `dtype` (identity for fp32), at the
 * points the eager graph materialises a tensor:
 *     hidden = round(x + round(gate[b] * mix[b, rowmap[l]]))          (rowmap int32[seqlen] or NULL = identity)
 *     mean, rstd of the row of hidden in fp32:  rstd = 1 / sqrt(mean((hidden - mean)^2) + eps)   (norm_msa: eps 1e-6)
 *     ln     = round((hidden - mean) * rstd)                         (LayerNorm without affine)
 *     q_in   = round(round(ln * round(1 + scale[b])) + shift[b])
 * mean and rstd (batch * seqlen, fp32) are stored when non-NULL.  gate / shift / scale are (batch, dim) views with row
 * stride mod_rs.  dim % 4 == 0, dim <= 2048; alignment as the block tail's.  batch == 0 or seqlen == 0 passes the checks and
 * launches nothing.  One 128-thread CTA per token row (the four-warps-per-row layout of the block tail). */
typedef struct {
    const void *x, *mix, *gate, *shift, *scale;
    const int32_t *rowmap;
    void *hidden, *q_in;
    float *mean, *rstd;
    int64_t mod_rs;
    int32_t batch, seqlen, dim, dtype;
    float eps;
} zg_text_prologue_params;

int zg_text_prologue_fwd(const zg_text_prologue_params *p, void *stream);

/* Backward of the above.  Inputs d_hidden (the gradient reaching hidden from the next block's tail, NULL = zero) and d_q
 * (the gradient of q_in); hidden, mean and rstd from the forward; mix read through rowmap as in the forward:
 *     d_ln = round(d_q * round(1 + scale[b]))        dshift[b] += sum_l d_q        dscale[b] += sum_l d_q * ln
 *     g    = (d_ln - (xhat * mean(d_ln * xhat) + mean(d_ln))) * rstd       xhat = (hidden - mean) * rstd   (LayerNorm bwd)
 *     dh   = round(d_hidden + round(g));   d_x = dh
 *     d_mix[b, rowmap[l]] = round(gate[b] * dh[b, l])                        dgate[b] += sum_l dh[b, l] * mix[b, rowmap[l]]
 * dgate / dshift / dscale are (batch, dim) fp32 accumulated with atomics (caller zero-fills; any may be NULL).  The kernel
 * runs nparts persistent 128-thread CTAs (1 <= nparts <= 65535) with the partition of zg_block_tail_bwd.  dim % 4 == 0,
 * dim <= 1024.  The _det twin follows the deterministic contract above: one partial row per warp index within a batch
 * element, the workspace holds 4 * nparts / batch rows of batch * dim floats (each rounded up to 16 bytes) for every
 * non-NULL column sum, and it needs 4 * nparts >= batch. */
typedef struct {
    const void *d_hidden, *d_q;
    const void *hidden, *mix, *gate, *scale;
    const float *mean, *rstd;
    const int32_t *rowmap;
    void *d_x, *d_mix;
    float *dgate, *dshift, *dscale;
    int64_t mod_rs;
    int32_t batch, seqlen, dim, dtype, nparts;
} zg_text_prologue_bwd_params;

int zg_text_prologue_bwd(const zg_text_prologue_bwd_params *p, void *stream);
int64_t zg_text_prologue_bwd_det_workspace_bytes(const zg_text_prologue_bwd_params *p);
int zg_text_prologue_bwd_det(const zg_text_prologue_bwd_params *p, void *workspace, int64_t workspace_bytes, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* ZIGMA_B200_H */
