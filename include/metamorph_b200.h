/* metamorph_b200 — C ABI of the H100 (sm_90a) hot-path kernels.
 *
 * The reference (facebookresearch/metamorph) has NO native/FFI layer: its hot path is Python calling
 * third-party torch / transformers ops (SURVEY.md F1, F3). This header is therefore the boundary the
 * build introduces (SURVEY.md section 8b): plain C symbols in metamorph_b200/_C.so, bound with ctypes from
 * the Python classes that mirror the reference API. Each entry cites the reference call site it replaces.
 *
 * Conventions
 *   - every function returns 0 on success, <0 on failure (-1 bad argument, -2 CUDA error, -3 wrong arch);
 *     mm_last_error() returns a thread-local message. No exceptions cross the ABI.
 *   - the caller owns every buffer (including workspaces); kernels never allocate or free.
 *   - all work is enqueued asynchronously on the given cudaStream_t; device pointers only.
 *   - mm_ce_fwd_bwd / mm_cosine_loss (with loss_sum), mm_rmsnorm_bwd (with dw_accum) and mm_sumsq_bf16_accum use library-owned device
 *     scratch private to (device, stream), allocated on a stream's first such call: calls on one stream share it in
 *     stream order, calls on different streams never do. The first call on a stream must not be inside graph capture.
 *   - matrices are row-major bf16 unless stated; `ld*` are row pitches in elements.
 */
#ifndef METAMORPH_B200_H
#define METAMORPH_B200_H
#include <cuda_runtime_api.h>
#ifdef __cplusplus
extern "C" {
#endif

const char* mm_last_error(void);
int mm_abi_version(void);
int mm_check_device(void); /* 0 iff the current device is sm_90 (H100) */

/* Dense contraction on Hopper tensor cores (TMA -> 128B-swizzled smem -> wgmma.mma_async -> registers -> epilogue).
 * Replaces every nn.Linear / F.linear on the path: HF LlamaAttention q/k/v/o_proj (modeling_llama.py:262-288),
 * LlamaMLP (:182-183), lm_head (metamorph_llama.py:398), mm_projector (metamorph_arch.py:159), vision_head
 * (metamorph_llama.py:433), SigLIP projections / MLP / patch-embed (modeling_siglip.py:178-184,285-326) and,
 * with MN-major operands, their autograd dgrad/wgrad.
 *   a_mn_major=0: A is [M,K];  =1: A stored [K,M] (A^T is used).   b_mn_major=0: B is [N,K] (C = A B^T);
 *   =1: B stored [K,N] (C = A B).  epilogue: 0 store, 1 +bias, 2 +bias,GELU(erf), 3 +bias,GELU(tanh),
 *   4 +residual, 5 +bias+residual, 6 SwiGLU over [16 gate|16 up] interleaved columns (C is [M,N/2], aux gets
 *   the raw [M,N] gate|up), 7 SwiGLU backward fused into the down_proj dgrad (acc = d act; aux = gate|up [M,2N]
 *   overwritten with its gradient; C = recomputed act). out_f32: C is fp32. accumulate: C += result. force_bn: 0 auto, 128, 256. */
int mm_gemm_bf16(const void* A, const void* B, void* C, const void* bias, const void* resid, void* aux,
                 long long M, long long N, long long K, long long lda, long long ldb, long long ldc,
                 long long ldr, long long ld_aux, int a_mn_major, int b_mn_major, int epilogue, int out_f32,
                 int accumulate, float alpha, int force_bn, cudaStream_t stream);

/* LlamaRMSNorm (modeling_llama.py:53-67) forward / backward (dx = dres_in + grad; dw_accum fp32 += ...). */
int mm_rmsnorm_fwd(const void* x, const void* w, void* y, long long M, long long H, float eps, cudaStream_t s);
int mm_rmsnorm_bwd(const void* dy, const void* x, const void* w, const void* dres_in, void* dx, float* dw_accum,
                   long long M, long long H, float eps, cudaStream_t s);
/* SigLIP LayerNorm (modeling_siglip.py:348,357). */
int mm_layernorm_fwd(const void* x, const void* w, const void* b, void* y, long long M, long long H, float eps,
                     cudaStream_t s);
/* apply_rotary_pos_emb (modeling_llama.py:146-168), in place on the first n_rot_heads heads of each row. */
int mm_rope_inplace(void* qkv, const int* pos, const float* cos_t, const float* sin_t, long long M, long long ld,
                    int n_rot_heads, int head_dim, int backward, cudaStream_t s);

/* Elementwise pieces: SwiGLU backward (LlamaMLP), erf-GELU fwd/bwd (projector / vision head), bias gradient,
 * SigLIP patch im2col (Conv2d k=s=14, modeling_siglip.py:178), position-embedding add, grad-norm partials. */
int mm_swiglu_bwd(const void* gu, const void* dact, void* dgu, void* act, long long M, long long I, cudaStream_t s);
int mm_gelu_fwd(const void* z, void* a, long long n, cudaStream_t s);
int mm_gelu_bwd(const void* z, const void* da, void* dz, long long n, cudaStream_t s);
int mm_colsum_accum(const void* x, float* out, long long R, long long N, long long ld, cudaStream_t s);
int mm_im2col_patch14(const void* img, void* out, int n_img, int image_size, int ldp, cudaStream_t s);
int mm_add_pos_emb(void* x, const void* pos, long long R, int P, int H, cudaStream_t s);
/* *out += sum x^2 (two launches: per-block partials, then a fixed-order add, so the result is the same bits on every run). */
int mm_sumsq_bf16_accum(const void* x, float* out, long long n, cudaStream_t s);

/* Image/text token gather-interleave (metamorph_arch.py:272-399) and its backward.
 * row_map[r] >= 0: embed_tokens row; -1: zero (padding); <= -2: image feature row -(row_map[r]) - 2. */
int mm_interleave_gather(const void* embed, const void* img, const int* row_map, void* out, long long R, int H,
                         cudaStream_t s);
int mm_interleave_scatter(const void* dout, const int* row_map, void* dembed, void* dimg, long long R, int H,
                          cudaStream_t s);
int mm_gather_rows(const void* x, const int* idx, void* out, long long R, int H, cudaStream_t s);
int mm_scatter_add_rows(void* x, const int* idx, const void* g, long long R, int H, cudaStream_t s);

/* SiglipVisionTower feature reduction: bilinear 27x27 -> TxT (fp32 taps) + F.normalize
 * (siglip_encoder.py:151-163, 206-208); row-wise L2 normalise (metamorph_llama.py:369-370). */
int mm_bilinear_l2norm(const void* x, void* y, int n_img, int in_side, int out_side, int C, int normalize,
                       float eps, cudaStream_t s);
int mm_l2norm_rows(const void* x, void* y, long long R, int C, float eps, cudaStream_t s);

/* Shifted cross-entropy forward+backward over an fp32 logits chunk (metamorph_llama.py:402-413);
 * -mean cosine similarity of the normalised vision-head output vs target (metamorph_llama.py:433-453);
 * argmax over the vocabulary (metamorph_llama.py:542). */
int mm_ce_fwd_bwd(const float* logits, long long ld, const int* labels, void* dlogits, long long ld_d,
                  float* loss_sum, float* lse_out, long long R, int V, float grad_scale, int ignore_index,
                  cudaStream_t s);
int mm_cosine_loss(const void* pred, const void* target, void* pred_norm, void* dpred, float* loss_sum,
                   long long R, int C, float grad_scale, cudaStream_t s);
long long mm_argmax_workspace_bytes(long long R);
int mm_argmax_rows(const float* logits, long long ld, long long R, int V, int* out, void* workspace,
                   long long workspace_bytes, cudaStream_t s);
/* Seeded sampling in place of the argmax of metamorph_llama.py:542, one token per row, with HF's
 * TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper (transformers generation/logits_process.py) decided by
 * value: z = l / T (NaN -> -inf); top-k keeps count(z_j > z_i) < k (ties kept; k <= 0 or k >= V: off); top-p keeps
 * mass(z_j > z_i) < p * mass(top-k set) with mass_j = round(exp(z_j - max z) * 2^40) added as 64-bit integers (relative
 * masses below ~1e-12 count as 0; p >= 1 or NaN: off; p <= 0: only the maximum). The token is the Gumbel-max
 * argmax_i z_i - log(-log u_i) over the kept set, lowest index on ties, u_i = (w + 0.5) 2^-32 with w word (i & 3) of
 * Philox4x32-10(counter (i >> 2, counter[r], 0, 0), key (seed[r] & 0xffffffff, seed[r] >> 32)): a pure function of the
 * row's logits bits and parameters, the same on every run, under graph replay and whatever rows share the call.
 * T <= 0 or NaN: exactly mm_argmax_rows' token. Always returns an index in [0, V) (0 for a row without a logit above
 * -inf). Every per-row array is a device pointer. One launch of R thread-block clusters of 8 CTAs; V <= 393216. */
int mm_sample_rows(const float* logits, long long ld, long long R, int V, const float* temperature, const int* top_k,
                   const float* top_p, const unsigned long long* seed, const int* counter, int* out, cudaStream_t s);
/* Log-probabilities of the tokens a decode step emitted, read after mm_decode_state_step[_slots]: for the model's raw
 * distribution over one fp32 logits row (NaN read as -inf, m = max l, S = sum_j exp(l_j - m)),
 * logprob(i) = l_i - m - ln S, rounded once to fp32 from an fp64 evaluation (S summed in fp64 from expf terms; within
 * 0.5 ulp + 2^-21 + 2^-51 |logprob| of the exact value). A row whose max is +inf is the point mass on its c +inf
 * entries (-ln c each, -inf elsewhere); a row with no logit above -inf reports NaN. Row r reports when
 * append_kind[r] == 0 (the step appended next_token = token[r] to ids_out), n_top[r] >= 0 (-1: skip) and
 * 0 <= n_ids[r] - 1 < max_ids; it then writes slot o = r * max_ids + n_ids[r] - 1 and nothing else:
 * lp_out[o] = logprob(token[r]) (NaN for a token outside [0, V)), and for k < min(n_top[r], 20)
 * top_ids[o * 20 + k], top_lp[o * 20 + k] = the k-th entry in order of logit descending, lowest index first among
 * ties (mm_argmax_rows' order); entries past V get id -1 and logprob -inf. The bits are a pure function of the row's
 * logits and V, and a token in the list has the same bits there as in lp_out. lp_out [R, max_ids],
 * top_ids / top_lp [R, max_ids, 20]; every pointer is a device pointer. One launch of R clusters of 8 CTAs;
 * V <= 393216. */
int mm_decode_logprobs(const float* logits, long long ld, long long R, int V, const int* append_kind, const int* token,
                       const int* n_ids, const int* n_top, int max_ids, float* lp_out, int* top_ids, float* top_lp,
                       cudaStream_t s);

/* torch.optim.AdamW step (train.py:82 --optim adamw_torch), fused over flat buffers; clip coefficient. */
int mm_adamw_step(void* p16, float* p32, float* m, float* v, const void* grad, int grad_f32, long long n, float lr,
                  float beta1, float beta2, float eps, float wd, int step, const float* grad_scale_ptr,
                  float grad_scale, cudaStream_t s);
/* Sharded-optimizer step with its all-gather fused in: AdamW on this rank's slice, and the updated bf16 slice is written
 * into EVERY rank's replica of the parameter buffer by the same kernel — through the NVSwitch multicast address of the
 * (symmetric) buffer (multimem.st) when multicast_p16 != NULL, else with one store per peer over NVLink P2P (peers = device
 * array of the n_peers buffer base pointers, slice_offset = first element of the slice). Replaces DeepSpeed ZeRO's
 * all-gather of updated parameters (scripts/zero2.json `allgather_bucket_size`).
 * grad_multicast = 1: `grad` is the multicast address of this rank's slice of the SYMMETRIC gradient buffers and is read
 * with multimem.ld_reduce (sum over all ranks inside the switch, fp32 accumulation): the reduce-scatter is fused in as
 * well, the bucket's whole [reduce-scatter -> AdamW -> all-gather] is one kernel (callers order it between two cross-rank
 * barriers: every rank's gradients complete before, every rank done reading after). */
int mm_adamw_step_bcast(void* multicast_p16, const void* const* peers, int n_peers, long long slice_offset, float* p32,
                        float* m, float* v, const void* grad, int grad_f32, int grad_multicast, long long n, float lr,
                        float beta1, float beta2, float eps, float wd, int step, const float* grad_scale_ptr,
                        float grad_scale, cudaStream_t s);
int mm_clip_coef(const float* sumsq, float* out2, float max_norm, cudaStream_t s);

/* Attention: LLaMA causal GQA (modeling_llama.py:199-220) forward/backward, SigLIP MHA forward
 * (modeling_siglip.py:229-249). q/k/v/o are [B*T, heads*head_dim] views with independent pitches.
 * wgmma / TMA flash attention for head_dim 128 (csrc/attention_tc.cu forward, csrc/attention_bwd_tc.cu backward:
 * a query-stationary dQ kernel + a key-stationary dK/dV kernel, no atomics -> bit-reproducible).
 * Rows >= seqlens[b] are outside the sequence: zero dQ/dK/dV, their dO is ignored. Backward workspace: lse*log2e and
 * delta, mm_attn_bwd_tc_workspace_bytes. */
long long mm_attn_bwd_tc_workspace_bytes(int B, int T, int Hq);
int mm_attn_fwd_tc(const void* q, const void* k, const void* v, void* o, float* lse, const int* seqlens,
                   long long ldq, long long ldk, long long ldv, long long ldo, int B, int T, int Hq, int Hkv,
                   int head_dim, int causal, float scale, cudaStream_t s);
int mm_attn_bwd_tc(const void* q, const void* k, const void* v, const void* o, const void* dout, const float* lse,
                   void* dq, void* dk, void* dv, const int* seqlens, long long ldq, long long ldk, long long ldv,
                   long long ldo, long long lddo, long long lddq, long long lddk, long long lddv, int B, int T,
                   int Hq, int Hkv, int head_dim, float scale, void* workspace, long long workspace_bytes,
                   cudaStream_t s);
/* Packed sequences (SURVEY.md section 8f N2; replaces right padding, metamorph_arch.py:361-399): block-diagonal causal
 * attention over n_seg sequences laid end to end, ONE launch for all of them. Sequence s = rows [seg_start[s],
 * seg_start[s] + seg_len[s]) of the [total_rows, width] operands; lse is [n_seg, Hq, max_len]; work lists are int pairs
 * (sequence, 128-row tile), heaviest first: query tiles for the forward and the dQ kernel, key tiles for dK/dV. */
int mm_attn_fwd_tc_varlen(const void* q, const void* k, const void* v, void* o, float* lse, const int* seg_start,
                          const int* seg_len, int n_seg, int max_len, const int* work, int n_work,
                          long long total_rows, long long ldq, long long ldk, long long ldv, long long ldo, int Hq,
                          int Hkv, int head_dim, float scale, cudaStream_t s);
int mm_attn_bwd_tc_varlen(const void* q, const void* k, const void* v, const void* o, const void* dout,
                          const float* lse, void* dq, void* dk, void* dv, const int* seg_start, const int* seg_len,
                          int n_seg, int max_len, const int* work_q, int n_work_q, const int* work_k, int n_work_k,
                          long long total_rows, long long ldq, long long ldk, long long ldv, long long ldo,
                          long long lddo, long long lddq, long long lddk, long long lddv, int Hq, int Hkv,
                          int head_dim, float scale, void* workspace, long long workspace_bytes, cudaStream_t s);

/* On-GPU SigLIP image pre-processing (SURVEY.md section 8f, row N1), bit-exact with the reference's CPU chain:
 * expand2square + processor.preprocess (metamorph/train/train.py:1189-1209) with the SigLIP processor of
 * multimodal_encoder/siglip_encoder.py:113-121 = Pillow BICUBIC resize (ImagingResample: two uint8 passes, 22-bit
 * fixed-point coefficients) + x 1/255 + normalise 0.5/0.5 + channels first.
 * mm_resize_coeff_build is a HOST function (no CUDA): it fills a host buffer with the coefficient table of one axis;
 * the caller copies it to the device. mm_siglip_preprocess: img uint8 [H][W][3], tmp uint8 [rows][out][3] scratch
 * (rows = padded side, or H), lut = 256 floats, out = [3][out][out] fp32 (or bf16). */
long long mm_resize_coeff_bytes(int in_size, int out_size);
int mm_resize_coeff_build(void* host_buf, int in_size, int out_size);
int mm_siglip_preprocess(const void* img, int H, int W, int pad_square, int fill, const void* coeff_x,
                         const void* coeff_y, int ksize_x, int ksize_y, int out_size, const float* lut, void* tmp,
                         void* out, int out_bf16, cudaStream_t s);

/* KV-cached decode step (replaces the no-cache loop of greedy_decode, metamorph_llama.py:502-597).
 * mm_skinny_gemm: y[m, N] = x[m, K] W[N, K]^T for 1 <= m <= 32 sequences (weights streamed once per call);
 * epilogue 0 store, 1 +bias, 2 +resid, 3 +bias then GELU(erf), 4 SwiGLU over 16-row interleaved gate/up (y is [m, N/2]). */
int mm_skinny_gemm(const void* x, const void* W, void* y, const void* bias, const void* resid, long long ldx,
                   long long ldw, long long ldy, long long ldr, int m, int N, int K, int epilogue, int out_f32,
                   cudaStream_t s);
/* mm_skinny_gemm_wide: the same product, arguments and epilogues for 1 <= m <= 128 sequences (wgmma, K split over a
 * thread-block cluster of up to 8 CTAs whose fp32 partials are added in rank order; no float atomics). The decode step
 * calls it for m > 32. Determinism: a row's output bits depend only on its own x row, W, N, K and the epilogue (and its
 * bias / residual row), never on m or the other rows, and repeated calls give the same bits. Against mm_skinny_gemm
 * (m <= 32) the results agree within bf16 rounding, not bit for bit. */
int mm_skinny_gemm_wide(const void* x, const void* W, void* y, const void* bias, const void* resid, long long ldx,
                        long long ldw, long long ldy, long long ldr, int m, int N, int K, int epilogue, int out_f32,
                        cudaStream_t s);
long long mm_decode_attn_workspace_bytes(int B, int Hq, int Hkv, int splits);
int mm_decode_attn(const void* qkv, long long ldqkv, void* kcache, void* vcache, const int* pos,
                   const float* cos_t, const float* sin_t, void* out, long long ldo, int B, int Hq, int Hkv,
                   int head_dim, int Tmax, float scale, void* workspace, long long workspace_bytes, int splits,
                   cudaStream_t s);
int mm_kv_prefill(const void* qkv, long long ld, void* kcache, void* vcache, int B, int T, int Hq, int Hkv,
                  int head_dim, int Tmax, cudaStream_t s);
/* Paged KV cache. kpool / vpool (one pair per layer): [num_blocks, Hkv, block_size, 128] bf16; block_table:
 * [B, max_blocks] int32 on the device, one row per sequence, shared by every layer. Logical position p of sequence b
 * lives in block block_table[b * max_blocks + p / block_size] at row p % block_size. block_size is a power of two in
 * [16, 256]. Every table entry the call can reach (those of positions 0..pos[b] for the attention, 0..T-1 for the
 * prefill) must lie in [0, num_blocks); the kernels do not check them.
 * mm_decode_attn_paged is mm_decode_attn with that addressing and the logical Tmax = max_blocks * block_size (which
 * sizes the shared-memory bound exactly as in the dense call; workspace: mm_decode_attn_workspace_bytes). It walks
 * the positions in the same split and order, so with equal splits its output and the appended K/V bits are those of
 * mm_decode_attn on the same logical cache. mm_kv_prefill_paged copies the post-RoPE K/V rows of a prefill pass of
 * ONE sequence (qkv rows [T, ld], positions 0..T-1) into the blocks of its table row (block_table_row points at that
 * row); the bits are mm_kv_prefill's. */
int mm_decode_attn_paged(const void* qkv, long long ldqkv, void* kpool, void* vpool, const int* block_table,
                         int max_blocks, int block_size, const int* pos, const float* cos_t, const float* sin_t,
                         void* out, long long ldo, int B, int Hq, int Hkv, int head_dim, float scale, void* workspace,
                         long long workspace_bytes, int splits, cudaStream_t s);
int mm_kv_prefill_paged(const void* qkv, long long ld, void* kpool, void* vpool, const int* block_table_row,
                        int max_blocks, int block_size, int T, int Hq, int Hkv, int head_dim, cudaStream_t s);
/* Prefill attention over a paged cache (prefix caching: a suffix attends to shared prefix blocks). Causal flash attention
 * of ONE sequence, head_dim 128, any GQA group, no lse: q [n_q, ldq] holds the query rows of positions
 * q_start .. q_start + n_q - 1, and keys / values 0 .. kv_len - 1 (kv_len = q_start + n_q) are read from kpool / vpool
 * [num_blocks, Hkv, block_size, 128] through block_table_row (max_blocks entries, same layout and block sizes as
 * mm_decode_attn_paged; every entry of positions < kv_len must lie in [0, num_blocks)). o: [n_q, ldo]. Pool rows at or
 * past kv_len are never used, whatever they hold (NaN included). Output row of position r is, bit for bit, row r of
 * mm_attn_fwd_tc(B=1, T=kv_len, causal) on the same post-RoPE K/V: query tiles are aligned to absolute multiples of 128,
 * so every row meets the same key tiles, masks and arithmetic as in the dense kernel. Arguments are checked (block
 * size, table, head_dim, q_start >= 0, n_q >= 1, kv_len <= max_blocks * block_size, alignment) before any launch. */
int mm_attn_fwd_tc_paged(const void* q, long long ldq, const void* kpool, const void* vpool, int num_blocks,
                         const int* block_table_row, int max_blocks, int block_size, void* o, long long ldo,
                         int q_start, int n_q, int Hq, int Hkv, int head_dim, float scale, cudaStream_t s);
/* FP8 KV cache (E4M3). Each (position, kv head) row of 128 values x is stored as q_i = RNE_e4m3(x_i 2^-e) with one fp32
 * scale 2^e: a = max |x_i|, e the least integer with a <= 448 2^e, at least -124; a zero row stores zeros with e = 0, a
 * row holding Inf or NaN stores 0x7f (E4M3 NaN) everywhere with e = 0; at e = 120 an entry that rounds to 256 (|x| >=
 * 1.9375 2^127, whose x-hat 2^128 would overflow) stores 240 instead. x-hat_i = float(q_i) 2^e is exact and a bf16
 * value. A row's bytes depend on that row alone. Byte caches are the bf16 layouts above; scales are addressed like the
 * rows: [B, Hkv, Tmax] dense, [num_blocks, Hkv, block_size] paged (scale index = element offset of the row / 128).
 * mm_decode_attn_fp8 / mm_decode_attn_paged_fp8: mm_decode_attn / mm_decode_attn_paged on such a cache. The owner of pos
 * quantises the rotated new k and the new v, appends bytes and scales and scores pos from their x-hat; with equal splits
 * the output bits are those of the bf16 call on a bf16 cache holding x-hat (appended rows included).
 * mm_kv_quant_prefill[_paged]: mm_kv_prefill[_paged] for such a cache; also overwrites the K and V columns of qkv with
 * x-hat (Q columns untouched), so a prefill's attention reads what the cache holds. qkv rows must be 8-byte aligned.
 * mm_kv_dequant_paged: staging block i <- x-hat of pool block block_table_row[i] for i < n_blocks, into bf16 staging
 * pools [>= n_blocks, Hkv, block_size, 128]. Every scale pointer must be non-null. */
int mm_decode_attn_fp8(const void* qkv, long long ldqkv, void* kcache, void* vcache, float* kscale, float* vscale,
                       const int* pos, const float* cos_t, const float* sin_t, void* out, long long ldo, int B, int Hq,
                       int Hkv, int head_dim, int Tmax, float scale, void* workspace, long long workspace_bytes,
                       int splits, cudaStream_t s);
int mm_decode_attn_paged_fp8(const void* qkv, long long ldqkv, void* kpool, void* vpool, float* kscale, float* vscale,
                             const int* block_table, int max_blocks, int block_size, const int* pos, const float* cos_t,
                             const float* sin_t, void* out, long long ldo, int B, int Hq, int Hkv, int head_dim,
                             float scale, void* workspace, long long workspace_bytes, int splits, cudaStream_t s);
int mm_kv_quant_prefill(void* qkv, long long ld, void* kcache, void* vcache, float* kscale, float* vscale, int B, int T,
                        int Hq, int Hkv, int head_dim, int Tmax, cudaStream_t s);
int mm_kv_quant_prefill_paged(void* qkv, long long ld, void* kpool, void* vpool, float* kscale, float* vscale,
                              const int* block_table_row, int max_blocks, int block_size, int T, int Hq, int Hkv,
                              int head_dim, cudaStream_t s);
int mm_kv_dequant_paged(const void* kpool, const void* vpool, const float* kscale, const float* vscale,
                        const int* block_table_row, int max_blocks, int block_size, int n_blocks, int Hkv,
                        int head_dim, void* kstage, void* vstage, cudaStream_t s);
/* FP8 weights (E4M3) for the weight-streaming GEMMs. A matrix W [N, K] (K a multiple of 128) is stored as bytes
 * q [N, K] (row stride ldq / ldw, in bytes) and fp32 scales [N, K / 128] (row stride lds): group j of row n,
 * W[n, 128 j .. 128 j + 127], is one row of the FP8 KV-cache rule above, so W-hat = float(q) * scale is exact and a bf16
 * value.
 * mm_weight_quant_fp8: W (bf16, row stride ldw elements) -> (q, scale); mm_weight_dequant_fp8: (q, scale) -> W-hat (bf16,
 * row stride ldw elements). One warp per group; row strides must be multiples of 4 and at least K.
 * mm_skinny_gemm_fp8 / mm_skinny_gemm_wide_fp8: mm_skinny_gemm / mm_skinny_gemm_wide with W given as (Wq, wscale), same
 * batch limits, epilogues and out_f32 / padded ldy. Every weight reaches the tensor cores as its exact bf16 value W-hat,
 * in the bf16 kernel's fragment slots and accumulation order (the same k chunks per warp, the same split-K and reduction),
 * so the output bits are those of the bf16 call on W-hat. Need K % 128 == 0, ldw % 16 == 0, lds >= K / 128, 16-byte
 * aligned x / Wq and a non-null, 4-byte aligned wscale; checked before any launch. */
int mm_weight_quant_fp8(const void* W, long long ldw, void* q, long long ldq, float* scale, long long lds, int N, int K,
                        cudaStream_t s);
int mm_weight_dequant_fp8(const void* q, long long ldq, const float* scale, long long lds, void* W, long long ldw, int N,
                          int K, cudaStream_t s);
int mm_skinny_gemm_fp8(const void* x, const void* Wq, const float* wscale, void* y, const void* bias, const void* resid,
                       long long ldx, long long ldw, long long lds, long long ldy, long long ldr, int m, int N, int K,
                       int epilogue, int out_f32, cudaStream_t s);
int mm_skinny_gemm_wide_fp8(const void* x, const void* Wq, const float* wscale, void* y, const void* bias,
                            const void* resid, long long ldx, long long ldw, long long lds, long long ldy, long long ldr,
                            int m, int N, int K, int epilogue, int out_f32, cudaStream_t s);
int mm_decode_state_step(int* in_image_mode, int* total_image_tokens, int* total_output, int* finished, int* pos,
                         int* n_ids, int* n_img, int* ids_out, int* append_kind, int* next_token,
                         const int* argmax_tok, const int* forced, int forced_ld, int step, int B,
                         int num_image_tokens, int max_new_tokens, int max_ids, int start_id, int end_id, int eos0,
                         int eos1, const void* pred_z, void* img_out, int max_img, int C, cudaStream_t s);
/* continuous batching (SURVEY 8f N4): per-slot output limit; a negative forced entry = free running */
int mm_decode_state_step_slots(int* in_image_mode, int* total_image_tokens, int* total_output, int* finished, int* pos,
                               int* n_ids, int* n_img, int* ids_out, int* append_kind, int* next_token,
                               const int* argmax_tok, const int* forced, int forced_ld, const int* max_new_slot, int B,
                               int num_image_tokens, int max_ids, int start_id, int end_id, int eos0, int eos1,
                               const void* pred_z, void* img_out, int max_img, int C, cudaStream_t s);
int mm_decode_next_input(const int* kind, const int* tok, const void* embed, const void* pred, void* x, int B,
                         int H, cudaStream_t s);
int mm_decode_select_hidden(const int* mode, const void* hidden, const void* pred, void* out, int B, int H,
                            cudaStream_t s);

#ifdef __cplusplus
}
#endif
#endif /* METAMORPH_B200_H */
