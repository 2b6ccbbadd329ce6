/* b200_e2eft_vae_attention.h — training entry points of libb200_e2eft.so for the VAE mid-block's single attention
 * head of width 512: the flash forward with its log-sum-exp, the row dot delta = rowsum(dout o out) and the fused
 * backward.  Declared beside the engine's main C ABI (include/b200_e2eft.h), whose conventions they follow: 0 ok,
 * < 0 invalid argument (b200_last_error_string() says which, checked before any launch), > 0 a cudaError_t; the caller
 * owns every buffer; nothing is allocated and nothing synchronises; every launch goes on `stream`. */
#pragma once

#ifdef __cplusplus
extern "C" {
#endif

/* b200_attention_d512 (include/b200_e2eft.h) with an optional log-sum-exp: out = softmax(scale Q K^T) V for one head
 * of width 512, and, when lse != NULL, lse [B][Lq] fp32 = log2(sum_j exp2(scale log2(e) S_ij)), the log2-domain
 * log-sum-exp of b200_attention's `lse`.  out has the same bits with and without lse, and b200_attention_d512 is
 * this call with lse = NULL.  Operands, strides and limits as b200_attention_d512; lse 4-byte aligned. */
int b200_attention_d512_lse(const void* q, long long q_bs, long long q_ls,
                            const void* k, long long k_bs, long long k_ls,
                            const void* v, long long v_bs, long long v_ls,
                            void* out, long long o_bs, long long o_ls,
                            int B, int Lq, int Lk, float scale, float* lse, void* stream);

/* delta [B][L] fp32 = sum over the 512 columns of a * c, a / c fp16 [B][L][>= 512] row-strided (element (b, l, d) at
 * base + b * bs + l * ls + d): the delta = rowsum(dout o out) of b200_attention_d512_bwd.  Strides multiples of 8
 * elements, row strides >= 512, a / c 16-byte aligned, delta 4-byte aligned, 1 <= B <= 65535, L >= 1. */
int b200_rowdot_d512(const void* a, long long a_bs, long long a_ls,
                     const void* c, long long c_bs, long long c_ls,
                     int B, int L, float* delta, void* stream);

/* Backward of b200_attention_d512_lse: dq, dk, dv of out = softmax(scale Q K^T) V for one head of width 512.
 * q / dout / dq are [B][Lq][>= 512], k / v / dk / dv [B][Lk][>= 512], fp16, row-strided like the forward's operands
 * (e.g. column blocks of fused [B, L, 1536] QKV and d(QKV) buffers); lse [B][Lq] is the forward's and delta [B][Lq] =
 * rowsum(dout o out) (b200_rowdot_d512).  Writes the 512 columns of the Lq rows of dq and of the Lk rows of dk and dv,
 * nothing else.  P = fp16(exp2(fmaf(S, scale log2(e), -lse))) and dS = fp16(fmaf(dP, scale, -scale delta) P) are
 * recomputed in registers and never stored, so memory stays O(B L); three kernels (dQ query-stationary, dK and dV
 * key-stationary) without atomics give the same bits on every call.
 * Strides multiples of 8 elements, row strides >= 512, every fp16 operand 16-byte aligned, lse / delta 4-byte
 * aligned, 1 <= B <= 65535, Lq, Lk >= 1. */
int b200_attention_d512_bwd(const void* q, long long q_bs, long long q_ls,
                            const void* k, long long k_bs, long long k_ls,
                            const void* v, long long v_bs, long long v_ls,
                            const void* dout, long long do_bs, long long do_ls,
                            const float* lse, const float* delta,
                            void* dq, long long dq_bs, long long dq_ls,
                            void* dk, long long dk_bs, long long dk_ls,
                            void* dv, long long dv_bs, long long dv_ls,
                            int B, int Lq, int Lk, float scale, void* stream);

#ifdef __cplusplus
}
#endif
