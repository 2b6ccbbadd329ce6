/* b200_e2eft_attention_bwd.h — the fused flash-attention backward of libb200_e2eft.so, a training entry point
 * declared beside the engine's main C ABI (include/b200_e2eft.h), whose conventions it follows: 0 ok, < 0 invalid
 * argument (b200_last_error_string() says which), > 0 a cudaError_t; every launch goes on `stream`. */
#pragma once

#ifdef __cplusplus
extern "C" {
#endif

/* Backward of b200_attention (include/b200_e2eft.h): dq, dk, dv of out = softmax(scale Q K^T) V for heads of width head_dim in
 * {40, 64, 80, 160}, with the same operand layout and kv_segments meaning.  dout is dL/dout [B][Lq][heads*head_dim]
 * (row-strided like q); lse [B][heads][Lq] is the forward's log2-domain log-sum-exp (b200_attention's `lse`) and
 * delta [B][heads][Lq] = sum_d dout * out per head (b200_rowdot_heads_d).  dq is written like q (Lq rows), dk / dv
 * like k / v (Lk rows of each batch element); nothing else is written.  P and dS are recomputed in registers and never
 * stored (memory O(B L C)); with kv_segments = 2, dk / dv of batch element e sum over the queries of e % (B/2) and
 * e % (B/2) + B/2.  Deterministic: two kernels without atomics, the same bits on every call.
 * Strides are multiples of 8 elements, q/k/v/dout/dq/dk/dv 16-byte aligned, 1 <= B, heads <= 65535.
 * Replaces the backward of xformers.ops.memory_efficient_attention (attention.py:497) in training. */
int b200_attention_bwd(const void* q, long long q_bs, long long q_ls,
                       const void* k, long long k_bs, long long k_ls,
                       const void* v, long long v_bs, long long v_ls,
                       const void* dout, long long do_bs, long long do_ls,
                       const float* lse, const float* delta,
                       void* dq, long long dq_bs, long long dq_ls,
                       void* dk, long long dk_bs, long long dk_ls,
                       void* dv, long long dv_bs, long long dv_ls,
                       int B, int heads, int head_dim, int Lq, int Lk, int kv_segments, float scale, void* stream);

#ifdef __cplusplus
}
#endif
