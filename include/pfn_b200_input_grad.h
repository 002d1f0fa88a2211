/*
 * pfn_b200_input_grad.h — input-gradient entry points of libpfn_b200.so, an extension of the C ABI of pfn_b200.h (which it
 * includes).  The declarations of pfn_b200.h are unchanged by it; a caller that does not include this header sees the same
 * library as before.
 */
#ifndef PFN_B200_INPUT_GRAD_H
#define PFN_B200_INPUT_GRAD_H

#include "pfn_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------------------
 * Context attention with a backward (the gradient of the query rows against cached training rows):
 *   keys(i) = the n cached training keys of dataset b (its first n_keys[b] when n_keys is set)  U  {query row i itself}
 * c      : the descriptor of pfn_attention_ctx_fwd_*, with the same meaning for every field.
 * n_keys : optional [B] device int32; null: every dataset has all n cached rows.  Values outside [0, c.n] are clamped
 *          into it.  With n_keys set the outputs equal those of pfn_attention_ctx_ragged_fwd_*, bit for bit.
 * lse    : [B*H, m] fp32 natural-log-sum-exp of each query row's scaled scores: written by the forward, read by the
 *          backward.  The forward's `out` equals pfn_attention_ctx_fwd_*'s bit for bit.
 * dout   : [m*B, H*dh] gradient of out (backward).
 * dqkv   : [m*B, 3*H*dh] written completely by the backward: dQ of every query row, and dK_i, dV_i of the row's own key.
 *          The cached keys are constants: the backward writes no gradient of kv.
 * delta  : [B*H, m] fp32 scratch of the backward: rowsum(dO * O).
 * _tc entry points: bf16, dh = 128, leading dims multiples of 8, 16-byte aligned bases; _simt: fp32 or bf16, dh <= 256.
 * ---------------------------------------------------------------------------------------------- */
typedef struct pfn_attn_ctx_grad_desc {
  pfn_attn_ctx_desc c;
  const int* n_keys;
  float* lse;
  const void* dout; int ld_dout;
  void* dqkv; int ld_dqkv;
  float* delta;
} pfn_attn_ctx_grad_desc;

int pfn_attention_ctx_grad_fwd_simt(const pfn_attn_ctx_grad_desc* d, void* stream);
int pfn_attention_ctx_grad_fwd_tc(const pfn_attn_ctx_grad_desc* d, void* stream);
int pfn_attention_ctx_bwd_simt(const pfn_attn_ctx_grad_desc* d, void* stream);
int pfn_attention_ctx_bwd_tc(const pfn_attn_ctx_grad_desc* d, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Input gradient of the embedding stage (pfn_embed_fwd / pfn_embed_ragged_fwd):
 *   dx[t,b,:] = dout[t,b,:] Wx                     for every row
 *   dy[t,b]   = dout[t,b,:] . wy  if t < sep (t < n_keys[b] when n_keys is set, clamped to [0, T]), else 0
 * dout [T*B, E] (dtype PFN_F32 or PFN_BF16), Wx [E, F], wy [E] fp32; dx [T*B, F], dy [T*B] fp32, overwritten.  F <= 64.
 * Each output is summed over e in one fixed order: two calls give the same bits.
 * ---------------------------------------------------------------------------------------------- */
int pfn_embed_input_bwd(const void* dout, int dtype, const float* Wx, const float* wy, float* dx, float* dy, int T, int B,
                        int F, int E, int sep, const int* n_keys, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* PFN_B200_INPUT_GRAD_H */
