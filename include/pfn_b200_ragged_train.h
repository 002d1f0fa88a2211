/*
 * pfn_b200_ragged_train.h — ragged-dataset training entry points of libpfn_b200.so, an extension of the C ABI of
 * pfn_b200.h (which it includes).  The declarations of pfn_b200.h are unchanged by it; a caller that does not include
 * this header sees the same library as before.
 */
#ifndef PFN_B200_RAGGED_TRAIN_H
#define PFN_B200_RAGGED_TRAIN_H

#include "pfn_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------------------
 * Ragged datasets in training: the masked attention (forward with lse, backward) where dataset b has its own
 * single_eval_pos s_b = n_keys[b] (n_keys a device int32 [B] array) in place of the scalar sep:
 *   keys(i) = {0..s_b-1}  U  ({i} if i >= s_b)
 * a : the descriptor the scalar entry points take (pfn_attention_fwd_* / pfn_attention_bwd_*), with the same meaning for
 *     every field but sep, which here is an upper bound of every s_b; values of n_keys outside [0, a.sep] are clamped
 *     into it.  The keys [s_b, a.sep) of dataset b are real rows of qkv: they must be finite on the tensor-core path.
 *     The least work is done with a.sep = max_b s_b.  Rows t >= s_b of dataset b get dK, dV from their own key only.
 * With every s_b equal to a.sep the outputs are those of the scalar entry points with sep = a.sep, bit for bit.
 * ---------------------------------------------------------------------------------------------- */
typedef struct pfn_attn_ragged_train_desc {
  pfn_attn_desc a;
  const int* n_keys;       /* [B] device, 0 <= n_keys[b] <= a.sep */
} pfn_attn_ragged_train_desc;

int pfn_attention_ragged_train_fwd_simt(const pfn_attn_ragged_train_desc* d, void* stream);
int pfn_attention_ragged_train_fwd_tc(const pfn_attn_ragged_train_desc* d, void* stream);
int pfn_attention_ragged_train_bwd_simt(const pfn_attn_ragged_train_desc* d, void* stream);
int pfn_attention_ragged_train_bwd_tc(const pfn_attn_ragged_train_desc* d, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Ragged embedding: pfn_embed_fwd / pfn_embed_bwd with the y embedding of dataset b on its rows t < n_keys[b]:
 *   out[t,b,:] = x[t,b,:] Wx^T + bx + (t < n_keys[b] ? y[t,b] wy + by : 0)
 * and dwy, dby summed over those rows only.  n_keys: device int32 [B], each in [0, T] (clamped into it).
 * ---------------------------------------------------------------------------------------------- */
int pfn_embed_ragged_fwd(const float* x, const float* y, const float* Wx, const float* bx, const float* wy,
                         const float* by, void* out, int out_dtype, int T, int B, int F, int E, const int* n_keys,
                         void* stream);
int pfn_embed_ragged_bwd(const void* dout, int dtype, const float* x, const float* y, float* dWx, float* dbx, float* dwy,
                         float* dby, int T, int B, int F, int E, const int* n_keys, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* PFN_B200_RAGGED_TRAIN_H */
