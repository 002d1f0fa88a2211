/*
 * pfn_b200_ragged.h — ragged-dataset attention entry points of libpfn_b200.so, an extension of the C ABI of pfn_b200.h
 * (which it includes).  The declarations of pfn_b200.h are unchanged by it; a caller that does not include this header
 * sees the same library as before.
 */
#ifndef PFN_B200_RAGGED_H
#define PFN_B200_RAGGED_H

#include "pfn_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------------------
 * Ragged datasets (forward only, no lse): the two attentions above where dataset b has its own key count
 * n_b = n_keys[b] in [0, T] (masked) or [0, n] (context), n_keys a device int32 [B] array, in place of sep / n:
 *   masked  : keys(i) = {0..n_b-1}  U  ({i} if i >= n_b)      rows i >= n_b of dataset b are its padding / query rows
 *   context : keys(i) = the first n_b cached keys of dataset b  U  {query row i itself}
 * Rows t >= n_b of the qkv (masked) or the cache (context) of dataset b are never a key; their values must be finite on the
 * tensor-core path (a masked key's probability is an exact 0, which still turns a NaN or Inf value into a NaN).
 * The other fields mean what they mean in pfn_attn_desc (T rows per dataset) and pfn_attn_ctx_desc, and the paths take
 * the same dtypes, head dims and layouts.  With every n_b equal to T (n) the outputs are those of
 * pfn_attention_fwd_* with sep = T (pfn_attention_ctx_fwd_*), bit for bit.
 * ---------------------------------------------------------------------------------------------- */
typedef struct pfn_attn_ragged_desc {
  int T, B, H, dh;         /* rows per dataset, batch, heads, head dim */
  int dtype;
  float scale;
  const void* qkv; int ld_qkv;
  void* out; int ld_out;
  const int* n_keys;       /* [B] device, 0 <= n_keys[b] <= T */
} pfn_attn_ragged_desc;

typedef struct pfn_attn_ctx_ragged_desc {
  int m, n, B, H, dh;      /* query rows, cached training rows (the longest training set), batch, heads, head dim */
  int dtype;
  float scale;
  const void* qkv; int ld_qkv;
  const void* kv; int ld_kv;
  void* out; int ld_out;
  const int* n_keys;       /* [B] device, 0 <= n_keys[b] <= n */
} pfn_attn_ctx_ragged_desc;

int pfn_attention_ragged_fwd_simt(const pfn_attn_ragged_desc* d, void* stream);
int pfn_attention_ragged_fwd_tc(const pfn_attn_ragged_desc* d, void* stream);
int pfn_attention_ctx_ragged_fwd_simt(const pfn_attn_ctx_ragged_desc* d, void* stream);
int pfn_attention_ctx_ragged_fwd_tc(const pfn_attn_ctx_ragged_desc* d, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* PFN_B200_RAGGED_H */
