"""Drop-in `transformer.TransformerModel` (reference transformer.py:13-91) whose forward runs on the sm_90a engine.

The module keeps `self.transformer_encoder = nn.TransformerEncoder(...)` purely as the *parameter container*:
identical state_dict keys (the five reference checkpoints under results/ load with strict=True), identical
construction-time RNG consumption and the reference's zero-init of `linear2` / `out_proj` — but its forward is
never called.  `forward()` routes embedding -> encoder stack -> decoder through `engine.*Fn`.
"""
import torch
import torch.nn as nn
from torch.nn import TransformerEncoder, TransformerEncoderLayer

from . import engine
from ._lib import draw_seed, drop_threshold as L_drop_threshold
from .positional_encodings import NoPositionalEncoding
from .utils import SeqBN


class TransformerModel(nn.Module):
    def __init__(self, encoder, n_out, ninp, nhead, nhid, nlayers, dropout=0.0, y_encoder=None, pos_encoder=None,
                 decoder=None, input_normalization=False):
        super().__init__()
        self.model_type = 'Transformer'
        layer = TransformerEncoderLayer(ninp, nhead, nhid, dropout, activation='gelu')
        self.transformer_encoder = TransformerEncoder(layer, nlayers, enable_nested_tensor=False)
        self.ninp = ninp
        self.nhead = nhead
        self.dropout = dropout
        self.encoder = encoder
        self.y_encoder = y_encoder
        self.pos_encoder = pos_encoder
        if decoder is not None:
            self.decoder = decoder(ninp, nhid, n_out)
        else:
            self.decoder = nn.Sequential(nn.Linear(ninp, nhid), nn.GELU(), nn.Linear(nhid, n_out))
        self.input_ln = SeqBN(ninp) if input_normalization else None
        self.precision = engine.default_precision()   # 'bf16' (tensor cores) or 'fp32' (parity mode)
        self.init_weights()

    # ---- static helpers kept for API compatibility (reference transformer.py:28-41) ----------------------
    @staticmethod
    def generate_square_subsequent_mask(sz):
        allowed = torch.tril(torch.ones(sz, sz, dtype=torch.bool))
        return torch.zeros(sz, sz).masked_fill(~allowed, float('-inf'))

    @staticmethod
    def generate_D_q_matrix(sz, query_size):
        """Additive mask: key j visible to row i iff j < sz - query_size or i == j.  The engine never builds this
        matrix (the structure is implied by `single_eval_pos`); it is provided for callers and tests."""
        train_size = sz - query_size
        if train_size < 0:               # the reference slices `mask[:, train_size:]`: negative counts from the end
            train_size = max(sz + train_size, 0)
        rows = torch.arange(sz).unsqueeze(1)
        cols = torch.arange(sz).unsqueeze(0)
        allowed = (cols < train_size) | (rows == cols)
        return torch.zeros(sz, sz).masked_fill(~allowed, float('-inf'))

    def init_weights(self):
        # reference transformer.py:43-53: attention out-projection and the second MLP matrix start at zero
        for layer in self.transformer_encoder.layers:
            for t in (layer.linear2.weight, layer.linear2.bias, layer.self_attn.out_proj.weight,
                      layer.self_attn.out_proj.bias):
                nn.init.zeros_(t)

    # ---- forward -------------------------------------------------------------------------------------------
    def _fused_embed_ok(self):
        return (isinstance(self.encoder, nn.Linear) and isinstance(self.y_encoder, nn.Linear)
                and self.y_encoder.in_features == 1 and self.encoder.bias is not None
                and self.y_encoder.bias is not None and self.input_ln is None and self.encoder.in_features <= 64
                and (self.pos_encoder is None or isinstance(self.pos_encoder, NoPositionalEncoding)))

    def _default_decoder(self):
        d = self.decoder
        return (isinstance(d, nn.Sequential) and len(d) == 3 and isinstance(d[0], nn.Linear)
                and isinstance(d[1], nn.GELU) and getattr(d[1], 'approximate', 'none') == 'none'
                and isinstance(d[2], nn.Linear) and d[0].bias is not None and d[2].bias is not None)

    def forward(self, src, src_mask=None, single_eval_pos=None):
        assert single_eval_pos is not None, 'Single eval pos is required now.'
        assert isinstance(src, tuple), 'the fused x/y input mode cannot be combined with single_eval_pos'
        x_src, y_src = src
        if src_mask is not None:
            # The kernels implement exactly the mask the reference builds when none is given (transformer.py:62-65:
            # generate_D_q_matrix(T, T - single_eval_pos)).  A caller that passes that very mask gets the same fast path; any
            # other attention pattern is rejected rather than silently replaced.
            sep_chk = int(single_eval_pos)
            T_chk = x_src.shape[0]
            sep_chk = min(max(sep_chk + T_chk, 0) if sep_chk < 0 else sep_chk, T_chk)
            expect = self.generate_D_q_matrix(T_chk, T_chk - sep_chk).to(src_mask.device)
            if src_mask.shape != expect.shape or not torch.equal(src_mask.to(expect.dtype), expect):
                raise NotImplementedError(
                    "src_mask differs from generate_D_q_matrix(T, T - single_eval_pos): the sm_90a attention kernels "
                    "implement that mask implicitly and no other (reference transformer.py:60)")
        if not x_src.is_cuda:
            raise RuntimeError(
                "TransformerModel.forward runs on hand-written sm_90a kernels only; inputs are on "
                f"{x_src.device}. Move model and data to a CUDA device (there is no CPU fallback).")
        T, B = x_src.shape[0], x_src.shape[1]
        sep = int(single_eval_pos)
        if sep < 0:                      # python slicing semantics of the reference (priors/omniglot.py:75 uses -1)
            sep = max(sep + T, 0)
        sep = min(sep, T)
        precision = self.precision
        dt = engine.act_dtype(precision)

        if self._fused_embed_ok():
            h = engine.EmbedFn.apply(x_src, y_src, self.encoder.weight, self.encoder.bias, self.y_encoder.weight,
                                     self.y_encoder.bias, sep, precision)
        else:
            xs = self.encoder(x_src)
            ys = self.y_encoder(y_src.unsqueeze(-1) if y_src.dim() == 2 else y_src)
            h = torch.cat([xs[:sep] + ys[:sep], xs[sep:]], 0)
            if self.input_ln is not None:
                h = self.input_ln(h)
            if self.pos_encoder is not None:
                h = self.pos_encoder(h)
            h = h.reshape(T * B, self.ninp).to(dt)

        params = []
        for layer in self.transformer_encoder.layers:
            params.extend(engine.layer_params(layer))
        drop = None
        if self.training and self.dropout > 0:
            # one seed per forward from torch's CPU generator (reproducible under torch.manual_seed, no device sync); the
            # kernels derive per-layer / per-site counter-based masks from it
            drop = (draw_seed(), L_drop_threshold(self.dropout))
        h = engine.EncoderStackFn.apply(h, T, B, sep, self.nhead, precision, torch.is_grad_enabled(), drop, *params)

        hq = h[sep * B:]
        if self._default_decoder():
            out = engine.DecoderFn.apply(hq, self.decoder[0].weight, self.decoder[0].bias, self.decoder[2].weight,
                                         self.decoder[2].bias, precision)
        else:
            out = self.decoder(hq.float())
        return out.reshape(T - sep, B, -1)
