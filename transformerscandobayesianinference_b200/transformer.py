"""Drop-in `transformer.TransformerModel` (reference transformer.py:13-91) whose forward runs on the sm_90a engine.

The module keeps `self.transformer_encoder = nn.TransformerEncoder(...)` purely as the *parameter container*:
identical state_dict keys (the five reference checkpoints under results/ load with strict=True), identical
construction-time RNG consumption and the reference's zero-init of `linear2` / `out_proj` — but its forward is
never called.  `forward()` routes embedding -> encoder stack -> decoder through `engine.*Fn`.

For inference against one training set, `encode_context(x_train, y_train)` runs the training rows once and keeps every
layer's K and V of them; `predict(ctx, x_query)` then scores any number of query sets against that context.  Under the
single_eval_pos mask a training row attends only to training rows and a query row to the training rows and itself, so
`predict` returns what `forward` returns for the concatenated sequence at single_eval_pos = n.  `predict` is
differentiable in x_query (with the context and the parameters held constant), so candidate points can be optimised by
gradient against one cached context; `forward` is differentiable in x and y as the reference's module is.  With
`encode_context(x_train, y_train, n_train)` the datasets of one batch have training sets of their own sizes: dataset b
uses rows [0, n_train[b]) and the rows after them are padding that never reaches an output.

`forward(src, single_eval_pos=seps)` with B values trains on datasets of different training-set sizes in one batch:
dataset b's rows attend under its own separator seps[b], and `query_rows(T, seps)` marks which of the returned rows are
its queries.
"""
import numbers

import torch
import torch.nn as nn
from torch.nn import TransformerEncoder, TransformerEncoderLayer

from . import decoders, engine
from ._lib import draw_seed, drop_threshold as L_drop_threshold
from .positional_encodings import NoPositionalEncoding
from .utils import SeqBN


def _require_cuda_input(x, method):
    if not x.is_cuda:
        raise RuntimeError(
            f"TransformerModel.{method} runs on hand-written sm_90a kernels only; inputs are on "
            f"{x.device}. Move model and data to a CUDA device (there is no CPU fallback).")


class TrainingContext:
    """What `TransformerModel.encode_context` keeps of n training rows: `kv` [nlayers, n*B, 2*E] holds each layer's K | V
    of the rows (token row t*B + b, the model's activation dtype), plus the shapes and the precision it was made with.
    `n_train` is None when every dataset has all n rows, else the int32 [B] device tensor of each dataset's row count.
    It holds no weights: `predict` uses the model it is called on.  `predict` never writes to it, and a backward through
    `predict` treats it as a constant: no gradient reaches the training rows through it (differentiate `forward` on the
    concatenated sequence for that)."""
    __slots__ = ("kv", "n", "B", "E", "nhead", "nlayers", "precision", "device", "n_train")

    def __init__(self, kv, n, B, E, nhead, nlayers, precision, device, n_train=None):
        self.kv, self.n, self.B, self.E, self.nhead, self.nlayers = kv, n, B, E, nhead, nlayers
        self.precision, self.device = precision, torch.device(device)
        self.n_train = n_train


def _dataset_ints(values, n, B, who, name, noun, rows):
    """values (B integers in [0, n]: a sequence or an integer tensor on any device) as a tuple of ints; ValueError
    otherwise.  who, name: the caller and its argument; noun: what the values are; rows: what n counts."""
    if torch.is_tensor(values):
        if values.dtype.is_floating_point or values.dtype.is_complex or values.dtype == torch.bool:
            raise ValueError(f"{who}: {name} must hold integers, got a {values.dtype} tensor")
        if values.dim() != 1:
            raise ValueError(f"{who}: {name} must be one-dimensional, got shape {tuple(values.shape)}")
        ints = values.tolist()
    else:
        ints = list(values)
        for v in ints:
            if isinstance(v, bool) or not isinstance(v, numbers.Integral):
                raise ValueError(f"{who}: {name} must hold integers, got {v!r}")
        ints = [int(v) for v in ints]
    if len(ints) != B:
        raise ValueError(f"{who}: {name} holds {len(ints)} {noun} for a batch of {B} datasets")
    bad = [v for v in ints if not 0 <= v <= n]
    if bad:
        raise ValueError(f"{who}: {name} values must lie in [0, {n}] ({rows}), got {bad[0]}")
    return tuple(ints)


def _training_set_sizes(n_train, n, B):
    """n_train (B integers in [0, n]: a sequence or an integer tensor on any device) as a tuple of ints; ValueError
    otherwise."""
    return _dataset_ints(n_train, n, B, "encode_context", "n_train", "sizes", "the rows of x_train")


def is_per_dataset(single_eval_pos):
    """True when single_eval_pos is one value per dataset (a sequence, or a tensor or array with a dimension) rather than
    one for the whole batch."""
    if torch.is_tensor(single_eval_pos) or hasattr(single_eval_pos, "ndim"):
        return single_eval_pos.ndim >= 1
    return isinstance(single_eval_pos, (list, tuple))


def dataset_seps(single_eval_pos, T, B, who="forward"):
    """The per-dataset single_eval_pos (B integers in [0, T]) as a tuple of ints; ValueError otherwise."""
    return _dataset_ints(single_eval_pos, T, B, who, "single_eval_pos", "values", "the sequence length")


def _call_params(linear, frozen):
    """(weight, bias) of an nn.Linear, detached when frozen."""
    return (linear.weight.detach(), linear.bias.detach()) if frozen else (linear.weight, linear.bias)


def _call_module(module, frozen, x):
    """module(x), with every parameter of the module detached for the call when frozen."""
    if not frozen:
        return module(x)
    return torch.func.functional_call(module, {k: p.detach() for k, p in module.named_parameters()}, (x,))


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

    def _embed(self, x_src, y_src, sep, frozen=False):
        """[T*B, E] activation-dtype input of the encoder stack: the x embedding of every row plus the y embedding of the
        rows t < sep (t < n_keys[b] in dataset b for an engine.RaggedSeps).  frozen: the encoders' parameters are
        constants of the call, so a backward reaches the inputs only."""
        T, B = x_src.shape[0], x_src.shape[1]
        precision = self.precision
        if self._fused_embed_ok():
            return engine.EmbedFn.apply(x_src, y_src, *_call_params(self.encoder, frozen),
                                        *_call_params(self.y_encoder, frozen), sep, precision)
        xs = _call_module(self.encoder, frozen, x_src)
        ys = _call_module(self.y_encoder, frozen, y_src.unsqueeze(-1) if y_src.dim() == 2 else y_src)
        if isinstance(sep, engine.RaggedSeps):
            train = torch.arange(T, device=xs.device).unsqueeze(1) < sep.n_keys.to(xs.device)
            h = torch.where(train.unsqueeze(-1), xs + ys, xs)
        else:
            h = torch.cat([xs[:sep] + ys[:sep], xs[sep:]], 0)
        if self.input_ln is not None:
            h = self.input_ln(h)
        if self.pos_encoder is not None:
            h = self.pos_encoder(h)
        return h.reshape(T * B, self.ninp).to(engine.act_dtype(precision))

    def _layer_params(self):
        params = []
        for layer in self.transformer_encoder.layers:
            params.extend(engine.layer_params(layer))
        return params

    def _decode(self, hq, rows, B, frozen=False):
        """Logits [rows, B, n_out] of the decoder on the output hq [rows*B, E] of the query rows.  frozen: the decoder's
        parameters are constants of the call."""
        precision = self.precision
        if self._default_decoder():
            out = engine.DecoderFn.apply(hq, *_call_params(self.decoder[0], frozen), *_call_params(self.decoder[2], frozen),
                                         precision)
        elif isinstance(self.decoder, (decoders.ScaledDecoder, decoders.FixedScaledDecoder)):
            out = self.decoder.fused(hq, (rows, B), precision, frozen)
        else:
            # any other head runs as its own torch ops on the sequence-first [T - sep, B, E] rows, the shape the reference
            # hands its decoder (reference transformer.py:85)
            out = _call_module(self.decoder, frozen, hq.float().view(rows, B, -1))
        return out.reshape(rows, B, -1)

    @staticmethod
    def query_rows(T, single_eval_pos):
        """Bool [T - s_min, B] mask of the rows of forward(..., single_eval_pos)'s output that are queries: row r of
        dataset b is sequence position s_min + r, a query when it is >= single_eval_pos[b].  s_min = min(single_eval_pos)
        for B values (the mask is then on their device, the CPU for a sequence); for a scalar every row is a query and
        the mask has one column."""
        if not is_per_dataset(single_eval_pos):
            sep = int(single_eval_pos)
            sep = min(max(sep + T, 0) if sep < 0 else sep, T)
            return torch.ones(T - sep, 1, dtype=torch.bool)
        n = len(single_eval_pos)
        seps = dataset_seps(single_eval_pos, T, n, "query_rows")
        dev = single_eval_pos.device if torch.is_tensor(single_eval_pos) else torch.device("cpu")
        s_min = min(seps) if seps else 0
        pos = torch.arange(s_min, T, device=dev).unsqueeze(1)
        return pos >= torch.tensor(seps, dtype=torch.long, device=dev).unsqueeze(0)

    def forward(self, src, src_mask=None, single_eval_pos=None):
        """Logits [T - sep, B, n_out] of the rows t >= single_eval_pos.  single_eval_pos may also be B integers in [0, T],
        one per dataset (a sequence, or an integer tensor on any device): dataset b's rows then attend under
        generate_D_q_matrix at its own value, the y embedding is added to its rows t < single_eval_pos[b], and the
        result has T - min(single_eval_pos) rows; `query_rows` marks which are the queries.  B equal values run the
        scalar path.  The logits are differentiable in x and y (src) as well as in the parameters: y's gradient is zero
        on the query rows t >= single_eval_pos[b], which have no y embedding."""
        assert single_eval_pos is not None, 'Single eval pos is required now.'
        assert isinstance(src, tuple), 'the fused x/y input mode cannot be combined with single_eval_pos'
        x_src, y_src = src
        if is_per_dataset(single_eval_pos):
            seps = dataset_seps(single_eval_pos, x_src.shape[0], x_src.shape[1])
            if src_mask is not None:
                raise NotImplementedError("forward: an explicit src_mask cannot be combined with one single_eval_pos per "
                                          "dataset (the kernels build the per-dataset mask themselves)")
            if len(set(seps)) > 1:
                return self._forward_ragged(x_src, y_src, seps)
            single_eval_pos = seps[0]
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
        _require_cuda_input(x_src, "forward")
        T, B = x_src.shape[0], x_src.shape[1]
        sep = int(single_eval_pos)
        if sep < 0:                      # python slicing semantics of the reference (priors/omniglot.py:75 uses -1)
            sep = max(sep + T, 0)
        sep = min(sep, T)
        precision = self.precision
        h = self._embed(x_src, y_src, sep)
        params = self._layer_params()
        drop = None
        if self.training and self.dropout > 0:
            # one seed per forward from torch's CPU generator (reproducible under torch.manual_seed, no device sync); the
            # kernels derive per-layer / per-site counter-based masks from it
            drop = (draw_seed(), L_drop_threshold(self.dropout))
        h = engine.EncoderStackFn.apply(h, T, B, sep, self.nhead, precision, torch.is_grad_enabled(), drop, *params)
        return self._decode(h[sep * B:], T - sep, B)

    def _forward_ragged(self, x_src, y_src, seps):
        """forward with one separator per dataset (seps: B ints, not all equal): the embedding and the attention take
        every value, the rest of the step runs on the rows from s_min = min(seps) as the scalar path does."""
        _require_cuda_input(x_src, "forward")
        T, B = x_src.shape[0], x_src.shape[1]
        n_keys = torch.tensor(seps, dtype=torch.int32).to(x_src.device, non_blocking=True)
        sep = engine.RaggedSeps(n_keys, min(seps), max(seps))
        h = self._embed(x_src, y_src, sep)
        drop = None
        if self.training and self.dropout > 0:
            drop = (draw_seed(), L_drop_threshold(self.dropout))
        h = engine.EncoderStackFn.apply(h, T, B, sep, self.nhead, self.precision, torch.is_grad_enabled(), drop,
                                        *self._layer_params())
        return self._decode(h[sep.s_min * B:], T - sep.s_min, B)

    # ---- inference against a cached training set -------------------------------------------------------------
    def _check_context_inference(self):
        """Raise ValueError for a configuration in which a query row's result depends on more than the training rows and
        itself, or is not the same in every call."""
        if self.input_ln is not None:
            raise ValueError("encode_context / predict: input_normalization=True is not supported: SeqBN normalises each "
                             "feature over all rows of the sequence, so the training rows would depend on the queries")
        if self.pos_encoder is not None and not isinstance(self.pos_encoder, NoPositionalEncoding):
            raise ValueError(f"encode_context / predict: positional encoder {type(self.pos_encoder).__name__} is not "
                             "supported: it adds a row of its table by position, so a query's result would depend on its "
                             "index in the sequence (use None or NoPositionalEncoding)")
        if self.training and self.dropout > 0:
            raise ValueError("encode_context / predict: training-mode dropout is not supported: its masks are keyed by "
                             "the row's position in the full sequence; call model.eval() first")

    def encode_context(self, x_train, y_train, n_train=None):
        """Run the n training rows x_train [n, B, F], y_train [n, B] (n >= 0) through the embedding and every encoder
        layer on their own (they never attend to a query row) and return a `TrainingContext` holding each layer's K and
        V of them.  No autograd: the context is a constant of every `predict`.  With n = 0 a query attends only to itself, as in forward(..., single_eval_pos=0).

        n_train (optional): B integers in [0, n], a sequence or an integer tensor on any device.  Dataset b then has the
        training rows [0, n_train[b]) and `predict` gives its queries what forward gives them on those rows alone, at
        single_eval_pos = n_train[b]; rows t >= n_train[b] are padding, whatever values they hold.  None (or every size
        equal to n) runs the same kernels as a call without it."""
        self._check_context_inference()
        if x_train.dim() != 3 or y_train.shape[:2] != x_train.shape[:2]:
            raise ValueError(f"encode_context: x_train must be [n, B, F] and y_train [n, B]; got {tuple(x_train.shape)} "
                             f"and {tuple(y_train.shape)}")
        n, B = x_train.shape[0], x_train.shape[1]
        sizes = None if n_train is None else _training_set_sizes(n_train, n, B)
        if sizes is not None and all(v == n for v in sizes):
            sizes = None
        _require_cuda_input(x_train, "encode_context")
        E, nlayers = self.ninp, len(self.transformer_encoder.layers)
        dt = engine.act_dtype(self.precision)
        n_keys = None
        with torch.no_grad():
            if sizes is not None:
                # the padding rows are zeroed before the embedding: a NaN or Inf there would survive a masked key's zero
                # probability inside the attention's P V product
                n_keys = torch.tensor(sizes, dtype=torch.int32, device=x_train.device)
                keep = torch.arange(n, device=x_train.device).unsqueeze(1) < n_keys
                x_train = torch.where(keep.unsqueeze(-1), x_train, 0)
                y_train = torch.where(keep.view(*keep.shape, *(1,) * (y_train.dim() - 2)), y_train, 0)
            if n == 0:
                kv = torch.empty(nlayers, 0, 2 * E, device=x_train.device, dtype=dt)
            else:
                h = self._embed(x_train, y_train, n)
                kv = engine.encode_context(h, n, B, self.nhead, self.precision, *self._layer_params(), n_keys=n_keys)
        return TrainingContext(kv, n, B, E, self.nhead, nlayers, self.precision, x_train.device, n_keys)

    def predict(self, ctx, x_query):
        """Logits [m, B, n_out] of the query rows x_query [m, B, F] (m >= 1) given the training rows `ctx` holds: what
        forward((cat(x_train, x_query), cat(y_train, anything)), single_eval_pos=n) returns.  `ctx` is only read, so one
        context serves any number of calls.

        With grad mode on and x_query.requires_grad the call builds a graph whose backward reaches x_query only: the
        context and every parameter of the model are constants of it, so a parameter's .grad is left as it was (with the
        cached K / V held fixed a weight gradient would only be a partial derivative).  The logits are the same bits
        either way; otherwise no graph is built."""
        self._check_context_inference()
        if not isinstance(ctx, TrainingContext):
            raise ValueError(f"predict: ctx must be a TrainingContext from encode_context, got {type(ctx).__name__}")
        if x_query.dim() != 3 or x_query.shape[0] < 1:
            raise ValueError(f"predict: x_query must be [m, B, F] with m >= 1; got {tuple(x_query.shape)}")
        m, B = x_query.shape[0], x_query.shape[1]
        want = {"B": B, "E": self.ninp, "nhead": self.nhead, "nlayers": len(self.transformer_encoder.layers),
                "precision": self.precision, "device": x_query.device}
        for name, value in want.items():
            have = getattr(ctx, name)
            if have != value:
                raise ValueError(f"predict: the context's {name} is {have} but the model and queries have {value}")
        _require_cuda_input(x_query, "predict")
        if torch.is_grad_enabled() and x_query.requires_grad:
            h = self._embed(x_query, x_query.new_zeros(m, B), 0, frozen=True)
            h = engine.QueryStackFn.apply(h, ctx.kv, ctx.n, B, self.nhead, self.precision, ctx.n_train,
                                          *(p.detach() for p in self._layer_params()))
            return self._decode(h, m, B, frozen=True)
        with torch.no_grad():
            h = self._embed(x_query, x_query.new_zeros(m, B), 0)
            h = engine.query_stack(h, ctx.kv, ctx.n, B, self.nhead, self.precision, *self._layer_params(),
                                   n_keys=ctx.n_train)
            return self._decode(h, m, B)
