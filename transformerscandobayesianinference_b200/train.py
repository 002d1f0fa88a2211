"""Drop-in `train.train` (reference train.py:22-135) on the sm_90a engine.

Same signature, defaults, prints and return value `(total_loss, positional_losses, model_on_cpu)`.  Differences that
do not change results: the model forward/backward and the criterion run on hand-written CUDA kernels; the mask is
never built; per-step `.item()` syncs are replaced by on-device accumulation read once per epoch; the prior loader
samples the NEXT batch on a side stream while this step runs; under torchrun (WORLD_SIZE > 1) `batch_size` is the
GLOBAL batch, sharded over ranks (each rank seeds its sampler differently) with one gradient all-reduce per
optimizer step (parallel.py).

`build_trainer(...)` returns the `Trainer` that `train()` drives; `bench.py` times exactly `Trainer.step`, i.e. the
public path, not a re-implementation of it.
"""
import inspect
import os
import time

import numpy as np
import torch
from torch import nn

from . import encoders, positional_encodings, parallel
from .bar_distribution import BarDistribution, FullSupportBarDistribution, get_bucket_limits  # noqa: F401
from .transformer import TransformerModel, dataset_seps, is_per_dataset
from .utils import (get_cosine_schedule_with_warmup, get_openai_lr, StoreDictKeyPair,  # noqa: F401
                    get_weighted_single_eval_pos_sampler, get_uniform_single_eval_pos_sampler)


class Losses():
    gaussian = nn.GaussianNLLLoss(full=True, reduction='none')
    mse = nn.MSELoss(reduction='none')
    ce = nn.CrossEntropyLoss(reduction='none')
    bce = nn.BCEWithLogitsLoss(reduction='none')
    get_BarDistribution = BarDistribution


def _is_bar(criterion):
    return isinstance(criterion, BarDistribution) or "BarDistribution" in criterion.__class__.__name__


def _loader_accepts_device(priordataloader_class):
    """True when the prior's `get_batch` takes a `device` keyword (all priors of this package do)."""
    fn = getattr(priordataloader_class, 'get_batch_method', None)
    if fn is None:
        return False
    try:
        return 'device' in inspect.signature(fn).parameters
    except (TypeError, ValueError):
        return False


class Trainer:
    """Everything `train()` builds (loader, model, criterion, optimizer, scheduler) plus the inner step
    (reference train.py:58-110).  One instance per process / rank."""

    def __init__(self, priordataloader_class, criterion, encoder_generator, emsize, nhid, nlayers, nhead, dropout,
                 epochs, steps_per_epoch, batch_size, bptt, lr, warmup_epochs, input_normalization,
                 y_encoder_generator, pos_encoder_generator, decoder, extra_prior_kwargs_dict, scheduler,
                 load_weights_from_this_state_dict, single_eval_pos_gen, gpu_device, aggregate_k_gradients):
        world = parallel.world_size()
        if world > 1 and torch.cuda.is_available():
            gpu_device = f'cuda:{torch.cuda.current_device()}'
        device = gpu_device if torch.cuda.is_available() else 'cpu:0'
        print(f'Using {device} device')
        assert batch_size % world == 0, f'global batch {batch_size} must be divisible by the world size {world}'
        self.world, self.rank = world, parallel.rank()
        self.batch_size = batch_size
        self.device = device
        self.bptt = bptt
        self.steps_per_epoch = steps_per_epoch
        self.aggregate_k_gradients = aggregate_k_gradients
        self.single_eval_pos_gen = single_eval_pos_gen
        self.criterion = criterion
        local_batch = batch_size // world
        prior_kwargs = dict(extra_prior_kwargs_dict)
        on_cuda = torch.device(device).type == 'cuda'
        # the prior samples where the model lives (the reference priors default to `utils.default_device` = cuda:0, which
        # is wrong for every rank but 0 and for gpu_device='cuda:1')
        if on_cuda and 'device' not in prior_kwargs and _loader_accepts_device(priordataloader_class):
            prior_kwargs['device'] = device
        self.dl = priordataloader_class(num_steps=steps_per_epoch, batch_size=local_batch, seq_len=bptt, **prior_kwargs)
        dl = self.dl

        encoder = encoder_generator(dl.num_features + 1 if dl.fuse_x_y else dl.num_features, emsize)
        n_out = dl.num_outputs
        if isinstance(criterion, nn.GaussianNLLLoss):
            n_out *= 2
        elif _is_bar(criterion):
            assert n_out == 1
            n_out = criterion.num_bars
        self.n_out = n_out
        model = TransformerModel(encoder, n_out, emsize, nhead, nhid, nlayers, dropout,
                                 y_encoder=y_encoder_generator(1, emsize), input_normalization=input_normalization,
                                 pos_encoder=(pos_encoder_generator or positional_encodings.NoPositionalEncoding)(emsize, bptt * 2),
                                 decoder=decoder)
        model.criterion = criterion
        if load_weights_from_this_state_dict is not None:
            model.load_state_dict(load_weights_from_this_state_dict)
        model.to(device)
        parallel.broadcast_parameters(model)
        self.model = model

        if world > 1:
            # Distinct prior draws per rank: every rank arrives here with the same torch / numpy generator state (same
            # default seed or the same user seed), so shift each by the rank.  Python's `random` stays shared: it drives the
            # single_eval_pos samplers, which must agree across ranks (and are broadcast per epoch anyway).
            base = torch.initial_seed()
            torch.manual_seed(base + self.rank)
            np.random.seed((int(np.random.get_state()[1][0]) + self.rank) % (2 ** 32))

        if lr is None:
            lr = get_openai_lr(model)
            print(f"Using OpenAI max lr of {lr}.")
        # reference train.py:55 torch.optim.Adam + :94 clip_grad_norm_(1.): on CUDA one fused clip + update (optim.py)
        if on_cuda and os.environ.get("PFN_B200_FUSED_ADAM", "1") != "0":       # (knob for A/B runs)
            from .optim import FusedClipAdam
            self.optimizer = FusedClipAdam(model.parameters(), lr=lr, max_grad_norm=1.)
        else:
            self.optimizer = torch.optim.Adam(model.parameters(), lr=lr, **({'fused': True} if on_cuda else {}))
        self.scheduler = scheduler(self.optimizer, warmup_epochs, epochs)
        self.params = [p for p in model.parameters() if p.requires_grad]
        self._micro = 0
        # data parallel: bucketed all-reduce overlapped with the backward (one micro-batch per optimizer step); with gradient
        # accumulation the accumulated buffer is reduced once at the end instead (reference semantics, train.py:92-97)
        self.reducer = parallel.OverlappedGradReducer() if (world > 1 and on_cuda and aggregate_k_gradients == 1) else None

    # ------------------------------------------------------------------------------------------------------------
    def local_seps(self, single_eval_pos, T):
        """(single_eval_pos for this rank's forward, this rank's values, global number of query rows) of one step.
        A scalar gives (itself, None, None).  B values for the global batch (batch_size of them, validated) give this
        rank's slice of them; the forward takes the slice, or the common value when all B are equal (the scalar step,
        whose loss is the mean: the count is then None).  A slice without a query row (every value T, while other ranks
        have some) runs the forward at T - 1, so that the rank still takes part in the gradient reduction; its one row
        per dataset is masked out of the loss."""
        if not is_per_dataset(single_eval_pos):
            return single_eval_pos, None, None
        seps = dataset_seps(single_eval_pos, T, self.batch_size, "Trainer.step")
        n_query = sum(T - s for s in seps)
        if n_query == 0:
            raise ValueError("Trainer.step: single_eval_pos leaves no query row in the batch")
        local = self.batch_size // self.world
        mine = seps[self.rank * local:(self.rank + 1) * local]
        if len(set(seps)) == 1:
            return seps[0], mine, None
        return (T - 1 if min(mine) == T else mine), mine, n_query

    @staticmethod
    def query_mask(T, rows, seps, device):
        """Bool [rows, len(seps)]: row r of the last `rows` sequence positions is a query of dataset b."""
        pos = torch.arange(T - rows, T, device=device).unsqueeze(1)
        return pos >= torch.tensor(seps, dtype=torch.long, device=device).unsqueeze(0)

    def step(self, data, targets, single_eval_pos):
        """One training step on one batch (reference train.py:64-97).  Returns (loss, losses) on the device; the
        optimizer steps every `aggregate_k_gradients`-th call.  single_eval_pos may be one value per dataset of the
        global batch: the per-row losses are then kept on each dataset's query rows only, and the loss is their sum over
        (global query rows / world), so that the data-parallel mean is the global batch's mean."""
        device, criterion, model, n_out = self.device, self.criterion, self.model, self.n_out
        T = targets.shape[0]
        single_eval_pos, mine, n_query = self.local_seps(single_eval_pos, T)
        data = tuple(e.to(device) for e in data) if isinstance(data, tuple) else data.to(device)
        output = model(data, single_eval_pos=single_eval_pos)
        self.forward_done_time = time.time()

        if n_query is not None:
            targets = targets[T - output.shape[0]:]
        elif single_eval_pos is not None:
            targets = targets[single_eval_pos:]
        if isinstance(criterion, nn.GaussianNLLLoss):
            assert output.shape[-1] == 2, \
                'need to write a little bit of code to handle multiple regression targets at once'
            mean_pred = output[..., 0]
            var_pred = output[..., 1].abs()
            losses = criterion(mean_pred.flatten(), targets.to(device).flatten(), var=var_pred.flatten())
        elif isinstance(criterion, (nn.MSELoss, nn.BCEWithLogitsLoss)):
            losses = criterion(output.flatten(), targets.to(device).flatten())
        else:
            losses = criterion(output.reshape(-1, n_out), targets.to(device).flatten())
        losses = losses.view(*output.shape[0:2]).squeeze(-1)

        if n_query is not None:
            query = self.query_mask(T, output.shape[0], mine, losses.device)
            loss = torch.where(query, losses.view(query.shape), 0.).sum() / (n_query / self.world)
        else:
            loss = losses.mean()
        if self.reducer is not None:
            from . import engine
            self.reducer.install(engine)
            try:
                loss.backward()
            finally:
                self.reducer.uninstall(engine)
        else:
            loss.backward()
        self._micro += 1
        if self._micro % self.aggregate_k_gradients == 0:
            if self.reducer is not None:
                self.reducer.finish(self.params)
            else:
                parallel.allreduce_gradients(self.params)
            if not getattr(self.optimizer, "max_grad_norm", 0):          # FusedClipAdam clips inside its step
                torch.nn.utils.clip_grad_norm_(model.parameters(), 1.)
            self.optimizer.step()
            self.optimizer.zero_grad()
        return loss, losses

    def draw_single_eval_positions(self, n):
        """One single_eval_pos per global step, identical on every rank (reference train.py:69)."""
        gen = self.single_eval_pos_gen
        seps = [gen() if callable(gen) else gen for _ in range(n)]
        return parallel.broadcast_object(seps)

    def train_epoch(self):
        model, dl, device, bptt = self.model, self.dl, self.device, self.bptt
        model.train()
        total_loss = torch.zeros((), device=device)
        pos_loss = torch.zeros(bptt, device=device)
        pos_count = torch.zeros(bptt, device=device)
        before_get_batch = time.time()
        assert len(dl) % self.aggregate_k_gradients == 0, \
            'Please set the number of steps per epoch s.t. `aggregate_k_gradients` divides it.'
        seps = self.draw_single_eval_positions(len(dl))
        time_to_get_batch = forward_time = step_time = 0.
        self._micro = 0
        ragged = False
        for batch, (data, targets) in enumerate(dl):
            time_to_get_batch = time.time() - before_get_batch
            before_forward = time.time()
            single_eval_pos = seps[batch]
            loss, losses = self.step(data, targets, single_eval_pos)
            single_eval_pos, mine, _ = self.local_seps(single_eval_pos, targets.shape[0])
            forward_time = self.forward_done_time - before_forward
            step_time = time.time() - before_forward

            ld = loss.detach()
            total_loss += ld
            if mine is not None:
                # a step with one value per dataset: each dataset's mean query-row loss in the bucket of its own value
                ragged = True
                query = self.query_mask(targets.shape[0], losses.numel() // len(mine), mine, device)
                n_q = query.sum(0)
                mean = torch.where(query, losses.detach().view(query.shape), 0.).sum(0) / n_q.clamp(min=1)
                idx = torch.tensor(mine, device=device)
                has = n_q > 0
                pos_loss.index_add_(0, idx[has], mean[has])
                pos_count.index_add_(0, idx[has], torch.ones_like(mean[has]))
            elif single_eval_pos is None:
                pos_loss += losses.mean(1).detach()
                pos_count += 1
            else:
                pos_loss[single_eval_pos] += ld
                pos_count[single_eval_pos] += 1
            before_get_batch = time.time()

        if _is_bar(self.criterion) and hasattr(self.criterion, 'check_support'):
            self.criterion.check_support()
        total_loss = parallel.allreduce_mean_scalar(total_loss)
        pos_loss = parallel.allreduce_mean_scalar(pos_loss)
        if ragged:      # the ranks' datasets fall in different buckets: the mean is their sum over the summed counts
            pos_count = parallel.allreduce_mean_scalar(pos_count)
        return (total_loss.item() / self.steps_per_epoch, (pos_loss / pos_count).tolist(), time_to_get_batch,
                forward_time, step_time)


def build_trainer(priordataloader_class, criterion, encoder_generator, emsize=200, nhid=200, nlayers=6, nhead=2,
                  dropout=0.2, epochs=10, steps_per_epoch=100, batch_size=200, bptt=10, lr=None, warmup_epochs=10,
                  input_normalization=False, y_encoder_generator=None, pos_encoder_generator=None, decoder=None,
                  extra_prior_kwargs_dict={}, scheduler=get_cosine_schedule_with_warmup,
                  load_weights_from_this_state_dict=None, validation_period=10, single_eval_pos_gen=None,
                  gpu_device='cuda:0', aggregate_k_gradients=1, verbose=True):
    """Same arguments as `train()`; returns the Trainer without running an epoch."""
    return Trainer(priordataloader_class, criterion, encoder_generator, emsize, nhid, nlayers, nhead, dropout, epochs,
                   steps_per_epoch, batch_size, bptt, lr, warmup_epochs, input_normalization, y_encoder_generator,
                   pos_encoder_generator, decoder, extra_prior_kwargs_dict, scheduler,
                   load_weights_from_this_state_dict, single_eval_pos_gen, gpu_device, aggregate_k_gradients)


def train(priordataloader_class, criterion, encoder_generator, emsize=200, nhid=200, nlayers=6, nhead=2, dropout=0.2,
          epochs=10, steps_per_epoch=100, batch_size=200, bptt=10, lr=None, warmup_epochs=10, input_normalization=False,
          y_encoder_generator=None, pos_encoder_generator=None, decoder=None, extra_prior_kwargs_dict={},
          scheduler=get_cosine_schedule_with_warmup, load_weights_from_this_state_dict=None, validation_period=10,
          single_eval_pos_gen=None, gpu_device='cuda:0', aggregate_k_gradients=1, verbose=True):
    tr = Trainer(priordataloader_class, criterion, encoder_generator, emsize, nhid, nlayers, nhead, dropout, epochs,
                 steps_per_epoch, batch_size, bptt, lr, warmup_epochs, input_normalization, y_encoder_generator,
                 pos_encoder_generator, decoder, extra_prior_kwargs_dict, scheduler, load_weights_from_this_state_dict,
                 single_eval_pos_gen, gpu_device, aggregate_k_gradients)
    model, dl, scheduler = tr.model, tr.dl, tr.scheduler

    total_loss = float('inf')
    total_positional_losses = float('inf')
    prev_defer = BarDistribution.defer_support_check
    BarDistribution.defer_support_check = True
    try:
        for epoch in range(1, epochs + 1):
            epoch_start_time = time.time()
            total_loss, total_positional_losses, time_to_get_batch, forward_time, step_time = tr.train_epoch()
            if hasattr(dl, 'validate') and epoch % validation_period == 0:
                with torch.no_grad():
                    val_score = dl.validate(model)
            else:
                val_score = None
            if verbose:
                print('-' * 89)
                print(
                    f'| end of epoch {epoch:3d} | time: {(time.time() - epoch_start_time):5.2f}s | mean loss {total_loss:5.2f} | '
                    f"pos losses {','.join([f'{l:5.2f}' for l in total_positional_losses])}, lr {scheduler.get_last_lr()[0]}"
                    f' data time {time_to_get_batch:5.2f} step time {step_time:5.2f}'
                    f' forward time {forward_time:5.2f}' + (f'val score {val_score}' if val_score is not None else ''))
                print('-' * 89)
            scheduler.step()
    finally:
        BarDistribution.defer_support_check = prev_defer
    return total_loss, total_positional_losses, model.to('cpu')


# ---- command line (reference train.py:137-287) --------------------------------------------------------------
# `python -m transformerscandobayesianinference_b200.train gp --loss_function barnll --min_y -3 --max_y 3 ...`
# Same positional / optional arguments, defaults and `--config file.yaml` override as the reference script; the choices the
# reference names but cannot construct (encoders 'mlp' / 'positional', prior 'stroke') are rejected up front.
_CLI_PRIORS = {'gp': 'fast_gp', 'mix_gp': 'fast_gp_mix', 'ridge': 'ridge'}
_CLI_POS_ENCODERS = {'none': None, 'sinus': 'PositionalEncoding', 'learned': 'LearnedPositionalEncoding',
                     'paired_scrambled_learned': 'PairedScrambledPositionalEncodings'}
_CLI_SAMPLERS = {'weighted': get_weighted_single_eval_pos_sampler, 'uniform': get_uniform_single_eval_pos_sampler}


def _cli_parser():
    import argparse
    ap = argparse.ArgumentParser(prog='train', description='Train a PFN on a prior (sm_90a engine).')
    ap.add_argument('prior', help='gp | mix_gp | ridge')
    ap.add_argument('--config', help='yaml file whose keys override the defaults below')
    ap.add_argument('--loss_function', default='barnll',
                    help='barnll | adaptivebarnll | adaptivefullsupportbarnll | ce | gaussnll | mse')
    ap.add_argument('--min_y', type=float, help='lower end of the bar distribution support (barnll)')
    ap.add_argument('--max_y', type=float, help='upper end of the bar distribution support (barnll)')
    ap.add_argument('--num_buckets', default=100, type=int)
    ap.add_argument('--extra_prior_kwargs_dict', default={'fuse_x_y': False}, action=StoreDictKeyPair, nargs='+',
                    metavar='KEY=VAL', help='forwarded to the prior DataLoader')
    ap.add_argument('--encoder', default='linear')
    ap.add_argument('--y_encoder', default='linear')
    ap.add_argument('--pos_encoder', default='sinus', help=' | '.join(_CLI_POS_ENCODERS))
    ap.add_argument('--bptt', default=10, type=int)
    ap.add_argument('--epochs', default=200, type=int)
    ap.add_argument('--warmup_epochs', default=50, type=int)
    ap.add_argument('--validation_period', default=10, type=int)
    ap.add_argument('--permutation_invariant_max_eval_pos', default=None, type=int)
    ap.add_argument('--permutation_invariant_sampling', default='weighted', help='weighted | uniform')
    ap.add_argument('--emsize', default=512, type=int)
    ap.add_argument('--nlayers', default=6, type=int)
    ap.add_argument('--nhid', default=None, type=int, help='default: 2 * emsize')
    ap.add_argument('--nhead', default=4, type=int)
    ap.add_argument('--dropout', default=.0, type=float)
    ap.add_argument('--steps_per_epoch', default=10, type=int)
    ap.add_argument('--batch_size', default=1000, type=int)
    ap.add_argument('--lr', '--learning_rate', default=.001, type=float)
    return ap


def resolve_cli(argv=None):
    """Parse the reference's command line into `(prior DataLoader class, criterion, encoder generator, train kwargs)`."""
    import importlib
    ap = _cli_parser()
    known, _ = ap.parse_known_args(argv)
    if known.config:
        import yaml
        with open(known.config) as f:
            ap.set_defaults(**yaml.safe_load(f))
    a = vars(ap.parse_args(argv))
    a.pop('config')
    if a['nhid'] is None:
        a['nhid'] = 2 * a['emsize']

    prior_name = a.pop('prior')
    if prior_name not in _CLI_PRIORS:
        raise NotImplementedError(f'Prior == {prior_name}.')
    prior = importlib.import_module(f'{__package__}.priors.{_CLI_PRIORS[prior_name]}').DataLoader

    def y_sample():
        dl = prior(num_steps=1, batch_size=a['batch_size'] * a['steps_per_epoch'], seq_len=a['bptt'],
                   **a['extra_prior_kwargs_dict'])
        ys = next(iter(dl))[-1]
        print(f'Creating Bar distribution with borders from y sample of size {ys.numel()}')
        return ys

    loss, nb, lo, hi = a.pop('loss_function'), a.pop('num_buckets'), a.pop('min_y'), a.pop('max_y')
    if loss == 'ce':
        criterion = nn.CrossEntropyLoss(reduction='none')
    elif loss == 'gaussnll':
        criterion = nn.GaussianNLLLoss(reduction='none', full=True)
    elif loss == 'mse':
        criterion = nn.MSELoss(reduction='none')
    elif loss == 'barnll':
        criterion = BarDistribution(borders=get_bucket_limits(nb, full_range=(lo, hi)))
    elif loss == 'adaptivebarnll':
        criterion = BarDistribution(borders=get_bucket_limits(nb, ys=y_sample(), full_range=(lo, hi)))
    elif loss == 'adaptivefullsupportbarnll':
        assert lo is None and hi is None, 'Please do not specify `min_y` and `max_y` with `adaptivefullsupportbarnll`.'
        criterion = FullSupportBarDistribution(borders=get_bucket_limits(nb, ys=y_sample()))
    else:
        raise NotImplementedError(f'loss_function == {loss}.')

    def encoder_generator(name):
        if name != 'linear':
            raise NotImplementedError(f'A {name} encoder is not valid.')
        return encoders.Linear

    enc, y_enc = encoder_generator(a.pop('encoder')), encoder_generator(a.pop('y_encoder'))
    pos = a.pop('pos_encoder')
    if pos not in _CLI_POS_ENCODERS:
        raise NotImplementedError(f'pos_encoder == {pos} is not valid.')
    pos_gen = getattr(positional_encodings, _CLI_POS_ENCODERS[pos]) if _CLI_POS_ENCODERS[pos] else None

    max_pos, sampling = a.pop('permutation_invariant_max_eval_pos'), a.pop('permutation_invariant_sampling')
    if max_pos is not None:
        if sampling not in _CLI_SAMPLERS:
            raise ValueError(f'permutation_invariant_sampling == {sampling}')
        a['single_eval_pos_gen'] = _CLI_SAMPLERS[sampling](max_pos)
    a.update(y_encoder_generator=y_enc, pos_encoder_generator=pos_gen)
    return prior, criterion, enc, a


def main(argv=None):
    prior, criterion, enc, kwargs = resolve_cli(argv)
    print('ARGS for `train`:', kwargs)
    return train(prior, criterion, enc, **kwargs)


if __name__ == '__main__':
    main()
