"""`mcmc_svi_transformer_on_bayesian` (reference mcmc_svi_transformer_on_bayesian.py): approximate inference for a
Bayesian neural network, the transformer against NUTS.

`BayesianModel` is the reference's two-layer network (:28-67: fc1 [embed, num_features], fc2 [2, embed], all weights and
biases N(0, 1), inputs N(0, 1), no nonlinearity between the layers, a categorical observation on the softmax), here
without pyro: a draw comes from csrc/bnn_prior.cu, and `eval_mcmc` runs one NUTS chain per dataset, all of them in ONE
launch of csrc/bnn_mcmc.cu (pyro 1.7's NUTS defaults as in the GP baseline; the reference runs the chains one after
another on the CPU).  `eval_transformer` evaluates all datasets in one forward pass.  PARITY WITH PYRO UNPINNED: pyro is
not installed where this is tested; the contract is the CPU restatement `oracle/gp_mcmc_oracle.nuts_chain` on the
potential of `oracle/bnn_oracle.py`, and the posterior predictive against importance sampling.

The module keeps the reference's function names, signatures, result-file names and file contents, so notebooks written
against it run; the helpers themselves are written for this package.  `eval_svi` (AutoDiagonalNormal + Trace_ELBO) and
SVGD are not provided: 'svi' and 'svgd' raise NotImplementedError in `training_steps` / `training_samples`.
`plot_features` (matplotlib at import) is not provided either.
"""
import argparse
import glob
import os
import time

import numpy as np
import scipy.stats as st
import torch
import torch.nn.functional as Fn

from . import _lib as L
from . import encoders, priors
from .train import train, Losses
from .utils import get_weighted_single_eval_pos_sampler

MCMC_MAX_TREE_DEPTH = L.GP_MCMC_MAX_DEPTH
SEQ_LEN = 300                                           # rows per toy dataset (reference :355)
MODEL_SIZES = {'small': (3, 5, 2), 'big': (8, 64, 2)}   # name -> (num_features, embed, nlayers) (reference :357-364)
TOY_DATASETS = 100                                      # datasets `generate_toy_data` draws (reference :196)
STEP_GRID = tuple(2 ** k for k in range(1, 13))         # warmup = samples of `training_steps`: 2 .. 4096 (reference :296)
TRAINING_ROWS_OF_STEP_GRID = 100                        # (reference :295)
DEFAULT_MCMC_STEPS = 512                                # warmup = samples of `training_samples` (reference :323-324)
# the transformer the paper trains for this task (reference :71-83); num_features and seq_len come from the model spec
TRANSFORMER_DEFAULTS = dict(lr=2.006434218345026e-05, epochs=400, dropout=0.0, emsize=256, batch_size=256, nlayers=5,
                            num_outputs=1, steps_per_epoch=100, nhead=4, nhid_factor=2)


class BayesianModel:
    """The reference's BayesianModel (:28-67) as a sampler: `model(seq_len=n)` returns one prior draw (x [n, F], obs [n]);
    every call draws fresh weights, as a pyro module does.  `nlayers` of the spec is ignored, as in the reference."""

    def __init__(self, model_spec, device='cuda'):
        self.device = device
        self.num_features = model_spec['num_features']
        self.embed = model_spec['embed']

    def forward(self, x=None, y=None, seq_len=1):
        if x is not None or y is not None:
            raise NotImplementedError("BayesianModel draws from the prior only; conditioning on (x, y) is what eval_mcmc does "
                                      "(sample_bnn_posterior)")
        xs, obs = priors.pyro.sample_bnn_prior(1, seq_len, self.num_features, self.embed, self.device)
        return xs[:, 0], obs[:, 0]

    __call__ = forward


def get_default_model_spec(size):
    """'small', 'big', or '<num_features>_<embed>_<nlayers>' -> the model spec dict (reference :354-370)."""
    num_features, embed, nlayers = MODEL_SIZES[size] if size in MODEL_SIZES else (int(v) for v in size.split('_')[:3])
    return {'nlayers': nlayers, 'embed': embed, 'num_features': num_features, 'seq_len': SEQ_LEN}


def get_default_evaluation_points():
    """Training-set sizes of the `training_samples` sweep: 2, 7, .., 97 (reference :372-373)."""
    return list(range(2, 100, 5))


def get_transformer_config(model_spec):
    """Hyperparameters of the transformer for a model spec (reference :70-83)."""
    return dict(TRANSFORMER_DEFAULTS, num_features=model_spec['num_features'], seq_len=model_spec['seq_len'])


def get_model(model_generator, config, should_train=True, device='cuda'):
    """`train()` on `priors.pyro.DataLoader` under the BCE loss with the given config; zero epochs when not
    `should_train` (reference :86-116).  Returns what `train` returns: (loss, positional losses, model)."""
    prior_kwargs = {'num_outputs': config['num_outputs'], 'num_features': config['num_features'], 'canonical_args': None,
                    'fuse_x_y': False, 'model': model_generator}
    return train(priors.pyro.DataLoader, Losses.bce, encoders.Linear,
                 emsize=config['emsize'], nhid=config['emsize'] * config['nhid_factor'], nlayers=config['nlayers'],
                 nhead=config['nhead'], dropout=config['dropout'], lr=config['lr'],
                 epochs=config['epochs'] if should_train else 0, warmup_epochs=config['epochs'] // 4,
                 steps_per_epoch=config['steps_per_epoch'], batch_size=config['batch_size'], bptt=config['seq_len'],
                 y_encoder_generator=encoders.Linear, pos_encoder_generator=None,
                 single_eval_pos_gen=get_weighted_single_eval_pos_sampler(100), extra_prior_kwargs_dict=prior_kwargs,
                 gpu_device=device, verbose=True)


def evaluate_preds(preds, y_test):
    """Scores of drawn classes preds['obs'] [S, m] against labels y_test [m] (reference :130-139): the accuracy of all
    S x m draws, the binary cross entropy of the per-row mean of the draws, and its squared error.  -> (acc, nll, mse)."""
    drawn = preds['obs'] > 0.5
    vote = drawn.float().mean(0)
    target = y_test.float()
    acc = (drawn == y_test).float().mean()
    return acc, Fn.binary_cross_entropy(vote, target), ((vote - target) ** 2).mean()


def compute_mean_and_conf_interval(accuracies, confidence=.95):
    """(mean, half-width of the two-sided Student-t interval of the mean) (reference :187-192)."""
    values = np.asarray(accuracies, dtype=float)
    half_width = st.sem(values) * st.t.ppf(0.5 + confidence / 2., len(values) - 1)
    return values.mean(), half_width


def load_results(path, task='steps'):
    """Reads every `{path}_*.npy` written by `training_steps` (task 'steps': (nll, acc, seconds)) or `training_samples`
    (otherwise: (training rows, nll, acc, seconds)) and returns (files, times, samples, means, conf) as arrays ordered by
    seconds for 'steps' and by training rows otherwise; means / conf are `compute_mean_and_conf_interval` of each file's
    NLLs; for 'steps' `samples` repeats the file names (reference :142-176)."""
    rows = []
    for name in glob.glob(f'{path}_*.npy'):
        print(name)
        record = list(np.load(name, allow_pickle=True))
        key = name if task == 'steps' else record.pop(0)
        nll, _, seconds = record
        rows.append((seconds if task == 'steps' else key, name, seconds, key) + compute_mean_and_conf_interval(nll))
    rows.sort(key=lambda r: r[0])
    columns = list(zip(*rows)) if rows else [()] * 6
    return tuple(np.array(c) for c in columns[1:])


def plot_with_confidence_intervals(ax_or_pyplot, x, mean, confidence, **common_kwargs):
    """A line with a translucent mean +- confidence band on the axis (or pyplot module) given (reference :178-184)."""
    ax_or_pyplot.plot(x, mean, **common_kwargs)
    band_kwargs = {k: v for k, v in common_kwargs.items() if k not in ('label', 'marker')}
    ax_or_pyplot.fill_between(x, mean - confidence, mean + confidence, alpha=.1, **band_kwargs)


def generate_toy_data(model, bptt, device='cpu'):
    """TOY_DATASETS draws of `model(seq_len=bptt)` after `torch.manual_seed(0)`, stacked: X [100, bptt, F], y [100, bptt]
    (reference :195-207)."""
    torch.manual_seed(0)
    xs, ys = zip(*(model(seq_len=bptt) for _ in range(TOY_DATASETS)))
    return torch.stack(xs).to(device), torch.stack(ys).to(device)


_KERNEL = "the Bayesian-NN NUTS baseline runs on the sm_90a kernel of csrc/bnn_mcmc.cu"


@torch.no_grad()
def sample_bnn_posterior(x_train, y_train, x_test, spec, num_samples, warmup_steps, seed, max_tree_depth=MCMC_MAX_TREE_DEPTH,
                         init=None, trace=False):
    """One pfn_bnn_mcmc launch: a NUTS chain per dataset on the posterior of the network weights theta = (W1 [E, F],
    b1 [E], W2 [2, E], b2 [2]) (flattened in that order, d values) given x_train [N, n, F], y_train [N, n] (0 / 1) on a CUDA
    device; `spec` holds 'num_features' and 'embed'.  Returns a dict of tensors with leading dim N: samples [N, S', d],
    probs [N, S', n_test] (class-1 probability of every row of x_test [N, n_test, F] under every sample), obs (one class
    drawn from each of them, fp32 0. / 1.), potential and
    grad [N, d] (U and dU/dtheta at the last state), step_size, accept (mean acceptance statistic of the sampling phase),
    diag [N, 6] int32 (columns L.GP_MCMC_DIAG_NAMES; not_pd counts non-finite potentials), and "seed".
    S' = max(num_samples, 1).  init [N, d] gives the starting theta; num_samples = warmup_steps = 0 then only evaluates U,
    its gradient and the probabilities at init.  trace=True adds "trace" [N, W + S, d + 2]: per iteration theta, the step
    size used and the tree depth."""
    F, E = int(spec['num_features']), int(spec['embed'])
    N, n, Fx = x_train.shape
    if Fx != F:
        raise ValueError(f"x_train has {Fx} features, the model spec {F}")
    d = E * F + 3 * E + 2
    if d > L.BNN_MAX_D:
        raise ValueError(f"the network has d = E F + 3 E + 2 = {d} weights, above the sampler's limit of {L.BNN_MAX_D}")
    if not 1 <= n <= L.BNN_MAX_N:
        raise ValueError(f"the sampler keeps the training rows in shared memory: n={n} outside [1, {L.BNN_MAX_N}]")
    if not 1 <= max_tree_depth <= L.GP_MCMC_MAX_DEPTH:
        raise ValueError(f"max_tree_depth={max_tree_depth} outside [1, {L.GP_MCMC_MAX_DEPTH}]")
    dev = L.compute_device(x_train.device, _KERNEL)
    seed = L.draw_seed(seed)
    n_test = 0 if x_test is None else x_test.shape[1]
    So = max(int(num_samples), 1)
    f64 = dict(dtype=torch.float64, device=dev)
    with L.on_device(dev):
        out = L.mcmc_outputs(N, d, num_samples, warmup_steps, trace, dev)
        out.update(probs=torch.empty(N, So, n_test, **f64), obs=torch.empty(N, So, n_test, dtype=torch.float32, device=dev))
        desc = L.bnn_mcmc_desc(N, n, n_test, F, E, num_samples, warmup_steps, seed, max_tree_depth)
        per_chain = L.bnn_mcmc_workspace(desc)
        workspace = torch.empty(N, per_chain, **f64) if per_chain else None
        th0 = None if init is None else init.to(dev, torch.float64).reshape(N, d).contiguous()
        xs = None if x_test is None else x_test.to(dev, torch.float32).contiguous()
        L.bnn_mcmc(x_train.to(dev, torch.float32).contiguous(), y_train.to(dev, torch.float32).contiguous(), xs, desc,
                   out["samples"], out["step_size"], out["accept"], out["diag"], init=th0, probs=out["probs"], obs=out["obs"],
                   potential=out["potential"], grad=out["grad"], trace=out.get("trace"), workspace=workspace)
    out["seed"] = seed
    return out


def _report_mcmc(diag):
    n_div, n_depth = L.mcmc_trouble(diag)
    if n_div or n_depth:
        print(f"eval_mcmc: {diag.shape[0]} chains: {n_div} sampling iterations diverged, {n_depth} iterations (warmup "
              f"included) hit the tree-depth cap")


@torch.no_grad()
def eval_mcmc(X, y, device, model_sampler, training_samples_n, warmup_steps, num_pred_samples, seed=None):
    """NUTS baseline (reference :249-267): X [N, T, F], y [N, T]; for every dataset a chain on its first
    `training_samples_n` rows, then `evaluate_preds` on the rest: per (sample, row) one class drawn from the sample's
    probabilities (what pyro's `predictive` returns as 'obs'), BCELoss of their mean over samples against the labels and
    the accuracy of the drawn classes.  Returns (nll [N], acc [N]) as numpy arrays.  All chains run in one launch.

    The chains always run on a CUDA device: `device='cpu'` (the default of `training_steps` / `training_samples`, as in
    the reference, which runs pyro there) selects the current CUDA device, and raises when there is none."""
    model = model_sampler()
    spec = {'num_features': model.num_features, 'embed': model.embed}
    dev = L.compute_device(device, _KERNEL)
    seed = L.draw_seed(seed)
    X, y = X.to(dev), y.to(dev)
    k = training_samples_n
    r = sample_bnn_posterior(X[:, :k], y[:, :k], X[:, k:], spec, num_pred_samples, warmup_steps, seed)
    _report_mcmc(r["diag"])
    scores = [evaluate_preds({'obs': obs_b}, y_b) for obs_b, y_b in zip(r["obs"], y[:, k:])]    # obs_b [S, n_test]
    acc, nll = (torch.stack([s[i] for s in scores]).cpu().numpy() for i in (0, 1))
    return nll, acc


@torch.no_grad()
def eval_transformer(X, y, device, model, training_samples_n):
    """The transformer on the same task (reference :270-291): X [N, T, F], y [N, T]; x standardised with the mean and
    unbiased std (+ 1e-6) of each dataset's training prefix; all N datasets in ONE forward pass (the reference loops over
    batches of one).  Returns (acc [N], nll [N], seconds of the forward pass, device synchronised)."""
    k = training_samples_n
    xs, ys = X.to(device).transpose(0, 1), y.to(device).float().transpose(0, 1).contiguous()    # sequence first
    prefix = xs[:k]
    xs = ((xs - prefix.mean(0)) / (prefix.std(0) + 1e-6)).contiguous()
    model = model.to(device)
    torch.cuda.synchronize(device)
    t0 = time.time()
    logits = model((xs, ys), single_eval_pos=k).squeeze(-1)
    torch.cuda.synchronize(device)
    seconds = time.time() - t0
    p = torch.sigmoid(logits.float().cpu())
    target = ys[k:].cpu()
    acc = ((p > 0.5) == (target > 0.5)).float().mean(0)
    nll = Fn.binary_cross_entropy(p, target, reduction='none').mean(0)
    return acc, nll, seconds


def _only_mcmc(method):
    if method != 'mcmc':
        raise NotImplementedError(f"method {method!r}: only 'mcmc' (NUTS, csrc/bnn_mcmc.cu) is implemented; the SVI "
                                  "(AutoDiagonalNormal + Trace_ELBO) and SVGD baselines are not")


def _timed_eval_to_file(path, overwrite, label, prefix, X, y, device, model_sampler, n_train, steps):
    """One `eval_mcmc` call whose (prefix..., nll, acc, seconds) record goes to `path`, unless the file exists."""
    if os.path.isfile(path) and not overwrite:
        print(f'already done {label}')
        return
    t0 = time.time()
    nll, acc = eval_mcmc(X, y, device, model_sampler, n_train, warmup_steps=steps, num_pred_samples=steps)
    seconds = time.time() - t0
    for name, values in (('NLL ', nll), ('ACC ', acc)):
        print(name, compute_mean_and_conf_interval(values))
    print('TIME ', seconds)
    record = np.empty(len(prefix) + 3, dtype=object)          # the reference saves a ragged tuple; numpy needs it spelled out
    record[:] = list(prefix) + [np.asarray(nll), np.asarray(acc), seconds]
    np.save(path, record)
    print(f'Saved results at {path}')


def training_steps(method, X, y, model_spec, device='cpu', path_interfix='', overwrite=False):
    """The baseline at 100 training rows for warmup = samples = 2, 4, .., 4096 (reference :294-319); one file
    `{path_interfix}/results_{method}_training_steps_{s}.npy` holding (nll, acc, seconds) per setting.  `model_spec` is the
    zero-argument model factory, as in the reference's calls."""
    _only_mcmc(method)
    for s in STEP_GRID:
        _timed_eval_to_file(f'{path_interfix}/results_{method}_training_steps_{s}.npy', overwrite, s, (), X, y, device,
                            model_spec, TRAINING_ROWS_OF_STEP_GRID, s)


def training_samples(method, X, y, model_spec, evaluation_points, steps=None, device='cpu', path_interfix='', overwrite=False):
    """The baseline at every training-set size of `evaluation_points` with warmup = samples = `steps` (default 512)
    (reference :322-351); one file `{path_interfix}/results_{method}_{steps}_training_samples_{n}.npy` holding
    (n, nll, acc, seconds) per size."""
    _only_mcmc(method)
    steps = steps or DEFAULT_MCMC_STEPS
    for n in evaluation_points:
        _timed_eval_to_file(f'{path_interfix}/results_{method}_{steps}_training_samples_{n}.npy', overwrite, n, (n,), X, y,
                            device, model_spec, n, steps)


def main(argv=None):
    """The reference's command line (:375-398): --solver, --task steps|samples, --model_size."""
    ap = argparse.ArgumentParser()
    ap.add_argument('--solver', default='mcmc', type=str)
    ap.add_argument('--task', default='steps', type=str, choices=('steps', 'samples'))
    ap.add_argument('--model_size', default='small', type=str)
    args = ap.parse_args(argv)
    spec, device = get_default_model_spec(args.model_size), 'cuda:0'
    sampler = lambda: BayesianModel(spec, device=device)
    X, y = generate_toy_data(sampler(), spec['seq_len'])
    out_dir = f'results/timing_{args.model_size}_model'
    os.makedirs(out_dir, exist_ok=True)
    if args.task == 'steps':
        training_steps(args.solver, X, y, sampler, device=device, path_interfix=out_dir)
    else:
        training_samples(args.solver, X, y, sampler, get_default_evaluation_points(), device=device, path_interfix=out_dir)


if __name__ == '__main__':
    main()
