"""Configuration: one dataclass per entry point, with the reference's knob names.

The reference has no flag system — its knobs are module-level constants edited
by hand (SURVEY §5.6; e.g. /root/reference/src/consensus_multi.py:8-59).  Every
constant is a dataclass field here with the same name and default, settable
from the command line as ``--K 8 --use_resnet --Nloop 2`` (booleans accept
``--flag`` / ``--no-flag`` / ``--flag=false``).  Fields that do not exist in the
reference (runtime placement, parity switches, synthetic-data options) are
grouped at the end of :class:`CommonConfig`.
"""
from __future__ import annotations

import argparse
import dataclasses
import math
from dataclasses import dataclass, field
from typing import Optional, Sequence, Type, TypeVar

T = TypeVar("T")


@dataclass
class CommonConfig:
    K: int = 10
    default_batch: int = 128
    Nloop: int = 12
    Nepoch: int = 1
    Nadmm: int = 3
    load_model: bool = False
    init_model: bool = True
    save_model: bool = True
    check_results: bool = True
    biased_input: bool = True
    be_verbose: bool = False
    use_resnet: bool = False
    use_cuda: bool = True
    # ---- new in this framework -------------------------------------------------
    model: str = ""                 # '', 'Net', 'Net1', 'Net2', 'ResNet18', 'ResNet9' ('' = follow use_resnet)
    optimizer: str = "adam"         # 'adam' | 'adamw' | 'sgd' | 'lbfgs' (the reference's commented-out alternative)
    # client optimizer (classifier drivers): torch.optim.SGD semantics with dampening 0 (optim/block_sgd.py), and
    # torch.optim.AdamW (optim/block_adam.py)
    lr: float = 0.0                 # 0 = the optimizer's default: 1e-3 for adam / adamw; sgd has none and needs lr > 0
    momentum: float = 0.0           # sgd only, in [0, 1)
    nesterov: bool = False          # sgd only, needs momentum > 0
    weight_decay: float = 0.0       # sgd / adamw, >= 0: sgd adds weight_decay * x to the gradient, adamw decays x by
                                    # 1 - lr * weight_decay before its step
    # client learning-rate schedule over communication rounds (optim/schedule.py; adam / adamw / sgd)
    lr_schedule: str = "const"      # 'const' | 'step' | 'cosine'
    lr_warmup: int = 0              # linear warmup over the first lr_warmup rounds, with any schedule
    lr_gamma: float = 0.1           # step only, in (0, 1]: the factor every lr_step_rounds rounds
    lr_step_rounds: int = 0         # step only, >= 1 (no default: 0 = unset)
    lr_min: float = 0.0             # cosine only, in [0, 1): the final rate is lr_min * lr
    clip_norm: float = 0.0          # > 0: clip the block's data-loss gradient to this norm before every step (0 = off)
    seed: int = 69                  # torch.manual_seed(69) at the top of every reference script
    data: str = "synthetic"         # 'synthetic' | 'torchvision' (needs local files, never downloads)
    data_seed: int = 1234
    data_noise: float = 0.6         # synthetic data: noise std relative to the class-template amplitude (harder when larger)
    train_size: int = 50000
    test_size: int = 10000
    data_on_device: bool = True     # dataset resident in HBM; False = pinned host + native batch assembler
    fix_shard_off_by_one: bool = False   # Q1
    intended_elastic_net_gate: bool = False  # Q2: regularise whenever the block holds dense-layer weights
    diagnostics: str = "post"       # Q17: 'post' (extra forward after the step) | 'pre'
    eval_bn: str = "batch"          # Q4: 'batch' (reference: train-mode BN at evaluation, running stats updated by test data) | 'running' (net.eval())
                                    # classifier drivers only: the VAE, VAE-CL and CPC networks have no BatchNorm and do not evaluate;
                                    # no effect with norm 'group' (GroupNorm has no running statistics)
    # normalisation of the ResNets: 'batch' (the reference) | 'group' = GroupNorm with norm_groups groups in every layer
    # (Wu & He 2018), which normalises each sample on its own and mixes no worker's data statistics into the model
    norm: str = "batch"
    norm_groups: int = 32           # must divide 64, the narrowest layer
    augment: bool = False           # random 4-pixel-padded crop + horizontal flip of training batches (classifier drivers only)
    # regularisers of the classifier drivers' training loss (timm's Mixup in batch mode, SoftTargetCrossEntropy): sample i
    # of a batch is mixed with sample n-1-i (data/cifar.py: mix_draws); 0 = off
    label_smoothing: float = 0.0    # epsilon in [0, 1): targets (1 - eps) onehot(y) + eps / C
    mixup_alpha: float = 0.0        # >= 0: mixup with lambda ~ Beta(alpha, alpha)
    cutmix_alpha: float = 0.0       # >= 0: CutMix with lambda ~ Beta(alpha, alpha); with mixup, one of the two per batch
    nan_guard: str = "raise"        # non-finite aggregation residual: 'raise' | 'warn' | 'off'
    collective: str = "auto"        # 'auto' | 'fused' | 'torch'
    fast: bool = True               # use the hand-written sm_90a kernels on CUDA devices
    graphs: bool = True             # CUDA-graph the per-minibatch step when possible
    distributed: bool = True        # honour torchrun env (one process per GPU); False = all K replicas here
    ckpt_dir: str = "."
    metrics_path: str = ""
    max_minibatches: int = 0        # >0 caps minibatches per round (smoke tests / benchmarks)
    resume: str = ""                # path of a true-resume record written by this framework: re-enter the schedule there
    resume_out: str = ""            # write the true-resume record here after every aggregation round ('' = never)
    streams: bool = True            # co-resident replicas (K > #GPUs) step concurrently on their own CUDA streams
    # training-set split over the K workers (classifier drivers): 'iid' = equal contiguous shards (the reference) |
    # 'dirichlet' = label skew, each class split in proportions p ~ Dir(dirichlet_alpha 1_K) (data/cifar.py: dirichlet_shards)
    partition: str = "iid"
    dirichlet_alpha: float = 0.5    # smaller = more skewed


@dataclass
class NoConsensusConfig(CommonConfig):
    Nepoch: int = 20
    Nloop: int = 1
    Nadmm: int = 1


SERVER_OPTS = ("none", "avgm", "adagrad", "adam", "yogi")


def check_server_opt(server_opt: str, server_lr: float, server_momentum: float, server_beta1: float, server_beta2: float,
                     server_tau: float) -> None:
    """Raise ``ValueError`` unless the server-optimizer settings of :class:`FederatedConfig` are valid."""
    if server_opt not in SERVER_OPTS:
        raise ValueError("server_opt must be one of %s, got %r" % (", ".join(SERVER_OPTS), server_opt))
    if not server_lr >= 0.0:
        raise ValueError("server_lr must be >= 0, got %r" % (server_lr,))
    for name, val in (("server_momentum", server_momentum), ("server_beta1", server_beta1), ("server_beta2", server_beta2)):
        if not 0.0 <= val < 1.0:
            raise ValueError("%s must lie in [0, 1), got %r" % (name, val))
    if not server_tau > 0.0:
        raise ValueError("server_tau must be > 0, got %r" % (server_tau,))


AGGREGATORS = ("mean", "median", "trimmed_mean")
ROBUST_MAX_K = 16                   # the robust rules sort the K values of a coordinate in registers
ATTACKS = ("signflip", "gaussian", "nan")


def trim_count(trim_fraction: float, K: int) -> int:
    """Values dropped at each end by the trimmed mean: ``floor(trim_fraction * K)`` (``scipy.stats.trim_mean``)."""
    return int(trim_fraction * K)


def check_aggregator(aggregator: str, trim_fraction: float, K: int) -> None:
    """Raise ``ValueError`` unless the aggregation rule of :class:`FederatedConfig` is valid for ``K`` workers."""
    if aggregator not in AGGREGATORS:
        raise ValueError("aggregator must be one of %s, got %r" % (", ".join(AGGREGATORS), aggregator))
    if not 0.0 <= trim_fraction < 0.5:
        raise ValueError("trim_fraction must lie in [0, 0.5), got %r" % (trim_fraction,))
    if aggregator != "mean" and K > ROBUST_MAX_K:
        raise ValueError("aggregator %r supports at most %d workers, got K = %d" % (aggregator, ROBUST_MAX_K, K))
    if aggregator == "trimmed_mean" and trim_count(trim_fraction, K) == 0:
        raise ValueError("trim_fraction %r trims nothing at K = %d (floor(trim_fraction * K) = 0): the trimmed mean would "
                         "be the mean" % (trim_fraction, K))


def check_byzantine(byzantine: int, attack: str, attack_scale: float, K: int) -> None:
    """Raise ``ValueError`` unless the simulated-attacker settings of :class:`FederatedConfig` are valid."""
    if not 0 <= byzantine < K:
        raise ValueError("byzantine must lie in [0, K) = [0, %d), got %r" % (K, byzantine))
    if attack not in ATTACKS:
        raise ValueError("attack must be one of %s, got %r" % (", ".join(ATTACKS), attack))
    if not attack_scale > 0.0:
        raise ValueError("attack_scale must be > 0, got %r" % (attack_scale,))


def check_dp(dp_clip: float, dp_noise: float, dp_delta: float, aggregator: str) -> None:
    """Raise ``ValueError`` unless the differential-privacy settings of :class:`FederatedConfig` are valid."""
    if not (math.isfinite(dp_clip) and dp_clip >= 0.0):
        raise ValueError("dp_clip must be finite and >= 0 (0 = off), got %r" % (dp_clip,))
    if not dp_noise >= 0.0:
        raise ValueError("dp_noise must be >= 0, got %r" % (dp_noise,))
    if not 0.0 < dp_delta < 1.0:
        raise ValueError("dp_delta must lie in (0, 1), got %r" % (dp_delta,))
    if dp_clip > 0.0 and aggregator != "mean":
        raise ValueError("dp_clip needs aggregator 'mean' (robust rules have a different sensitivity), got aggregator %r"
                         % (aggregator,))


NORMS = ("batch", "group")
NORM_MODELS = ("ResNet18", "ResNet9")      # the models with a normalisation layer


def check_norm(norm: str, norm_groups: int, model: str) -> None:
    """Raise ``ValueError`` unless the normalisation settings of :class:`CommonConfig` are valid for ``model``."""
    if norm not in NORMS:
        raise ValueError("norm must be one of %s, got %r" % (", ".join(NORMS), norm))
    if not (isinstance(norm_groups, int) and norm_groups >= 1 and 64 % norm_groups == 0):
        raise ValueError("norm_groups must divide 64 (the narrowest layer), got %r" % (norm_groups,))
    if norm != "batch" and model not in NORM_MODELS:
        raise ValueError("norm %r needs a model with normalisation layers (%s), got model %r"
                         % (norm, ", ".join(NORM_MODELS), model))


OPTIMIZERS = ("adam", "adamw", "sgd", "lbfgs")
ADAM_LR = 1e-3                      # the reference's client learning rate
LR_SCHEDULES = ("const", "step", "cosine")
# the client-recipe fields (schedule and clipping) and their defaults
CLIENT_RECIPE_DEFAULTS = (("lr_schedule", "const"), ("lr_warmup", 0), ("lr_gamma", 0.1), ("lr_step_rounds", 0),
                          ("lr_min", 0.0), ("clip_norm", 0.0))


def check_client_opt(optimizer: str, lr: float, momentum: float, nesterov: bool, weight_decay: float,
                     lr_schedule: str = "const", lr_warmup: int = 0, lr_gamma: float = 0.1, lr_step_rounds: int = 0,
                     lr_min: float = 0.0, clip_norm: float = 0.0) -> None:
    """Raise ``ValueError`` unless the client-optimizer settings of :class:`CommonConfig` are valid."""
    if optimizer not in OPTIMIZERS:
        raise ValueError("optimizer must be one of %s, got %r" % (", ".join(OPTIMIZERS), optimizer))
    if not (math.isfinite(lr) and lr >= 0.0):
        raise ValueError("lr must be finite and >= 0 (0 = the optimizer's default), got %r" % (lr,))
    if optimizer == "lbfgs" and lr != 0.0:
        raise ValueError("lr cannot be set with optimizer 'lbfgs' (its line search sets the step length), got lr %r" % (lr,))
    if optimizer == "sgd" and lr == 0.0:
        raise ValueError("optimizer 'sgd' has no default learning rate: set lr > 0")
    if not 0.0 <= momentum < 1.0:
        raise ValueError("momentum must lie in [0, 1), got %r" % (momentum,))
    if not (math.isfinite(weight_decay) and weight_decay >= 0.0):
        raise ValueError("weight_decay must be finite and >= 0, got %r" % (weight_decay,))
    for name, val, default in (("momentum", momentum, 0.0), ("nesterov", nesterov, False)):
        if val != default and optimizer != "sgd":
            raise ValueError("%s needs optimizer 'sgd', got optimizer %r" % (name, optimizer))
    if weight_decay != 0.0 and optimizer not in ("sgd", "adamw"):
        raise ValueError("weight_decay needs optimizer 'sgd' or 'adamw' (coupled L2 decay for Adam is not offered), "
                         "got optimizer %r" % (optimizer,))
    if nesterov and momentum == 0.0:
        raise ValueError("nesterov needs momentum > 0, got momentum %r" % (momentum,))
    # learning-rate schedule and clipping
    if lr_schedule not in LR_SCHEDULES:
        raise ValueError("lr_schedule must be one of %s, got %r" % (", ".join(LR_SCHEDULES), lr_schedule))
    if not (isinstance(lr_warmup, int) and lr_warmup >= 0):
        raise ValueError("lr_warmup must be an integer >= 0, got %r" % (lr_warmup,))
    if not 0.0 < lr_gamma <= 1.0:
        raise ValueError("lr_gamma must lie in (0, 1], got %r" % (lr_gamma,))
    if not (isinstance(lr_step_rounds, int) and lr_step_rounds >= 0):
        raise ValueError("lr_step_rounds must be an integer >= 0 (0 = unset), got %r" % (lr_step_rounds,))
    if not 0.0 <= lr_min < 1.0:
        raise ValueError("lr_min must lie in [0, 1), got %r" % (lr_min,))
    if not (math.isfinite(clip_norm) and clip_norm >= 0.0):
        raise ValueError("clip_norm must be finite and >= 0 (0 = off), got %r" % (clip_norm,))
    if lr_schedule == "step" and lr_step_rounds < 1:
        raise ValueError("lr_schedule 'step' needs lr_step_rounds >= 1, got lr_step_rounds %r" % (lr_step_rounds,))
    for name, val, default, owner in (("lr_gamma", lr_gamma, 0.1, "step"), ("lr_step_rounds", lr_step_rounds, 0, "step"),
                                      ("lr_min", lr_min, 0.0, "cosine")):
        if val != default and lr_schedule != owner:
            raise ValueError("%s belongs to lr_schedule %r, got lr_schedule %r" % (name, owner, lr_schedule))
    if optimizer == "lbfgs":
        for name, val, default in (("lr_schedule", lr_schedule, "const"), ("lr_warmup", lr_warmup, 0),
                                   ("clip_norm", clip_norm, 0.0)):
            if val != default:
                raise ValueError("%s cannot be set with optimizer 'lbfgs' (its line search sets the step), got %s %r"
                                 % (name, name, val))


MIX_DEFAULTS = (("label_smoothing", 0.0), ("mixup_alpha", 0.0), ("cutmix_alpha", 0.0))


def check_mix(label_smoothing: float, mixup_alpha: float, cutmix_alpha: float) -> None:
    """Raise ``ValueError`` unless the label-smoothing, mixup and CutMix settings of :class:`CommonConfig` are valid."""
    if not 0.0 <= label_smoothing < 1.0:
        raise ValueError("label_smoothing must lie in [0, 1), got %r" % (label_smoothing,))
    for name, val in (("mixup_alpha", mixup_alpha), ("cutmix_alpha", cutmix_alpha)):
        if not (math.isfinite(val) and val >= 0.0):
            raise ValueError("%s must be finite and >= 0 (0 = off), got %r" % (name, val))


PARTITIONS = ("iid", "dirichlet")


def check_partition(partition: str, dirichlet_alpha: float) -> None:
    """Raise ``ValueError`` unless the training-set split of :class:`CommonConfig` is valid."""
    if partition not in PARTITIONS:
        raise ValueError("partition must be one of %s, got %r" % (", ".join(PARTITIONS), partition))
    if not (math.isfinite(dirichlet_alpha) and dirichlet_alpha > 0.0):
        raise ValueError("dirichlet_alpha must be finite and > 0, got %r" % (dirichlet_alpha,))


def sampled_rounds(clients_per_round: int, K: int, partition: str) -> bool:
    """Whether federated averaging runs its sampled, sample-weighted rounds: a strict subset of the workers per round,
    or unequal (Dirichlet) shards, whose sample counts weight the average."""
    return 0 < clients_per_round < K or partition == "dirichlet"


def check_sampling(clients_per_round: int, K: int, partition: str, aggregator: str, dp_clip: float,
                   compress_bits: int, compress_topk: float = 0.0) -> None:
    """Raise ``ValueError`` unless the client-sampling settings of :class:`FederatedConfig` are valid."""
    if not 0 <= clients_per_round <= K:
        raise ValueError("clients_per_round must lie in [0, K] = [0, %d] (0 = all), got %r" % (K, clients_per_round))
    if not sampled_rounds(clients_per_round, K, partition):
        return
    what = "clients_per_round %d" % clients_per_round if 0 < clients_per_round < K else "partition 'dirichlet'"
    if aggregator != "mean":
        raise ValueError("%s needs aggregator 'mean' (sample-weighted averaging), got aggregator %r" % (what, aggregator))
    if dp_clip > 0.0:
        raise ValueError("%s cannot be combined with dp_clip > 0 (the accountant has no privacy amplification by "
                         "subsampling), got dp_clip %r" % (what, dp_clip))
    if compress_bits:
        raise ValueError("%s cannot be combined with compress_bits, got compress_bits %r" % (what, compress_bits))
    if compress_topk:
        raise ValueError("%s cannot be combined with compress_topk, got compress_topk %r" % (what, compress_topk))


def check_compress(compress_bits: int, compress_ef: bool, dp_clip: float, aggregator: str,
                   compress_topk: float = 0.0) -> None:
    """Raise ``ValueError`` unless the update-compression settings of :class:`FederatedConfig` are valid."""
    if compress_bits not in (0, 8, 4):
        raise ValueError("compress_bits must be 0 (off), 8 or 4, got %r" % (compress_bits,))
    if not (compress_topk == 0.0 or 0.0 < compress_topk < 1.0):
        raise ValueError("compress_topk must be 0 (off) or lie in (0, 1), got %r" % (compress_topk,))
    if compress_topk and compress_bits:
        raise ValueError("compress_topk cannot be combined with compress_bits (the selected values are sent in fp32), got "
                         "compress_bits %r" % (compress_bits,))
    if compress_ef and not (compress_bits or compress_topk):
        raise ValueError("compress_ef needs compress_bits 8 or 4 or compress_topk > 0 (error feedback of uncompressed "
                         "updates is always 0)")
    if compress_topk and dp_clip > 0.0:
        raise ValueError("compress_topk cannot be combined with dp_clip > 0, got dp_clip %r" % (dp_clip,))
    if compress_topk and aggregator != "mean":
        raise ValueError("compress_topk needs aggregator 'mean', got aggregator %r" % (aggregator,))
    if compress_bits and dp_clip > 0.0:
        raise ValueError("compress_bits cannot be combined with dp_clip > 0 (quantized updates no longer have the clipped "
                         "sensitivity), got dp_clip %r" % (dp_clip,))
    if compress_bits and aggregator != "mean":
        raise ValueError("compress_bits needs aggregator 'mean', got aggregator %r" % (aggregator,))


def check_secagg(secagg: bool, secagg_clip: float, K: int, aggregator: str, dp_clip: float, compress_bits: int,
                 clients_per_round: int, partition: str, compress_topk: float = 0.0) -> None:
    """Raise ``ValueError`` unless the secure-aggregation settings of :class:`FederatedConfig` are valid."""
    if not secagg:
        return
    from .algo.secagg import frac_bits

    frac_bits(secagg_clip, max(K, 2))                 # names secagg_clip: not finite and > 0, or no scale 2^f in range
    if K < 2:
        raise ValueError("secagg needs K >= 2 (a lone worker's payload is unmasked), got K = %d" % K)
    if aggregator != "mean":
        raise ValueError("secagg needs aggregator 'mean' (the server sees only the sum), got aggregator %r" % (aggregator,))
    if dp_clip > 0.0:
        raise ValueError("secagg cannot be combined with dp_clip > 0, got dp_clip %r" % (dp_clip,))
    if compress_bits:
        raise ValueError("secagg cannot be combined with compress_bits, got compress_bits %r" % (compress_bits,))
    if compress_topk:
        raise ValueError("secagg cannot be combined with compress_topk, got compress_topk %r" % (compress_topk,))
    if sampled_rounds(clients_per_round, K, partition):
        what = "clients_per_round %d" % clients_per_round if 0 < clients_per_round < K else "partition 'dirichlet'"
        raise ValueError("secagg cannot be combined with sampled rounds (every worker takes part in every round), got %s"
                         % what)


def check_scaffold(scaffold: bool, aggregator: str, dp_clip: float, compress_bits: int, secagg: bool,
                   optimizer: Optional[str] = None, compress_topk: float = 0.0) -> None:
    """Raise ``ValueError`` unless the SCAFFOLD settings of :class:`FederatedConfig` are valid.  ``optimizer`` None: not
    checked (the aggregation strategy does not know the client optimizer)."""
    if not scaffold:
        return
    if optimizer is not None and optimizer != "sgd":
        raise ValueError("scaffold needs optimizer 'sgd' (its control-variate update assumes SGD local steps), got "
                         "optimizer %r" % (optimizer,))
    if aggregator != "mean":
        raise ValueError("scaffold needs aggregator 'mean' (the control variates are averaged), got aggregator %r"
                         % (aggregator,))
    for name, val, on in (("dp_clip", dp_clip, dp_clip > 0.0), ("compress_bits", compress_bits, bool(compress_bits)),
                          ("compress_topk", compress_topk, bool(compress_topk)), ("secagg", secagg, bool(secagg))):
        if on:
            raise ValueError("scaffold cannot be combined with %s (the control-variate update needs the workers' models "
                             "as trained, which %s changes), got %s %r" % (name, name, name, val))


@dataclass
class FederatedConfig(CommonConfig):
    lambda1: float = 0.0001
    lambda2: float = 0.0001
    # server optimizer on the round's mean change (FedAvgM, FedAdagrad, FedAdam, FedYogi); 'none' = plain FedAvg
    server_opt: str = "none"        # 'none' | 'avgm' | 'adagrad' | 'adam' | 'yogi'
    server_lr: float = 0.0          # 0 = the variant's default: 1.0 for avgm, 1e-2 for adagrad / adam / yogi
    server_momentum: float = 0.9    # avgm
    server_beta1: float = 0.9       # adagrad / adam / yogi
    server_beta2: float = 0.99      # adam / yogi
    server_tau: float = 1e-3        # adaptivity floor: z += lr m / (sqrt(v) + tau); v starts at tau^2
    # Byzantine-robust aggregation: coordinate-wise order statistic over the K workers instead of their mean
    aggregator: str = "mean"        # 'mean' | 'median' | 'trimmed_mean'
    trim_fraction: float = 0.1      # trimmed_mean: drop floor(trim_fraction * K) values at each end
    # simulated Byzantine workers K - byzantine .. K - 1 (worker 0 stays honest), applied before every aggregation
    byzantine: int = 0
    attack: str = "signflip"        # 'signflip': x <- z - s (x - z) | 'gaussian': x <- z + s N(0, 1) | 'nan': x <- NaN
    attack_scale: float = 4.0       # s
    # client-level differential privacy (DP-FedAvg): clip every worker's block update to C = dp_clip * sqrt(N), add
    # N(0, (dp_noise C / K)^2) noise to the mean (algo/privacy.py)
    dp_clip: float = 0.0            # 0 = off
    dp_noise: float = 1.0           # noise multiplier sigma (0 = clipping only)
    dp_delta: float = 1e-5          # delta at which epsilon is reported
    # compressed client updates (QSGD / FedPAQ): every worker uploads its block update as stochastically rounded codes with
    # one float32 scale per 128 coordinates (algo/compress.py); the new model is still broadcast in fp32
    compress_bits: int = 0          # 0 = off | 8 | 4
    compress_ef: bool = False       # error feedback: each worker carries its quantization error into its next update
    # top-k sparsified client updates: every worker uploads the max(1, ceil(r N)) largest-magnitude coordinates of its
    # block update, unchanged (algo/compress.py: topk_select); with compress_ef the rest is carried into its next update
    compress_topk: float = 0.0      # r: 0 = off, else 0 < r < 1
    # client sampling (FedAvg partial participation): each round trains and averages a uniform random subset of this many
    # workers, weighted by their sample counts (algo/sampling.py); 0 = all K.  --partition dirichlet weights all K by n_k
    clients_per_round: int = 0
    # secure aggregation (SecAgg): every worker uploads its block update as int32 fixed-point codes of clamp(u, -R, R)
    # masked with pairwise ChaCha20 keystreams that cancel in the sum (algo/secagg.py); pair keys are derived from --seed
    secagg: bool = False
    secagg_clip: float = 1.0        # R
    # SCAFFOLD control variates (algo/scaffold.py): every SGD step adds c - c_i to the gradient, which corrects client drift
    scaffold: bool = False

    def __post_init__(self):
        check_server_opt(self.server_opt, self.server_lr, self.server_momentum, self.server_beta1, self.server_beta2,
                         self.server_tau)
        check_aggregator(self.aggregator, self.trim_fraction, self.K)
        check_byzantine(self.byzantine, self.attack, self.attack_scale, self.K)
        check_dp(self.dp_clip, self.dp_noise, self.dp_delta, self.aggregator)
        check_compress(self.compress_bits, self.compress_ef, self.dp_clip, self.aggregator, self.compress_topk)
        check_partition(self.partition, self.dirichlet_alpha)
        check_sampling(self.clients_per_round, self.K, self.partition, self.aggregator, self.dp_clip, self.compress_bits,
                       self.compress_topk)
        check_secagg(self.secagg, self.secagg_clip, self.K, self.aggregator, self.dp_clip, self.compress_bits,
                     self.clients_per_round, self.partition, self.compress_topk)
        check_scaffold(self.scaffold, self.aggregator, self.dp_clip, self.compress_bits, self.secagg, self.optimizer,
                       self.compress_topk)


@dataclass
class FedProxConfig(CommonConfig):
    Nadmm: int = 5
    lambda1: float = 0.0001
    lambda2: float = 0.0001
    admm_rho0: float = 1.0


@dataclass
class ConsensusConfig(CommonConfig):
    Nadmm: int = 5
    lambda1: float = 0.0001
    lambda2: float = 0.0001
    admm_rho0: float = 0.1
    bb_update: bool = False
    bb_period_T: int = 2
    bb_alphacorrmin: float = 0.2
    bb_epsilon: float = 1e-3
    bb_rhomax: float = 0.1
    bb_seed_yhat0_zero: bool = False    # Q9


@dataclass
class VAEConfig(CommonConfig):
    Nadmm: int = 3
    be_verbose: bool = True             # the VAE driver prints every minibatch unconditionally
    check_results: bool = False


@dataclass
class VAECLConfig(CommonConfig):
    K: int = 1
    Kc: int = 10
    Lc: int = 32
    Nloop: int = 1
    Nadmm: int = 1
    lambda2: float = 0.001
    be_verbose: bool = True
    check_results: bool = False
    batched_clusters: bool = True


@dataclass
class CPCConfig(CommonConfig):
    K: int = 4
    Lc: int = 256
    Rc: int = 32
    batch_size: int = 128
    Nloop: int = 1
    Niter: int = 10
    Nadmm: int = 1
    load_model: bool = True
    init_model: bool = False
    be_verbose: bool = True
    check_results: bool = False
    # synthetic LOFAR source (the reference reads HDF5 files from a Colab drive)
    file_list: str = ""                 # comma separated .h5 paths ('' = synthetic)
    sap_list: str = ""                  # comma separated SAP ids
    nbase: int = 64
    ntime: int = 64
    nfreq: int = 64
    patch_layout: str = "batch_major"   # Q13: 'batch_major' | 'reference'


# ----------------------------------------------------------------------------
def _str2bool(v: str) -> bool:
    if v.lower() in ("1", "true", "yes", "y", "on"):
        return True
    if v.lower() in ("0", "false", "no", "n", "off"):
        return False
    raise argparse.ArgumentTypeError("expected a boolean, got %r" % v)


def build_parser(cls: Type[T], prog: Optional[str] = None) -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(prog=prog, description=(cls.__doc__ or "").strip() or None)
    for f in dataclasses.fields(cls):
        name = "--" + f.name
        if f.type in (bool, "bool"):
            p.add_argument(name, nargs="?", const=True, default=f.default, type=_str2bool)
            p.add_argument("--no-" + f.name, dest=f.name, action="store_false")
        else:
            typ = {"int": int, "float": float, "str": str}.get(f.type if isinstance(f.type, str) else f.type.__name__, str)
            p.add_argument(name, type=typ, default=f.default)
    return p


def parse_config(cls: Type[T], argv: Optional[Sequence[str]] = None, prog: Optional[str] = None) -> T:
    ns = build_parser(cls, prog).parse_args(argv)
    return cls(**vars(ns))


def override(cfg: T, **kw) -> T:
    return dataclasses.replace(cfg, **kw)
