"""Loss functions of the seven drivers (SURVEY §2.6), vectorised.

The reference evaluates the VAE-CL costs with Python loops over the batch
(/root/reference/src/federated_vae_cl.py:101-140: ~5 000 tiny kernels per step)
and InfoNCE with a P^2 loop of ``torch.dot`` (federated_cpc.py:161-178).  The
same quantities are computed here as a few batched tensor expressions — and, on
the GPU, as single fused kernels (``csrc/loss_kernels.cu``) behind
``torch.autograd.Function``s.  The ``*_reference`` variants are literal
transcriptions of the math with loops, kept as test oracles.
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Tuple

import torch
import torch.nn.functional as F

from . import functional as FX


# ----------------------------------------------------------------------------
# classifier
# ----------------------------------------------------------------------------
def cross_entropy(logits: torch.Tensor, labels: torch.Tensor, label_smoothing: float = 0.0,
                  lam: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Mean softmax cross-entropy (``nn.CrossEntropyLoss()`` of federated_multi.py:132).

    With ``label_smoothing`` eps or a mixed batch's ``lam`` (a one-element tensor, ``lam_eff`` of ``data.cifar.mix_draws``)
    the target of sample ``i`` is ``lam s(y_i) + (1 - lam) s(y_{B-1-i})`` with ``s(y) = (1 - eps) onehot(y) + eps / C``
    (timm's ``SoftTargetCrossEntropy`` of mixed, smoothed targets), i.e.
    ``lam CE_eps(z, y) + (1 - lam) CE_eps(z, y.flip(0))``.  Without either the hard-label kernels run as before."""
    plain = label_smoothing == 0.0 and lam is None
    if logits.is_cuda and FX.fast_path_enabled():
        from . import cuda_ops

        if cuda_ops.cross_entropy_supported(logits):
            if plain:
                return cuda_ops.cross_entropy(logits, labels)
            return cuda_ops.soft_cross_entropy(logits, labels, lam, label_smoothing)
    if plain:
        return F.cross_entropy(logits, labels)
    loss = F.cross_entropy(logits, labels, label_smoothing=label_smoothing)
    if lam is None:
        return loss
    lam = lam.reshape(())
    return lam * loss + (1.0 - lam) * F.cross_entropy(logits, labels.flip(0), label_smoothing=label_smoothing)


# ----------------------------------------------------------------------------
# VAE (federated_vae.py:96-108)
# ----------------------------------------------------------------------------
def vae_loss(recon_x: torch.Tensor, x: torch.Tensor, mu: torch.Tensor, logvar: torch.Tensor) -> torch.Tensor:
    """``sum (recon-x)^2  - 1/2 sum(1 + logvar - mu^2 - exp(logvar))``."""
    if recon_x.is_cuda and FX.fast_path_enabled():
        from . import cuda_ops

        return cuda_ops.vae_loss(recon_x, x, mu, logvar)
    mse = torch.sum((recon_x - x) ** 2)
    kld = -0.5 * torch.sum(1 + logvar - mu.pow(2) - logvar.exp())
    return mse + kld


# ----------------------------------------------------------------------------
# variational clustering (federated_vae_cl.py:101-162)
# ----------------------------------------------------------------------------
def _stack(d, K: int) -> torch.Tensor:
    if torch.is_tensor(d):
        return d
    return torch.stack([d[k] for k in range(K)], dim=0)


def vae_cl_costs(ekhat, mu_xi, sig2_xi, mu_b, sig2_b, mu_th, sig2_th, x) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """Per-cluster costs ``(c1, c2, c21, c3)``, each of shape ``[Kc]``.

    ``ekhat [B,Kc]`` = q(k|x); dict/stacked ``[Kc,B,...]`` tensors for the rest.
    """
    Kc = ekhat.shape[1]
    B = x.shape[0]
    pk = ekhat.t()                                            # [Kc,B]
    mu_th, sig2_th = _stack(mu_th, Kc), _stack(sig2_th, Kc)   # [Kc,B,3,32,32]
    mu_xi, sig2_xi = _stack(mu_xi, Kc), _stack(sig2_xi, Kc)   # [Kc,B,L]
    mu_b, sig2_b = _stack(mu_b, Kc), _stack(sig2_b, Kc)
    # c1: E_q(k)[ -log p(x|theta) ]  (weighted Gaussian NLL).  On the GPU the [Kc, B, 3072] -> [Kc, B] reduction (the only
    # large tensors of this loss: 2 x 15.7 MB at Kc = 10, B = 128) is ONE kernel forward and one backward (SURVEY G11).
    if x.is_cuda and FX.fast_path_enabled() and x.dtype == torch.float32:
        from . import cuda_ops

        nll_rows = cuda_ops.gauss_nll_rows(x, mu_th, sig2_th)
    else:
        nll = (x.unsqueeze(0) - mu_th).pow(2) / (2 * sig2_th) + 0.5 * torch.log(sig2_th * (2 * math.pi))
        nll_rows = nll.flatten(2).sum(-1)
    c1 = (pk * nll_rows).sum(-1) / B
    # c2: sample-wise entropy of q(k|x)
    c2 = -(pk * torch.log(pk + 1e-9)).sum(-1) / B
    # c21: reciprocal of the batch-wise entropy term
    pbar = pk.mean(-1)
    c21 = 1.0 / (-pbar * torch.log(pbar + 1e-9) + 1e-9)
    # c3: E_q(k)[ KL(q(z|x,k) || p(z|k)) ]
    ratio = sig2_xi / sig2_b
    kl = ratio - torch.log(ratio) + (mu_b - mu_xi).pow(2) / sig2_b - 1
    c3 = 0.5 * (pk * kl.sum(-1)).sum(-1) / B
    return c1, c2, c21, c3


def vae_cl_loss(ekhat, mu_xi, sig2_xi, mu_b, sig2_b, mu_th, sig2_th, x, alpha: float = 10.0, beta: float = 1.0) -> torch.Tensor:
    """``sum_k c1 + alpha (c2 + c3) + beta c21`` (alpha=10, beta=1 in the reference)."""
    c1, c2, c21, c3 = vae_cl_costs(ekhat, mu_xi, sig2_xi, mu_b, sig2_b, mu_th, sig2_th, x)
    return (c1 + alpha * (c2 + c3) + beta * c21).sum()


def vae_cl_loss_reference(ekhat, mu_xi, sig2_xi, mu_b, sig2_b, mu_th, sig2_th, x, alpha=10.0, beta=1.0) -> torch.Tensor:
    """Loop oracle: per-sample accumulation exactly as written in the reference's formulas."""
    Kc, B = ekhat.shape[1], x.shape[0]
    total = x.new_zeros(())
    for k in range(Kc):
        pk = ekhat[:, k]
        err = (x - mu_th[k]).pow(2) / (2 * sig2_th[k])
        lg = 0.5 * torch.log(sig2_th[k] * 2 * math.pi)
        c1 = sum(pk[b] * torch.sum(err[b] + lg[b]) for b in range(B)) / B
        c2 = sum(-pk[b] * torch.log(pk[b] + 1e-9) for b in range(B)) / B
        pbar = torch.mean(pk, 0)
        c21 = 1 / (-pbar * torch.log(pbar + 1e-9) + 1e-9)
        md = (mu_b[k] - mu_xi[k]).pow(2) / sig2_b[k]
        sr = sig2_xi[k] / sig2_b[k]
        c3 = sum(0.5 * pk[b] * torch.sum(sr[b] - torch.log(sr[b]) + md[b] - 1) for b in range(B)) / B
        total = total + c1 + alpha * (c2 + c3) + beta * c21
    return total


# ----------------------------------------------------------------------------
# InfoNCE (federated_cpc.py:149-180)
# ----------------------------------------------------------------------------
def info_nce(z: torch.Tensor, zhat: torch.Tensor) -> torch.Tensor:
    """Contrastive loss over the patch grid.

    ``z, zhat: [B, C, px, py]``.  With ``Z = z.view(-1, P)`` (rows = B*C, one column
    per patch) the score matrix is the cosine Gram ``G = normalize(Z)^T normalize(Zhat)``
    (a P x P x (B*C) GEMM) and ``loss = -sum_i log(softmax(G_i)[i] + 1e-6)``.
    """
    assert z.shape == zhat.shape
    if z.is_cuda and FX.fast_path_enabled():
        from . import cuda_ops

        if cuda_ops.info_nce_supported(z):
            return cuda_ops.info_nce(z, zhat)
    P = z.shape[2] * z.shape[3]
    Z = z.reshape(-1, P)
    Zh = zhat.reshape(-1, P)
    G = (Z / Z.norm(dim=0, keepdim=True)).t() @ (Zh / Zh.norm(dim=0, keepdim=True))
    prob = torch.softmax(G, dim=1).diagonal()
    return -torch.log(prob + 1e-6).sum()


def info_nce_reference(z: torch.Tensor, zhat: torch.Tensor) -> torch.Tensor:
    """Loop oracle (P^2 dot products) for tests at small P."""
    P = z.shape[2] * z.shape[3]
    Z, Zh = z.reshape(-1, P), zhat.reshape(-1, P)
    zz = z.new_zeros(P, P)
    for i in range(P):
        for j in range(P):
            zz[i, j] = torch.dot(Z[:, i], Zh[:, j]) / (torch.norm(Z[:, i]) * torch.norm(Zh[:, j]))
    loss = z.new_zeros(())
    for i in range(P):
        num = torch.exp(zz[i, i])
        den = torch.exp(zz[i]).sum()
        loss = loss - torch.log(num / den + 1e-6)
    return loss
