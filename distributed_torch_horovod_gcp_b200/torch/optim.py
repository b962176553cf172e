"""Optimizers the fused engine runs besides torch's own: the layer-wise adaptive ``hvd.LARS`` and ``hvd.LAMB``,
and ``hvd.Muon`` (at the end of this module).

Both scale each tensor's update by a trust ratio ``‖w‖ / ‖update‖`` so that large-batch training keeps a
similar relative step size in every layer.  ``step()`` here is the eager, pure-torch definition: it runs on
CPU / Gloo and on the generic ``DistributedOptimizer`` path.  Wrapped in ``hvd.DistributedOptimizer`` on CUDA,
the fused engine runs the same update inside its bucket kernels (``parallel/fused_engine.py``), with the
norms taken over the reduced gradient while it is on chip.

Every param group takes ``adaptive`` (default True).  ``adaptive=False`` fixes the trust ratio at 1; put
biases and BatchNorm / LayerNorm parameters in such a group, usually with ``weight_decay=0``.  Gradients
are treated as dense; parameters without a gradient are skipped.
"""
from __future__ import annotations

import math

import torch


def _check(group: dict, betas: bool):
    lr, wd = group["lr"], group["weight_decay"]
    if not 0.0 <= lr:
        raise ValueError(f"Invalid learning rate: {lr}")
    if not 0.0 <= wd:
        raise ValueError(f"Invalid weight_decay value: {wd}")
    if group.get("maximize", False):
        raise ValueError("maximize=True is not supported")
    if betas:
        b1, b2 = group["betas"]
        if not 0.0 <= b1 < 1.0:
            raise ValueError(f"Invalid beta parameter at index 0: {b1}")
        if not 0.0 <= b2 < 1.0:
            raise ValueError(f"Invalid beta parameter at index 1: {b2}")
        if not 0.0 <= group["eps"]:
            raise ValueError(f"Invalid epsilon value: {group['eps']}")
    else:
        if not 0.0 <= group["momentum"] < 1.0:
            raise ValueError(f"Invalid momentum value: {group['momentum']}")
        if not 0.0 <= group["trust_coefficient"]:
            raise ValueError(f"Invalid trust_coefficient value: {group['trust_coefficient']}")


def _trust(w: torch.Tensor, d: torch.Tensor, coef: float) -> torch.Tensor:
    """coef * ‖w‖ / ‖d‖ when both norms are > 0, else 1 (fp32, on the parameter's device)."""
    wn = torch.linalg.vector_norm(w.float())
    dn = torch.linalg.vector_norm(d.float())
    one = torch.ones_like(wn)
    return torch.where((wn > 0) & (dn > 0), coef * wn / dn, one)


class LARS(torch.optim.Optimizer):
    """LARS in the MLPerf ResNet reference form (You et al. 2017).  For each tensor ``w`` with gradient ``g``:

    ``g' = g + weight_decay * w``; ``trust = trust_coefficient * ‖w‖ / ‖g'‖`` (1 if either norm is 0 or the
    group has ``adaptive=False``); ``v = momentum * v + lr * trust * g'`` (v starts at 0); ``w -= v``.

    State per parameter: ``momentum_buffer``.
    """

    def __init__(self, params, lr: float = 1e-3, momentum: float = 0.9, weight_decay: float = 0.0,
                 trust_coefficient: float = 0.001, adaptive: bool = True, maximize: bool = False):
        defaults = dict(lr=lr, momentum=momentum, weight_decay=weight_decay,
                        trust_coefficient=trust_coefficient, adaptive=adaptive, maximize=maximize)
        _check(defaults, betas=False)
        super().__init__(params, defaults)

    def add_param_group(self, param_group):
        super().add_param_group(param_group)
        _check(self.param_groups[-1], betas=False)

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            lr, mu, wd = group["lr"], group["momentum"], group["weight_decay"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                w = p if p.dtype == torch.float32 else p.float()
                d = p.grad.float()
                if wd != 0.0:
                    d = d.add(w, alpha=wd)
                trust = _trust(w, d, group["trust_coefficient"]) if group["adaptive"] else 1.0
                st = self.state[p]
                buf = st.get("momentum_buffer")
                if buf is None:
                    buf = st["momentum_buffer"] = torch.zeros_like(w, memory_format=torch.preserve_format)
                buf.mul_(mu).add_(d * (lr * trust))
                if w is p:
                    p.sub_(buf)
                else:
                    p.copy_(w.sub_(buf))
        return loss


class LAMB(torch.optim.Optimizer):
    """LAMB (You et al. 2019), without gradient pre-normalisation.  For each tensor ``w`` with gradient ``g``,
    at step ``t`` (starting at 1):

    ``m = b1 * m + (1 - b1) * g``; ``v = b2 * v + (1 - b2) * g²``;
    ``r = (m / (1 - b1^t)) / (sqrt(v) / sqrt(1 - b2^t) + eps) + weight_decay * w``;
    ``trust = ‖w‖ / ‖r‖`` (1 if either norm is 0 or the group has ``adaptive=False``); ``w -= lr * trust * r``.

    State per parameter: ``step``, ``exp_avg``, ``exp_avg_sq``.
    """

    def __init__(self, params, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-6,
                 weight_decay: float = 0.01, adaptive: bool = True, maximize: bool = False):
        defaults = dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay, adaptive=adaptive,
                        maximize=maximize)
        _check(defaults, betas=True)
        super().__init__(params, defaults)

    def add_param_group(self, param_group):
        super().add_param_group(param_group)
        _check(self.param_groups[-1], betas=True)

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            lr, wd, eps = group["lr"], group["weight_decay"], group["eps"]
            b1, b2 = group["betas"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                w = p if p.dtype == torch.float32 else p.float()
                g = p.grad.float()
                st = self.state[p]
                if "step" not in st:
                    st["step"] = torch.tensor(0.0)
                    st["exp_avg"] = torch.zeros_like(w, memory_format=torch.preserve_format)
                    st["exp_avg_sq"] = torch.zeros_like(w, memory_format=torch.preserve_format)
                st["step"] += 1
                t = float(st["step"])
                m, v = st["exp_avg"], st["exp_avg_sq"]
                m.lerp_(g, 1.0 - b1)
                v.mul_(b2).addcmul_(g, g, value=1.0 - b2)
                bc1 = 1.0 - b1 ** t
                bc2_sqrt = (1.0 - b2 ** t) ** 0.5
                r = (m / bc1) / (v.sqrt() / bc2_sqrt + eps)
                if wd != 0.0:
                    r.add_(w, alpha=wd)
                trust = _trust(w, r, 1.0) if group["adaptive"] else 1.0
                if w is p:
                    p.sub_(r * (lr * trust))
                else:
                    p.copy_(w.sub_(r * (lr * trust)))
        return loss


MUON_ADJUST_LR_FNS = (None, "original", "match_rms_adamw")


def muon_lr_ratio(adjust_lr_fn, shape) -> float:
    """Muon's learning-rate factor f of a [A, B] matrix: ``sqrt(max(1, A / B))`` for ``None`` / ``"original"``,
    ``0.2 * sqrt(max(A, B))`` for ``"match_rms_adamw"`` (which gives the update the RMS of an AdamW update)."""
    A, B = shape[:2]
    if adjust_lr_fn is None or adjust_lr_fn == "original":
        return math.sqrt(max(1, A / B))
    return 0.2 * math.sqrt(max(A, B))


def newton_schulz(u: torch.Tensor, ns_coefficients, ns_steps: int, eps: float) -> torch.Tensor:
    """The quintic Newton–Schulz orthogonalisation of ``torch.optim.Muon``, op for op: in bf16, on the transpose
    of a tall matrix, after dividing by the Frobenius norm clamped to ``eps``."""
    a, b, c = ns_coefficients
    x = u.bfloat16()
    tall = u.size(0) > u.size(1)
    if tall:
        x = x.T
    x.div_(x.norm().clamp(min=eps))
    for _ in range(ns_steps):
        gram = x @ x.T
        h = torch.addmm(gram, gram, gram, beta=b, alpha=c)
        x = torch.addmm(x, h, x, beta=a)
    return x.T if tall else x


def _check_muon(group: dict):
    _check({"lr": group["lr"], "weight_decay": group["weight_decay"], "maximize": group.get("maximize", False),
            "betas": group["betas"], "eps": group["adam_eps"]}, betas=True)
    if not 0.0 <= group["eps"]:
        raise ValueError(f"Invalid epsilon value: {group['eps']}")
    if not 0.0 <= group["momentum"] < 1.0:
        raise ValueError(f"Invalid momentum value: {group['momentum']}")
    if not (isinstance(group["ns_steps"], int) and 1 <= group["ns_steps"] <= 99):
        raise ValueError(f"Invalid ns_steps value: {group['ns_steps']} (1..99)")
    if group["adjust_lr_fn"] not in MUON_ADJUST_LR_FNS:
        raise ValueError(f"Adjust learning rate function {group['adjust_lr_fn']} is not supported")
    if len(tuple(group["ns_coefficients"])) != 3:
        raise ValueError("ns_coefficients must be three values (a, b, c)")
    if group["use_muon"]:
        for p in group["params"]:
            if p.dim() != 2:
                raise ValueError(f"Muon groups take 2-D parameters only, got one of size {tuple(p.shape)}; put it "
                                 "in a group with use_muon=False")


class Muon(torch.optim.Optimizer):
    """Muon (Jordan et al. 2024) for the matrices of a model, with AdamW for everything else, in one optimizer.

    Each param group has ``use_muon`` (default True).  Muon groups take 2-D parameters only and follow the code
    of ``torch.optim.Muon`` (torch 2.11); for each matrix ``w`` with gradient ``g``:

    ``buf.lerp_(g, 1 - momentum)``; ``u = g.lerp(buf, momentum)`` with ``nesterov``, else ``buf``;
    ``O = NS(u)`` (``newton_schulz``); ``w *= 1 - lr * weight_decay``; ``w -= lr * f * O`` with ``f`` from
    ``adjust_lr_fn`` (``muon_lr_ratio``).

    ``use_muon=False`` groups follow ``torch.optim.AdamW`` with the group's ``lr``, ``betas``, ``adam_eps`` and
    ``weight_decay``.  State per parameter: ``momentum_buffer`` (Muon), ``step``, ``exp_avg``, ``exp_avg_sq``
    (AdamW).  Wrapped in ``hvd.DistributedOptimizer`` on CUDA, the fused engine runs both rules from the bucket
    hooks, with the Newton–Schulz iterations on the wgmma GEMM (``parallel/fused_engine.py``).
    """

    def __init__(self, params, lr: float = 1e-3, weight_decay: float = 0.1, momentum: float = 0.95,
                 nesterov: bool = True, ns_coefficients=(3.4445, -4.775, 2.0315), eps: float = 1e-7,
                 ns_steps: int = 5, adjust_lr_fn=None, betas=(0.9, 0.95), adam_eps: float = 1e-8,
                 maximize: bool = False):
        defaults = dict(lr=lr, weight_decay=weight_decay, momentum=momentum, nesterov=nesterov,
                        ns_coefficients=tuple(ns_coefficients), eps=eps, ns_steps=ns_steps,
                        adjust_lr_fn=adjust_lr_fn, betas=tuple(betas), adam_eps=adam_eps, use_muon=True,
                        maximize=maximize)
        _check_muon({**defaults, "params": []})
        super().__init__(params, defaults)

    def add_param_group(self, param_group):
        super().add_param_group(param_group)
        _check_muon(self.param_groups[-1])

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            if group["use_muon"]:
                self._muon_group(group)
            else:
                self._adamw_group(group)
        return loss

    def _muon_group(self, group):
        lr, wd, mu = group["lr"], group["weight_decay"], group["momentum"]
        for p in group["params"]:
            if p.grad is None:
                continue
            g = p.grad
            st = self.state[p]
            if "momentum_buffer" not in st:
                st["momentum_buffer"] = torch.zeros_like(g, memory_format=torch.preserve_format)
            buf = st["momentum_buffer"]
            buf.lerp_(g, 1 - mu)
            u = g.lerp(buf, mu) if group["nesterov"] else buf
            o = newton_schulz(u, group["ns_coefficients"], group["ns_steps"], group["eps"])
            p.mul_(1 - lr * wd)
            p.add_(o, alpha=-(lr * muon_lr_ratio(group["adjust_lr_fn"], p.shape)))

    def _adamw_group(self, group):
        lr, wd, eps = group["lr"], group["weight_decay"], group["adam_eps"]
        b1, b2 = group["betas"]
        for p in group["params"]:
            if p.grad is None:
                continue
            g = p.grad
            st = self.state[p]
            if "step" not in st:
                st["step"] = torch.tensor(0.0)
                st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
            st["step"] += 1
            t = st["step"].item()
            m, v = st["exp_avg"], st["exp_avg_sq"]
            p.mul_(1 - lr * wd)
            m.lerp_(g, 1 - b1)
            v.mul_(b2).addcmul_(g, g, value=1 - b2)
            bc1 = 1 - b1 ** t
            bc2_sqrt = (1 - b2 ** t) ** 0.5
            denom = (v.sqrt() / bc2_sqrt).add_(eps)
            p.addcdiv_(m, denom, value=-(lr / bc1))
