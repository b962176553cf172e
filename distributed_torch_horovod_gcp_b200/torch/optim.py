"""Layer-wise adaptive optimizers: ``hvd.LARS`` and ``hvd.LAMB``.

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
