"""Element-wise error bounds against float64 references, shared by the kernel numerics tests.

A test computes the operation in float64 from the exact low-precision inputs the kernel saw (``ref64``)
and a bound on the kernel's error derived from the roundings the kernel performs: a sum of magnitude
terms (float64 tensors, broadcast against ``ref64``), each with its own coefficient.  Nothing is fitted
to observed errors, so a bound that holds does not flake, and one that breaks is a finding.

The worst err/bound ratio of every group is kept and printed by ``report_ratios`` (the test modules
call it at module teardown; run pytest with ``-s`` to see it).
"""
import numpy as np
import torch

U32 = 2.0 ** -24          # unit roundoff of fp32
U_BF16 = 2.0 ** -8        # relative rounding error of a bf16 store

_WORST = {}


def report_ratios():
    """Print the worst err/bound ratio of each group checked since the last report."""
    for k in sorted(_WORST):
        print(f"\n[err/bound] {k}: max {_WORST[k]:.3e}", end="")
    print()
    _WORST.clear()


def assert_within_bound(out, ref64, mag64=None, n_terms=0, out_bf16=False, group="misc", terms=()):
    """|out - ref64| <= 2 * n_terms * 2^-24 * mag64 (+ 2^-8 * |ref64| for a bf16 output)
    + sum(coef * mag for coef, mag in terms), elementwise.

    ``ref64``: the operation in float64 on the inputs the kernel saw; ``mag64``: the same operation on
    absolute values.  The first term bounds any fp32 summation order and rounding of ``n_terms`` terms.
    ``terms`` adds further (coefficient, magnitude) pairs; a coefficient may be a tensor (e.g. per row)."""
    out64 = out.detach().double()
    err = (out64 - ref64).abs()
    bound = torch.zeros_like(err)
    if mag64 is not None:
        bound = bound + 2.0 * n_terms * U32 * mag64
    if out_bf16:
        bound = bound + U_BF16 * ref64.abs()
    for coef, mag in terms:
        bound = bound + coef * mag
    ratio = torch.where(bound > 0, err / bound.clamp_min(1e-300),
                        torch.where(err > 0, torch.full_like(err, float("inf")), torch.zeros_like(err)))
    # NaN anywhere (out or reference) is a failure, never a pass
    ratio = torch.where(torch.isnan(ratio), torch.full_like(ratio, float("inf")), ratio)
    worst = int(torch.argmax(ratio))
    r = float(ratio.reshape(-1)[worst])
    _WORST[group] = max(_WORST.get(group, 0.0), r)
    if not r <= 1.0:
        idx = np.unravel_index(worst, tuple(ratio.shape))
        raise AssertionError(
            f"{group}: {int((ratio > 1).sum())} element(s) outside the fp64 bound; worst at {tuple(map(int, idx))}: "
            f"out={float(out64[idx]):.9g} ref={float(ref64[idx]):.9g} err/bound={r:.3g}")
