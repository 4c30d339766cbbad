"""CPU oracle of the sparse optimizer (train.py --optimizer_type sparse_adam) -- TEST INFRASTRUCTURE ONLY, nothing under
gaussian-splatting_b200/ imports it.

* ``SparseGaussianAdamOracle``: a torch restatement of the accel branch's SparseGaussianAdam (train.py:180-183,
  scene/gaussian_model.py:194-196).  UNVERIFIED_VS_REFERENCE: the accel branch's source is absent from /root/reference; the
  semantics are the recalled ones the product states (diff_gaussian_rasterization/sparse_adam.py): betas (0.9, 0.999), no
  bias correction, rows with visibility False untouched (parameter and both moments), torch.optim.Adam's state keys,
  ``step`` never advanced.
* ``SparseModelOracle``: oracle.model_oracle.ModelOracle (the reference class's training state) with that optimizer in
  place of torch.optim.Adam, stepped as train.py:181-182 does: ``step(visible, N)``.

tests/golden/make_golden_sparse.py injects the first into the reference's own scene/gaussian_model.py to record
tests/golden/reference_sparse_adam.npz; the second replays that fixture."""
from __future__ import annotations

from typing import Dict

import torch

from oracle.model_oracle import GROUPS, ModelOracle


class SparseGaussianAdamOracle(torch.optim.Adam):
    def __init__(self, params, lr, eps):
        super().__init__(params=params, lr=lr, eps=eps)

    @torch.no_grad()
    def step(self, visibility: torch.Tensor, N: int):
        vis = visibility.reshape(-1).bool()
        assert vis.numel() == int(N)
        f32 = lambda x: torch.tensor(x, dtype=torch.float32)       # coefficients in float32, as a float kernel holds them
        b1, b2 = f32(0.9), f32(0.999)
        for group in self.param_groups:
            assert len(group["params"]) == 1
            p = group["params"][0]
            if p.grad is None:
                continue
            st = self.state[p]
            if len(st) == 0:
                st["step"] = torch.tensor(0.0, dtype=torch.float32)
                st["exp_avg"] = torch.zeros_like(p)
                st["exp_avg_sq"] = torch.zeros_like(p)
            g, m, v = p.grad[vis], st["exp_avg"][vis], st["exp_avg_sq"][vis]
            m = m + (1.0 - b1) * (g - m)
            v = v * b2 + ((1.0 - b2) * g) * g
            st["exp_avg"][vis], st["exp_avg_sq"][vis] = m, v
            p[vis] = p[vis] - f32(group["lr"]) * (m / (v.sqrt() + f32(group["eps"])))


class SparseModelOracle(ModelOracle):
    """ModelOracle with optimizer_type "sparse_adam" (gaussian_model.py:194-196): ``optimizer_cls`` (default the oracle
    above) over the same six groups; every optimizer-state surgery of ModelOracle works on it unchanged."""

    def __init__(self, *args, optimizer_cls=SparseGaussianAdamOracle, **kw):
        super().__init__(*args, **kw)
        groups = [{"params": [self.p[g["name"]]], "lr": g["lr"], "name": g["name"]} for g in self.adam.param_groups]
        assert [g["name"] for g in groups] == list(GROUPS)
        self.adam = optimizer_cls(groups, lr=0.0, eps=1e-15)

    def optimizer_step(self, visible: torch.Tensor) -> None:  # type: ignore[override]
        """train.py:181-183: visible = radii > 0 ([N] bool), N = radii.shape[0]."""
        self.adam.step(visible, visible.shape[0])
        self.adam.zero_grad(set_to_none=True)

    def step(self, iteration: int, act_grads: Dict[str, torch.Tensor], visible: torch.Tensor) -> None:  # type: ignore[override]
        self.backward(iteration, act_grads)
        self.optimizer_step(visible)
