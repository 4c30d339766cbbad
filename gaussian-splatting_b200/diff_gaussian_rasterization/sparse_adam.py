"""``SparseGaussianAdam``: the optimizer of ``train.py --optimizer_type sparse_adam`` (train.py:180-183,
scene/gaussian_model.py:194-196), stepping only the gaussians that were visible in the view.

Semantics [RECALL, UNVERIFIED_VS_REFERENCE] -- the accel branch's source is absent from /root/reference, so this states
what that optimizer is recalled to do, the same way gaussian_store's ``optimizer_type="sparse_adam"`` mode does:
  * betas (0.9, 0.999), each group's own ``lr`` and ``eps``, NO bias correction:
        m += (1-b1)(g - m);  v = b2 v + (1-b2) g^2;  p -= lr * m / (sqrt(v) + eps)
  * rows whose ``visibility`` is False keep their parameter AND both moments untouched (no decay);
  * the state's ``step`` is created (torch.optim.Adam's key) but never advanced.

The state is torch.optim.Adam's (``step``, ``exp_avg``, ``exp_avg_sq`` per parameter), created lazily on the first step, so
the reference's optimizer-state surgery (replace_tensor_to_optimizer, _prune_optimizer, cat_tensors_to_optimizer) and
capture() / restore() work on it unchanged.  Every stepped group goes into ONE CUDA launch (gsb_sparse_adam_step, csrc/
optim.cu: the store's sparse update, the same device function) with no host synchronisation.
"""
from __future__ import annotations

import torch

import diff_gaussian_rasterization as _pkg

__all__ = ["SparseGaussianAdam"]

BETAS = (0.9, 0.999)


def _check_dense(t: torch.Tensor, what: str) -> None:
    _pkg._require_cuda(t)
    if t.dtype != torch.float32 or not t.is_contiguous():
        raise ValueError(f"SparseGaussianAdam: {what} must be a contiguous float32 tensor (got {t.dtype}, "
                         f"contiguous={t.is_contiguous()})")


class SparseGaussianAdam(torch.optim.Adam):
    def __init__(self, params, lr, eps):
        super().__init__(params=params, lr=lr, eps=eps)

    @torch.no_grad()
    def step(self, visibility: torch.Tensor, N: int):
        """Updates the rows ``i`` with ``visibility[i]`` of every group whose parameter has a gradient.  Every such
        parameter is [N, ...]; ``visibility`` is [N] (bool, e.g. ``radii > 0``, or uint8) on the parameters' device."""
        N = int(N)
        _pkg._require_cuda(visibility)
        if visibility.numel() != N:
            raise ValueError(f"SparseGaussianAdam.step: visibility has {visibility.numel()} entries, N = {N}")
        todo = []
        for group in self.param_groups:
            if len(group["params"]) != 1:
                raise ValueError("SparseGaussianAdam: every parameter group must hold exactly one tensor")
            p = group["params"][0]
            if p.grad is None:
                continue
            _check_dense(p, f"parameter of group {group.get('name', len(todo))!r}")
            _check_dense(p.grad, f"gradient of group {group.get('name', len(todo))!r}")
            if p.dim() == 0 or p.shape[0] != N or p.grad.shape != p.shape:
                raise ValueError(f"SparseGaussianAdam.step: group {group.get('name', '')!r} has shape {tuple(p.shape)} "
                                 f"(gradient {tuple(p.grad.shape)}), expected [N = {N}, ...]")
            state = self.state[p]
            if len(state) == 0:
                state["step"] = torch.tensor(0.0, dtype=torch.float32)
                state["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
            m, v = state["exp_avg"], state["exp_avg_sq"]
            _check_dense(m, "exp_avg")
            _check_dense(v, "exp_avg_sq")
            if m.shape != p.shape or v.shape != p.shape:
                raise ValueError(f"SparseGaussianAdam.step: moments of group {group.get('name', '')!r} do not match its parameter")
            todo.append((p, p.grad, m, v, group["lr"], group["eps"]))
        for k in range(0, len(todo), _pkg.MAX_SPARSE_GROUPS):
            _pkg.sparse_adam_step(todo[k:k + _pkg.MAX_SPARSE_GROUPS], visibility, N, *BETAS)
