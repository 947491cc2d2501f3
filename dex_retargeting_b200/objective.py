"""The retargeting objective as a differentiable torch function of the joint vectors (learning-based retargeting: the
objective a solve minimises, used as a training loss).

`retargeting_cost(opt, qpos, ...)` returns, per frame, L(x) + norm_delta |x - last_qpos|^2 at the GIVEN joint vectors
`qpos` [B,opt_dof] (`Optimizer.objective_batch`, one `dexr_eval_objective` launch); backward returns
grad_output[:, None] * d cost / d qpos from the same launch.  Derivatives with respect to the keypoints, the fixed joints
or the anchor are not computed: those arguments must not require grad.
"""
from __future__ import annotations

import torch
from torch.autograd.function import once_differentiable


class _RetargetingCost(torch.autograd.Function):
    @staticmethod
    def forward(ctx, qpos, opt, kwargs):
        _, cost, grad = opt.objective_batch(qpos.detach(), want_grad=ctx.needs_input_grad[0], **kwargs)
        ctx.save_for_backward(grad)
        return cost

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        (grad,) = ctx.saved_tensors
        return grad_output[:, None] * grad, None, None


def retargeting_cost(opt, qpos, *, keypoints=None, ref_value=None, fixed_qpos=None, last_qpos=None, projected=None,
                     raw_hand=None):
    """cost [B] of optimizer `opt` at `qpos` [B,opt_dof] (float32 CUDA tensors as for `Optimizer.objective_batch`),
    differentiable in `qpos`.  `projected` (DexPilot flags) is read and updated in place by the forward call."""
    for name, t in (("keypoints", keypoints), ("ref_value", ref_value), ("fixed_qpos", fixed_qpos), ("last_qpos", last_qpos)):
        if t is not None and t.requires_grad:
            raise ValueError(f"{name} requires grad, but retargeting_cost is only differentiable in qpos: detach it")
    kwargs = dict(keypoints=keypoints, ref_value=ref_value, fixed_qpos=fixed_qpos, last_qpos=last_qpos, projected=projected,
                  raw_hand=raw_hand)
    return _RetargetingCost.apply(qpos, opt, kwargs)
