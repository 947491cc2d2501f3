"""The retargeting objective as a differentiable torch function of the joint vectors (learning-based retargeting: the
objective a solve minimises, used as a training loss).

`retargeting_cost(opt, qpos, ...)` returns, per frame, L(x) + norm_delta |x - last_qpos|^2 at the GIVEN joint vectors
`qpos` [B,opt_dof] (`Optimizer.objective_batch`, one `dexr_eval_objective` launch); backward returns
grad_output[:, None] * d cost / d qpos from the same launch.  Derivatives with respect to the keypoints, the fixed joints
or the anchor are not computed: those arguments must not require grad.

`differentiable_retarget(opt, ...)` is the other direction: the solve's answer as a differentiable function of the keypoints
(or ref_value), the fixed joints and the anchor (`Optimizer.retarget_batch` forward, `Optimizer.retarget_batch_vjp` backward):
a hand-pose network trained with a loss on the robot joint angles backpropagates through the retargeting with it.

`differentiable_retarget_sequences(seq, keypoints, state)` does the same for whole streams with `SeqRetargeting`'s
semantics (clipped warm start, carried solution, mimic, low-pass filter): forward one recorded `retarget_sequences` launch,
backward one `retarget_sequences_vjp` launch through every frame of every stream.  The returned state carries the graph,
so chained calls backpropagate across chunk boundaries.
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


class _DifferentiableRetarget(torch.autograd.Function):
    @staticmethod
    def forward(ctx, targets, fixed_qpos, last_qpos, opt, cfg):
        by_kp, projected, clip_init = cfg["by_kp"], cfg["projected"], cfg["clip_init"]
        tgt = dict(keypoints=targets) if by_kp else dict(ref_value=targets)
        if projected is None and opt.retargeting_type == "DEXPILOT":
            # the backward needs the flags the solve leaves; every frame starts unprojected, as with no flag buffer
            projected = torch.zeros((targets.shape[0], opt._objective_spec().len_proj), dtype=torch.uint8,
                                    device=targets.device)
        kw = {k: v.detach() for k, v in tgt.items()}
        if cfg["raw_hand"] is not None:
            kw["raw_hand"] = cfg["raw_hand"]
        qpos = opt.retarget_batch(fixed_qpos=None if fixed_qpos is None else fixed_qpos.detach(), last_qpos=last_qpos.detach(),
                                  projected=projected, clip_init=clip_init, **kw)
        flags = None if projected is None else projected.clone()
        ctx.opt, ctx.by_kp = opt, by_kp
        ctx.save_for_backward(qpos, targets.detach(), None if fixed_qpos is None else fixed_qpos.detach(), last_qpos.detach(),
                              flags)
        return qpos

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_qpos):
        qpos, targets, fixed_qpos, last_qpos, flags = ctx.saved_tensors
        tgt = dict(keypoints=targets) if ctx.by_kp else dict(ref_value=targets)
        g_tgt, g_fixed, g_last = ctx.opt.retarget_batch_vjp(grad_qpos.contiguous(), qpos, fixed_qpos=fixed_qpos,
                                                            last_qpos=last_qpos, projected=flags, **tgt)
        return g_tgt, g_fixed, g_last, None, None


def differentiable_retarget(opt, *, keypoints=None, ref_value=None, fixed_qpos=None, last_qpos, projected=None,
                            clip_init=False, raw_hand=None):
    """qpos [B,opt_dof] = `opt.retarget_batch(...)` (float32 CUDA tensors as there), differentiable in `keypoints` or
    `ref_value`, in `fixed_qpos` and in `last_qpos` as the anchor of the norm_delta term (its warm-start role only picks the
    basin).  backward() is one `Optimizer.retarget_batch_vjp` launch: the implicit-function derivative of the converged
    solution (active bounds get zero sensitivity; a frame that ended at max_iters gets the derivative of the linearisation at
    its answer; one whose free Hessian is not positive definite gets zero gradients).  `projected` (DexPilot flags) is updated
    in place by the solve, as by `retarget_batch`; the backward uses a copy of the flags the solve left.
    Chaining calls with one frame's output as the next call's `last_qpos` backpropagates through a stream fed frame by
    frame.  Raw detector landmarks (`raw_hand`) are solved but not differentiated: pre-process them first."""
    if (keypoints is None) == (ref_value is None):
        raise ValueError("give exactly one of keypoints / ref_value")
    targets = keypoints if keypoints is not None else ref_value
    if raw_hand is not None and any(t is not None and t.requires_grad for t in (targets, fixed_qpos, last_qpos)):
        raise ValueError("raw_hand: raw-landmark pre-processing is not differentiated; pre-process the keypoints "
                         "(dexr_preprocess_keypoints) and pass them without raw_hand")
    cfg = dict(by_kp=keypoints is not None, projected=projected, clip_init=clip_init, raw_hand=raw_hand)
    return _DifferentiableRetarget.apply(targets, fixed_qpos, last_qpos, opt, cfg)


class _DifferentiableRetargetSequences(torch.autograd.Function):
    @staticmethod
    def forward(ctx, keypoints, fixed_qpos, last_qpos, filter_state, seq, cfg):
        from .seq_retarget import StreamState

        st = cfg["state"]
        new = StreamState(last_qpos=last_qpos.detach().clone(), filter_state=filter_state.detach().clone(),
                          filter_init=st.filter_init.clone(), projected=None if st.projected is None else st.projected.clone(),
                          damping=None if st.damping is None else st.damping.clone())
        S, T = int(keypoints.shape[0]), int(keypoints.shape[1])
        tape = seq.make_sequence_tape(S, T)
        kp = keypoints.detach().contiguous()
        fixed = None if fixed_qpos is None else fixed_qpos.detach().contiguous()
        out, _ = seq.retarget_sequences(kp, new, fixed_qpos=fixed, tape=tape)
        ctx.seq, ctx.tape = seq, tape
        ctx.save_for_backward(kp, fixed, last_qpos.detach().contiguous(), st.filter_init.clone())
        ctx.set_materialize_grads(False)
        cfg["new_state"] = new
        return out, new.last_qpos, new.filter_state

    @staticmethod
    @once_differentiable
    def backward(ctx, g_out, g_last, g_filter):
        keypoints, fixed, last0, finit0 = ctx.saved_tensors
        c = (lambda g: None if g is None else g.contiguous())
        g_kp, g_fixed, g_last0, g_filter0 = ctx.seq.retarget_sequences_vjp(
            keypoints, ctx.tape, last0, finit0, grad_robot_qpos=c(g_out), grad_last_qpos=c(g_last),
            grad_filter_state=c(g_filter), fixed_qpos=fixed)
        return g_kp, g_fixed, g_last0, g_filter0, None, None


def differentiable_retarget_sequences(seq, keypoints, state=None, fixed_qpos=None, *, raw_hand=None):
    """(robot_qpos [S,T,dof], new_state) = `seq.retarget_sequences(keypoints, state, fixed_qpos)` (float32 CUDA tensors as
    there), differentiable in `keypoints`, `fixed_qpos`, `state.last_qpos` and `state.filter_state`.  `state` (None: fresh
    streams, `seq.make_stream_state`) is not modified: autograd keeps it, and a new `StreamState` comes back whose
    `last_qpos` and `filter_state` carry the graph -- feed it to the next call for full or truncated (detach it)
    backpropagation through time over long recordings.  backward() is one `retarget_sequences_vjp` launch: every frame's
    implicit-function derivative at its solution and clipped anchor, the anchor chain through the clip and the low-pass
    filter (see `SeqRetargeting.retarget_sequences_vjp`).  Raw detector landmarks (`raw_hand`) are solved but not
    differentiated: pre-process them first."""
    from .seq_retarget import StreamState

    S = int(keypoints.shape[0])
    state = seq.make_stream_state(S) if state is None else state
    if raw_hand is not None:
        if any(t is not None and t.requires_grad for t in (keypoints, fixed_qpos, state.last_qpos, state.filter_state)):
            raise ValueError("raw_hand: raw-landmark pre-processing is not differentiated; pre-process the keypoints "
                             "(dexr_preprocess_keypoints) and pass them without raw_hand")
        new = StreamState(**{k: (None if getattr(state, k) is None else getattr(state, k).clone()) for k in StreamState._FIELDS})
        out, new = seq.retarget_sequences(keypoints, new, fixed_qpos=fixed_qpos, raw_hand=raw_hand)
        return out, new
    cfg = dict(state=state)
    out, last, filt = _DifferentiableRetargetSequences.apply(keypoints, fixed_qpos, state.last_qpos, state.filter_state, seq,
                                                             cfg)
    new = cfg["new_state"]
    return out, StreamState(last_qpos=last, filter_state=filt, filter_init=new.filter_init, projected=new.projected,
                            damping=new.damping)


class _DifferentiableRetargetPackedSequences(torch.autograd.Function):
    @staticmethod
    def forward(ctx, keypoints, fixed_qpos, last_qpos, filter_state, seq, cfg):
        from .seq_retarget import StreamState

        st, layout = cfg["state"], cfg["layout"]
        new = StreamState(last_qpos=last_qpos.detach().clone(), filter_state=filter_state.detach().clone(),
                          filter_init=st.filter_init.clone(), projected=None if st.projected is None else st.projected.clone(),
                          damping=None if st.damping is None else st.damping.clone())
        tape = seq.make_packed_sequence_tape(layout)
        kp = keypoints.detach().contiguous()
        fixed = None if fixed_qpos is None else fixed_qpos.detach().contiguous()
        out, _ = seq.retarget_packed_sequences(kp, layout, new, fixed_qpos=fixed, tape=tape)
        ctx.seq, ctx.tape, ctx.layout = seq, tape, layout
        ctx.save_for_backward(kp, fixed, last_qpos.detach().contiguous(), st.filter_init.clone())
        ctx.set_materialize_grads(False)
        cfg["new_state"] = new
        return out, new.last_qpos, new.filter_state

    @staticmethod
    @once_differentiable
    def backward(ctx, g_out, g_last, g_filter):
        keypoints, fixed, last0, finit0 = ctx.saved_tensors
        c = (lambda g: None if g is None else g.contiguous())
        g_kp, g_fixed, g_last0, g_filter0 = ctx.seq.retarget_packed_sequences_vjp(
            keypoints, ctx.layout, ctx.tape, last0, finit0, grad_robot_qpos=c(g_out), grad_last_qpos=c(g_last),
            grad_filter_state=c(g_filter), fixed_qpos=fixed)
        return g_kp, g_fixed, g_last0, g_filter0, None, None


def differentiable_retarget_packed_sequences(seq, keypoints, layout, state=None, fixed_qpos=None, *, raw_hand=None):
    """(robot_qpos [N,dof], new_state) = `seq.retarget_packed_sequences(keypoints, layout, state, fixed_qpos)` for streams of
    any lengths packed end to end (`seq.pack_streams`), differentiable in `keypoints` [N,21,3], `fixed_qpos` [N,n_fixed],
    `state.last_qpos` and `state.filter_state` ([S,...]).  The contract of `differentiable_retarget_sequences`: `state` is
    not modified, and the returned state carries the graph across chunks.  backward() is one
    `retarget_packed_sequences_vjp` launch.  Raw detector landmarks (`raw_hand`) are solved but not differentiated."""
    from .seq_retarget import StreamState

    state = seq.make_stream_state(layout.num_streams) if state is None else state
    if raw_hand is not None:
        if any(t is not None and t.requires_grad for t in (keypoints, fixed_qpos, state.last_qpos, state.filter_state)):
            raise ValueError("raw_hand: raw-landmark pre-processing is not differentiated; pre-process the keypoints "
                             "(dexr_preprocess_keypoints) and pass them without raw_hand")
        new = StreamState(**{k: (None if getattr(state, k) is None else getattr(state, k).clone()) for k in StreamState._FIELDS})
        return seq.retarget_packed_sequences(keypoints, layout, new, fixed_qpos=fixed_qpos, raw_hand=raw_hand)
    cfg = dict(state=state, layout=layout)
    out, last, filt = _DifferentiableRetargetPackedSequences.apply(keypoints, fixed_qpos, state.last_qpos,
                                                                   state.filter_state, seq, cfg)
    new = cfg["new_state"]
    return out, StreamState(last_qpos=last, filter_state=filt, filter_init=new.filter_init, projected=new.projected,
                            damping=new.damping)


class _DifferentiableSmoothPackedSequences(torch.autograd.Function):
    @staticmethod
    def forward(ctx, keypoints, fixed_qpos, last_qpos, seq, cfg):
        from .seq_retarget import StreamState

        st, layout = cfg["state"], cfg["layout"]
        kp = keypoints.detach().contiguous()
        fixed = None if fixed_qpos is None else fixed_qpos.detach().contiguous()
        last0 = last_qpos.detach().contiguous()
        proj0 = None if st.projected is None else st.projected.clone()
        view = StreamState(last_qpos=last0, filter_state=st.filter_state.detach(), filter_init=st.filter_init,
                           projected=proj0, damping=None if st.damping is None else st.damping.detach())
        rq, q, status = seq.smooth_packed_sequences(kp, layout, view, fixed_qpos=fixed, qpos_init=cfg["qpos_init"],
                                                    smooth_weight=cfg["smooth_weight"], accel_weight=cfg["accel_weight"])
        ctx.seq, ctx.layout, ctx.smooth_weight, ctx.accel_weight = seq, layout, cfg["smooth_weight"], cfg["accel_weight"]
        ctx.save_for_backward(kp, fixed, last0, proj0, q)
        ctx.set_materialize_grads(False)
        ctx.mark_non_differentiable(status)
        return rq, q, status

    @staticmethod
    @once_differentiable
    def backward(ctx, g_rq, g_q, _g_status):
        kp, fixed, last0, proj0, q = ctx.saved_tensors
        c = (lambda g: None if g is None else g.contiguous())
        g_kp, g_fixed, g_last = ctx.seq.smooth_packed_sequences_vjp(
            kp, ctx.layout, q, last0, proj0, grad_qpos=c(g_q), grad_robot_qpos=c(g_rq), fixed_qpos=fixed,
            smooth_weight=ctx.smooth_weight, accel_weight=ctx.accel_weight)
        return g_kp, g_fixed, g_last, None, None


def differentiable_smooth_packed_sequences(seq, keypoints, layout, state=None, fixed_qpos=None, *, qpos_init=None,
                                           smooth_weight=None, accel_weight=None):
    """(robot_qpos [N,dof], qpos [N,opt_dof], status [N]) = `seq.smooth_packed_sequences(keypoints, layout, state, ...)`
    (recorded clips packed end to end, `seq.pack_streams`; float32 CUDA tensors as there), differentiable in `keypoints`
    [N,21,3], `fixed_qpos` [N,n_fixed] and the anchor `state.last_qpos` [S,opt_dof], through both robot_qpos and qpos.
    `state` (None: fresh streams) is read only, as by the forward.  backward() is one `smooth_packed_sequences_vjp`
    launch: the implicit-function derivative of the smoothed clips, one linear solve with the stacked Hessian per stream.
    The gradient is not causal: a loss on one frame reaches the keypoints of the whole clip.  The DexPilot flags, the
    starting trajectory `qpos_init`, `smooth_weight` and `accel_weight` (the acceleration penalty of
    `smooth_packed_sequences`; None or 0: none) are not differentiated: they, and the state's other tensors, must not
    require grad."""
    state = seq.make_stream_state(layout.num_streams) if state is None else state
    for name, t in (("qpos_init", qpos_init), ("smooth_weight", smooth_weight), ("accel_weight", accel_weight),
                    ("state.filter_state", state.filter_state), ("state.damping", state.damping)):
        if isinstance(t, torch.Tensor) and t.requires_grad:
            raise ValueError(f"{name} requires grad, but the smoother is not differentiated in it: detach it")
    if isinstance(smooth_weight, torch.Tensor):
        smooth_weight = float(smooth_weight)
    if isinstance(accel_weight, torch.Tensor):
        accel_weight = float(accel_weight)
    cfg = dict(state=state, layout=layout, qpos_init=qpos_init, smooth_weight=smooth_weight, accel_weight=accel_weight)
    return _DifferentiableSmoothPackedSequences.apply(keypoints, fixed_qpos, state.last_qpos, seq, cfg)


def _fixed_lag_copy(state):
    """A detached copy of a FixedLagState (the forward updates its state in place; autograd keeps the original)."""
    from .seq_retarget import FixedLagState

    return FixedLagState(lag=state.lag, accel_weight=float(state.accel_weight),
                         **{k: (None if getattr(state, k) is None else getattr(state, k).detach().clone())
                            for k in FixedLagState._FIELDS})


class _DifferentiableRetargetFixedLag(torch.autograd.Function):
    @staticmethod
    def forward(ctx, keypoints, fixed_qpos, last_qpos, window_keypoints, window_fixed_qpos, window_qpos, seq, cfg):
        state0 = _fixed_lag_copy(cfg["state"])
        new = _fixed_lag_copy(state0)
        S, K = int(keypoints.shape[0]), int(keypoints.shape[1])
        tape = seq.make_fixed_lag_tape(S, K, state0.lag)
        kp = keypoints.detach().contiguous()
        fixed = None if fixed_qpos is None else fixed_qpos.detach().contiguous()
        rq, q, status = seq.retarget_fixed_lag(kp, new, fixed_qpos=fixed, smooth_weight=cfg["smooth_weight"], tape=tape)
        ctx.seq, ctx.tape, ctx.state0, ctx.smooth_weight = seq, tape, state0, cfg["smooth_weight"]
        ctx.save_for_backward(kp, fixed)
        ctx.set_materialize_grads(False)
        ctx.mark_non_differentiable(status)
        cfg["new_state"] = new
        return rq, q, status, new.last_qpos, new.window_keypoints, new.window_fixed_qpos, new.window_qpos

    @staticmethod
    @once_differentiable
    def backward(ctx, g_rq, g_q, _g_status, g_last, g_wkp, g_wfix, g_wq):
        kp, fixed = ctx.saved_tensors
        c = (lambda g: None if g is None else g.contiguous())
        g_kp, g_fixed, g_last0, g_wkp0, g_wfix0, g_wq0, _ = ctx.seq.retarget_fixed_lag_vjp(
            kp, ctx.tape, ctx.state0, fixed_qpos=fixed, grad_qpos=c(g_q), grad_robot_qpos=c(g_rq),
            grad_last_qpos_out=c(g_last), grad_window_qpos_out=c(g_wq), grad_window_keypoints_out=c(g_wkp),
            grad_window_fixed_qpos_out=c(g_wfix), smooth_weight=ctx.smooth_weight)
        return g_kp, g_fixed, g_last0, g_wkp0, g_wfix0, g_wq0, None, None


def differentiable_retarget_fixed_lag(seq, keypoints, state, fixed_qpos=None, *, smooth_weight=None):
    """(robot_qpos [S,K,dof], qpos [S,K,opt_dof], status [S,K], new_state) = `seq.retarget_fixed_lag(keypoints, state,
    ...)` (float32 CUDA tensors as there), differentiable in `keypoints`, `fixed_qpos` and the state's `last_qpos`,
    `window_keypoints`, `window_fixed_qpos` and `window_qpos`.  The contract of `differentiable_retarget_sequences`: `state`
    is not modified, and the returned FixedLagState's last_qpos and window tensors carry the graph, so chunks of a live
    stream backpropagate across call boundaries (detach the state for truncated backpropagation).  backward() is one
    `retarget_fixed_lag_vjp` launch: each emitting window's smoother VJP, the anchor chain through the committed frames.
    PENDING rows (NaN) get no gradient.  The DexPilot flags and `smooth_weight` are not differentiated.  A state with an
    acceleration penalty is refused (ValueError): its backward is `differentiable_retarget_fixed_lag_accel`."""
    from .seq_retarget import FixedLagState, _refuse_accel_backward

    _refuse_accel_backward(state, "differentiable_retarget_fixed_lag")
    if isinstance(smooth_weight, torch.Tensor):
        if smooth_weight.requires_grad:
            raise ValueError("smooth_weight requires grad, but fixed-lag smoothing is not differentiated in it: detach it")
        smooth_weight = float(smooth_weight)
    cfg = dict(state=state, smooth_weight=smooth_weight)
    rq, q, status, last, wkp, wfix, wq = _DifferentiableRetargetFixedLag.apply(
        keypoints, fixed_qpos, state.last_qpos, state.window_keypoints, state.window_fixed_qpos, state.window_qpos, seq, cfg)
    new = cfg["new_state"]
    return rq, q, status, FixedLagState(lag=new.lag, last_qpos=last, projected=new.projected, window_keypoints=wkp,
                                        window_fixed_qpos=wfix, window_qpos=wq, window_len=new.window_len)


class _DifferentiableFlushFixedLag(torch.autograd.Function):
    @staticmethod
    def forward(ctx, last_qpos, window_keypoints, window_fixed_qpos, window_qpos, seq, cfg):
        state0 = _fixed_lag_copy(cfg["state"])
        new = _fixed_lag_copy(state0)
        rq, q, count = seq.flush_fixed_lag(new)
        ctx.seq, ctx.state0 = seq, state0
        ctx.set_materialize_grads(False)
        ctx.mark_non_differentiable(count)
        cfg["new_state"] = new
        return rq, q, count, new.last_qpos, new.window_keypoints, new.window_fixed_qpos, new.window_qpos

    @staticmethod
    @once_differentiable
    def backward(ctx, g_rq, g_q, _g_count, g_last, g_wkp, g_wfix, g_wq):
        c = (lambda g: None if g is None else g.contiguous())
        g_last0, g_wkp0, g_wfix0, g_wq0 = ctx.seq.flush_fixed_lag_vjp(
            ctx.state0, grad_qpos=c(g_q), grad_robot_qpos=c(g_rq), grad_last_qpos_out=c(g_last),
            grad_window_qpos_out=c(g_wq), grad_window_keypoints_out=c(g_wkp), grad_window_fixed_qpos_out=c(g_wfix))
        return g_last0, g_wkp0, g_wfix0, g_wq0, None, None


def differentiable_flush_fixed_lag(seq, state):
    """(robot_qpos [S,L,dof], qpos [S,L,opt_dof], count [S], new_state) = `seq.flush_fixed_lag(state)`, differentiable in
    the state's `last_qpos` and window tensors (the flushed rows are its held slots of window_qpos).  `state` is not
    modified; the returned state carries the graph as `differentiable_retarget_fixed_lag`'s does.  A state with an
    acceleration penalty is refused (ValueError), as there: its backward is `differentiable_flush_fixed_lag_accel`."""
    from .seq_retarget import FixedLagState, _refuse_accel_backward

    _refuse_accel_backward(state, "differentiable_flush_fixed_lag")
    cfg = dict(state=state)
    rq, q, count, last, wkp, wfix, wq = _DifferentiableFlushFixedLag.apply(
        state.last_qpos, state.window_keypoints, state.window_fixed_qpos, state.window_qpos, seq, cfg)
    new = cfg["new_state"]
    return rq, q, count, FixedLagState(lag=new.lag, last_qpos=last, projected=new.projected, window_keypoints=wkp,
                                       window_fixed_qpos=wfix, window_qpos=wq, window_len=new.window_len)


def _accel_weight_of(state, what):
    """The state's acceleration weight as a float: it is not differentiated, so a tensor that requires grad is refused."""
    c = state.accel_weight
    if isinstance(c, torch.Tensor):
        if c.requires_grad:
            raise ValueError(f"{what}: accel_weight requires grad, but fixed-lag smoothing is not differentiated in it: "
                             "detach it")
        c = float(c)
    if not c:
        raise ValueError(f"{what}: the state has no acceleration penalty (accel_weight = 0): use "
                         f"{what.replace('_accel', '')}")
    return float(c)


def _accel_copy(state, c):
    new = _fixed_lag_copy(state)
    new.accel_weight = c
    return new


class _DifferentiableRetargetFixedLagAccel(torch.autograd.Function):
    @staticmethod
    def forward(ctx, keypoints, fixed_qpos, last_qpos, window_keypoints, window_fixed_qpos, window_qpos, prev_qpos, seq, cfg):
        state0 = _accel_copy(cfg["state"], cfg["accel_weight"])
        new = _fixed_lag_copy(state0)
        S, K = int(keypoints.shape[0]), int(keypoints.shape[1])
        tape = seq.make_fixed_lag_tape(S, K, state0.lag, accel_weight=state0.accel_weight)
        kp = keypoints.detach().contiguous()
        fixed = None if fixed_qpos is None else fixed_qpos.detach().contiguous()
        rq, q, status = seq.retarget_fixed_lag(kp, new, fixed_qpos=fixed, smooth_weight=cfg["smooth_weight"], tape=tape)
        ctx.seq, ctx.tape, ctx.state0, ctx.smooth_weight = seq, tape, state0, cfg["smooth_weight"]
        ctx.save_for_backward(kp, fixed)
        ctx.set_materialize_grads(False)
        ctx.mark_non_differentiable(status)
        cfg["new_state"] = new
        return (rq, q, status, new.last_qpos, new.window_keypoints, new.window_fixed_qpos, new.window_qpos,
                new.prev_qpos)

    @staticmethod
    @once_differentiable
    def backward(ctx, g_rq, g_q, _g_status, g_last, g_wkp, g_wfix, g_wq, g_prev):
        kp, fixed = ctx.saved_tensors
        c = (lambda g: None if g is None else g.contiguous())
        g_kp, g_fixed, g_last0, g_wkp0, g_wfix0, g_wq0, _, g_prev0 = ctx.seq.retarget_fixed_lag_accel_vjp(
            kp, ctx.tape, ctx.state0, fixed_qpos=fixed, grad_qpos=c(g_q), grad_robot_qpos=c(g_rq),
            grad_last_qpos_out=c(g_last), grad_prev_qpos_out=c(g_prev), grad_window_qpos_out=c(g_wq),
            grad_window_keypoints_out=c(g_wkp), grad_window_fixed_qpos_out=c(g_wfix), smooth_weight=ctx.smooth_weight)
        return g_kp, g_fixed, g_last0, g_wkp0, g_wfix0, g_wq0, g_prev0, None, None


def _accel_state_out(new, last, wkp, wfix, wq, prev):
    from .seq_retarget import FixedLagState

    return FixedLagState(lag=new.lag, last_qpos=last, projected=new.projected, window_keypoints=wkp, window_fixed_qpos=wfix,
                         window_qpos=wq, window_len=new.window_len, accel_weight=new.accel_weight, prev_qpos=prev,
                         has_prev=new.has_prev)


def differentiable_retarget_fixed_lag_accel(seq, keypoints, state, fixed_qpos=None, *, smooth_weight=None):
    """`differentiable_retarget_fixed_lag` for an accelerated state (`make_fixed_lag_state(S, L, accel_weight=c)`, c > 0):
    (robot_qpos, qpos, status, new_state) = `seq.retarget_fixed_lag(keypoints, state, ...)`, differentiable in
    `keypoints`, `fixed_qpos` and the state's `last_qpos`, `prev_qpos` and window tensors.  The returned state carries
    accel_weight, has_prev and the graph through last_qpos, prev_qpos and the windows, so chunks backpropagate across call
    boundaries.  backward() is one `retarget_fixed_lag_accel_vjp` launch.  The DexPilot flags, `smooth_weight`, c and
    has_prev are not differentiated (a c or smooth_weight tensor that requires grad is refused)."""
    if isinstance(smooth_weight, torch.Tensor):
        if smooth_weight.requires_grad:
            raise ValueError("smooth_weight requires grad, but fixed-lag smoothing is not differentiated in it: detach it")
        smooth_weight = float(smooth_weight)
    accel = _accel_weight_of(state, "differentiable_retarget_fixed_lag_accel")
    cfg = dict(state=state, smooth_weight=smooth_weight, accel_weight=accel)
    rq, q, status, last, wkp, wfix, wq, prev = _DifferentiableRetargetFixedLagAccel.apply(
        keypoints, fixed_qpos, state.last_qpos, state.window_keypoints, state.window_fixed_qpos, state.window_qpos,
        state.prev_qpos, seq, cfg)
    return rq, q, status, _accel_state_out(cfg["new_state"], last, wkp, wfix, wq, prev)


class _DifferentiableFlushFixedLagAccel(torch.autograd.Function):
    @staticmethod
    def forward(ctx, last_qpos, window_keypoints, window_fixed_qpos, window_qpos, prev_qpos, seq, cfg):
        state0 = _accel_copy(cfg["state"], cfg["accel_weight"])
        new = _fixed_lag_copy(state0)
        rq, q, count = seq.flush_fixed_lag(new)
        ctx.seq, ctx.state0 = seq, state0
        ctx.set_materialize_grads(False)
        ctx.mark_non_differentiable(count)
        cfg["new_state"] = new
        return rq, q, count, new.last_qpos, new.window_keypoints, new.window_fixed_qpos, new.window_qpos, new.prev_qpos

    @staticmethod
    @once_differentiable
    def backward(ctx, g_rq, g_q, _g_count, g_last, g_wkp, g_wfix, g_wq, g_prev):
        c = (lambda g: None if g is None else g.contiguous())
        g_last0, g_wkp0, g_wfix0, g_wq0, g_prev0 = ctx.seq.flush_fixed_lag_accel_vjp(
            ctx.state0, grad_qpos=c(g_q), grad_robot_qpos=c(g_rq), grad_last_qpos_out=c(g_last),
            grad_prev_qpos_out=c(g_prev), grad_window_qpos_out=c(g_wq), grad_window_keypoints_out=c(g_wkp),
            grad_window_fixed_qpos_out=c(g_wfix))
        return g_last0, g_wkp0, g_wfix0, g_wq0, g_prev0, None, None


def differentiable_flush_fixed_lag_accel(seq, state):
    """`differentiable_flush_fixed_lag` for an accelerated state: differentiable in the state's `last_qpos`, `prev_qpos`
    and window tensors; the returned state carries accel_weight, has_prev and the graph as
    `differentiable_retarget_fixed_lag_accel`'s does."""
    accel = _accel_weight_of(state, "differentiable_flush_fixed_lag_accel")
    cfg = dict(state=state, accel_weight=accel)
    rq, q, count, last, wkp, wfix, wq, prev = _DifferentiableFlushFixedLagAccel.apply(
        state.last_qpos, state.window_keypoints, state.window_fixed_qpos, state.window_qpos, state.prev_qpos, seq, cfg)
    return rq, q, count, _accel_state_out(cfg["new_state"], last, wkp, wfix, wq, prev)
