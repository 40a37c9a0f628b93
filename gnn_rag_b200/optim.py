"""Gradient clipping + Adam as two kernels over a tensor list (csrc/optim.cu), for a captured training step.

The reference ends each training iteration with ``clip_grad_norm_(model.parameters(), gradient_clip)`` and
``Adam.step()`` (gnn/train_model.py:91-92, 221-230).  Run eagerly, that tail is a dozen multi-tensor launches and
their Python dispatch after every step.  :class:`ClipAdam` runs it as gr_grad_sumsq + gr_clip_adam, which a CUDA graph
can capture, and reproduces torch bit for bit: ``clip_grads_with_norm_`` given the norm the kernels compute, and
``torch.optim.adam._multi_tensor_adam``, the default CUDA path of ``torch.optim.Adam`` (foreach, not capturable).

The optimizer state stays torch's: ``exp_avg`` and ``exp_avg_sq`` are the tensors in ``opt.state`` (the kernels
update them in place), and the CPU ``step`` tensors advance on the host, so ``opt.state_dict()``, checkpoints and
eager ``opt.step()`` calls between graphed steps keep working.  The per-step scalars (bias corrections, ``lr`` and the
group's other hyperparameters) are computed on the host in float64, exactly as ``_multi_tensor_adam`` computes them,
and uploaded before each launch without a host synchronisation; a scheduler that changes ``lr`` needs no new capture.
Optimizer step hooks do not run."""
import numpy as np
import torch
from torch.optim.optimizer import _get_scalar_dtype

from . import ops

_FLAGS = ("amsgrad", "maximize", "decoupled_weight_decay", "capturable", "differentiable")


def check_optimizer(opt, params, max_norm):
    """Raise ``ValueError`` unless ``opt`` (or None) and ``max_norm`` can run as :class:`ClipAdam` for a model whose
    parameters are ``params``: ``opt`` must be exactly ``torch.optim.Adam`` over fp32 parameters of the model, without
    amsgrad, maximize, decoupled weight decay, capturable, differentiable or fused (which rounds differently), with
    float ``lr`` and betas; ``max_norm`` needs an optimizer and must be > 0."""
    if opt is None:
        if max_norm is not None:
            raise ValueError("max_norm clips inside the optimizer step: it needs an optimizer")
        return
    if type(opt) is not torch.optim.Adam:
        raise ValueError("the fused optimizer step is torch.optim.Adam's; got %s" % type(opt).__name__)
    if max_norm is not None and not float(max_norm) > 0:
        raise ValueError("max_norm must be > 0, got %r" % (max_norm,))
    mine = {id(p) for p in params}
    for group in opt.param_groups:
        for flag in _FLAGS:
            if group.get(flag, False):
                raise ValueError("the fused Adam step does not implement %s=True" % flag)
        if group.get("fused"):
            raise ValueError("fused=True Adam rounds differently from the foreach path the kernels reproduce")
        if isinstance(group["lr"], torch.Tensor) or any(isinstance(b, torch.Tensor) for b in group["betas"]):
            raise ValueError("the fused Adam step takes a float lr and betas, not tensors")
        for p in group["params"]:
            if id(p) not in mine:
                raise ValueError("the optimizer holds a parameter that is not the model's")
            if p.dtype != torch.float32:
                raise ValueError("the fused Adam step updates fp32 parameters, got %s" % p.dtype)


def init_state(opt, params):
    """Create the missing state of every parameter in ``params`` as ``Adam._init_group`` does (CPU ``step`` 0, zero
    ``exp_avg`` / ``exp_avg_sq``)."""
    for p in params:
        state = opt.state[p]
        if len(state) == 0:
            state["step"] = torch.tensor(0.0, dtype=_get_scalar_dtype())
            state["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
            state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)


def state_key(opt):
    """The ``data_ptr`` of every state tensor of ``opt`` (None for a parameter without state): ``load_state_dict``
    replaces them, and a captured step must then be captured again."""
    out = []
    for group in opt.param_groups:
        for p in group["params"]:
            st = opt.state.get(p)
            out.append(None if not st else tuple(st[k].data_ptr() for k in ("step", "exp_avg", "exp_avg_sq")))
    return tuple(out)


def adam_scalars(lr, beta1, beta2, eps, weight_decay, step):
    """The fp32 scalar row of one tensor at (already advanced) ``step``: the float64 values ``_multi_tensor_adam``
    computes on the host, each rounded once to fp32 as torch hands them to its foreach kernels."""
    bias_correction1 = 1 - beta1 ** step
    bias_correction2 = 1 - beta2 ** step
    step_size = (lr / bias_correction1) * -1
    bias_correction2_sqrt = bias_correction2 ** 0.5
    return np.array([1 - beta1, beta2, 1 - beta2, eps, weight_decay, step_size, bias_correction2_sqrt, 0.0],
                    dtype=np.float32)


def _any_weight_decay(opt):
    return any(g["weight_decay"] != 0 for g in opt.param_groups)


class ClipAdam:
    """``clip_grad_norm_(params, max_norm)`` + ``opt.step()`` over the gradients ``grads`` of ``params`` as two
    launches (:func:`ops.clip_adam`).

    ``params`` are the parameters that have a gradient (the norm covers all of them, as ``clip_grad_norm_`` over the
    model's parameters does); those the optimizer holds are updated, the others only clipped.  ``grads`` are the
    tensors the kernels read and write as ``p.grad``, fixed for the lifetime of the object (a captured backward's
    gradient tensors).  Call :meth:`prepare` before every :meth:`launch` (or replay of a graph that captured it): it
    advances the CPU ``step`` tensors, uploads that step's scalars and bumps the ``_version`` of every parameter it
    updates (:meth:`advance` does too, for a whole epoch of replays).  ``grad_norm`` (device fp32 scalar) holds the
    total norm after a launch with ``max_norm``; it is None without."""

    def __init__(self, opt, params, grads, max_norm=None):
        check_optimizer(opt, params, max_norm)
        self.opt, self.max_norm = opt, None if max_norm is None else float(max_norm)
        group_of = {id(p): gi for gi, g in enumerate(opt.param_groups) for p in g["params"]}
        rows = [(p, g) for p, g in zip(params, grads) if g is not None
                and (self.max_norm is not None or id(p) in group_of)]
        init_state(opt, [p for p, _ in rows if id(p) in group_of])
        dev = params[0].device if params else torch.device("cuda")
        E = ops.adam_chunk_elems()
        chunks = []
        self._adam_rows, self._groups, self._steps = [], [], []
        for r, (p, _g) in enumerate(rows):
            if id(p) in group_of:
                st = opt.state[p]
                for k in ("exp_avg", "exp_avg_sq"):
                    t = st[k]
                    if not (t.is_cuda and t.dtype == torch.float32 and t.shape == p.shape and t.is_contiguous()):
                        raise ValueError("Adam state %s must be a contiguous fp32 CUDA tensor like its parameter" % k)
                if st["step"].is_cuda:
                    raise ValueError("Adam state step must be a CPU tensor (a capturable or fused Adam's is not)")
                self._adam_rows.append(r)
                self._groups.append(group_of[id(p)])
                self._steps.append(st["step"])
            chunks += [(r, k) for k in range((p.numel() + E - 1) // E)]
        self.params = [p for p, _ in rows]
        self._updated = [self.params[r] for r in self._adam_rows]
        self._wd = _any_weight_decay(opt)
        T, C = len(rows), len(chunks)
        self._table = torch.zeros(T, 6, dtype=torch.int64, device=dev)
        self.bind([g for _, g in rows])
        self._chunks = torch.tensor(chunks, dtype=torch.int32).reshape(C, 2).to(dev)
        self._scalars = torch.zeros(T, 8, dtype=torch.float32, device=dev)
        self._host = np.zeros((T, 8), dtype=np.float32)
        if self.max_norm is not None:
            self._slots = torch.empty(max(C, 1), dtype=torch.float64, device=dev)
            self.grad_norm = torch.empty((), dtype=torch.float32, device=dev)
        else:
            self._slots = self.grad_norm = None

    def bind(self, grads):
        """Point the kernels at ``grads`` (one per row, as ``params``): the tensor table is written here, once (a
        synchronous copy), so a captured launch reads it unchanged on every replay."""
        table, adam = [], set(self._adam_rows)
        for r, (p, g) in enumerate(zip(self.params, grads)):
            if not (p.is_contiguous() and g is not None and g.is_contiguous() and g.shape == p.shape
                    and g.dtype == torch.float32 and g.device == p.device):
                raise ValueError("the fused Adam step needs contiguous fp32 parameters and gradients of their shape")
            ptrs = [p.data_ptr(), g.data_ptr(), 0, 0]
            if r in adam:
                st = self.opt.state[p]
                ptrs[2:] = [st["exp_avg"].data_ptr(), st["exp_avg_sq"].data_ptr()]
            aligned = all(x % 16 == 0 for x in ptrs if x)
            table.append(ptrs + [p.numel(), ops.ADAM_ALIGNED16 if aligned else 0])
        self._table.copy_(torch.tensor(table, dtype=torch.int64).reshape(self._table.shape))

    def prepare(self):
        """Advance the ``step`` of every updated parameter (``torch._foreach_add_``, as Adam does for CPU steps) and
        upload this step's scalars (a pageable H2D copy on the current stream: no host synchronisation)."""
        self._check_groups()
        groups = self.opt.param_groups
        if self._steps:
            torch._foreach_add_(self._steps, torch.tensor(1.0, device="cpu"), alpha=1.0)
        memo = {}
        for r, gi, step in zip(self._adam_rows, self._groups, self._steps):
            t = step.item()
            row = memo.get((gi, t))
            if row is None:
                g = groups[gi]
                beta1, beta2 = g["betas"]
                row = memo[(gi, t)] = adam_scalars(g["lr"], beta1, beta2, g["eps"], g["weight_decay"], t)
            self._host[r] = row
        self._scalars.copy_(torch.from_numpy(self._host.copy()), non_blocking=True)
        self._bump_versions()
        self.opt._opt_called = True          # an LR scheduler's check that the optimizer stepped before it

    def _bump_versions(self):
        """Move the version counter of every parameter this object updates, as an in-place torch op would: the kernels
        write them through raw pointers, and the weight formats cached per version (``ops._cached``) and the
        serving graphs keyed on versions (``GraphedStep``) must see the new values."""
        torch.autograd.graph.increment_version(self._updated)

    def _check_groups(self):
        groups = self.opt.param_groups
        if any(isinstance(g["lr"], torch.Tensor) for g in groups):
            raise ValueError("the fused Adam step takes a float lr, not a tensor")
        if _any_weight_decay(self.opt) != self._wd:
            raise ValueError("a group's weight_decay moved between zero and non-zero: build a new ClipAdam")

    def layout(self):
        """What the scalar rows depend on besides the hyperparameters: the updated rows, their groups and ``step``
        tensors.  Two objects with the same layout take the same :meth:`epoch_scalars`."""
        return self._scalars.shape[0], tuple(self._adam_rows), tuple(self._groups), tuple(id(s) for s in self._steps)

    def epoch_scalars(self, steps):
        """The scalar rows of the next ``steps`` :meth:`prepare` calls, fp32 [steps, T, 8], without advancing anything:
        the same float64 host arithmetic per step, with the current ``lr`` and hyperparameters."""
        self._check_groups()
        groups = self.opt.param_groups
        out = np.zeros((steps, self._scalars.shape[0], 8), dtype=np.float32)
        memo = {}
        for r, gi, step in zip(self._adam_rows, self._groups, self._steps):
            t0 = step.item()
            rows = memo.get((gi, t0))
            if rows is None:
                g = groups[gi]
                beta1, beta2 = g["betas"]
                rows = memo[(gi, t0)] = np.stack(
                    [adam_scalars(g["lr"], beta1, beta2, g["eps"], g["weight_decay"], t0 + s + 1) for s in range(steps)]
                ) if steps else np.zeros((0, 8), dtype=np.float32)
            out[:, r] = rows
        return out

    def advance(self, steps):
        """Advance the ``step`` of every updated parameter by ``steps`` at once, as ``steps`` calls of :meth:`prepare`
        do (the counts are integers, exact in the step tensors' dtype up to 2^24)."""
        if self._steps and steps:
            torch._foreach_add_(self._steps, torch.tensor(float(steps), device="cpu"), alpha=1.0)
            self._bump_versions()
        self.opt._opt_called = True

    def launch(self):
        """Enqueue gr_grad_sumsq (with max_norm) and gr_clip_adam on the current stream."""
        ops.clip_adam(self._table, self._scalars, self._chunks, self._slots,
                      0.0 if self.max_norm is None else self.max_norm, self.grad_norm, self._wd)

    def step(self):
        """:meth:`prepare` + :meth:`launch`: one eager optimizer step over the current gradients."""
        self.prepare()
        self.launch()
