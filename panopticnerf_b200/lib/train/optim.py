"""FusedAdam: torch.optim.Adam's update on the library's kernel (pnr_adam_step), one launch per parameter group.

Each group's parameters, gradients and moments live in flat fp32 buffers on the device: `p.data` is a view into the
group's parameter buffer and `p.grad` a view into its gradient buffer, which backward accumulates into in place.  With a
communicator (`comm`: `parallel.TileGather` or any object with `world`, `allgather(t) -> [world, *t.shape]` and
`broadcast(t)`), `step()` all-gathers every rank's flat gradient and the kernel sums the slices in rank order before the
update, so every replica computes the same bits; without one it runs with a single slice."""
from __future__ import annotations

import ctypes as C
import math
from typing import List, Optional

import torch

from ... import _capi

_REFUSED = ("amsgrad", "maximize", "capturable", "differentiable")
_ALIGN = 64      # each parameter starts 256 bytes into the flat buffers, as aligned as its own allocation was for the
                 # vector loads that read it (the hash-grid table's float2 / float4 corners); padding stays zero


class FusedAdam(torch.optim.Optimizer):
    """Adam (param groups with lr, betas, eps, weight_decay; torch's LR schedulers apply unchanged).  state_dict() has
    torch.optim.Adam's layout ('step', 'exp_avg', 'exp_avg_sq' per parameter), so a checkpoint's optimiser entry loads
    into either optimiser.  zero_grad() zeroes the flat gradients in place whatever set_to_none says: a gradient that
    backward replaced instead of accumulating into its view (or that is missing) is refused at step().  Every
    parameter is updated every step, as torch does for a zero gradient."""

    def __init__(self, params, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 0.0,
                 amsgrad: bool = False, *, maximize: bool = False, capturable: bool = False,
                 differentiable: bool = False, comm=None):
        for name, value in zip(_REFUSED, (amsgrad, maximize, capturable, differentiable)):
            if value:
                raise ValueError(f"FusedAdam: {name}=True is not supported")
        if not 0.0 <= lr or not math.isfinite(lr):
            raise ValueError(f"FusedAdam: invalid lr {lr}")
        if not 0.0 <= eps or not math.isfinite(eps):
            raise ValueError(f"FusedAdam: invalid eps {eps}")
        if not all(0.0 <= b < 1.0 for b in betas) or len(betas) != 2:
            raise ValueError(f"FusedAdam: invalid betas {betas}")
        if not 0.0 <= weight_decay or not math.isfinite(weight_decay):
            raise ValueError(f"FusedAdam: invalid weight_decay {weight_decay}")
        defaults = dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay, amsgrad=False, maximize=False,
                        capturable=False, differentiable=False)
        self.comm = comm
        self._flat: List[dict] = []
        super().__init__(params, defaults)          # add_param_group flattens each group
        if comm is not None:
            for f in self._flat:
                for k in ("param", "exp_avg", "exp_avg_sq"):
                    comm.broadcast(f[k])

    # ---------------------------------------------------------------------------------------------- set-up
    @staticmethod
    def _check_group(group):
        for name in _REFUSED:
            if group.get(name):
                raise ValueError(f"FusedAdam: {name}=True is not supported")
        for p in group["params"]:
            if p.dtype != torch.float32:
                raise ValueError(f"FusedAdam: parameters must be float32, got {p.dtype}")
            if not p.is_cuda:
                raise ValueError(f"FusedAdam: parameters must be CUDA tensors, got a {p.device} parameter (no CPU path)")
            if p.is_sparse:
                raise ValueError("FusedAdam: sparse parameters are not supported")

    def add_param_group(self, param_group):
        super().add_param_group(param_group)
        self._check_group(self.param_groups[-1])
        self._flatten(self.param_groups[-1])

    def _flatten(self, group):
        params = group["params"]
        dev = params[0].device
        if any(p.device != dev for p in params):
            raise ValueError("FusedAdam: the parameters of one group must be on one device")
        offsets, P = [], 0
        for p in params:
            offsets.append(P)
            P += (p.numel() + _ALIGN - 1) // _ALIGN * _ALIGN
        f = {k: torch.zeros(P, dtype=torch.float32, device=dev) for k in ("param", "grad", "exp_avg", "exp_avg_sq")}
        f["P"], f["views"], f["data"], f["offsets"] = P, [], [], offsets
        with torch.no_grad():
            for p, off in zip(params, offsets):
                n = p.numel()
                f["param"][off:off + n].copy_(p.detach().reshape(-1))
                p.data = f["param"][off:off + n].view_as(p)
                p.grad = f["grad"][off:off + n].view_as(p)
                st = self.state[p]
                st["step"] = torch.tensor(0.0)
                st["exp_avg"] = f["exp_avg"][off:off + n].view_as(p)
                st["exp_avg_sq"] = f["exp_avg_sq"][off:off + n].view_as(p)
                f["views"].append(p.grad)
                f["data"].append(p.data)
        self._flat.append(f)

    # ---------------------------------------------------------------------------------------------- gradients
    def zero_grad(self, set_to_none: bool = True):
        """Zero the flat gradients in place (never None: backward accumulates into the views)."""
        for f in self._flat:
            f["grad"].zero_()

    def flat_grads(self) -> List[torch.Tensor]:
        """Each group's flat gradient [P] (after checking that every .grad is still its view)."""
        for group, f in zip(self.param_groups, self._flat):
            for p, view in zip(group["params"], f["views"]):
                if p.grad is not None and p.grad.is_sparse:
                    raise ValueError("FusedAdam: sparse gradients are not supported")
                if p.grad is None or p.grad.data_ptr() != view.data_ptr() or p.grad.shape != view.shape:
                    raise RuntimeError("FusedAdam: a parameter's .grad is no longer its view into the flat gradient "
                                       "(set to None or replaced by backward): zero gradients with "
                                       "FusedAdam.zero_grad(), never set them to None")
        return [f["grad"] for f in self._flat]

    def _check_params(self):
        """Every parameter still is its view into the flat parameter buffer: after module.to(), a load_state_dict with
        assign=True or any other replacement of p.data the kernel would update a buffer that nothing reads."""
        for group, f in zip(self.param_groups, self._flat):
            for p, view in zip(group["params"], f["data"]):
                if p.device != view.device or p.data_ptr() != view.data_ptr() or p.shape != view.shape:
                    raise RuntimeError("FusedAdam: a parameter's data is no longer its view into the flat parameter "
                                       "buffer (moved or replaced after the optimiser was built): build the optimiser "
                                       "after moving the module, and load weights in place")

    # ---------------------------------------------------------------------------------------------- update
    @torch.no_grad()
    def step(self, closure=None):
        """All-gather the flat gradients (with a communicator) and update every group: one pnr_adam_step each."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        grads = self.flat_grads()
        if self.comm is not None:
            stacked = [self.comm.allgather(g) for g in grads]
        else:
            stacked = [g.reshape(1, -1) for g in grads]
        self.step_gathered(stacked)
        return loss

    @torch.no_grad()
    def step_gathered(self, stacked: List[torch.Tensor], grad_sum: Optional[List[torch.Tensor]] = None):
        """The update from each group's gradient slices stacked [G, P] (rows summed in order): what step() runs after
        the exchange, and how G ranks' step is reproduced in one process."""
        if len(stacked) != len(self._flat):
            raise ValueError(f"FusedAdam.step_gathered: {len(stacked)} gradient stacks for {len(self._flat)} groups")
        self._check_params()
        for i, (group, f, s) in enumerate(zip(self.param_groups, self._flat, stacked)):
            if s.dim() != 2 or s.shape[1] != f["P"] or s.dtype != torch.float32 or s.device != f["param"].device:
                raise ValueError(f"FusedAdam.step_gathered: group {i} expects [G, {f['P']}] float32 on "
                                 f"{f['param'].device}, got {s.dtype} {tuple(s.shape)} on {s.device}")
            s = s if s.stride(1) == 1 and s.stride(0) >= f["P"] else s.contiguous()
            params = group["params"]
            state = self.state[params[0]]
            t = float(state["step"]) + 1.0
            for p in params:
                self.state[p]["step"].fill_(t)
            beta1, beta2 = group["betas"]
            lr = group["lr"]
            lr = float(lr) if not torch.is_tensor(lr) else float(lr.item())
            a = _capi.PnrAdamArgs()
            a.P, a.ld_grad, a.G = f["P"], s.stride(0) if s.shape[0] > 1 else f["P"], s.shape[0]
            a.beta1, a.beta2 = float(beta1), float(beta2)
            a.eps, a.weight_decay = float(group["eps"]), float(group["weight_decay"])
            a.step_size = lr / (1.0 - beta1 ** t)
            a.bc2_sqrt = (1.0 - beta2 ** t) ** 0.5
            gs = grad_sum[i] if grad_sum is not None else None
            with torch.cuda.device(f["param"].device):
                _capi.check(_capi.lib().pnr_adam_step(
                    s.data_ptr(), f["param"].data_ptr(), f["exp_avg"].data_ptr(), f["exp_avg_sq"].data_ptr(),
                    C.byref(a), _capi.ptr(gs, torch.float32, "grad_sum"), _capi.stream_ptr()), "pnr_adam_step")
            # the kernel wrote through data_ptr(): bump the version counters, which Network.pack() reads to repack
            for p in params:
                torch.autograd.graph.increment_version(p)

    # ---------------------------------------------------------------------------------------------- checkpoints
    def state_dict(self):
        """torch.optim.Adam's layout; the moments are copies (a loaded optimiser never writes into these buffers)."""
        sd = super().state_dict()
        sd["state"] = {k: {n: v.detach().clone() for n, v in st.items()} for k, st in sd["state"].items()}
        return sd

    def load_state_dict(self, state_dict):
        """Load a FusedAdam or torch.optim.Adam state_dict: moments are copied into the flat buffers."""
        super().load_state_dict(state_dict)
        for group, f in zip(self.param_groups, self._flat):
            self._check_group(group)
            steps = set()
            for p, off in zip(group["params"], f["offsets"]):
                n = p.numel()
                st = self.state[p]
                for k in ("exp_avg", "exp_avg_sq"):
                    buf = f[k][off:off + n]
                    if k in st:
                        buf.copy_(st[k].detach().reshape(-1))
                    else:
                        buf.zero_()
                    st[k] = buf.view_as(p)
                step = float(st["step"]) if "step" in st else 0.0
                st["step"] = torch.tensor(step)
                steps.add(step)
            if len(steps) > 1:
                raise ValueError(f"FusedAdam.load_state_dict: the parameters of one group are at different steps {steps}")
        if self.comm is not None:
            for f in self._flat:
                for k in ("exp_avg", "exp_avg_sq"):
                    self.comm.broadcast(f[k])
