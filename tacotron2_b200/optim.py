"""Fused gradient clipping + Adam for train.py:229-236.

    grad_norm = torch.nn.utils.clip_grad_norm_(model.parameters(), hparams.grad_clip_thresh)    # train.py:232-233
    optimizer.step()                                                                             # train.py:236

become ONE call, ``grad_norm = optimizer.step(max_norm=hparams.grad_clip_thresh)``: three multi-tensor launches in
libt2b200 (sum of squares, norm / clip coefficient, update) instead of torch's per-operation foreach kernels.  Same
arithmetic as ``clip_grad_norm_`` + ``torch.optim.Adam`` (L2 weight decay, bias correction); state_dict layout is
torch.optim.Adam's (``exp_avg``, ``exp_avg_sq``, ``step``), so checkpoints interchange (train.py:99-113)."""
import ctypes as C

import torch

from . import _capi
from ._engine import bump_weights_generation


class FusedClipAdam(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))
        self._ws = _capi.Workspace()

    @torch.no_grad()
    def step(self, closure=None, max_norm=None):
        """Clips the gradients of ALL parameters to ``max_norm`` (None / <= 0: no clipping), then one Adam update per
        param group.  Returns the total gradient norm before clipping (0-dim CUDA tensor; .item() syncs)."""
        if closure is not None:
            raise RuntimeError("FusedClipAdam does not support closures")
        L = _capi.lib()
        groups = [(g, [p for p in g["params"] if p.grad is not None]) for g in self.param_groups]
        all_p = [p for _, ps in groups for p in ps]
        if not all_p:
            return None
        dev = all_p[0].device
        for p in all_p:
            if p.dtype != torch.float32 or p.grad.dtype != torch.float32 or not p.is_cuda:
                raise RuntimeError("FusedClipAdam: fp32 CUDA parameters and gradients only")
            if not p.is_contiguous():
                raise RuntimeError("FusedClipAdam: parameters must be contiguous")
            if not p.grad.is_contiguous():
                p.grad = p.grad.contiguous()
            st = self.state[p]
            if not st:
                st["step"] = torch.tensor(0.0)
                st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
        norm = torch.zeros((), device=dev, dtype=torch.float32)
        total = sum(p.numel() for p in all_p)
        ws = self._ws.get("adam", L.t2_clip_adam_workspace_bytes(total, len(all_p)), dev)
        first = True
        for g, ps in groups:
            if not ps:
                continue
            # one group = one launch set; the clip coefficient is computed over ALL parameters (first launch set);
            # further groups get max_norm = 0 after their gradients were pre-scaled -> keep it simple: single group
            if not first:
                raise RuntimeError("FusedClipAdam: one param group only (train.py uses one)")
            first = False
            n = len(ps)
            arr = lambda ts: (C.c_void_p * n)(*[t.data_ptr() for t in ts])
            # "step" is a CPU scalar tensor here; checkpoints written by older torch.optim.Adam hold a Python int
            steps = {int(float(self.state[p]["step"])) for p in ps}
            if len(steps) != 1:
                raise RuntimeError("FusedClipAdam: parameters with different step counts %s (a parameter skipped "
                                   "updates because its .grad was None); one bias correction per launch" % sorted(steps))
            step = steps.pop() + 1
            a = _capi.T2AdamArgs()
            a.n = n
            pa, ga = arr(ps), arr([p.grad for p in ps])
            ma, va = arr([self.state[p]["exp_avg"] for p in ps]), arr([self.state[p]["exp_avg_sq"] for p in ps])
            ne = (C.c_int64 * n)(*[p.numel() for p in ps])
            a.params, a.grads, a.exp_avg, a.exp_avg_sq, a.numel = pa, ga, ma, va, ne
            a.lr, (a.beta1, a.beta2) = float(g["lr"]), [float(b) for b in g["betas"]]
            a.eps, a.weight_decay = float(g["eps"]), float(g["weight_decay"])
            a.max_norm = float(max_norm) if max_norm else 0.0
            a.step = step
            a.grad_norm = norm.data_ptr()
            a.ws, a.ws_bytes = ws.data_ptr(), ws.numel()
            _capi.call(L.t2_clip_adam_step, dev, C.byref(a))
            for p in ps:
                st = self.state[p]
                st["step"] = st["step"] + 1 if torch.is_tensor(st["step"]) else torch.tensor(float(st["step"]) + 1.0)
        bump_weights_generation()       # parameters changed underneath torch's version counters
        return norm


class AmpFusedClipAdam(torch.optim.Optimizer):
    """The reference's "fp16" training flow (Apex AMP O2: train.py:173-176, 222-236) as one fused optimizer step.

        model, optimizer = tacotron2_b200.amp.initialize(model, optimizer, opt_level="O2")     # instead of apex.amp
        ...
        with tacotron2_b200.amp.scale_loss(loss, optimizer) as scaled_loss:                   # train.py:223-224
            scaled_loss.backward()
        grad_norm = optimizer.step(max_norm=hparams.grad_clip_thresh)                         # train.py:229-236 in one call

    The model holds fp16 parameters (BatchNorm stays fp32, like O2's keep_batchnorm_fp32), this optimizer holds the fp32
    masters.  ``step`` = unscale the fp16 gradients, overflow check, ``clip_grad_norm_`` over the unscaled gradients, Adam on
    the masters, fp16 write-back, dynamic loss-scale update (overflow: skip + scale / 2; ``growth_interval`` = 2000 good
    steps: scale x 2) -- three multi-tensor launches in libt2b200 and no host synchronisation; whether a step was skipped is
    known on the device only (``last_step_skipped()`` reads it back).  state_dict layout: torch.optim.Adam's per-parameter
    ``exp_avg`` / ``exp_avg_sq`` / ``step`` plus ``master`` and the scaler state."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, init_scale=2.0 ** 16,
                 growth_interval=2000, growth_factor=2.0, backoff_factor=0.5):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))
        if len(self.param_groups) != 1:
            raise RuntimeError("AmpFusedClipAdam: one param group only (train.py uses one)")
        self.growth_interval, self.growth_factor, self.backoff_factor = int(growth_interval), float(growth_factor), float(backoff_factor)
        self._init_scale = float(init_scale)
        self._dev_state = None          # device floats: [loss scale, good steps, optimizer steps taken, last step skipped]
        self._skipped = None
        self._ws = _capi.Workspace()

    def _state_tensor(self, dev):
        if self._dev_state is None or self._dev_state.device != dev:
            self._dev_state = torch.tensor([self._init_scale, 0.0, 0.0, 0.0], device=dev, dtype=torch.float32)
            self._skipped = torch.zeros(1, device=dev, dtype=torch.int32)
        return self._dev_state

    def _params(self):
        return [p for p in self.param_groups[0]["params"] if p.requires_grad]

    def _ensure_masters(self):
        for p in self._params():
            st = self.state[p]
            if "master" not in st:
                st["master"] = p.detach().clone().float() if p.dtype != torch.float32 else p.detach()
                st["exp_avg"] = torch.zeros_like(st["master"])
                st["exp_avg_sq"] = torch.zeros_like(st["master"])

    def master_params(self):
        """The fp32 copies the update is applied to (apex ``amp.master_params(optimizer)``)."""
        self._ensure_masters()
        return [self.state[p]["master"] for p in self._params()]

    def loss_scale(self):
        """Current loss scale as a 0-dim device tensor (no synchronisation)."""
        dev = self._params()[0].device
        return self._state_tensor(dev)[0]

    def scale_loss(self, loss):
        return loss * self._state_tensor(loss.device)[0].to(loss.dtype)

    def last_step_skipped(self):
        """True if the last step() found inf / nan gradients and skipped the update (synchronises)."""
        return bool(self._skipped is not None and int(self._skipped.item()) == 1)

    def steps_taken(self):
        return int(self._dev_state[2].item()) if self._dev_state is not None else 0

    @torch.no_grad()
    def step(self, closure=None, max_norm=None):
        if closure is not None:
            raise RuntimeError("AmpFusedClipAdam does not support closures")
        L = _capi.lib()
        g = self.param_groups[0]
        ps = [p for p in self._params() if p.grad is not None]
        if not ps:
            return None
        self._ensure_masters()
        dev = ps[0].device
        state = self._state_tensor(dev)
        n = len(ps)
        for p in ps:
            if not p.is_cuda or p.dtype not in (torch.float16, torch.float32) or p.grad.dtype not in (torch.float16, torch.float32):
                raise RuntimeError("AmpFusedClipAdam: fp16 / fp32 CUDA parameters and gradients only")
            if not p.is_contiguous():
                raise RuntimeError("AmpFusedClipAdam: parameters must be contiguous")
            if not p.grad.is_contiguous():
                p.grad = p.grad.contiguous()
        arr = lambda ts: (C.c_void_p * n)(*[t.data_ptr() for t in ts])
        flags = lambda ts: (C.c_int32 * n)(*[1 if t.dtype == torch.float16 else 0 for t in ts])
        a = _capi.T2AmpAdamArgs()
        a.n = n
        keep = (arr(ps), flags(ps), arr([p.grad for p in ps]), flags([p.grad for p in ps]),
                arr([self.state[p]["master"] for p in ps]), arr([self.state[p]["exp_avg"] for p in ps]),
                arr([self.state[p]["exp_avg_sq"] for p in ps]), (C.c_int64 * n)(*[p.numel() for p in ps]))
        (a.model_params, a.param_is_half, a.grads, a.grad_is_half, a.master, a.exp_avg, a.exp_avg_sq, a.numel) = keep
        a.lr, (a.beta1, a.beta2) = float(g["lr"]), [float(b) for b in g["betas"]]
        a.eps, a.weight_decay = float(g["eps"]), float(g["weight_decay"])
        a.max_norm = float(max_norm) if max_norm else 0.0
        a.growth_interval, a.growth_factor, a.backoff_factor = self.growth_interval, self.growth_factor, self.backoff_factor
        norm = torch.zeros((), device=dev, dtype=torch.float32)
        a.state, a.grad_norm, a.skipped = state.data_ptr(), norm.data_ptr(), self._skipped.data_ptr()
        ws = self._ws.get("adam", L.t2_amp_adam_workspace_bytes(sum(p.numel() for p in ps), n), dev)
        a.ws, a.ws_bytes = ws.data_ptr(), ws.numel()
        _capi.call(L.t2_amp_adam_step, dev, C.byref(a))
        bump_weights_generation()
        return norm

    def state_dict(self):
        self._ensure_masters()
        if self._dev_state is not None:
            steps = float(self._dev_state[2].item())
            for p in self._params():
                self.state[p]["step"] = torch.tensor(steps)
        sd = super().state_dict()
        sd["amp_scaler"] = (self._dev_state.cpu().tolist() if self._dev_state is not None else [self._init_scale, 0.0, 0.0, 0.0])
        return sd

    def load_state_dict(self, sd):
        sd = dict(sd)
        scaler = sd.pop("amp_scaler", None)
        super().load_state_dict(sd)
        if scaler is not None:
            dev = self._params()[0].device
            self._dev_state = torch.tensor([float(x) for x in scaler], device=dev, dtype=torch.float32)
            self._skipped = torch.zeros(1, device=dev, dtype=torch.int32)
