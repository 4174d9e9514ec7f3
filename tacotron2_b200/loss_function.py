"""Tacotron2Loss (loss_function.py:8-19) as a thin caller of libt2b200's fused loss kernel (t2_tacotron2_loss): one pass
over the model outputs gives the loss AND the gradient seeds d_mel / d_mel_postnet / d_gate; backward only scales them."""
import ctypes as C

import torch
from torch import nn

from . import _capi


class _FusedLossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, mel, post, gate, mel_target, gate_target):
        if not mel.is_cuda:
            raise RuntimeError("tacotron2_b200.Tacotron2Loss: CUDA tensors only (there is no CPU path)")
        L = _capi.lib()
        f32 = dict(device=mel.device, dtype=torch.float32)
        mel_c, post_c, gate_c = (x.detach().to(torch.float32).contiguous() for x in (mel, post, gate))
        tgt, gt = mel_target.detach().to(**f32).contiguous(), gate_target.detach().to(**f32).contiguous()
        B, Cm, T = mel_c.shape
        if post_c.shape != mel_c.shape or tgt.shape != mel_c.shape or gate_c.numel() != B * T or gt.numel() != B * T:
            raise RuntimeError("Tacotron2Loss: shapes %s %s %s %s %s" % (tuple(mel.shape), tuple(post.shape), tuple(gate.shape),
                                                                        tuple(mel_target.shape), tuple(gate_target.shape)))
        need = [ctx.needs_input_grad[i] for i in range(3)]
        d = [torch.empty_like(x) if n else None for x, n in zip((mel_c, post_c, gate_c), need)]
        out = torch.empty(4, **f32)
        ws = _capi.byte_buffer(L.t2_loss_workspace_bytes(), mel.device)
        a = _capi.T2LossArgs(mel_c.data_ptr(), post_c.data_ptr(), gate_c.data_ptr(), tgt.data_ptr(), gt.data_ptr(), None,
                             int(B), int(Cm), int(T), out.data_ptr(), *(x.data_ptr() if x is not None else None for x in d),
                             ws.data_ptr(), ws.numel())
        _capi.call(L.t2_tacotron2_loss, mel.device, C.byref(a))
        ctx.seeds = d
        ctx.dtypes = (mel.dtype, post.dtype, gate.dtype)
        ctx.gate_shape = gate.shape
        ctx.terms = out[1:]
        return out[0]

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g):
        d_mel, d_post, d_gate = ctx.seeds
        ctx.seeds = None
        res = []
        for x, dt in zip((d_mel, d_post, d_gate), ctx.dtypes):
            res.append((x * g).to(dt) if x is not None else None)
        if res[2] is not None:
            res[2] = res[2].view(ctx.gate_shape)
        return res[0], res[1], res[2], None, None


class Tacotron2Loss(nn.Module):
    """loss_function.py:8-19: MSE(mel_out, mel_target) + MSE(mel_out_postnet, mel_target) + BCEWithLogits(gate_out, gate_target)."""

    def forward(self, model_output, targets):
        mel_target, gate_target = targets[0], targets[1]
        mel_out, mel_out_postnet, gate_out, _ = model_output
        return _FusedLossFn.apply(mel_out, mel_out_postnet, gate_out, mel_target, gate_target)
