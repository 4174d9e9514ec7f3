"""Precision study (build-container tool, not product): how do reduced-precision GEMM operands
propagate through the autoregressive decoder recurrence?  Uses the oracle's ``mm`` hook to
round operands before an fp32-accumulated matmul.  Drives DESIGN.md section "precision"."""
import os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import tacotron2_oracle as O
from oracle.ref_import import default_hparams, import_reference_model

def q(x, mode):
    if mode == 'fp32': return x
    if mode == 'fp16': return x.half().float()
    if mode == 'bf16': return x.bfloat16().float()
    if mode == 'tf32':
        i = x.view(torch.int32); i = (i + 0x1000) & ~0x1fff  # round-to-nearest 10-bit mantissa
        return i.view(torch.float32)
    if mode == 'bf16x2':
        h = x.bfloat16().float(); return h + (x - h).bfloat16().float()
    if mode == 'fp16x2':
        h = x.half().float(); return h + (x - h).half().float()
    raise ValueError(mode)

def make_mm(wmode, xmode):
    def mm(x, w):
        return (q(x, xmode).double() @ q(w, wmode).double().t()).float()
    return mm

if __name__ == '__main__':
    m = import_reference_model()
    torch.manual_seed(1234)
    model = m.Tacotron2(default_hparams()).eval()
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    B, T_enc, steps = 4, 150, int(sys.argv[1]) if len(sys.argv) > 1 else 200
    g = torch.Generator().manual_seed(0)
    text = torch.randint(0, 148, (B, T_enc), generator=g)
    with torch.no_grad():
        memory = O.encoder(sd, sd['embedding.weight'][text].transpose(1, 2))
        keep = torch.rand(steps, 2, B, 256, generator=g) < 0.5
        ref = O.decoder_inference(sd, memory, keep, 1.0, steps)
        for wmode, xmode in [('fp32', 'fp32'), ('fp16', 'fp16'), ('bf16', 'bf16'), ('tf32', 'tf32'),
                             ('fp16', 'fp16x2'), ('fp16x2', 'fp16'), ('bf16x2', 'bf16x2'), ('fp16x2', 'fp16x2')]:
            out = O.decoder_inference(sd, memory, keep, 1.0, steps, mm=make_mm(wmode, xmode))
            errs = []
            for a, b in zip(ref[:3], out[:3]):
                errs.append(((a - b).abs().max() / a.abs().max()).item())
            # per-frame relative error on mel
            pf = ((ref[0] - out[0]).abs().amax(1) / ref[0].abs().amax(1)).max().item()
            print(f"W={wmode:7s} X={xmode:7s} mel {errs[0]:.2e} (per-frame {pf:.2e}) gate {errs[1]:.2e} align {errs[2]:.2e}")
