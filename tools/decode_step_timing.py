"""Per-step time of the decoder step API on the GPU: decode() and prenet + decode() at B = 1 and 64, T_enc = 150, next
to Decoder.inference's time per step and the reference step (the fp32 oracle port, oracle/tacotron2_oracle.py) in eager
PyTorch on the same card.  CUDA events over 200 steps after 20 warm-up steps.  Prints the card's name and power limit.

    python tools/decode_step_timing.py [--steps 200]"""
import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import tacotron2_b200 as t2  # noqa: E402
from oracle import tacotron2_oracle as O  # noqa: E402
from tests.common import synth_state_dict  # noqa: E402


def timed(fn, steps, warmup=20):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return 1000.0 * a.elapsed_time(b) / steps       # us per step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("decode_step_timing: no CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    print("device: %s (%s)" % (torch.cuda.get_device_name(), q[0] if q else "power limit unknown"))
    sd = synth_state_dict(41, scale=2.0)
    model = t2.Tacotron2(t2.create_hparams())
    model.load_state_dict(sd)
    model = model.cuda().eval()
    dec = model.decoder
    sdg = {k: v.cuda() for k, v in sd.items()}
    T = 150
    for B in (1, 64):
        memory = torch.randn(B, T, 512, device="cuda")
        x0 = torch.zeros(B, 80, device="cuda")
        with torch.no_grad():
            dec.initialize_decoder_states(memory, None)
            px = dec.prenet(x0)
            step = timed(lambda: dec.decode(px), args.steps)
            dec.initialize_decoder_states(memory, None)
            both = timed(lambda: dec.decode(dec.prenet(x0)), args.steps)
            dec.max_decoder_steps, dec.gate_threshold = args.steps, 1.0
            dec.inference(memory)
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            dec.inference(memory)
            b.record()
            torch.cuda.synchronize()
            infer = 1000.0 * a.elapsed_time(b) / args.steps
            st = O.init_decoder_state(sdg, memory)
            keep = torch.ones(B, 256, device="cuda")
            ref = timed(lambda: O.decode_step(sdg, st, memory, O.prenet(sdg, x0, keep, keep)), args.steps)
        print("B=%d T_enc=%d: decode %.1f us, prenet + decode %.1f us, Decoder.inference %.1f us/step, "
              "reference step (eager PyTorch fp32) %.1f us" % (B, T, step, both, infer, ref))


if __name__ == "__main__":
    main()
