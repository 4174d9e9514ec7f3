"""Records the SHA-256 digests of the published WaveGlow's outputs (tests/waveglow_configs.published_digests) on the
GPU, as JSON.  Run on a build that is to be the yardstick; tests/test_gpu_waveglow_configs.py checks later builds
against tests/golden/waveglow_published_sha256.json.

    python tools/waveglow_published_digests.py [--out tests/golden/waveglow_published_sha256.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden", "waveglow_published_sha256.json"))
    args = ap.parse_args()
    import torch
    from tests.waveglow_configs import published_digests
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    d = dict(device=gpu or torch.cuda.get_device_name(0), digests=published_digests())
    with open(args.out, "w") as f:
        json.dump(d, f, indent=1, sort_keys=True)
        f.write("\n")
    print(json.dumps(d, indent=1, sort_keys=True))


if __name__ == "__main__":
    main()
