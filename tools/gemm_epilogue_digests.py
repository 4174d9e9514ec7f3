"""Records the SHA-256 digests of outputs that reach every wg_gemm instantiation not pinned by
tests/golden/waveglow_published_sha256.json (tests/test_gpu_gemm_epilogue_bits.digests) on the GPU, as JSON.  Run on
a build that is to be the yardstick; tests/test_gpu_gemm_epilogue_bits.py checks later builds against
tests/golden/gemm_epilogue_sha256.json.

    T2B200_LIB=<the yardstick build's libt2b200.so> python tools/gemm_epilogue_digests.py [--out FILE] [--repeat 2]

With --repeat N the cases run N times in one process; a case whose digest differs between runs is reported and left
out, since it cannot pin bits.
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
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden", "gemm_epilogue_sha256.json"))
    ap.add_argument("--repeat", type=int, default=2)
    args = ap.parse_args()
    import torch
    from tests.test_gpu_gemm_epilogue_bits import digests
    runs = [digests() for _ in range(max(1, args.repeat))]
    unstable = sorted(k for k in runs[0] if any(r[k] != runs[0][k] for r in runs[1:]))
    if unstable:
        print("not reproducible run to run, left out: %s" % unstable)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    d = dict(device=gpu or torch.cuda.get_device_name(0),
             digests={k: v for k, v in runs[0].items() if k not in unstable})
    with open(args.out, "w") as f:
        json.dump(d, f, indent=1, sort_keys=True)
        f.write("\n")
    print(json.dumps(d, indent=1, sort_keys=True))


if __name__ == "__main__":
    main()
