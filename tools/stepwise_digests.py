"""Record the stepwise decoder's output digests for a build (tests/test_gpu_decode_step.py::stepwise_digests).

    T2B200_LIB=<a build's libt2b200.so> python tools/stepwise_digests.py OUT.json

tests/golden/decoder_stepwise_sha256.json holds the digests of the build before the stepwise loop body became
decoder_step(); test_stepwise_run_keeps_its_bits compares every later build with them."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tests.test_gpu_decode_step import stepwise_digests  # noqa: E402

if __name__ == "__main__":
    d = stepwise_digests()
    with open(sys.argv[1], "w") as f:
        json.dump(d, f, indent=1, sort_keys=True)
    print(json.dumps(d, sort_keys=True))
