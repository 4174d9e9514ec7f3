"""Write tests/golden/waveglow_infer_bits_b64_t800.npz: for each case of
tests/test_gpu_waveglow_stream.bits_cases(), the digest of WaveGlow.infer's whole output and 4096 sampled samples, as
computed by the build that tacotron2_b200 loads.  The committed fixture was written by the build of commit f1d22d5, the
last one before t2_waveglow_infer became the window call; the test requires every later build to reproduce it bit for
bit.

    python tools/make_waveglow_bits.py [OUT_DIR] [--package DIR]        (needs a GPU)

--package DIR: import tacotron2_b200 (Python and its built library) from DIR instead of this tree.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def main():
    args = sys.argv[1:]
    if "--package" in args:
        i = args.index("--package")
        sys.path.insert(0, os.path.abspath(args[i + 1]))
        del args[i:i + 2]
    import numpy as np
    import tacotron2_b200
    print("tacotron2_b200 from", os.path.dirname(tacotron2_b200.__file__))
    from tests.common import GOLDEN_DIR, tensor_digest
    from tests.test_gpu_waveglow_stream import BITS_FIXTURE, bits_cases, bits_outputs, bits_sample
    out_dir = args[0] if args else GOLDEN_DIR
    arrays = {}
    for name, half, philox in bits_cases():
        out = bits_outputs(half, philox)
        arrays[name + "_digest"] = np.array(tensor_digest(out))
        arrays[name + "_samples"] = bits_sample(out).numpy()
        print(name, arrays[name + "_digest"])
    os.makedirs(out_dir, exist_ok=True)
    np.savez_compressed(os.path.join(out_dir, BITS_FIXTURE + ".npz"), **arrays)


if __name__ == "__main__":
    main()
