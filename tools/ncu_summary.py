"""Turns an `ncu --set full` report of the persistent decoder kernel into the committed evidence:
    python tools/ncu_summary.py gpurun_out/prof_dec.ncu-rep <steps in the captured launch> profiles/r02_decoder_ncu_summary.md
writes the markdown metric table and profiles/decoder_traffic.json = {source_sha16, dram_bytes_per_step, ...} that
bench.py's roofline.traffic reads (and nulls when decoder_persistent.cu no longer hashes to source_sha16)."""
import csv
import hashlib
import io
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WANT = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_sector_hit_rate.pct",
        "lts__throughput.avg.pct_of_peak_sustained_elapsed", "l1tex__m_xbar2l1tex_read_bytes.sum",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread", "launch__grid_size",
        "smsp__inst_executed.sum", "launch__shared_mem_per_block_dynamic"]
UNIT = {"Gbyte": 1e9, "Mbyte": 1e6, "Kbyte": 1e3, "byte": 1.0, "Tbyte": 1e12}


def main():
    rep, steps, out_md = sys.argv[1], int(sys.argv[2]), sys.argv[3]
    kernel = sys.argv[4] if len(sys.argv) > 4 else "decoder_persistent_kernel"
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units = rows[0], rows[1]
    data = [r for r in rows[2:] if any(kernel in c for c in r)]
    assert data, "no launch of %s in %s" % (kernel, rep)
    r = data[-1]
    vals = {}
    for name, unit, v in zip(hdr, units, r):
        if name in WANT:
            vals[name] = (v, unit)
    lines = ["| metric | value | unit |", "|---|---|---|"] + ["| %s | %s | %s |" % (k, vals[k][0], vals[k][1]) for k in WANT if k in vals]

    def to_bytes(key):
        v, u = vals[key]
        return float(v.replace(",", "")) * UNIT.get(u, 1.0)
    dram = to_bytes("dram__bytes_read.sum") + to_bytes("dram__bytes_write.sum")
    dur = vals["gpu__time_duration.sum"]
    src = open(os.path.join(ROOT, "tacotron2_b200", "csrc", "decoder_persistent.cu"), "rb").read()
    traffic = {"source_sha16": hashlib.sha256(src).hexdigest()[:16], "kernel": kernel, "steps_in_capture": steps,
               "dram_bytes_per_launch": dram, "dram_bytes_per_step": dram / steps, "duration": "%s %s" % dur,
               "capture": "ncu --set full --clock-control none, %s (%d decoder steps in the launch); %s" % (os.path.basename(rep), steps, os.path.basename(out_md))}
    if kernel == "decoder_persistent_kernel":
        os.makedirs(os.path.join(ROOT, "profiles"), exist_ok=True)
        json.dump(traffic, open(os.path.join(ROOT, "profiles", "decoder_traffic.json"), "w"), indent=1)
    with open(out_md, "a") as f:
        f.write("\n".join(lines) + "\n\nDRAM traffic %.3f GB per launch = %.2f MB per decoder step (%d steps).\n" % (dram / 1e9, dram / steps / 1e6, steps))
    print("\n".join(lines))
    print(json.dumps(traffic))


if __name__ == "__main__":
    main()
