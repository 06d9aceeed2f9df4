#!/usr/bin/env python
"""``ncu --page raw --csv`` export (made on the GPU box by scripts/ncu_zoo.sh) → the tracked markdown table under profiles/.

    python scripts/ncu_csv_summary.py gpurun_out/ncu/ncu_zoo_raw.csv > profiles/ncu_summary.md
"""
import csv
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COLS = {
    "dur_us": "gpu__time_duration.sum", "rd": "dram__bytes_read.sum", "wr": "dram__bytes_write.sum", "dram_pct": "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "sm_pct": "sm__throughput.avg.pct_of_peak_sustained_elapsed", "regs": "launch__registers_per_thread", "warps_pct": "sm__warps_active.avg.pct_of_peak_sustained_active",
    "tensor_pct": "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "l2_pct": "lts__throughput.avg.pct_of_peak_sustained_elapsed",
    "occ_theory": "sm__maximum_warps_per_active_cycle_pct", "smem": "launch__shared_mem_per_block_dynamic", "waves": "launch__waves_per_multiprocessor",
}
SCALE = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "Tbyte": 1e12, "ns": 1e-3, "us": 1.0, "ms": 1e3, "s": 1e6, "nsecond": 1e-3, "usecond": 1.0, "msecond": 1e3, "second": 1e6}


def num(x):
    try:
        return float(str(x).replace(",", ""))
    except ValueError:
        return float("nan")


def main(path):
    rows = list(csv.reader(open(path)))
    hdr, units, body = rows[0], rows[1], rows[2:]
    ix = {}
    for k, name in COLS.items():
        c = [i for i, h in enumerate(hdr) if h == name]
        ix[k] = c[0] if c else None
    peak = 3350.0  # GB/s, H100 SXM data sheet; MEASURED_PEAKS.json overrides
    try:
        peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]
    except Exception:  # noqa: BLE001
        pass
    name_i, grid_i, block_i = hdr.index("Kernel Name"), hdr.index("Grid Size"), hdr.index("Block Size")
    print("# ncu captures of the hand-written kernels (H100, `ncu --set full --clock-control none`, one launch each, cold L2)\n")
    print(f"Source: `{os.path.relpath(path, ROOT)}` — exported on the GPU box by `scripts/ncu_zoo.sh` from one `scripts/kernel_zoo.py` run (world = 1: the peer")
    print("kernels run with this GPU as their only peer, so their loads/stores land in local HBM; ncu serialises kernels and cannot wrap a multi-rank job).")
    print(f"`HBM frac` = (DRAM bytes read + written) / duration / {peak:.1f} GB/s (measured copy peak, MEASURED_PEAKS.json). Durations under ncu are cold-cache, single")
    print("launch; event-timed numbers (L2 flushed, median of 5, clocks recorded) come from `scripts/kernel_zoo.py`.\n")
    print("| kernel | grid x block | regs | dur µs | DRAM rd MB | DRAM wr MB | achieved GB/s | HBM frac | DRAM % | L2 % | SM % | warps active % | tensor pipe % |")
    print("|---|---|---|---|---|---|---|---|---|---|---|---|---|")
    for r in body:
        def g(k):
            i = ix[k]
            if i is None:
                return float("nan")
            return num(r[i]) * SCALE.get(units[i], 1.0)
        dur, rd, wr = g("dur_us"), g("rd"), g("wr")
        gbps = (rd + wr) / dur / 1e3 if dur == dur and dur > 0 else float("nan")
        nm = r[name_i]
        nm = nm.split("(")[0]
        print(f"| `{nm}` | {r[grid_i].strip()} x {r[block_i].strip()} | {g('regs'):.0f} | {dur:.1f} | {rd / 1e6:.1f} | {wr / 1e6:.1f} | {gbps:.0f} | {gbps / peak:.2f} | {g('dram_pct'):.1f} | "
              f"{g('l2_pct'):.1f} | {g('sm_pct'):.1f} | {g('warps_pct'):.1f} | {g('tensor_pct'):.1f} |")


if __name__ == "__main__":
    main(sys.argv[1])
