"""Turn an .ncu-rep (ncu --set full --import-source on) into a plain-text summary.

    python tools/ncu_export.py mel.ncu-rep mel_summary.txt --frames 441344 --note "..."
"""
import argparse, csv, io, subprocess, sys, collections, re

KEYS = [
    "gpu__time_duration.sum", "sm__cycles_elapsed.avg", "launch__grid_size", "launch__block_size",
    "launch__registers_per_thread", "launch__shared_mem_per_block_dynamic", "dram__bytes_read.sum", "dram__bytes_write.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "smsp__inst_executed.sum",
    "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active",
    "sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active", "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum",
    "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed",
    "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "sm__warps_active.avg.pct_of_peak_sustained_active",
    "lts__t_bytes.sum", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
]


def ncu(args):
    return subprocess.run(["ncu"] + args, capture_output=True, text=True, check=True).stdout


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("rep"); ap.add_argument("out"); ap.add_argument("--frames", type=float, default=0); ap.add_argument("--note", default="")
    a = ap.parse_args()
    raw = list(csv.reader(io.StringIO(ncu(["-i", a.rep, "--page", "raw", "--csv"]))))
    h, u, v = raw[0], raw[1], raw[2]
    idx = {k: i for i, k in enumerate(h)}
    lines = [f"# {a.rep}", f"# {a.note}", f"kernel: {v[idx['Kernel Name']]}", ""]
    for k in KEYS:
        if k in idx:
            lines.append(f"{k:82s} {u[idx[k]]:>16s} {v[idx[k]]}")
    rd, wr = float(v[idx["dram__bytes_read.sum"]]), float(v[idx["dram__bytes_write.sum"]])
    ur, uw = u[idx["dram__bytes_read.sum"]], u[idx["dram__bytes_write.sum"]]
    scale = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}
    tot = rd * scale[ur] + wr * scale[uw]
    dur = float(v[idx["gpu__time_duration.sum"]]) * {"ns": 1e-9, "us": 1e-6, "ms": 1e-3, "s": 1}[u[idx["gpu__time_duration.sum"]]]
    lines += ["", f"DRAM traffic per launch (read+write): {tot/1e9:.4f} GB   -> {tot/dur/1e9:.1f} GB/s during this (profiled, cold) launch"]
    src = list(csv.reader(io.StringIO(ncu(["-i", a.rep, "--page", "source", "--csv", "--print-source", "sass"]))))
    hdr = src[1]; si = {k: i for i, k in enumerate(hdr)}
    ops = collections.Counter(); stall = collections.Counter(); total = samples = 0
    scols = [c for c in hdr if c.startswith("stall_") and "Not Issued" not in c]
    for r in src[2:]:
        if len(r) < len(hdr): continue
        ex = int(r[si["Instructions Executed"]] or 0); total += ex; samples += int(r[si["# Samples"]] or 0)
        m = re.match(r"(@!?U?P\d+\s+)?([A-Z0-9_]+)", r[si["Source"]].strip())
        ops[m.group(2) if m else "?"] += ex
        for c in scols: stall[c] += int(r[si[c]] or 0)
    div = a.frames or 1
    lines += ["", f"warp-instructions executed: {total}" + (f"   ({total/div:.1f} per frame)" if a.frames else ""), "opcode mix (warp-instr, per frame, share):"]
    for op, c in ops.most_common(16):
        lines.append(f"  {op:10s} {c:12d} {c/div:9.1f} {100*c/total:5.1f}%")
    lines += ["", "warp stall sampling (share of samples):"]
    for k, c in stall.most_common(10):
        lines.append(f"  {k:26s} {100*c/max(1,samples):5.1f}%")
    open(a.out, "w").write("\n".join(lines) + "\n")
    print("\n".join(lines))


if __name__ == "__main__":
    main()
