"""Turn Nsight Compute outputs into markdown summaries.
  python tools/summarize_ncu.py launches <launches.csv> <summary.md>
  python tools/summarize_ncu.py full <report.ncu-rep> <summary.md>
"""
import collections
import csv
import re
import subprocess
import sys


def launches(src, dst):
    rows = list(csv.reader(open(src)))
    hi = next(i for i, r in enumerate(rows) if "Kernel Name" in r)
    hdr = rows[hi]
    k, v, u = hdr.index("Kernel Name"), hdr.index("Metric Value"), hdr.index("Metric Unit")
    agg, n = collections.OrderedDict(), 0
    for r in rows[hi + 1:]:
        if len(r) <= v:
            continue
        name = re.sub(r"\(.*", "", r[k]).replace("void ", "").replace("ddnm::", "")
        t = float(r[v].replace(",", ""))
        t = t / 1e3 if r[u] == "ns" else (t * 1e3 if r[u] == "ms" else t)
        a = agg.setdefault(name, [0, 0.0])
        a[0] += 1
        a[1] += t
        n += 1
    tot = sum(a[1] for a in agg.values())
    with open(dst, "w") as f:
        f.write(f"# ncu launch list summary ({src})\n\n`ncu --metrics gpu__time_duration.sum --clock-control none` — per-launch device time, "
                f"cold-cache and serialised: compare SHARES, not absolutes.\n\n{n} launches, {tot / 1e3:.2f} ms total.\n\n"
                "| kernel | launches | total us | share |\n|---|---:|---:|---:|\n")
        for name, (c, t) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
            f.write(f"| `{name}` | {c} | {t:.1f} | {t / tot * 100:.1f}% |\n")
    print(open(dst).read())


WANT = ["gpu__time_duration.sum", "launch__grid_size", "launch__registers_per_thread", "launch__shared_mem_per_block_dynamic",
        "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_tensor_subpipe_hmma.avg.pct_of_peak_sustained_active",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "lts__t_sector_hit_rate.pct", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
        "l1tex__throughput.avg.pct_of_peak_sustained_elapsed", "sm__cycles_elapsed.avg.per_second", "lts__t_bytes.sum",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "smsp__cycles_active.avg",
        # shared-memory side of the tensor pipe: operand wavefronts read by wgmma, bank reads (MMA operands) / writes (TMA fill)
        "l1tex__data_pipe_tc_wavefronts_mem_shared.sum.pct_of_peak_sustained_elapsed", "l1tex__data_bank_reads.avg.pct_of_peak_sustained_elapsed",
        "l1tex__data_bank_writes.avg.pct_of_peak_sustained_elapsed"]


def full(src, dst, peak_gbs=None):
    """src: a .ncu-rep, or the `--page raw --csv` export of one made where the report was captured."""
    if src.endswith(".csv"):
        out = open(src).read()
    else:
        out = subprocess.run(["ncu", "-i", src, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    hdr, units = rows[0], rows[1]
    idx = {h: i for i, h in enumerate(hdr)}
    with open(dst, "w") as f:
        f.write(f"# ncu --set full summary ({src})\n\n")
        for r in rows[2:]:
            f.write(f"## {r[idx['Kernel Name']][:90]}  grid {r[idx['Grid Size']]} block {r[idx['Block Size']]}\n\n| metric | value | unit |\n|---|---:|---|\n")
            for w in WANT:
                if w in idx:
                    f.write(f"| {w} | {r[idx[w]]} | {units[idx[w]]} |\n")
            try:   # achieved DRAM bandwidth of the launch against the measured copy peak (MEASURED_PEAKS.json)
                def val(name):
                    x, u = float(r[idx[name]].replace(",", "")), units[idx[name]]
                    return x * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "ns": 1e-9, "us": 1e-6, "ms": 1e-3, "s": 1}[u]
                byts = val("dram__bytes_read.sum") + val("dram__bytes_write.sum")
                sec = val("gpu__time_duration.sum")
                gbs = byts / sec / 1e9
                pk = peak_gbs or __import__("json").load(open("MEASURED_PEAKS.json"))["hbm_gbs"]
                f.write(f"| **DRAM traffic / duration** | {gbs:.0f} | GB/s = {gbs / pk * 100:.0f} % of the measured {pk:.0f} GB/s copy peak |\n")
            except Exception:
                pass
            f.write("\n")
    print(open(dst).read())


def traffic(src, dst):
    """Per-launch DRAM traffic of the captured conv_tc_kernel launches -> the JSON bench.py reads for roofline.traffic."""
    import json
    out = subprocess.run(["ncu", "-i", src, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    hdr, units = rows[0], rows[1]
    idx = {h: i for i, h in enumerate(hdr)}

    def val(r, name, want):
        x, u = float(r[idx[name]].replace(",", "")), units[idx[name]]
        scale = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "ns": 1e-6, "us": 1e-3, "ms": 1, "%": 1, "Ghz": 1, "Mhz": 1e-3}[u]
        return x * scale

    ls = []
    for r in rows[2:]:
        ls.append(dict(kernel=r[idx["Kernel Name"]][:28], ms=val(r, "gpu__time_duration.sum", "ms"),
                       dram_read=val(r, "dram__bytes_read.sum", "byte"), dram_write=val(r, "dram__bytes_write.sum", "byte"),
                       tensor_active_pct=val(r, "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "%"),
                       l2_hit_pct=val(r, "lts__t_sector_hit_rate.pct", "%"), sm_ghz=val(r, "sm__cycles_elapsed.avg.per_second", "Ghz")))
    # the dominant launch of the celeba B=16 forward: up.0 conv1 (3x3, 256 -> 128 channels at 256x256), the longest captured
    top = max(ls, key=lambda l: l["ms"])
    B, H, Cin, Cout = 16, 256, 256, 128
    alg = B * H * H * Cin * 2 * 2 + B * H * H * Cout * 4 + 9 * Cin * Cout * 2 * 2   # fp16 hi+lo planes in, fp32 out, hi+lo weights
    doc = dict(source=" ".join(sys.argv[4:]) or src, launches=ls,
               algorithmic_bytes={"conv1_256to128_at_256x256_B16": alg},
               top_launch=dict(name="up.0.block.N.conv1 (3x3, 256->128 @256x256, B=16)", traffic_bytes=top["dram_read"] + top["dram_write"],
                               algorithmic_bytes=alg, tensor_pipe_active_pct=top["tensor_active_pct"], ms=top["ms"]))
    json.dump(doc, open(dst, "w"), indent=1)
    print(json.dumps(doc["top_launch"], indent=1))


if __name__ == "__main__":
    {"launches": launches, "full": full, "traffic": traffic}[sys.argv[1]](sys.argv[2], sys.argv[3])
