"""profiles/conv_traffic.json from an ncu launch list that carries DRAM byte counters.

    ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum --clock-control none -c 700 --csv \
        --log-file gpurun_out/launches.csv python bench.py --steps 2 --warmup 3 --no-cpu-baseline
    python tools/traffic_from_ncu.py gpurun_out/launches.csv profiles/conv_traffic.json

One step = the launches between two consecutive set_int_kernel launches that contain the mel kernels (the with-mel forward
graph + paste).  Sums dram__bytes_read + dram__bytes_write over the conv kernels (conv_halo_umma, conv_gather_umma,
stem_umma, splitk_finalize) of that step; bench.py reports the figure as roofline.traffic.  ncu serialises the kernels and
runs them cold, so this is an upper bound of the traffic inside a graph replay (no L2 reuse between layers is visible).
"""
import csv
import json
import sys


def main(src, dst):
    rows = [r for r in csv.reader(open(src)) if len(r) > 10]
    hdr = rows[0]
    ik, im, iv, iid, iu = hdr.index("Kernel Name"), hdr.index("Metric Name"), hdr.index("Metric Value"), hdr.index("ID"), hdr.index("Metric Unit")
    scale = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "ns": 1e-3, "us": 1.0, "ms": 1e3}   # bytes / microseconds
    launches = {}
    for r in rows[1:]:
        try:
            v = float(r[iv].replace(",", "")) * scale.get(r[iu], 1.0)
        except ValueError:
            continue
        d = launches.setdefault(int(r[iid]), {"name": r[ik]})
        d[r[im]] = v
    ids = sorted(launches)
    marks = [i for i in ids if "set_int" in launches[i]["name"]]
    step = None
    for a, b in zip(marks, marks[1:]):
        names = [launches[i]["name"] for i in ids if a <= i < b]
        if any(("mel_fused" in n or "mel_stft" in n) for n in names) and any("paste" in n for n in names):
            step = (a, b)                                  # keep the last complete step
    if step is None:
        raise SystemExit("no complete step (set_int .. mel .. paste) in the launch list")
    conv_b = other_b = conv_us = other_us = 0.0
    per_kernel = {}
    for i in ids:
        if not (step[0] <= i < step[1]):
            continue
        L = launches[i]
        by = L.get("dram__bytes_read.sum", 0.0) + L.get("dram__bytes_write.sum", 0.0)
        us = L.get("gpu__time_duration.sum", 0.0)
        is_conv = any(k in L["name"] for k in ("conv_halo_", "conv_ystack_", "conv_gather_", "stem_umma", "splitk_finalize"))
        short = L["name"].split("(")[0].replace("void ", "").replace("ltb::", "")
        pk = per_kernel.setdefault(short, [0, 0.0, 0.0])
        pk[0] += 1
        pk[1] += us
        pk[2] += by
        if is_conv:
            conv_b += by
            conv_us += us
        else:
            other_b += by
            other_us += us
    out = {"dram_bytes_per_step": int(conv_b), "conv_kernel_us_per_step_ncu": round(conv_us, 1),
           "other_dram_bytes_per_step": int(other_b), "other_kernel_us_per_step_ncu": round(other_us, 1),
           "source": src, "launch_ids": list(step),
           "per_kernel": {k: {"launches": v[0], "us": round(v[1], 1), "dram_MB": round(v[2] / 1e6, 2)} for k, v in sorted(per_kernel.items(), key=lambda kv: -kv[1][1])},
           "note": "sum of dram__bytes_read+write over the conv kernels of one B=16 step, ncu (serialised, cold L2)"}
    json.dump(out, open(dst, "w"), indent=1)
    print(json.dumps({k: out[k] for k in ("dram_bytes_per_step", "conv_kernel_us_per_step_ncu", "other_dram_bytes_per_step")}))


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2])
