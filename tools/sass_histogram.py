"""Per-kernel SASS opcode histogram of libltb200.so -> profiles/<tag>_sass_histogram.md.

The library itself is git-ignored (built in-tree by `python -m livetalking_b200.build`), so this table is the tracked evidence
that the shipped kernels are wgmma / TMA code:
  HGMMA    wgmma.mma_async (fp16)       UTMALDG  cp.async.bulk.tensor (TMA load)     UTMASTG  TMA store
  WARPSYNC / BAR: warpgroup fences      SYNCS    mbarrier arrive / try_wait          LDGSTS   cp.async (16-byte gather)
    python tools/sass_histogram.py [tag]"""
import collections
import os
import re
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OPS = ["HGMMA", "UTMALDG", "UTMASTG", "SYNCS", "LDGSTS", "BAR.SYNC", "SHFL", "STG", "LDG", "HFMA2", "DFMA", "FFMA", "IMAD"]


def main():
    tag = sys.argv[1] if len(sys.argv) > 1 else "r02"
    lib = os.path.join(ROOT, "livetalking_b200", "lib", "libltb200.so")
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    sass = subprocess.run([cuobjdump, "-sass", lib], capture_output=True, text=True, check=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)[1:]
    rows = []
    for f in funcs:
        name = f.split("\n", 1)[0].strip()
        dem = subprocess.run(["c++filt", name], capture_output=True, text=True).stdout.strip() or name
        dem = re.sub(r"\(.*", "", dem).replace("ltb::", "")
        dem = re.sub(r"^void ", "", dem)
        cnt = collections.Counter()
        n = 0
        for line in f.split("\n"):
            m = re.search(r"/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_.]*)", line)
            if not m:
                continue
            n += 1
            op = m.group(1)
            for o in OPS:
                if op.startswith(o):
                    cnt[o] += 1
                    break
        rows.append((dem, n, cnt))
    rows.sort(key=lambda r: (-r[2]["HGMMA"], r[0]))
    out = os.path.join(ROOT, "profiles", f"{tag}_sass_histogram.md")
    with open(out, "w") as fh:
        fh.write(f"# SASS opcode histogram of libltb200.so ({tag}; `python tools/sass_histogram.py {tag}`; sm_90a, nvcc "
                 "-gencode arch=compute_90a,code=sm_90a)\n\n")
        fh.write("| kernel | SASS instr | " + " | ".join(OPS) + " |\n|---|---|" + "---|" * len(OPS) + "\n")
        tot = collections.Counter()
        for dem, n, cnt in rows:
            fh.write(f"| `{dem}` | {n} | " + " | ".join(str(cnt[o]) if cnt[o] else "" for o in OPS) + " |\n")
            tot.update(cnt)
        fh.write(f"| **total ({len(rows)} kernels)** | {sum(r[1] for r in rows)} | " + " | ".join(str(tot[o]) for o in OPS) + " |\n")
    print(out, {o: tot[o] for o in OPS[:5]})


if __name__ == "__main__":
    main()
