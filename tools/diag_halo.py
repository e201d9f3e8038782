"""Where does the time of a halo-conv layer go?  (diagnostic tool, not part of the product path)

Builds lib/libltb200_diag.so with -DLTB_HALO_DIAG (conv_halo.cu then honours the LTB_HALO_DIAG environment variable at
plan time: bit0 no epilogue global I/O, bit1 no epilogue work, bit2 no MMAs, bit3 no A (halo) loads, bit4 no B (weight)
loads) and times the wav2lip256 decoder's 3x3 convs at batch 16 with each role knocked out in turn.  Each line starts with the
kernel instance Ctx.conv_plan picks for that shape (the fused 1x1 head of L53 exists only inside the engine's forward plan:
`tools/diag_layers.py --forward` times it there).

    python tools/diag_halo.py --build          # here (cross-compile)
    python tools/diag_halo.py                  # on the GPU box
"""
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402


def main():
    from livetalking_b200 import build
    if "--build" in sys.argv:
        print(build.build(defines=("LTB_HALO_DIAG",), tag="_diag"))
        return
    from livetalking_b200 import _capi
    if not os.environ.get("LTB_DIAG_NORMAL_LIB"):     # LTB_DIAG_NORMAL_LIB=1: time / profile the product library (variant 0 only)
        _capi.LIB_PATH = os.path.join(os.path.dirname(_capi.LIB_PATH), "libltb200_diag.so")
    from livetalking_b200 import ops
    ctx = ops.Ctx()
    rng = np.random.default_rng(0)
    cases = [  # name, N, H, Cin, Cout, residual
        ("L52 64->64 res @256", 16, 256, 64, 64, True),
        ("L53 80->32     @256", 16, 256, 80, 32, False),
        ("L49 128->128 res @128", 16, 128, 128, 128, True),
        ("L46 256->256 res @64", 16, 64, 256, 256, True),
        ("L43 384->384 res @32", 16, 32, 384, 384, True),
    ]
    variants = [0, 1, 2, 4, 8, 16, 24, 4 | 2, 8 | 16 | 2, 4 | 8 | 16, 4 | 8 | 16 | 2]
    if os.environ.get("LTB_DIAG_ONLY"):          # e.g. "0:0" = first case, variant 0 (for an ncu capture)
        ci, v = os.environ["LTB_DIAG_ONLY"].split(":")
        cases, variants = [cases[int(ci)]], [int(v)]
    # a residual case runs twice: residual = the conv input itself (taken from the halo tiles in shared memory) and
    # residual = a copy of it (read from global memory)
    cases = [(name + (" copy" if copy else ""), N, H, cin, cout, res, copy) for name, N, H, cin, cout, res in cases
             for copy in ((False, True) if res else (False,))]
    for name, N, H, cin, cout, res, copy in cases:
        xh = (rng.standard_normal((N * H * H, cin)) * 0.5).astype(np.float16)
        x = ctx.upload(xh)
        w = ops.ConvWeight(ctx, (rng.standard_normal((cout, cin, 3, 3)) * 0.05).astype(np.float32), np.zeros(cout, np.float32))
        out = ctx.alloc((N * H * H, cout), np.float16)
        r = (ctx.upload(xh) if copy else x) if (res and cin == cout) else None
        flops = 2.0 * N * H * H * 9 * cin * cout
        plan = ctx.conv_plan(x, w, out, N=N, IH=H, IW=H, OH=H, OW=H, pad=(1, 1), res=r, relu=True)
        inst = "kernel%d<%d,%d,%d,%d,RC=%d>" % (plan["kernel"], plan["bn"], plan["nsub"], plan["nacc"], plan["taps"], plan["resident_chunks"])
        line = [name]
        for v in variants:
            os.environ["LTB_HALO_DIAG"] = str(v)
            for _ in range(3):
                ctx.conv(x, w, out, N=N, IH=H, IW=H, OH=H, OW=H, pad=(1, 1), res=r, relu=True)
            ctx.sync()
            reps = 40
            t0 = time.perf_counter()
            for _ in range(reps):
                ctx.conv(x, w, out, N=N, IH=H, IW=H, OH=H, OW=H, pad=(1, 1), res=r, relu=True)
            ctx.sync()
            us = (time.perf_counter() - t0) / reps * 1e6
            line.append(f"dbg{v}:{us:.1f}us")
        print(inst, " ".join(line), f"| full = {flops / 1e6 / float(line[1].split(':')[1][:-2]):.0f} TF/s", flush=True)


if __name__ == "__main__":
    main()
