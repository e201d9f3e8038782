"""Knock-out timings of the wav2lip256 decoder's ConvT / conv layer shapes (diagnostic tool, not part of the product path).

    python -m livetalking_b200.build --diag          # here (cross-compile lib/libltb200_diag.so with -DLTB_HALO_DIAG)
    python tools/diag_layers.py                      # on the GPU box
    python tools/diag_layers.py --forward            # the same knock-outs on every op of the real batch-16 forward plan

For every shape: full kernel, then with one role knocked out (LTB_HALO_DIAG bits: 1 no epilogue global I/O, 2 no epilogue,
4 no MMAs, 8 no A (halo) loads, 16 no B (weight) loads) — what the remaining time is tells which resource bounds the layer.
--forward: per-op event timings (median of 5 eager profiling passes) of the wav2lip256 batch-16 forward, fused 1x1 head and
all, under LTB_HALO_DIAG 0 / 1 / 2, and the sum over the halo-kernel ops of (dbg0 - dbg1) and (dbg0 - dbg2).
--forward --ab VAR: the same per-op timings with the A/B switch VAR (e.g. LTB_CONV_ROWPAIR) on and off, in one process
(with LTB_DIAG_NORMAL_LIB=1 the product library runs)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402


def main():
    from livetalking_b200 import _capi
    if not os.environ.get("LTB_DIAG_NORMAL_LIB"):
        _capi.LIB_PATH = os.path.join(os.path.dirname(_capi.LIB_PATH), "libltb200_diag.so")
    from livetalking_b200 import engine
    engine.set_device(0)
    if "--forward" in sys.argv:
        return forward(engine)
    rng = np.random.default_rng(0)
    cases = [  # name, N, H, Cin, Cout, transposed, residual
        ("L50 ConvT 160->64 @128", 16, 128, 160, 64, True, False),
        ("L47 ConvT 320->128 @64", 16, 64, 320, 128, True, False),
        ("L44 ConvT 512->256 @32", 16, 32, 512, 256, True, False),
        ("L41 ConvT 768->384 @16", 16, 16, 768, 384, True, False),
        ("L42 conv 384->384 @32 res", 16, 32, 384, 384, False, True),
        ("L45 conv 256->256 @64 res", 16, 64, 256, 256, False, True),
        ("L48 conv 128->128 @128 res", 16, 128, 128, 128, False, True),
        ("L51 conv 64->64 @256 res", 16, 256, 64, 64, False, True),
        ("L53 conv 80->32 @256", 16, 256, 80, 32, False, False),
        ("L39 conv 512->512 @16 res", 16, 16, 512, 512, False, True),
        ("L25 conv 256->256 @16 res", 16, 16, 256, 256, False, True),
        ("L28 conv 512->512 @8 res", 16, 8, 512, 512, False, True),
    ]
    variants = [0, 1, 2, 4, 8, 16, 24, 6, 30]
    sel = os.environ.get("LTB_DIAG_CASES")
    if sel:
        cases = [cases[int(i)] for i in sel.split(",")]
    for name, N, H, cin, cout, tr, res in cases:
        x = (rng.standard_normal((N, H, H, cin)) * 0.5).astype(np.float16)
        w = (rng.standard_normal((cin, cout, 3, 3) if tr else (cout, cin, 3, 3)) * 0.05).astype(np.float32)
        b = np.zeros(cout, np.float32)
        r = x if (res and cin == cout) else None
        flops = 2.0 * N * H * H * 9 * cin * cout
        line = [name]
        base = None
        for v in variants:
            os.environ["LTB_HALO_DIAG"] = str(v)
            _, ms = engine.conv2d_f16(x, w, b, stride=(2, 2) if tr else (1, 1), pad=1, transposed=tr, relu=True, res=r, reps=30)
            if v == 0:
                base = ms
            line.append(f"dbg{v}:{ms * 1000:.1f}us")
        print(" ".join(line), f"| full = {flops / 1e9 / base:.0f} TF/s", flush=True)


def forward(engine):
    from livetalking_b200 import synth
    from livetalking_b200.w2l_pack import pack_state_dict
    model = engine.W2LModel(pack_state_dict(synth.random_state_dict(0)))
    av = engine.W2LAvatar(*synth.synthetic_avatar(n=16, H=720, W=1280, bbox=(200, 520, 480, 800)))
    med = {}
    ab = sys.argv[sys.argv.index("--ab") + 1] if "--ab" in sys.argv else None
    settings = [(ab, "1"), (ab, "0")] if ab else [("LTB_HALO_DIAG", str(v)) for v in (0, 1, 2)]
    for v, (var, val) in enumerate(settings):
        os.environ[var] = val    # read when the session plans its convs
        sess = engine.W2LSession(model, av, 16)
        sess.mel_step(synth.sine_audio(2.0)[:(10 + 10 + 2 * 16) * 320], want_output=False)   # one step's PCM window
        sess.profile_ops(0)
        passes = [sess.profile_ops(0) for _ in range(5)]
        kinds, flops = passes[0][2], passes[0][1]
        med[v] = np.median(np.stack([ms for ms, _, _ in passes]), axis=0)
        sess.close()
    halo = kinds == 4   # kind 4: a TMA conv kernel (halo, ping-pong or row-pair)
    if ab:
        print(f"op kind GFLOP  {ab}=1_us {ab}=0_us")
        for i in range(len(kinds)):
            if halo[i]:
                print(f"{i:3d} {kinds[i]} {flops[i] / 1e9:7.1f} {med[0][i] * 1e3:7.1f} {med[1][i] * 1e3:7.1f}")
        print(f"all ops {ab}=1 {med[0].sum() * 1e3:.1f} us | {ab}=0 {med[1].sum() * 1e3:.1f} us", flush=True)
        return
    print("op kind GFLOP  dbg0_us dbg1_us dbg2_us")
    for i in range(len(kinds)):
        if halo[i]:
            print(f"{i:3d} {kinds[i]} {flops[i] / 1e9:7.1f} {med[0][i] * 1e3:7.1f} {med[1][i] * 1e3:7.1f} {med[2][i] * 1e3:7.1f}")
    tot = med[0].sum() * 1e3
    rec, ceil = ((med[0] - med[1])[halo].sum() * 1e3, (med[0] - med[2])[halo].sum() * 1e3)
    print(f"all ops {tot:.1f} us | halo ops {med[0][halo].sum() * 1e3:.1f} us | sum(dbg0-dbg1) {rec:.1f} us ({100 * rec / tot:.1f} %)"
          f" | sum(dbg0-dbg2) {ceil:.1f} us ({100 * ceil / tot:.1f} %)", flush=True)


if __name__ == "__main__":
    main()
