"""GPU: a halo conv whose Cin is not a multiple of 64 writes exactly the bits of the same conv with its input channels and
weights zero-padded to the next multiple of 64.

The halo kernel loads Cin in K chunks of 64 channels; TMA zero-fills the channels >= Cin of the last chunk, and when that
chunk holds at most 32 channels the consumers of the BN <= 64 instances issue only its first two K steps (16 channels each).  The padded conv has no
ragged chunk and issues every K step of every chunk, so equal bits show that the skipped steps added nothing.  Rows cover every
halo path with a ragged last chunk: 3x3 with streamed and one or two resident weight chunks, sub-pixel ConvT (streamed and
resident), fused upsample + 3x3, stride 2 and GEMM mode, at remainders of 16 and 32 channels (skipped steps) and 40 and 48
(all four steps), Cin below 64, and the wav2lip256 decoder's 80 and 160.  The input slices sit between sentinel channels, so a
read past Cin would show.  The fused wav2lip head on the 80-channel
output conv is checked against the separate head kernel by test_gpu_w2l_layers.py."""
import numpy as np
import pytest
import torch
from test_gpu_conv_variants import (H100_SMS, SENT_IN, SENT_OUT, H, _bits, _check_model, _conv, _convT, _expected, _gemm, _key_id,
                                    _pack_convT, _reference, _shape_weight, _slice_buf, _up)

CASES = [
    # 3x3, streamed weights
    (H(32, 2, 1, 9), _conv(6, 128, 20, 16, 96)),
    (H(32, 2, 1, 9), _conv(6, 128, 20, 32, 96)),
    (H(32, 2, 1, 9), _conv(6, 128, 20, 48, 96)),
    (H(32, 2, 1, 9), _conv(6, 128, 20, 80, 96)),
    (H(32, 2, 1, 9), _conv(6, 128, 20, 112, 96)),
    (H(32, 2, 1, 9), _conv(6, 128, 20, 160, 96)),
    (H(32, 1, 1, 9), _conv(8, 20, 20, 80, 96)),
    (H(64, 2, 1, 9), _conv(6, 128, 20, 96, 192)),
    (H(64, 1, 1, 9), _conv(6, 20, 12, 48, 384)),
    (H(128, 2, 1, 9), _conv(5, 128, 36, 80, 256)),
    # 3x3, resident weights (one or two K chunks)
    (H(32, 2, 1, 9, 1), _conv(4, 128, 132, 16, 32)),
    (H(32, 2, 1, 9, 1), _conv(4, 128, 132, 48, 32)),
    (H(64, 2, 1, 9, 1), _conv(4, 128, 132, 32, 64)),
    (H(32, 2, 1, 9, 2), _conv(4, 128, 132, 80, 32)),
    (H(32, 2, 1, 9, 2), _conv(4, 128, 132, 112, 32)),
    # sub-pixel ConvT
    (H(64, 1, 4, 9), _convT(16, 8, 20, 80, 192)),
    (H(64, 1, 4, 9), _convT(16, 8, 20, 160, 192)),
    (H(32, 1, 4, 9), _convT(16, 8, 20, 48, 96)),
    (H(64, 1, 4, 9, 1), _convT(16, 8, 132, 32, 64)),
    (H(64, 1, 4, 9, 2), _convT(16, 8, 132, 80, 64)),
    (H(32, 1, 4, 9, 1), _convT(16, 8, 132, 16, 32)),
    (H(32, 1, 4, 9, 2), _convT(16, 8, 132, 112, 32)),
    # nearest-2x upsample + 3x3
    (H(64, 1, 4, 16), _up(3, 24, 60, 16, 192)),
    (H(64, 1, 4, 16), _up(3, 24, 60, 80, 192)),
    # 3x3 stride 2 (Cin >= 64)
    (H(64, 1, 1, 10), _conv(3, 72, 72, 80, 192, stride=2)),
    (H(64, 1, 1, 10), _conv(3, 72, 72, 112, 192, stride=2)),
    (H(32, 1, 1, 10), _conv(3, 72, 72, 96, 96, stride=2)),
    # GEMM mode (1x1)
    (H(128, 1, 1, 1), _gemm(2, 36, 120, 40, 256)),
    (H(64, 2, 1, 1), _gemm(1, 100, 120, 96, 192)),
    (H(64, 1, 1, 1), _gemm(1, 24, 120, 80, 384)),
    (H(32, 2, 1, 1), _gemm(1, 100, 120, 48, 96)),
    (H(32, 1, 1, 1), _gemm(3, 10, 70, 112, 256)),
]
IDS = [f"{_key_id(k)}-Cin{r['Cin']}" for k, r in CASES]


@pytest.fixture(scope="module")
def ctx():
    from livetalking_b200 import engine
    from livetalking_b200.ops import Ctx
    engine.set_device(0)
    c = Ctx()
    yield c
    c.close()


def _run(ctx, row, x, w, b, r, relu):
    """Plan and run the row's op on fp16 x (N, IH, IW, Cin) and w (conv: Cout, Cin, k, k; ConvT: Cin, Cout, 3, 3), fp32 b and
    an fp16 residual r (or None).  -> (planned variant, fp16 output)"""
    from livetalking_b200.ops import ConvWeight
    kind, N, IH, IW, k, s, p = (row[n] for n in ("kind", "N", "IH", "IW", "k", "stride", "pad"))
    Cin, Cout = x.shape[-1], b.shape[0]
    OH, OW = (2 * IH, 2 * IW) if kind in ("convT", "up") else ((IH + 2 * p - k) // s + 1, (IW + 2 * p - k) // s + 1)
    xv, xt, _ = _slice_buf(ctx, x.numpy(), Cin + 24, 8, SENT_IN)
    ov, ot, _ = _slice_buf(ctx, np.full((N, OH, OW, Cout), np.nan, np.float16), Cout + 16, 8, SENT_OUT)
    temps = [xt, ot]
    geo = dict(N=N, IH=IH, IW=IW, OH=OH, OW=OW, stride=(s, s), pad=(p, p), relu=relu, res=None, upsample2x=kind == "up",
               transposed=kind == "convT")
    if r is not None:
        geo["res"], rt, _ = _slice_buf(ctx, r.numpy(), Cout + 8, 8, SENT_IN)
        temps.append(rt)
    try:
        if kind == "up":
            cw = ConvWeight(ctx, w.float().numpy(), b.numpy(), tap_major=False)
            temps += [cw.w, cw.bias] + list(cw.upconv(ctx))
        else:
            if kind == "convT":
                rows, view = _pack_convT(w.numpy())
                wt, wtap = ctx.upload(rows), ctx.upload(view)
                temps += [wt, wtap]
            else:
                wt, wtap = ctx.upload(np.ascontiguousarray(w.permute(0, 2, 3, 1).reshape(Cout, k * k * Cin).numpy())), None
                temps.append(wt)
                if k == 3:
                    wtap = ctx.alloc((9, Cout, Cin))
                    temps.append(wtap)
                    ctx.w_tap_major(wt, wtap, Cout, Cin)
            bt = ctx.upload(b.numpy())
            temps.append(bt)
            cw = _shape_weight(Cout, Cin, k, wt, wtap, bt)
        variant = ctx.conv_plan(xv, cw, ov, **geo)
        ctx.conv(xv, cw, ov, **geo)
        got = ctx.download(ot)[..., 8:8 + Cout]
        ctx.sync()
    finally:
        for t in temps:
            ctx.free(t)
    return variant, got


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(CASES)), ids=IDS)
def test_ragged_cin_is_bit_identical_to_zero_padded_cin(ctx, case):
    assert torch.cuda.get_device_properties(0).multi_processor_count == H100_SMS, "the rows' variants assume the 132-SM H100 SXM"
    key, row = CASES[case]
    N, IH, IW, Cin, Cout, k = (row[n] for n in ("N", "IH", "IW", "Cin", "Cout", "k"))
    assert Cin % 64, "a ragged row"
    pad = -Cin % 64
    g = torch.Generator().manual_seed(700 + case)
    x = (torch.randn(N, IH, IW, Cin, generator=g) * 0.7 + 0.4).half()
    tr = row["kind"] == "convT"
    w = (torch.randn(*((Cin, Cout) if tr else (Cout, Cin)), k, k, generator=g) * (2.0 / (Cin * k * k)) ** 0.5).half()
    b = torch.randn(Cout, generator=g) * 0.2
    relu, with_res = case % 2 == 0, case % 3 != 2
    parts = _reference(row, x.double().permute(0, 3, 1, 2), w.double())
    r = (torch.randn(*parts[0].shape, generator=g) * 0.5).half() if with_res else None

    variant, got = _run(ctx, row, x, w, b, r, relu)
    x_pad = torch.cat([x, torch.zeros(N, IH, IW, pad, dtype=x.dtype)], dim=-1)
    w_pad = torch.cat([w, torch.zeros(*((pad, Cout) if tr else (Cout, pad)), k, k, dtype=w.dtype)], dim=0 if tr else 1)
    variant_pad, got_pad = _run(ctx, row, x_pad, w_pad, b, r, relu)

    want = _expected(key)
    assert variant == want and variant_pad == want, f"planned {variant} (Cin {Cin}) and {variant_pad} (Cin {Cin + pad}), expected {want}"
    _check_model(got, parts, b.double().numpy(), None if r is None else r.numpy(), relu, row, variant, IDS[case])
    diff = _bits(got) != _bits(got_pad)
    assert not diff.any(), (f"{IDS[case]}: {int(diff.sum())} outputs differ from the zero-padded Cin {Cin + pad}, first at "
                            f"{np.argwhere(diff)[0]}")
