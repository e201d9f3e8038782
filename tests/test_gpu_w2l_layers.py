"""GPU: every layer of the wav2lip256 engine (csrc/w2l_engine.cu) against float64, each computed from the GPU's own fp16 input.

A `keep_layers` session keeps every activation in its own buffer.  For each of the 54 Conv / ConvT + BN blocks and the head,
the layer's input is rebuilt from the read-back fp16 tensors of the layers that feed it (the concat of decoder and skip
outputs for the first layer of each decoder block), and the layer is recomputed in float64 with PyTorch in the reference's
own layout: `F.conv2d` / `F.conv_transpose2d` on [Cout, Cin, kh, kw] / [Cin, Cout, kh, kw] weights, never the engine's packed
[Cout][tap][Cin], sub-pixel, stem or k4 layouts.  The weights are the BN-folded weights rounded to fp16 (layer 0: fp32), the
bias is the folded bias in fp32: exactly what the weight blob holds.  The stem's input is the prepared image rebuilt on the
host (mirror-index gather, u8 * fp32(1/255) rounded to fp16, 3 masked channels with rows >= 128 zeroed, then 3 full ones,
zero padding 3), so the stem check also checks `w2l_prep_faces_kernel`.  Every output element of the checked images is
compared, borders included.

Error bound per output element, A = sum |w| |x| (a second float64 conv on absolute values), b the bias, r the residual,
pre = conv + b, ref = relu(pre (+ r)), u = 2^-11 (fp16), v = 2^-24 (fp32):

    |out - ref| <= 1.25 * ( eps_acc(K) A                     tensor-core accumulation over the layer's K chain
                          + 3 v (A + |b| + |r|)              fp32 adds of bias and residual in the epilogue
                          + u |ref| + 2^-25                  the fp16 output rounding (normal / subnormal)
                          [+ u |pre| + 2^-25]                halo kernel with a residual: it rounds fp16(acc + b) first and then
                                                             adds the residual in fp16 (conv_halo.cu, add_res)
                          [+ ks v (A + |b|)] )               gather kernel: split-K finalize sums ks fp32 partial slices;
                                                             ks <= min(32, K / 128) is the most the planner can choose

  * eps_acc(K) = 18 ceil(K / 16) 2^-23.  Assumption (not measured on the H100): each k16 wgmma step forms its 16 fp16
    products exactly and adds them and the fp32 accumulator after aligning all 17 addends to the largest, truncating each
    aligned addend and the normalised result by at most one fp32 ulp (2^-23 of the step's largest magnitude, which is at
    most the running sum of absolute values).  That is 18 ulps per step over ceil(K / 16) steps.  K is the accumulation
    chain: Cin k^2 for convs, 4 Cin for the stride-2 ConvTs (the widest sub-pixel phase), Cin for the k4 ConvT on the 1x1
    map (one GEMM row per output position) and 7 x 64 for the stem (7 kernel rows of 8 pixels x 8 channels).
  * Layer 0 (`w2l_audio_conv0_kernel`) runs on CUDA cores: an fp32 FMA chain from the bias over 9 taps, so its accumulation
    term is 10 v (A + |b|), with the same output rounding.
  * Head: pred = 255 sigmoid(z), z = hb + sum_c hw_c h_c as an fp32 FMA chain over 32 channels of the fp16 layer-53 output.
    |dz| <= 33 v (|hb| + sum |hw h|); the slope of 255 sigmoid is at most 255 / 4; `expf` is within 2 ulp (no fast math)
    and 1 + e, the division and * 255 round once each, so the sigmoid adds at most 8 v |pred|.
  * 1.25 absorbs the second-order terms the linearisation drops.

Runs: B = 16 on the benchmarked plan (halo kernels, stem on tensor cores), B = 3 (ragged tiles, other split-K and variant
choices) and B = 2 on the engine's gather plan (`no_halo`, the fallback when the stem plan cannot be made), where the stem
runs on the gather kernel as a 7-tap conv with Cin = 64 over the image's 8-channel pixel pitch.  `profile_ops` proves which
path each run took.  The avatar holds a full-range random u8 face and two smooth faces, the batch index makes the mirror
sequence turn inside the batch, and the mel windows contain values of exactly +-4.

The production plan (ring buffers, head and sigmoid fused into layer 53's halo epilogue, CUDA graph, PDL) must produce a
`pred` bit-identical to the inspected plan's at B = 16 and B = 3."""
import math
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

SAFETY = 1.25
U16 = 2.0 ** -11
SUB16 = 2.0 ** -25
V32 = 2.0 ** -24
ULP32 = 2.0 ** -23

# profile_ops kinds
GATHER, PREP, AUDIO0, HEAD, HALO, STEM, MEL = 0, 1, 2, 3, 4, 5, 6
STEM_LAYER = 13
# first layer of each decoder block (and the output block) -> the encoder layer whose output is concatenated after the
# decoder's: torch.cat((x, feats[-1]), dim=1)
SKIP = {34: 32, 36: 30, 38: 28, 41: 26, 44: 23, 47: 20, 50: 16, 53: 13}

# run -> (batch, index, checked images, no_halo)
RUNS = {
    "b16": (16, 2, (0, 15), False),   # faces 2 (smooth) and 0 (random): mirror_index(3, 2 + b) turns at b = 1 and b = 4
    "b3": (3, 4, (0, 1, 2), False),   # faces 1, 0, 0: the sequence turns between b = 1 and b = 2
    "b2_gather": (2, 0, (0,), True),  # face 0 (random)
}


def _faces():
    from oracle import wav2lip_ref as R
    _, img = R.synth_inputs(2, seed=31)
    smooth = (img[:, 3:6].permute(0, 2, 3, 1).numpy() * 255.0).round().astype(np.uint8)
    rnd = np.random.default_rng(2024).integers(0, 256, (256, 256, 3), dtype=np.uint8)
    rnd[0, 0], rnd[255, 255], rnd[127, 3], rnd[128, 7] = 255, 255, (255, 0, 255), (0, 255, 0)
    return [rnd, smooth[0], smooth[1]]


def _mel(B):
    rng = np.random.default_rng(100 + B)
    mel = rng.uniform(-4.0, 4.0, (B, 80, 16)).astype(np.float32)
    mel[:, ::7, ::5] = 4.0
    mel[:, 3::11, 2::3] = -4.0
    mel[:, :, 15] = np.where(np.arange(80) % 2 == 0, 4.0, -4.0)   # the last column, whose neighbour is the zero padding
    mel[:, 79, :] = -4.0
    return mel


@pytest.fixture(scope="module")
def model(w2l_state_dict):
    from livetalking_b200 import engine
    engine.set_device(0)
    m = engine.W2LModel.from_state_dict(w2l_state_dict)
    yield m
    m.close()


@pytest.fixture(scope="module")
def avatar():
    from livetalking_b200 import engine
    faces = _faces()
    frames = np.random.default_rng(5).integers(0, 256, (len(faces), 64, 64, 3), dtype=np.uint8)
    av = engine.W2LAvatar(faces, frames, [(0, 64, 0, 64)] * len(faces))
    yield av
    av.close()


@pytest.fixture(scope="module")
def weights(w2l_state_dict):
    """Per layer: (spec, float64 weight in PyTorch layout rounded as the blob holds it, float64 of the fp32 bias); head."""
    from livetalking_b200.w2l_pack import fold_bn
    from oracle import wav2lip_ref as R
    sd = {k.replace("module.", ""): v for k, v in w2l_state_dict.items()}
    out = []
    for li, (prefix, spec) in enumerate(R.layer_list()):
        w, b = fold_bn(sd, prefix, spec[0])
        w = w.astype(np.float32 if li == 0 else np.float16)
        out.append((spec, torch.from_numpy(w.astype(np.float64)), torch.from_numpy(b.astype(np.float32).astype(np.float64))))
    hw = torch.from_numpy(sd["output_block.1.weight"].numpy().reshape(3, 32).astype(np.float32).astype(np.float64))
    hb = torch.from_numpy(sd["output_block.1.bias"].numpy().astype(np.float32).astype(np.float64))
    return out, (hw, hb)


def _nchw(a):
    """NHWC array (fp16 / fp32) -> float64 NCHW tensor."""
    return torch.from_numpy(np.ascontiguousarray(a).astype(np.float64)).permute(0, 3, 1, 2)


def _prepared_image(faces, index, imgs):
    """The stem's input for the checked images, as w2l_prep_faces_kernel builds it (before the zero padding)."""
    from oracle.paste_ref import mirror_index
    out = []
    for b in imgs:
        f = faces[mirror_index(len(faces), index + b)]
        v = (f.astype(np.float32) * np.float32(1.0 / 255.0)).astype(np.float16)
        masked = v.copy()
        masked[128:] = 0
        out.append(np.concatenate([masked, v], axis=2))
    return _nchw(np.stack(out))


def _chain_k(li, spec):
    kind, cin, cout, k = spec[:4]
    if li == STEM_LAYER:
        return 7 * 64
    if kind == "t":
        return cin if k == 4 else 4 * cin
    return cin * k * k


def _layer_ops(kinds):
    """profile_ops index of each layer's op: mel, audio conv0, L1..L12, prep, stem, L14..L53 (+ the separate head)."""
    assert kinds[0] == MEL and kinds[1] == AUDIO0 and kinds[14] == PREP, kinds
    return [1] + [li + 1 for li in range(1, 13)] + [15] + [li + 2 for li in range(14, 54)]


def _check_layer(li, spec, w, b, x, got, kind):
    """float64 reference of layer li on input x (NCHW) and the bound above; returns (worst err / bound, where)."""
    ctype, cin, cout, k, s, p, op, res = spec
    if ctype == "c":
        conv = F.conv2d(x, w, stride=s, padding=p)
        A = F.conv2d(x.abs(), w.abs(), stride=s, padding=p)
    else:
        conv = F.conv_transpose2d(x, w, stride=s, padding=p, output_padding=op)
        A = F.conv_transpose2d(x.abs(), w.abs(), stride=s, padding=p, output_padding=op)
    bb = b[None, :, None, None]
    pre = conv + bb
    r = x if res else torch.zeros_like(pre)
    ref = torch.relu(pre + r)
    K = _chain_k(li, spec)
    if kind == AUDIO0:
        acc = 10 * V32 * (A + bb.abs())
    else:
        acc = 18 * math.ceil(K / 16) * ULP32 * A + 3 * V32 * (A + bb.abs() + r.abs())
    bound = acc + U16 * ref.abs() + SUB16
    if kind == HALO and res:
        bound = bound + U16 * pre.abs() + SUB16
    if kind == GATHER:
        bound = bound + min(32, K // 128) * V32 * (A + bb.abs())
    bound = SAFETY * bound
    assert got.shape == ref.shape, (li, tuple(got.shape), tuple(ref.shape))
    assert torch.isfinite(got).all(), f"layer {li}: non-finite output"
    ratio = (got - ref).abs() / bound
    worst = float(ratio.max())
    where = np.unravel_index(int(ratio.argmax()), tuple(ratio.shape))
    return worst, (where, float(got[where]), float(ref[where]), float(bound[where]))


@pytest.mark.parametrize("run", list(RUNS))
def test_every_layer_against_float64(model, avatar, weights, run):
    from livetalking_b200 import engine
    B, index, imgs, no_halo = RUNS[run]
    layers, (hw, hb) = weights
    mel = _mel(B)
    t0 = time.time()
    s = engine.W2LSession(model, avatar, B, keep_layers=True, no_halo=no_halo)
    try:
        kinds = s.profile_ops(index)[2]
        pred = s.infer(index, mel)
        outs = {li: s.layer_output(li)[list(imgs)] for li in range(54)}
    finally:
        s.close()
    t_gpu = time.time() - t0

    # which path ran
    ops = _layer_ops(kinds)
    assert len(kinds) == 57 and kinds[56] == HEAD, kinds          # keep_layers: the 1x1 head is its own kernel
    lk = [int(kinds[o]) for o in ops]
    if no_halo:
        assert not np.isin(kinds, (HALO, STEM)).any(), kinds
        assert lk[STEM_LAYER] == GATHER
    else:
        assert lk[STEM_LAYER] == STEM and lk[53] == HALO, lk
    assert np.isfinite(pred).all()

    faces = [avatar.faces[i] for i in range(avatar.n)]
    got = {li: _nchw(outs[li]) for li in outs}
    report, bad = [], []
    for li, (spec, w, b) in enumerate(layers):
        if li == 0:
            x = torch.from_numpy(mel[list(imgs)].astype(np.float64))[:, None]
        elif li == STEM_LAYER:
            x = _prepared_image(faces, index, imgs)
        elif li == 33:
            x = got[12]
        elif li in SKIP:
            x = torch.cat([got[li - 1], got[SKIP[li]]], dim=1)
        else:
            x = got[li - 1]
        worst, info = _check_layer(li, spec, w, b, x, got[li], lk[li])
        report.append((li, lk[li], worst))
        if worst > 1.0:
            bad.append((li, worst, info))
    # head on layer 53's fp16 output
    h = got[53]
    z = torch.einsum("oc,nchw->nohw", hw, h) + hb[None, :, None, None]
    Ah = torch.einsum("oc,nchw->nohw", hw.abs(), h.abs()) + hb.abs()[None, :, None, None]
    want = 255.0 * torch.sigmoid(z)
    bound = SAFETY * (255.0 / 4.0 * 33 * V32 * Ah + 8 * V32 * want)
    gp = torch.from_numpy(pred[list(imgs)].astype(np.float64)).permute(0, 3, 1, 2)
    ratio = (gp - want).abs() / bound
    report.append(("head", HEAD, float(ratio.max())))
    if float(ratio.max()) > 1.0:
        where = np.unravel_index(int(ratio.argmax()), tuple(ratio.shape))
        bad.append(("head", float(ratio.max()), (where, float(gp[where]), float(want[where]), float(bound[where]))))

    print(f"\n[{run}] B={B} index={index} images={imgs} no_halo={no_halo}: GPU + read-back {t_gpu:.1f} s, "
          f"float64 reference {time.time() - t0 - t_gpu:.1f} s")
    names = {GATHER: "gather", HALO: "halo", STEM: "stem", AUDIO0: "audio0", HEAD: "head"}
    for li, kd, worst in report:
        print(f"  L{li:>4} {names[kd]:>6}  worst err/bound {worst:.3f}" if li != "head" else
              f"  {li:>5} {names[kd]:>6}  worst err/bound {worst:.3f}")
    top = max(report, key=lambda r: r[2])
    print(f"  [{run}] largest err/bound {top[2]:.3f} at {top[0]}")
    assert not bad, f"[{run}] outside the bound (layer, err/bound, (image, c, y, x), got, want, bound): " + "; ".join(
        f"{li}: {r:.2f} {info}" for li, r, info in bad[:8])


@pytest.mark.parametrize("run", ["b16", "b3"])
def test_production_plan_equals_inspected_plan(model, avatar, run):
    """Ring buffers, the head fused into layer 53's halo epilogue, the CUDA graph and PDL change no bit of pred."""
    from livetalking_b200 import engine
    B, index, _, _ = RUNS[run]
    mel = _mel(B)
    keep = engine.W2LSession(model, avatar, B, keep_layers=True)
    try:
        keep_kinds = keep.profile_ops(index)[2]
        want = keep.infer(index, mel)
    finally:
        keep.close()
    prod = engine.W2LSession(model, avatar, B)
    try:
        prod_kinds = prod.profile_ops(index)[2]
        got = [prod.infer(index, mel) for _ in range(2)]
    finally:
        prod.close()
    assert int((keep_kinds == HEAD).sum()) == 1 and int((prod_kinds == HEAD).sum()) == 0, (keep_kinds, prod_kinds)
    assert len(prod_kinds) == len(keep_kinds) - 1
    assert np.isfinite(want).all()
    for g in got:
        diff = g.view(np.uint32) != want.view(np.uint32)
        assert not diff.any(), (f"[{run}] {int(diff.sum())} pred values differ, max |diff| "
                                f"{float(np.abs(g - want).max())} at {np.argwhere(diff)[:4].tolist()}")
