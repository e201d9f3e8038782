"""GPU: every sub-pixel halo conv instance (NACC == 4: ConvT TAPS = 9 and nearest-2x upsample + conv TAPS = 16; BN 64 and 32;
streamed, one and two resident K chunks; ragged Cin) writes exactly the bits it wrote when each halo view fed its adjacent
phase slots with one wide wgmma and the tensor pipe was drained after every view.

The MMAs now go one N = BN wgmma per (view, phase slot), in the same per-slot order, so every accumulator element sees the
same sequence of fp32 additions.  golden/halo_subpixel_sha256.json holds the SHA-256 of each row's fp16 output as that earlier
issue order computed it on an H100 from the same seeded inputs; each row is also checked against float64."""
import hashlib
import json
import os

import pytest
from test_gpu_conv_variants import H, VARIANTS, _bits, _check_model, _convT, _expected, _key_id, _run_row, _up

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "halo_subpixel_sha256.json")

ROWS = {f"{_key_id(k)}-Cin{r['Cin']}": (k, r) for k, r in VARIANTS.items() if k[0] == "halo" and k[3] == 4}
# ragged K: 160 channels = two full chunks and a zero-filled one (streamed weights only: resident variants hold <= 2 chunks)
ROWS.update({
    f"{_key_id(H(64, 1, 4, 9))}-Cin160": (H(64, 1, 4, 9), _convT(16, 8, 20, 160, 192)),
    f"{_key_id(H(32, 1, 4, 9))}-Cin160": (H(32, 1, 4, 9), _convT(16, 8, 20, 160, 96)),
    f"{_key_id(H(64, 1, 4, 16))}-Cin160": (H(64, 1, 4, 16), _up(3, 24, 60, 160, 192)),
})
IDS = sorted(ROWS)


def digest(ctx, rid):
    """(planned variant, SHA-256 of the output bits, output, float64 reference parts) of row rid on its fixed seed."""
    key, row = ROWS[rid]
    i = IDS.index(rid)
    (variant, got, ref, _, _), temps = _run_row(ctx, row, seed=500 + i, relu=i % 2 == 0, with_res=i % 3 != 2)
    for t in temps:
        ctx.free(t)
    return variant, hashlib.sha256(_bits(got).tobytes()).hexdigest(), got, ref


@pytest.fixture(scope="module")
def ctx():
    from livetalking_b200 import engine
    from livetalking_b200.ops import Ctx
    engine.set_device(0)
    c = Ctx()
    yield c
    c.close()


def test_golden_covers_every_row():
    with open(GOLDEN) as f:
        assert sorted(json.load(f)) == IDS


@pytest.mark.gpu
@pytest.mark.parametrize("rid", IDS)
def test_subpixel_instance_is_bit_identical_to_the_wide_view_issue(ctx, rid):
    import torch
    assert torch.cuda.get_device_properties(0).multi_processor_count == 132, "the rows' variants assume the 132-SM H100 SXM"
    with open(GOLDEN) as f:
        want = json.load(f)[rid]
    variant, sha, got, ref = digest(ctx, rid)
    assert variant == _expected(ROWS[rid][0]), f"{rid}: planned {variant}"
    parts, bias, r = ref
    worst = _check_model(got, parts, bias, r, IDS.index(rid) % 2 == 0, ROWS[rid][1], variant, rid)["worst"]
    assert sha == want, f"{rid}: output bits differ from the wide-view issue's (worst err / bound vs float64 {worst:.3f})"
