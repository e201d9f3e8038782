"""GPU parity tests proper: the CUDA wav2lip256 path (through the C ABI) against the CPU oracle.

Bars: model forward PSNR >= 40 dB after the reference's own u8 truncation (north_star), mel within 1e-5 of the float64
oracle, paste-back bit-exact.  Every layer on its own against float64: tests/test_gpu_w2l_layers.py."""
import os
import sys
import zlib

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))


def _faces_from_inputs(img):
    """oracle synth_inputs img (B,6,256,256) in [0,1] (k/255 exactly) -> list of u8 BGR faces (B,256,256,3)."""
    f = (img[:, 3:6].permute(0, 2, 3, 1).numpy() * 255.0).round().astype(np.uint8)
    return [f[i] for i in range(f.shape[0])]


def _avatar(faces, H=360, W=640, boxes=None):
    from livetalking_b200 import engine
    n = len(faces)
    rng = np.random.default_rng(11)
    frames = rng.integers(0, 256, (n, H, W, 3), dtype=np.uint8)
    if boxes is None:
        boxes = [(20 + 3 * i, 20 + 3 * i + 200 + 7 * i, 100 + i, 100 + i + 190 + 5 * i) for i in range(n)]
    return engine.W2LAvatar(faces, frames, boxes), frames, np.asarray(boxes, np.int32)


@pytest.fixture(scope="module")
def model(w2l_state_dict):
    from livetalking_b200 import engine
    engine.set_device(0)
    m = engine.W2LModel.from_state_dict(w2l_state_dict)
    yield m
    m.close()


def test_forward_psnr_against_oracle(model, w2l_state_dict):
    """The whole forward against the CPU fp32 oracle run end to end.  Each layer is checked on its own against float64 in
    tests/test_gpu_w2l_layers.py."""
    from livetalking_b200 import engine
    from oracle import wav2lip_ref as R
    B = 2
    mel, img = R.synth_inputs(B, seed=5)
    ref = R.wav2lip_forward(w2l_state_dict, mel, img)
    av, _, _ = _avatar(_faces_from_inputs(img))
    s = engine.W2LSession(model, av, B, keep_layers=True)
    pred = s.infer(0, mel.numpy().reshape(B, 80, 16))
    want = ref.permute(0, 2, 3, 1).numpy() * 255.0
    psnr = R.psnr_u8(pred.astype(np.uint8), want.astype(np.uint8))
    assert psnr >= 40.0, psnr
    assert np.abs(pred - want).max() < 6.0
    s.close()
    av.close()


def test_forward_matches_reference_golden(model, golden_dir):
    """pred of the CUDA path vs the frame produced by the UNMODIFIED reference module (committed fixture)."""
    from livetalking_b200 import engine
    from oracle import wav2lip_ref as R
    g = np.load(os.path.join(golden_dir, "w2l_golden.npz"))
    mel, img = R.synth_inputs(1, seed=int(g["seed"][1]))
    av, _, _ = _avatar(_faces_from_inputs(img))
    s = engine.W2LSession(model, av, 1)
    pred = s.infer(0, mel.numpy().reshape(1, 80, 16))
    psnr = R.psnr_u8(pred.astype(np.uint8), g["pred_u8"])
    assert psnr >= 40.0, psnr
    np.testing.assert_allclose(pred[:, ::4, ::4, :], g["pred_f32_sub"], atol=6.0)
    s.close()
    av.close()


def test_pdl_graph_equals_plain_launches(model):
    """Programmatic dependent launch (conv kernels start before their predecessor ends, gated by griddepcontrol.wait) must
    not change a single value: PDL graph vs plain graph vs eager launches, replayed several times at B=16."""
    from livetalking_b200 import engine
    from oracle import wav2lip_ref as R
    mel, img = R.synth_inputs(2, seed=21)
    av, _, _ = _avatar(_faces_from_inputs(img))
    melB = np.tile(mel.numpy().reshape(2, 80, 16), (8, 1, 1))
    plain = engine.W2LSession(model, av, 16, no_pdl=True)
    want = plain.infer(3, melB)
    plain.close()
    pdl = engine.W2LSession(model, av, 16)
    for _ in range(4):
        got = pdl.infer(3, melB)
        assert np.array_equal(got, want)
    pdl.close()
    eager = engine.W2LSession(model, av, 16, no_graph=True)
    assert np.array_equal(eager.infer(3, melB), want)
    eager.close()
    av.close()


def test_full_batch16_properties(model, w2l_state_dict):
    """BASELINE config 2 size (B=16): determinism, batch-size independence, mirror_index face gather."""
    from livetalking_b200 import engine
    from oracle import wav2lip_ref as R
    from oracle.paste_ref import mirror_index
    mel, img = R.synth_inputs(3, seed=9)
    faces = _faces_from_inputs(img)
    av, _, _ = _avatar(faces)
    melB = np.tile(mel.numpy().reshape(3, 80, 16), (6, 1, 1))[:16]
    s16 = engine.W2LSession(model, av, 16)
    p1 = s16.infer(4, melB)
    p2 = s16.infer(4, melB)
    assert np.array_equal(p1, p2)                       # replay-stable: split-K partials go to per-split slices, summed in order
    s1 = engine.W2LSession(model, av, 1)
    for slot in (0, 5, 15):
        fidx = mirror_index(3, 4 + slot)
        # B=1 session: index chosen so that mirror_index(3, index) == fidx
        q = s1.infer(fidx, melB[slot:slot + 1])
        assert np.abs(q[0] - p1[slot]).max() <= 1.0 and R.psnr_u8(q[0].astype(np.uint8), p1[slot].astype(np.uint8)) >= 50.0, slot  # batch-size independent
    # and against the oracle for one slot
    slot = 7
    fidx = mirror_index(3, 4 + slot)
    want = R.wav2lip_forward(w2l_state_dict, torch.from_numpy(melB[slot:slot + 1]).reshape(1, 1, 80, 16),
                             img[fidx:fidx + 1]).permute(0, 2, 3, 1).numpy() * 255.0
    assert R.psnr_u8(p1[slot].astype(np.uint8), want[0].astype(np.uint8)) >= 40.0
    s16.close()
    s1.close()
    av.close()


def test_mel_matches_oracle_and_golden(model, golden_dir):
    from livetalking_b200 import engine
    from oracle import mel_ref as M
    faces = [np.zeros((256, 256, 3), np.uint8)]
    av, _, _ = _avatar(faces)
    g = np.load(os.path.join(golden_dir, "mel_golden.npz"))
    s = engine.W2LSession(model, av, 16)
    got = s.mel_step(g["pcm"])
    np.testing.assert_allclose(got, M.mel_step(g["pcm"], 16), atol=1e-5)
    np.testing.assert_allclose(got, g["windows"], atol=3e-5)
    # BASELINE synthetic audio: 0.5*sin(2 pi 440 t); silence; noise; batch 1 (36 frames -> tail clamp never hit)
    t = np.arange(16640) / 16000.0
    for pcm in (0.5 * np.sin(2 * np.pi * 440 * t), np.zeros_like(t), np.random.default_rng(3).standard_normal(t.size) * 0.2):
        pcm = pcm.astype(np.float32)
        np.testing.assert_allclose(s.mel_step(pcm), M.mel_step(pcm, 16), atol=1e-5)
    s.close()
    s1 = engine.W2LSession(model, av, 1)
    pcm = (np.random.default_rng(4).standard_normal(7040) * 0.1).astype(np.float32)
    np.testing.assert_allclose(s1.mel_step(pcm), M.mel_step(pcm, 1), atol=1e-5)
    with pytest.raises(engine.LtbError):
        s1.mel_step(pcm[:-1])                           # wrong buffer length is an error, not UB
    s1.close()
    av.close()


def test_paste_back_bit_exact(model, golden_dir):
    import make_golden as G
    from livetalking_b200 import engine
    from oracle import paste_ref as P
    g = np.load(os.path.join(golden_dir, "paste_golden.npz"))
    boxes = [tuple(int(v) for v in b) for b in g["boxes"]]
    n = len(boxes)
    faces = [np.zeros((256, 256, 3), np.uint8)] * n
    frames = np.stack([G.synth_frame(300, 300)] * n)
    av = engine.W2LAvatar(faces, frames, boxes)
    s = engine.W2LSession(model, av, 1)
    pred = s.infer(0, np.zeros((1, 80, 16), np.float32))[0]      # whatever the net predicts: float, fractional
    for idx, box in enumerate(boxes):
        got = s.paste(0, idx)
        want = P.w2l_paste_back(pred, frames[idx], box)
        assert np.array_equal(got, want), (idx, box, int(np.abs(got.astype(int) - want).max()))
    s.close()
    av.close()


def test_paste_vectorised_rows(model):
    """W % 16 == 0 takes the 128-bit row path (w2l_paste_vec_kernel): generic, 2x-decimation (INTER_AREA) and 1:1 boxes with
    unaligned edges, batch with mirror_index, bit-exact against the OpenCV restatement."""
    from livetalking_b200 import engine
    from oracle import paste_ref as P
    rng = np.random.default_rng(11)
    n, H, W = 4, 288, 320
    faces = [rng.integers(0, 256, (256, 256, 3), dtype=np.uint8) for _ in range(n)]
    frames = rng.integers(0, 256, (n, H, W, 3), dtype=np.uint8)
    boxes = [(3, 283, 5, 317), (7, 135, 33, 161), (16, 272, 37, 293), (100, 131, 15, 18)]   # generic, 128x128, 256x256, sliver
    av = engine.W2LAvatar(faces, frames, boxes)
    s = engine.W2LSession(model, av, 6)
    pred = s.infer(1, rng.standard_normal((6, 80, 16)).astype(np.float32))
    got = s.paste_batch(1)
    for i in range(6):
        idx = P.mirror_index(n, 1 + i)
        want = P.w2l_paste_back(pred[i], frames[idx], boxes[idx])
        assert np.array_equal(got[i], want), (i, idx, int(np.abs(got[i].astype(int) - want).max()))
    s.close()
    av.close()


def test_paste_batch_and_odd_width(model):
    from livetalking_b200 import engine
    from oracle import paste_ref as P
    rng = np.random.default_rng(5)
    n, H, W = 3, 123, 211                                         # W*3 not a multiple of 4
    faces = [rng.integers(0, 256, (256, 256, 3), dtype=np.uint8) for _ in range(n)]
    frames = rng.integers(0, 256, (n, H, W, 3), dtype=np.uint8)
    boxes = [(1, 101, 2, 209), (0, 123, 0, 211), (50, 60, 60, 75)]
    av = engine.W2LAvatar(faces, frames, boxes)
    s = engine.W2LSession(model, av, 4)
    pred = s.infer(2, rng.standard_normal((4, 80, 16)).astype(np.float32))
    got = s.paste_batch(2)
    for i in range(4):
        idx = P.mirror_index(n, 2 + i)
        assert np.array_equal(got[i], P.w2l_paste_back(pred[i], frames[idx], boxes[idx])), i
    with pytest.raises(engine.LtbError):
        s.paste(9, 0)
    with pytest.raises(engine.LtbError):
        s.paste(0, 99)
    s.close()
    av.close()
    with pytest.raises(engine.LtbError):
        engine.W2LAvatar(faces, frames, [(0, 500, 0, 10)] * 3)     # bbox outside the frame


def test_cross_session_slots_match_single_session(w2l_state_dict):
    """ltb_w2l_infer_slots (SURVEY §8 f1): slots carrying frames of DIFFERENT avatars in one launch.  (1) a batch whose slots
    are one avatar's consecutive frames is bit-identical to that avatar's own session; (2) in a mixed batch every slot is
    bit-identical to the same request in a homogeneous batch — slots do not influence each other."""
    from livetalking_b200 import engine
    from oracle import paste_ref as P
    engine.set_device(0)
    rng = np.random.default_rng(11)
    H, W, Bm = 96, 160, 8
    model = engine.W2LModel.from_state_dict(w2l_state_dict)
    avs = []
    for n in (5, 3):
        faces = rng.integers(0, 256, (n, 256, 256, 3), dtype=np.uint8)
        frames = rng.integers(0, 256, (n, H, W, 3), dtype=np.uint8)
        coords = [(4 + i, 84 + i, 10 + 3 * i, 110 + 3 * i) for i in range(n)]
        avs.append(engine.W2LAvatar(list(faces), frames, coords))
    mels = np.clip(rng.standard_normal((Bm, 80, 16)), -4, 4).astype(np.float32)
    own = engine.W2LSession(model, avs[0], Bm)
    mux = engine.W2LSession(model, avs[1], Bm, slots=True)          # its own avatar only fixes the frame size
    index = 3
    own.infer(index, mels, want_pred=False)
    want = own.paste_batch(index)
    got = mux.infer_slots([(avs[0], P.mirror_index(5, index + i), mels[i]) for i in range(Bm)])
    assert np.array_equal(got, want)
    mixed = [(avs[i % 2], (2 * i + 1) % avs[i % 2].n, mels[i]) for i in range(Bm)]
    got = mux.infer_slots(mixed)
    for i in (0, 1, 4, 7):
        solo = mux.infer_slots([mixed[i]] * Bm)
        assert np.array_equal(got[i], solo[i]), f"slot {i} was influenced by its neighbours"
    part = mux.infer_slots(mixed[:3])                               # partially filled batch
    assert part.shape == (3, H, W, 3) and np.array_equal(part, got[:3])
    with pytest.raises(Exception):
        own.infer_slots(mixed)                                      # not a slots session
    # a mel-only session extracts features but owns no network
    asr = engine.W2LSession(model, avs[0], 4, mel_only=True)
    pcm = (0.3 * rng.standard_normal((10 + 10 + 8) * 320)).astype(np.float32)
    from oracle import mel_ref
    np.testing.assert_allclose(asr.mel_step(pcm), mel_ref.mel_step(pcm, 4), atol=1e-5)
    with pytest.raises(Exception):
        asr.infer(0, np.zeros((4, 80, 16), np.float32))
    for o in (asr, mux, own, *avs, model):
        o.close()
