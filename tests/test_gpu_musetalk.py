"""GPU: the MuseTalk path (UNet + VAE decode / encode + blend paste-back, assembled from engine ops through the C ABI)
against the CPU fp32 oracle restatement.  NB oracle/musetalk_ref.py: the diffusers architecture is not in the reference
tree — parity here is against our restatement of the published layout ("parity unpinned")."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _avatar(ctx, lat, n, H=300, W=400, seed=0):
    from livetalking_b200.musetalk import MuseTalkAvatar
    rng = np.random.default_rng(seed)
    frames = rng.integers(0, 256, (n, H, W, 3), dtype=np.uint8)
    coords = [(120 + 3 * i, 60 + 2 * i, 120 + 3 * i + 150 + 7 * i, 60 + 2 * i + 170 + 5 * i) for i in range(n)]   # x1,y1,x2,y2
    crops, masks = [], []
    for (x1, y1, x2, y2) in coords:
        xs, ys, xe, ye = max(0, x1 - 40), max(0, y1 - 30), min(W, x2 + 40), min(H, y2 + 30)
        crops.append((xs, ys, xe, ye))
        mh, mw = ye - ys, xe - xs
        yy = np.linspace(0, 1, mh)[:, None] * np.ones((1, mw))
        soft = (np.clip((yy - 0.35) * 4, 0, 1) * 255).astype(np.uint8)
        masks.append(np.stack([soft, soft, soft], -1))
    return MuseTalkAvatar(ctx, frames, masks, coords, crops, [lat[i:i + 1] for i in range(n)]), frames, coords, crops, masks


def _cmp_taps(ctx, taps, otaps, tol_max=4e-2, tol_mean=1e-2):
    bad = []
    for k, ot in otaps.items():
        got = ctx.download(taps[k]).astype(np.float32)
        want = ot.permute(0, 2, 3, 1).numpy()
        assert got.shape == want.shape, (k, got.shape, want.shape)
        assert np.isfinite(got).all(), k
        rel = np.abs(got - want).max() / max(1e-6, np.abs(want).max())
        mrel = np.abs(got - want).mean() / max(1e-6, np.abs(want).mean())
        if rel > tol_max or mrel > tol_mean:
            bad.append(f"{k}:{rel:.4f}:{mrel:.5f}")
    assert not bad, "taps out of tolerance (name:max-rel:mean-rel): " + "; ".join(bad)


@pytest.fixture(scope="module")
def small_nets():
    from oracle import musetalk_ref as M
    return M.UNET_SMALL, M.VAE_SMALL, M.synth_unet_state_dict(M.UNET_SMALL), M.synth_vae_state_dict(M.VAE_SMALL)


def test_small_unet_vae_decode_parity_and_blend(small_nets):
    from livetalking_b200 import engine
    from livetalking_b200.musetalk import MuseTalkModel, MuseTalkSession
    from livetalking_b200.ops import Ctx
    from oracle import musetalk_ref as M
    from oracle import paste_ref as P
    from oracle.wav2lip_ref import psnr_u8
    ucfg, vcfg, us, vs = small_nets
    engine.set_device(0)
    B = 2
    lat, aud = M.synth_latents_and_audio(B, seed=4)
    otaps = {}
    pred = M.unet_forward(us, ucfg, lat, M.positional_encoding(aud), taps=otaps)
    vt = {}
    M.vae_decode(vs, vcfg, pred / vcfg.scaling_factor, taps=vt)
    otaps.update(vt)
    want_u8 = M.decode_latents_u8(vs, vcfg, pred)
    ctx = Ctx()
    model = MuseTalkModel(ctx, us, vs, ucfg, vcfg)
    av, frames, coords, crops, masks = _avatar(ctx, lat.numpy(), B)
    s = MuseTalkSession(model, av, B, keep_taps=True)
    got_u8 = s.infer(0, aud.numpy())
    _cmp_taps(ctx, s.taps, otaps)
    got_lat = ctx.download(s.pred16).astype(np.float32)[..., :4]
    np.testing.assert_allclose(got_lat, pred.permute(0, 2, 3, 1).numpy(), atol=6e-2)
    assert got_u8.shape == (B, 256, 256, 3) and got_u8.dtype == np.uint8
    assert psnr_u8(got_u8, want_u8) >= 40.0, psnr_u8(got_u8, want_u8)
    # replay determinism + mirror index gather (index 1 -> latents [1, 1 mirrored -> 0]... with n=2: idx 1, then 1 (turn 1: 2-0-1))
    again = s.infer(0, aud.numpy())           # graph replay; GroupNorm statistics use float atomics -> last-bit jitter only
    assert np.abs(again.astype(int) - got_u8.astype(int)).max() <= 2 and psnr_u8(again, got_u8) >= 55.0
    # paste-back: bit-exact blend of the engine's own (latest) prediction
    got_u8 = again
    for slot in range(B):
        idx = P.mirror_index(B, slot)
        got = s.paste(slot, idx)
        want = P.mt_paste_back(got_u8[slot], frames[idx], coords[idx], masks[idx], crops[idx])
        assert np.array_equal(got, want), (slot, int(np.abs(got.astype(int) - want).max()))
    allf = s.paste_batch(0)
    for slot in range(B):
        idx = P.mirror_index(B, slot)
        assert np.array_equal(allf[slot], P.mt_paste_back(got_u8[slot], frames[idx], coords[idx], masks[idx], crops[idx]))
    host_pred = np.random.default_rng(1).integers(0, 256, (256, 256, 3), dtype=np.uint8)
    assert np.array_equal(s.paste_pred(host_pred, 1), P.mt_paste_back(host_pred, frames[1], coords[1], masks[1], crops[1]))
    ctx.close()


def test_small_nets_at_64x64_latents_512_images(small_nets):
    """BASELINE configs[4]: 512x512 crops = 64x64 latents (the reference hard-wires 256, avatars/musetalk/models/vae.py:15; the
    engine is parametrised on the avatar's latent size).  UNet + VAE decode parity, then the blend paste-back of a 512x512
    prediction (resize source side 512) against the oracle."""
    from livetalking_b200 import engine
    from livetalking_b200.musetalk import MuseTalkModel, MuseTalkSession
    from livetalking_b200.ops import Ctx
    from oracle import musetalk_ref as M
    from oracle import paste_ref as P
    from oracle.wav2lip_ref import psnr_u8
    ucfg, vcfg, us, vs = small_nets
    engine.set_device(0)
    B = 2
    lat, aud = M.synth_latents_and_audio(B, hw=64, seed=12)
    with torch.no_grad():
        pred = M.unet_forward(us, ucfg, lat, M.positional_encoding(aud))
        want_u8 = M.decode_latents_u8(vs, vcfg, pred)
    assert want_u8.shape == (B, 512, 512, 3)
    ctx = Ctx()
    model = MuseTalkModel(ctx, us, vs, ucfg, vcfg, with_encoder=False)
    av, frames, coords, crops, masks = _avatar(ctx, lat.numpy(), B, H=700, W=900)
    assert av.lat_hw == 64
    s = MuseTalkSession(model, av, B)
    got_u8 = s.infer(0, aud.numpy())
    assert got_u8.shape == (B, 512, 512, 3)
    got_lat = ctx.download(s.pred16).astype(np.float32)[..., :4]
    np.testing.assert_allclose(got_lat, pred.permute(0, 2, 3, 1).numpy(), atol=6e-2)
    assert psnr_u8(got_u8, want_u8) >= 40.0, psnr_u8(got_u8, want_u8)
    allf = s.paste_batch(0)
    for slot in range(B):
        idx = P.mirror_index(B, slot)
        assert np.array_equal(allf[slot], P.mt_paste_back(got_u8[slot], frames[idx], coords[idx], masks[idx], crops[idx]))
    host_pred = np.random.default_rng(3).integers(0, 256, (512, 512, 3), dtype=np.uint8)
    assert np.array_equal(s.paste_pred(host_pred, 1), P.mt_paste_back(host_pred, frames[1], coords[1], masks[1], crops[1]))
    s.close()
    ctx.close()


def test_small_vae_encode_parity(small_nets):
    from livetalking_b200 import engine
    from livetalking_b200.musetalk import MuseTalkModel, encode_avatar_latents
    from livetalking_b200.ops import Ctx
    from oracle import musetalk_ref as M
    ucfg, vcfg, us, vs = small_nets
    engine.set_device(0)
    rng = np.random.default_rng(2)
    low = rng.integers(0, 256, (2, 32, 32, 3)).astype(np.float32)
    imgs = np.clip(np.kron(low, np.ones((1, 8, 8, 1), np.float32)) + rng.integers(-6, 7, (2, 256, 256, 3)), 0, 255).astype(np.uint8)
    ctx = Ctx()
    model = MuseTalkModel(ctx, us, vs, ucfg, vcfg)
    got = encode_avatar_latents(model, imgs).astype(np.float32)
    want = np.concatenate([M.latents_for_unet(vs, vcfg, imgs[i]).numpy() for i in range(2)], 0)
    assert got.shape == want.shape == (2, 8, 32, 32)
    err = np.abs(got - want)
    assert err.max() <= 0.02 + 0.04 * np.abs(want).max(), (err.max(), np.abs(want).max())
    assert err.mean() <= 0.01 * max(1e-3, np.abs(want).mean()) + 2e-3
    ctx.close()


@pytest.mark.parametrize("B", [1, 8], ids=["B1", "B8_configs2"])
def test_full_width_networks(B):
    """The real MuseTalk widths (UNet 320/640/1280/1280 with head_dim 40 -> padded 48, sd-vae 128/256/512/512) at B = 1 and at
    BASELINE configs[2]'s batch 8 (different tile / split-K / wave configurations than B = 1)."""
    from livetalking_b200 import engine
    from livetalking_b200.musetalk import MuseTalkModel, MuseTalkSession
    from livetalking_b200.ops import Ctx
    from oracle import musetalk_ref as M
    from oracle.wav2lip_ref import psnr_u8
    engine.set_device(0)
    us = M.synth_unet_state_dict(M.UNET_FULL, fast=True)
    vs = M.synth_vae_state_dict(M.VAE_FULL, fast=True)
    assert M.count_params(us) == 849_947_844 and M.count_params(vs) == 83_653_863     # published parameter counts
    lat, aud = M.synth_latents_and_audio(B, seed=9)
    with torch.no_grad():
        pred = M.unet_forward(us, M.UNET_FULL, lat, M.positional_encoding(aud))
        want_u8 = M.decode_latents_u8(vs, M.VAE_FULL, pred)
    ctx = Ctx()
    model = MuseTalkModel(ctx, us, vs, M.UNET_FULL, M.VAE_FULL, with_encoder=False)
    av, *_ = _avatar(ctx, lat.numpy(), B)
    s = MuseTalkSession(model, av, B)
    got_u8 = s.infer(0, aud.numpy())
    assert got_u8.shape == (B, 256, 256, 3)
    got_lat = ctx.download(s.pred16).astype(np.float32)[..., :4]
    want_lat = pred.permute(0, 2, 3, 1).numpy()
    assert np.abs(got_lat - want_lat).max() <= 0.08 * max(1.0, np.abs(want_lat).max())
    assert psnr_u8(got_u8, want_u8) >= 40.0, psnr_u8(got_u8, want_u8)
    ctx.close()


def test_fused_groupnorm_statistics_path(small_nets):
    """ltb_conv_op.gn_stats: statistics accumulated by the conv epilogue (or its fallback pass) must give the same network
    output as the separate statistics kernel."""
    from livetalking_b200 import engine
    from livetalking_b200 import musetalk as MT
    from livetalking_b200.ops import Ctx
    from oracle import musetalk_ref as M
    from oracle.wav2lip_ref import psnr_u8
    ucfg, vcfg, us, vs = small_nets
    engine.set_device(0)
    lat, aud = M.synth_latents_and_audio(1, seed=6)
    outs = []
    for fuse in (False, True):
        MT.Builder.FUSE_GN_STATS = fuse
        try:
            ctx = Ctx()
            model = MT.MuseTalkModel(ctx, us, vs, ucfg, vcfg, with_encoder=False)
            av, *_ = _avatar(ctx, lat.numpy(), 1)
            s = MT.MuseTalkSession(model, av, 1)
            outs.append(s.infer(0, aud.numpy()))
            ctx.close()
        finally:
            MT.Builder.FUSE_GN_STATS = False
    assert psnr_u8(outs[0], outs[1]) >= 48.0
    want = M.decode_latents_u8(vs, vcfg, M.unet_forward(us, ucfg, lat, M.positional_encoding(aud)))
    assert psnr_u8(outs[1], want) >= 40.0


@pytest.mark.parametrize("shape", [(2, 12, 10, 64, 64), (1, 32, 32, 128, 128), (3, 8, 8, 320, 192)], ids=["ragged", "2tiles_n", "5chunks"])
def test_fused_upsample_conv_matches_interpolate_plus_conv(shape):
    """Upsample2D (F.interpolate nearest 2x + conv3x3 p1) as four sub-pixel 2x2 convs over the low-res map (ops.ConvWeight.upconv,
    conv_halo.cu TAPS = 16) against plain PyTorch fp32 of the same op.  Tolerance: fp16 in/out, fp32 accumulate, and the pre-summed
    taps are rounded to fp16 once (|err| <= 3e-2 + 1.5e-2 |ref|)."""
    import torch.nn.functional as F
    from livetalking_b200 import engine
    from livetalking_b200.ops import ConvWeight, Ctx
    engine.set_device(0)
    N, H, W, cin, cout = shape
    g = torch.Generator().manual_seed(sum(shape))
    x = (torch.randn(N, cin, H, W, generator=g) * 0.7).half()
    w = torch.randn(cout, cin, 3, 3, generator=g) * (2.0 / (cin * 9)) ** 0.5
    b = torch.randn(cout, generator=g) * 0.2
    ref = F.conv2d(F.interpolate(x.float(), scale_factor=2.0, mode="nearest"), w.half().float(), b, padding=1)
    ref = ref.permute(0, 2, 3, 1).contiguous().numpy()
    ctx = Ctx()
    cw = ConvWeight(ctx, w.numpy(), b.numpy())
    assert cw.upconv_supported()
    dx = ctx.upload(x.permute(0, 2, 3, 1).contiguous().numpy())
    out = ctx.alloc((N, 2 * H, 2 * W, cout), np.float16, zero=True)
    ctx.conv(dx, cw, out, N=N, IH=H, IW=W, OH=2 * H, OW=2 * W, pad=(1, 1), upsample2x=True)
    got = ctx.download(out).astype(np.float32)
    err = np.abs(got - ref)
    assert (err <= 3e-2 + 1.5e-2 * np.abs(ref)).all(), f"max err {err.max():.4f} at {np.unravel_index(err.argmax(), err.shape)}"
    assert err.mean() < 3e-3
    ctx.close()


@pytest.mark.parametrize("shape", [
    # B, H, d, nq, kv_rows, valid, self-attention layout (fused qkv buffer) or separate q / kv buffers
    (2, 8, 48, 1024, 1024, 1024, True),     # UNet 32x32 self-attention (d 40 padded to 48): 8 key tiles, 2 passes
    (1, 6, 64, 1500, 1500, 1500, True),     # Whisper-tiny encoder: ragged last query tile and key tile (1500 = 11*128 + 92)
    (3, 8, 80, 256, 64, 50, False),         # UNet cross-attention: 50 valid audio tokens of 64 rows, two K chunks
    (2, 8, 160, 64, 64, 64, True),          # 8x8 level: three K chunks, single-stage K ring
    (1, 8, 160, 16, 16, 16, True),          # mid block at 4x4: 16 queries, 16 keys
    (1, 2, 16, 130, 200, 137, False),       # smallest head dim; nothing aligned
], ids=["self1024_d48", "whisper1500_d64", "cross50_d80", "self64_d160", "mid16_d160", "ragged_d16"])
def test_fused_attention_matches_torch(shape):
    """softmax(scale QK^T)V as ONE wgmma kernel (csrc/attn_fused.cu) against plain PyTorch fp32 on the same fp16 inputs.
    Tolerance: probabilities are rounded to fp16 before the PV product (like the unfused path stored them), fp32 accumulate, fp16 out:
    |err| <= 4e-3 + 1e-2 |ref|."""
    from livetalking_b200 import engine
    from livetalking_b200.ops import Ctx, DevTensor
    engine.set_device(0)
    B, H, d, nq, kv_rows, valid, fused_qkv = shape
    g = torch.Generator().manual_seed(sum(shape[:6]))
    Hd = H * d
    scale = float(d) ** -0.5
    if fused_qkv:
        assert kv_rows == nq
        qkv = (torch.randn(B, nq, 3 * Hd, generator=g) * 1.5).half()
        q, k, v = qkv[..., :Hd], qkv[..., Hd:2 * Hd], qkv[..., 2 * Hd:]
    else:
        q = (torch.randn(B, nq, Hd, generator=g) * 1.5).half()
        kv = (torch.randn(B, kv_rows, 2 * Hd, generator=g) * 1.5).half()
        k, v = kv[..., :Hd], kv[..., Hd:]
    qh = q.float().view(B, nq, H, d).permute(0, 2, 1, 3)
    kh = k.float().view(B, kv_rows, H, d).permute(0, 2, 1, 3)[:, :, :valid]
    vh = v.float().view(B, kv_rows, H, d).permute(0, 2, 1, 3)[:, :, :valid]
    ref = torch.softmax(qh @ kh.transpose(-1, -2) * scale, -1) @ vh                     # B,H,nq,d
    ref = ref.permute(0, 2, 1, 3).reshape(B * nq, Hd).numpy()
    ctx = Ctx()
    n_pad = (kv_rows + 15) // 16 * 16
    if fused_qkv:
        dq = ctx.upload(qkv.contiguous().numpy())
        q_ptr, q_pitch, k_ptr, v_ptr, kv_pitch = dq.ptr, 3 * Hd, dq.ptr + 2 * Hd, dq.ptr + 4 * Hd, 3 * Hd
    else:
        dq, dkv = ctx.upload(q.contiguous().numpy()), ctx.upload(kv.contiguous().numpy())
        q_ptr, q_pitch, k_ptr, v_ptr, kv_pitch = dq.ptr, Hd, dkv.ptr, dkv.ptr + 2 * Hd, 2 * Hd
    vt = ctx.alloc((B * H, d, n_pad), np.float16, zero=True)
    ctx.transpose_heads(v_ptr, B, kv_rows, kv_pitch, H, d, n_pad, vt)
    out = ctx.alloc((B * nq, Hd), np.float16, zero=True)
    ctx.attention(q_ptr, q_pitch, k_ptr, kv_pitch, kv_rows, vt, n_pad, B, H, nq, valid, d, scale, out)
    got = ctx.download(out).astype(np.float32)
    err = np.abs(got - ref)
    assert np.isfinite(got).all()
    assert (err <= 4e-3 + 1e-2 * np.abs(ref)).all(), f"max err {err.max():.5f} at {np.unravel_index(err.argmax(), err.shape)}"
    ctx.close()


def test_cross_session_batch_matches_per_session(small_nets):
    """MuseTalkBatchSession (G sessions x Bs frames in ONE graph of batch G*Bs, per-group avatar + frame index) against the same
    sessions run one by one through MuseTalkSession: network output within the tile-configuration jitter (the batched launch may
    pick other tile shapes: fp32 accumulation order differs; <= 2 u8 steps, PSNR >= 50 dB) and each group's paste-back BIT-EXACT
    against the blend oracle applied to the batch's own prediction with that group's avatar assets."""
    from livetalking_b200 import engine
    from livetalking_b200.musetalk import MuseTalkBatchSession, MuseTalkModel, MuseTalkSession
    from livetalking_b200.ops import Ctx
    from oracle import musetalk_ref as M
    from oracle import paste_ref as P
    from oracle.wav2lip_ref import psnr_u8
    ucfg, vcfg, us, vs = small_nets
    engine.set_device(0)
    G, Bs, n = 3, 2, 5
    ctx = Ctx()
    model = MuseTalkModel(ctx, us, vs, ucfg, vcfg)
    avs, assets = [], []
    for g in range(G):
        lat, _ = M.synth_latents_and_audio(n, seed=10 + g)
        av, frames, coords, crops, masks = _avatar(ctx, lat.numpy(), n, H=300 + 20 * g, W=400 - 16 * g, seed=g)
        avs.append(av)
        assets.append((frames, coords, crops, masks))
    _, aud = M.synth_latents_and_audio(G * Bs, seed=77)
    aud = aud.numpy()
    indices = [3, 0, 7]                                     # 7 > n: mirror-indexed like the reference (basereal mirror_index)
    bs = MuseTalkBatchSession(model, 32, G, Bs)
    reqs = [(avs[g], indices[g], aud[g * Bs:(g + 1) * Bs]) for g in range(G)]
    outs = bs.step(reqs)
    pred_b = bs.ctx.download(bs.image_u8)
    for g in range(G):
        s = MuseTalkSession(model, avs[g], Bs)
        pred_s = s.infer(indices[g], aud[g * Bs:(g + 1) * Bs])
        got = pred_b[g * Bs:(g + 1) * Bs]
        assert np.abs(got.astype(int) - pred_s.astype(int)).max() <= 2 and psnr_u8(got, pred_s) >= 50.0, (g, psnr_u8(got, pred_s))
        frames, coords, crops, masks = assets[g]
        assert outs[g].shape == (Bs, frames.shape[1], frames.shape[2], 3)
        for i in range(Bs):
            idx = P.mirror_index(n, indices[g] + i)
            want = P.mt_paste_back(got[i], frames[idx], coords[idx], masks[idx], crops[idx])
            assert np.array_equal(outs[g][i], want), (g, i)
        s.close()
    again = bs.step([(avs[g], indices[g], None) for g in range(G)])           # features resident: replay
    for g in range(G):
        assert np.abs(again[g].astype(int) - outs[g].astype(int)).max() <= 2
    # a partial round with the sessions in other groups: any session may occupy any group
    preds = bs.infer_groups([reqs[2], reqs[0]])
    assert len(preds) == 2 and preds[0].shape == (Bs, 256, 256, 3)
    assert np.abs(preds[0].astype(int) - pred_b[2 * Bs:3 * Bs].astype(int)).max() <= 2
    assert np.abs(preds[1].astype(int) - pred_b[0:Bs].astype(int)).max() <= 2
    bs.close()
    ctx.close()
