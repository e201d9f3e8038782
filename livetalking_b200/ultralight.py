"""UltraLight avatar path on the B200 engine (SURVEY §8 row f4) — replaces the per-avatar U-Net of
avatars/ultralight/unet.py (``Model(6, 'hubert')``) and the glue of ``LightReal.inference_batch`` / ``paste_back_frame``
(avatars/ultralight_avatar.py:141-184).

The network is MobileNet-style: every InvertedResidual is 1x1 conv -> depthwise 3x3 -> 1x1 conv with BatchNorm after each
(unet.py:7-37).  BatchNorm (eval) is folded into the preceding convolution at load time; the 1x1 convs (97 % of the FLOPs) and the
two dense stride-2 3x3 convs of the audio branch run on the tcgen05 implicit-GEMM kernels, the depthwise convs / bilinear
upsampling / input glue / paste-back on the HBM-bound kernels of csrc/ultralight.cu.  ``torch.cat`` never copies: producers write
straight into channel slices of the concat buffers.  One CUDA graph per (session, batch size).

Cross-session batching (``UltraLightBatchSession``): the network belongs to the avatar, so a batch of several sessions runs every
layer as a *grouped* op — the weights of up to S avatars are stacked slot by slot in an ``UltraLightBank`` and image n of the
batch reads slot ``group_slot[n // Bs]`` from a device table, so one captured graph serves any assignment of avatars to groups.
``UltraLightSession`` is its one-group form bound to one avatar: no bank, the avatar's own network on the ungrouped ops."""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import numpy as np

from .graph import Builder, GraphSession, _ceil16, _np
from .ops import ConvWeight, Ctx, DevTensor, ul_prep_table

CH = [32, 64, 128, 256, 512]          # unet.py:188
FACE, CROP, INSET = 160, 168, 4       # network input side, stored crop side, crop[4:164] (ultralight_avatar.py:148)
BN_EPS = 1e-5


def _fold(sd, conv_w: np.ndarray, conv_b: Optional[np.ndarray], bn: str):
    """conv (+bias) followed by eval BatchNorm -> (w', b'):  y = (conv(x) + b - mean) * gamma / sqrt(var + eps) + beta."""
    g, beta, mean, var = (_np(sd[f"{bn}.{k}"]) for k in ("weight", "bias", "running_mean", "running_var"))
    s = g / np.sqrt(var + BN_EPS)
    b = beta - mean * s if conv_b is None else beta + (conv_b - mean) * s
    return conv_w * s.reshape(-1, *([1] * (conv_w.ndim - 1))), b.astype(np.float32)


class _IR:
    """One InvertedResidual (unet.py:7-37) with folded BatchNorms, channel counts padded to multiples of 16."""

    def __init__(self, ctx: Ctx, sd, p: str, inp: int, oup: int, stride: int, res: bool, expand: int = 2):
        hid = inp * expand
        self.inp_p, self.hid_p, self.oup, self.stride, self.res = _ceil16(inp), _ceil16(hid), oup, stride, res
        assert oup % 16 == 0
        w1, b1 = _fold(sd, _np(sd[p + ".conv.0.weight"]), None, p + ".conv.1")
        self.pw1 = ConvWeight(ctx, w1, b1, pad_cin=self.inp_p, pad_cout=self.hid_p, tap_major=False)
        wd, bd = _fold(sd, _np(sd[p + ".conv.3.weight"]), None, p + ".conv.4")              # (hid, 1, 3, 3)
        wt = np.zeros((9, self.hid_p), np.float16)
        wt[:, :hid] = wd.reshape(hid, 9).T
        bt = np.zeros(self.hid_p, np.float32)
        bt[:hid] = bd
        self.dw_w, self.dw_b = ctx.upload(wt), ctx.upload(bt)
        w2, b2 = _fold(sd, _np(sd[p + ".conv.6.weight"]), None, p + ".conv.7")
        self.pw2 = ConvWeight(ctx, w2, b2, pad_cin=self.hid_p, tap_major=False)


class UltraLightModel:
    """Device-resident ``Model(6, 'hubert')`` built from its state_dict (``ultralight.pth``, ultralight_avatar.py:69-70)."""

    def __init__(self, ctx: Ctx, sd: Dict):
        self.ctx = ctx
        ir = lambda p, i, o, s=1, r=False: _IR(ctx, sd, p, i, o, s, r)  # noqa: E731
        dc = lambda p, i, o, s: [ir(p + ".double_conv.0", i, o, s), ir(p + ".double_conv.1", o, o, 1, True)]  # noqa: E731  (DoubleConvDW)
        a = "audio_model"
        self.a1, self.a2 = ir(a + ".conv1", 16, CH[1]), ir(a + ".conv2", CH[1], CH[2])
        self.a3 = ConvWeight(ctx, *_fold(sd, _np(sd[a + ".conv3.weight"]), _np(sd[a + ".conv3.bias"]), a + ".bn3"))
        self.a4 = ir(a + ".conv4", CH[3], CH[3], 1, True)
        self.a5 = ConvWeight(ctx, *_fold(sd, _np(sd[a + ".conv5.weight"]), _np(sd[a + ".conv5.bias"]), a + ".bn5"), tap_major=False)
        self.a6, self.a7 = ir(a + ".conv6", CH[4], CH[4], 1, True), ir(a + ".conv7", CH[4], CH[4], 1, True)
        self.fuse = dc("fuse_conv.0", CH[4] * 2, CH[4], 1) + dc("fuse_conv.1", CH[4], CH[3], 1)
        self.inc = ir("inc.inconv.0", 6, CH[0])
        self.down = [dc(f"down{i + 1}.maxpool_conv.0", CH[i], CH[i + 1], 2) for i in range(4)]
        self.up = [dc(f"up{i + 1}.conv", c_in, c_out, 1)
                   for i, (c_in, c_out) in enumerate(((CH[4], CH[3] // 2), (CH[3], CH[2] // 2), (CH[2], CH[1] // 2), (CH[1], CH[0])))]
        self.head_w = ctx.upload(_np(sd["outc.conv.weight"]).reshape(3, CH[0]).astype(np.float32))
        self.head_b = ctx.upload(_np(sd["outc.conv.bias"]).astype(np.float32))
        ctx.sync()

    def blocks(self) -> List[_IR]:
        return [self.a1, self.a2, self.a4, self.a6, self.a7, *self.fuse, self.inc, *(k for d in self.down for k in d),
                *(k for u in self.up for k in u)]

    def weight_tensors(self) -> List[DevTensor]:
        """Every device weight tensor the forward reads, in a fixed order (the slot layout of UltraLightBank)."""
        ts = []
        for blk in self.blocks():
            ts += [blk.pw1.w, blk.pw1.bias, blk.dw_w, blk.dw_b, blk.pw2.w, blk.pw2.bias]
        return ts + [self.a3.w, self.a3.bias, self.a5.w, self.a5.bias, self.head_w, self.head_b]

    # ---- emitters (ops go to the builder's ctx = the session's stream; weights are read-only)
    @staticmethod
    def _ir(b: Builder, blk: _IR, x: DevTensor, out: Optional[DevTensor] = None, grp: Optional["_Grouping"] = None) -> DevTensor:
        ctx = b.ctx
        N, H, W, _ = x.shape
        rows = N * H * W
        h1 = b.new(N, H, W, blk.hid_p)
        OH, OW = (H - 1) // blk.stride + 1, (W - 1) // blk.stride + 1
        h2 = b.new(N, OH, OW, blk.hid_p)
        if out is None:
            out = b.new(N, OH, OW, blk.oup)
        orow = N * OH * OW
        res = x if blk.res else None
        if grp is None:
            ctx.conv(x, blk.pw1, h1, N=1, IH=1, IW=rows, OH=1, OW=rows, relu=True)
            ctx.dwconv3x3(h1, N, H, W, blk.dw_w, blk.dw_b, blk.stride, True, h2)
            ctx.conv(h2, blk.pw2, out, N=1, IH=1, IW=orow, OH=1, OW=orow, res=res)
        else:   # grouped: N = images, so that image n maps to group n // Bs
            ctx.conv(x, blk.pw1, h1, N=N, IH=H, IW=W, OH=H, OW=W, relu=True, **grp.conv(blk.pw1))
            ctx.dwconv3x3(h1, N, H, W, *grp.dw(blk.dw_w, blk.dw_b), blk.stride, True, h2, group=grp.dw_group(blk.dw_w, blk.dw_b))
            ctx.conv(h2, blk.pw2, out, N=N, IH=OH, IW=OW, OH=OH, OW=OW, res=res, **grp.conv(blk.pw2))
        return out

    def _dc(self, b: Builder, blks: List[_IR], x: DevTensor, out: Optional[DevTensor] = None, grp: Optional["_Grouping"] = None) -> DevTensor:
        for i, blk in enumerate(blks):
            x = self._ir(b, blk, x, out if i == len(blks) - 1 else None, grp)
        return x

    def emit(self, b: Builder, img16: DevTensor, audio16: DevTensor, pred: DevTensor, taps: Optional[dict] = None,
             grp: Optional["_Grouping"] = None):
        """img16 (B,160,160,16) fp16 NHWC (6 real channels), audio16 (B,32,32,16) -> pred f32 (B,160,160,3) = sigmoid x 255.
        Model.forward, unet.py:208-226.  grp: grouped form — every op reads the weights of its image's bank slot (this model only
        supplies the shapes)."""
        ctx = b.ctx
        g_conv = (lambda cw: grp.conv(cw)) if grp is not None else (lambda cw: {})   # noqa: E731
        B = img16.shape[0]
        view = lambda buf, c0, c: DevTensor(buf.ptr, buf.shape[:3] + (c,), pitch=buf.shape[3], c_off=c0)  # noqa: E731
        # concat buffers: [upsampled | skip] (torch.cat([x1, x2]), unet.py:88) and [x5 | audio] (unet.py:217)
        cat = [b.new(B, FACE >> i, FACE >> i, 2 * CH[i]) for i in range(4)]                  # up4..up1 inputs at 160, 80, 40, 20
        cat5 = b.new(B, 10, 10, 2 * CH[4])
        skips = [view(cat[i], CH[i], CH[i]) for i in range(4)]                              # x1..x4 live in the second half
        x = self._ir(b, self.inc, img16, skips[0], grp)
        for i in range(3):
            x = self._dc(b, self.down[i], x, skips[i + 1], grp)
        x5 = self._dc(b, self.down[3], x, view(cat5, 0, CH[4]), grp)
        # audio branch, AudioConvHubert.forward (unet.py:164-181)
        a = self._ir(b, self.a2, self._ir(b, self.a1, audio16, None, grp), None, grp)
        a3 = b.new(B, 16, 16, CH[3])
        ctx.conv(a, self.a3, a3, N=B, IH=32, IW=32, OH=16, OW=16, stride=(2, 2), pad=(1, 1), relu=True, **g_conv(self.a3))
        a4 = self._ir(b, self.a4, a3, None, grp)
        a5 = b.new(B, 10, 10, CH[4])
        ctx.conv(a4, self.a5, a5, N=B, IH=16, IW=16, OH=10, OW=10, stride=(2, 2), pad=(3, 3), relu=True, **g_conv(self.a5))
        af = self._ir(b, self.a7, self._ir(b, self.a6, a5, None, grp), view(cat5, CH[4], CH[4]), grp)
        f = self._dc(b, self.fuse, cat5, None, grp)
        if taps is not None:
            taps.update(x5=x5, audio=af, fuse=f)
        # Up.forward x 4 (unet.py:81-90): sizes are exact doubles, so the F.pad is a no-op
        for i in range(4):
            lvl = 3 - i
            H = FACE >> (lvl + 1)
            ctx.upsample_bilinear2x(f, B, H, H, view(cat[lvl], 0, CH[lvl]))
            f = self._dc(b, self.up[i], cat[lvl], None, grp)
            if taps is not None:
                taps[f"u{i + 1}"] = f
        if grp is None:
            ctx.head_sigmoid255(f, self.head_w, self.head_b, B * FACE * FACE, pred)
        else:
            ctx.head_sigmoid255(f, *grp.dw(self.head_w, self.head_b), B * FACE * FACE, pred, group=grp.dw_group(self.head_w, self.head_b),
                                hw=FACE * FACE)
        return pred


class UltraLightAvatar:
    """Avatar assets resident in HBM (replaces load_avatar's lists, ultralight_avatar.py:63-82): full frames, 168x168 face crops,
    bbox (x1,y1,x2,y2) — and, as in the reference, the avatar's OWN network (``ultralight.pth`` lives in the avatar directory)."""

    def __init__(self, ctx: Ctx, model: UltraLightModel, frames, faces, coords):
        frames = np.ascontiguousarray(np.asarray(frames), np.uint8)
        faces = np.ascontiguousarray(np.asarray(faces), np.uint8)
        self.n, self.H, self.W = frames.shape[0], frames.shape[1], frames.shape[2]
        if faces.shape != (self.n, CROP, CROP, 3):
            raise ValueError(f"UltraLight face crops must be ({self.n},{CROP},{CROP},3) uint8, got {faces.shape}")
        self.coords_host = np.ascontiguousarray(np.asarray(coords), np.int32).reshape(self.n, 4)
        for x1, y1, x2, y2 in self.coords_host:
            if not (0 <= x1 < x2 <= self.W and 0 <= y1 < y2 <= self.H):
                raise ValueError("avatar bbox outside the frame")
        self.ctx, self.model = ctx, model
        self.frames, self.faces, self.coords = ctx.upload(frames), ctx.upload(faces), ctx.upload(self.coords_host)


class UltraLightBank:
    """The weights of up to ``slots`` UltraLight networks, stacked slot by slot: one device buffer (slots, *shape) per weight tensor
    of ``UltraLightModel.weight_tensors()``.  ``slot_of(model)`` loads a network on a miss (stream-ordered device-to-device copies from
    its resident weights) into a free slot or the least recently used one.  Used by one dispatcher thread only: no lock.
    alloc(shape, dtype, zero=...): where the stacked buffers come from (ctx.alloc unless given; the batch session passes its own)."""

    def __init__(self, ctx: Ctx, template: UltraLightModel, slots: int, alloc=None):
        self.ctx, self.slots = ctx, int(slots)
        if self.slots < 1:
            raise ValueError("UltraLightBank needs at least one slot")
        ts = template.weight_tensors()
        self._layout = [(t.shape, t.dtype) for t in ts]
        self._index = {id(t): i for i, t in enumerate(ts)}
        self._bufs = [(alloc or ctx.alloc)((self.slots,) + t.shape, t.dtype, zero=True) for t in ts]
        self.nbytes = sum(b.nbytes for b in self._bufs)
        self._model: List[Optional[UltraLightModel]] = [None] * self.slots
        self._used = [0] * self.slots                   # tick of the last slot_of() that returned the slot; 0 = never
        self._tick = 0
        self.loads = 0

    def stacked(self, t: DevTensor) -> DevTensor:
        """The bank buffer (slots, *t.shape) of the template tensor t."""
        return self._bufs[self._index[id(t)]]

    def slot_of(self, model: UltraLightModel, keep: Sequence[int] = ()) -> int:
        """Slot holding `model`'s weights; on a miss the network is loaded into an empty slot or, failing that, the least recently
        used slot not listed in `keep` (the slots the current batch already uses)."""
        self._tick += 1
        for s, m in enumerate(self._model):
            if m is model:
                self._used[s] = self._tick
                return s
        free = [s for s in range(self.slots) if s not in keep]
        if not free:
            raise RuntimeError(f"UltraLightBank: all {self.slots} slots are in use by this batch")
        s = min(free, key=lambda k: self._used[k])
        ts = model.weight_tensors()
        if [(t.shape, t.dtype) for t in ts] != self._layout:
            raise ValueError("UltraLightBank: the network's weight shapes differ from the bank's")
        for t, buf in zip(ts, self._bufs):
            self.ctx.d2d(buf.ptr + s * t.nbytes, t.ptr, t.nbytes)
        self._model[s], self._used[s] = model, self._tick
        self.loads += 1
        return s


class _Grouping:
    """Arguments of the grouped ops: weights from `bank`, image n uses slot table[n // images]."""

    def __init__(self, bank: UltraLightBank, table: DevTensor, images: int):
        self.bank, self.table, self.images = bank, table, int(images)

    def conv(self, cw: ConvWeight) -> dict:
        w, b = self.bank.stacked(cw.w), self.bank.stacked(cw.bias)
        return dict(w_ptr=w.ptr, bias_ptr=b.ptr, group=(self.table, self.images, self.bank.slots, cw.cout * cw.ktot, cw.cout))

    def dw(self, w: DevTensor, b: DevTensor):
        return self.bank.stacked(w), self.bank.stacked(b)

    def dw_group(self, w: DevTensor, b: DevTensor) -> tuple:
        return (self.table, self.images, int(np.prod(w.shape)), int(np.prod(b.shape)))


class UltraLightBatchSession(GraphSession):
    """Cross-session batching for UltraLight: up to G sessions x Bs frames run as ONE captured prep + U-Net + head graph of batch
    G*Bs.  A *group request* is (UltraLightAvatar, first frame index, HuBERT features (Bs, 16, 1024) or None = resident).  Each
    avatar brings its own network: the graph's ops are grouped, group g reads the weights of bank slot group_slot[g] and its crops
    from its own avatar (a per-group prep descriptor), both device tables written before every launch.  Groups beyond the
    requests of a call keep their last slot and a blank crop source; their output is discarded.  `batch` / `infer_slots` make it a
    mux for plugin.batcher.CrossSessionBatcher; infer_groups returns composited frames, or float32 predictions with return_pred.

    avatar: bind the session to this one avatar (groups = 1).  There is no bank then: the graph runs the avatar's own network on
    the ungrouped ops, its crops indexed by the d_index scalar, and its output frames are allocated here.
    keep_taps: `taps` holds intermediate activations of the U-Net (else None)."""

    def __init__(self, template: UltraLightModel, groups: int, frames_per_session: int, slots: Optional[int] = None,
                 return_pred: bool = False, *, ctx: Optional[Ctx] = None, keep_taps: bool = False,
                 avatar: Optional[UltraLightAvatar] = None):
        super().__init__(ctx)
        self.G, self.Bs, self.return_pred, self.avatar = int(groups), int(frames_per_session), bool(return_pred), avatar
        self.batch = self.G                                  # CrossSessionBatcher: requests per engine call
        self.B = B = self.G * self.Bs
        try:
            ctx = self.ctx
            if avatar is not None:
                if self.G != 1:
                    raise ValueError("a session bound to an avatar has one group")
                self.d_index = self.alloc((4,), np.int32, zero=True)
            else:
                self.bank = UltraLightBank(ctx, template, slots if slots is not None else 2 * self.G, alloc=self.alloc)
                if self.bank.slots < self.G:
                    raise ValueError(f"the bank needs at least {self.G} slots")
                self.d_slot = self.alloc((self.G,), np.int32, zero=True)
                self._slot_host = np.zeros(self.G, np.int32)
                self._blank = self.alloc((1, CROP, CROP, 3), np.uint8, zero=True)      # crop source of the groups a call leaves empty
                self._prep = [(self._blank, 1, 0)] * self.G
                table = ul_prep_table(self._prep)
                self.d_prep = self.alloc(table.shape, table.dtype)
                ctx.h2d(self.d_prep, table)
            self.audio16 = self.alloc((B, 32, 32, 16), np.float16, zero=True)           # NHWC view of audiofeat.reshape(16, 32, 32)
            self.img16 = self.alloc((B, FACE, FACE, 16), np.float16, zero=True)
            self.pred = self.alloc((B, FACE, FACE, 3), np.float32, zero=True)
            self._frames_out: Dict[tuple, DevTensor] = {}
            if avatar is not None:
                self.frames_out = self._out(0, avatar)
            self.taps = {} if keep_taps else None
            self._audio_host = np.zeros((B, 1024, 16), np.float16)

            def emit(b: Builder):
                if avatar is not None:
                    ctx.ul_prep(avatar.faces, avatar.n, self.d_index, B, self.img16)
                    avatar.model.emit(b, self.img16, self.audio16, self.pred, self.taps)
                else:
                    ctx.ul_prep_grouped(self.d_prep, self.Bs, B, self.img16)
                    template.emit(b, self.img16, self.audio16, self.pred, self.taps, _Grouping(self.bank, self.d_slot, self.Bs))

            self.capture(emit)
        except BaseException:
            self.close()
            raise

    def _check(self, requests):
        if not 1 <= len(requests) <= self.G:
            raise ValueError(f"1..{self.G} group requests per call, got {len(requests)}")
        if self.avatar is not None and requests[0][0] is not self.avatar:
            raise ValueError("the session is bound to another avatar")

    def _launch(self, requests: Sequence[tuple]):
        """requests[g] = (UltraLightAvatar, first frame index, features (Bs,16,1024) | None = resident in audio16 rows of group g):
        stage the features, write the frame index (bound avatar) or the slot and prep tables, launch the graph."""
        if self.graph is None:
            raise RuntimeError(f"{type(self).__name__}: paste-only (or closed) session has no network graph")
        self._check(requests)
        ctx, Bs = self.ctx, self.Bs
        stage = False
        for g, (av, index, feats) in enumerate(requests):
            if feats is not None:
                a = np.asarray(feats, np.float32)
                if a.shape != (Bs, 16, 1024):
                    raise ValueError(f"audio features must be ({Bs},16,1024), got {a.shape}")
                self._audio_host[g * Bs:(g + 1) * Bs] = a.transpose(0, 2, 1)
                stage = True
        if stage:
            ctx.h2d(self.audio16, self._audio_host[:len(requests) * Bs], sync=False)
        if self.avatar is not None:
            ctx.set_i32(self.d_index, int(requests[0][1]))
        else:
            keep: List[int] = []
            for g, (av, index, _f) in enumerate(requests):
                s = self.bank.slot_of(av.model, keep)
                keep.append(s)
                self._slot_host[g] = s
                self._prep[g] = (av.faces, av.n, int(index))
            for g in range(len(requests), self.G):
                self._prep[g] = (self._blank, 1, 0)
            ctx.h2d(self.d_slot, self._slot_host, sync=False)
            ctx.h2d(self.d_prep, ul_prep_table(self._prep), sync=False)
        self.graph.launch()

    infer_async = _launch

    def _out(self, g: int, av: UltraLightAvatar) -> DevTensor:
        key = (g, av.H, av.W)
        if key not in self._frames_out:
            self._frames_out[key] = self.alloc((self.Bs, av.H, av.W, 3), np.uint8, zero=True)
        return self._frames_out[key]

    def paste_async(self, requests: Sequence[tuple]) -> List[DevTensor]:
        """Paste-back of every group's predictions into its own avatar's frames (LightReal.paste_back_frame x Bs per group)."""
        self._check(requests)
        outs = []
        for g, (av, index, _f) in enumerate(requests):
            out = self._out(g, av)
            self.ctx.ul_paste(av.frames, av.faces, av.coords, self.pred, out, av.n, av.H, av.W, int(index), -1, g * self.Bs, self.Bs)
            outs.append(out)
        return outs

    def step_async(self, requests: Sequence[tuple]):
        self._launch(requests)
        self.paste_async(requests)

    def infer_groups(self, requests: Sequence[tuple]) -> List[np.ndarray]:
        """-> per request its (Bs, H, W, 3) uint8 composited frames, or with return_pred its float32 (Bs, 160, 160, 3) predictions
        (what LightReal.inference_batch returns for that session)."""
        with self.ctx.lock:
            self._launch(requests)
            if self.return_pred:
                n = len(requests) * self.Bs
                pred = self.ctx.download(DevTensor(self.pred.ptr, (n, FACE, FACE, 3), np.float32))
                return [pred[g * self.Bs:(g + 1) * self.Bs] for g in range(len(requests))]
            outs = [self.ctx.download(t, sync=False) for t in self.paste_async(requests)]
            self.ctx.sync()
            return outs

    infer_slots = infer_groups


class UltraLightSession(UltraLightBatchSession):
    """One avatar stream at a fixed batch size: UltraLightBatchSession with one group, bound to `avatar` (its own network on the
    ungrouped ops)."""

    def __init__(self, avatar: UltraLightAvatar, batch: int, keep_taps: bool = False, ctx: Optional[Ctx] = None, paste_only: bool = False):
        """paste_only: no ctx, network graph or activation arena — only paste_pred() works (cross-session mode: this session's
        U-Net pass runs in a shared UltraLightBatchSession)."""
        if paste_only:
            GraphSession.__init__(self, ctx, with_ctx=False)
            self.avatar, self.B = avatar, int(batch)
            return
        super().__init__(avatar.model, 1, batch, ctx=ctx, keep_taps=keep_taps, avatar=avatar)

    # ---- LightReal.inference_batch (ultralight_avatar.py:141-169)
    def infer_async(self, index: int, audio_feats: Optional[np.ndarray] = None):
        """audio_feats: (B, 16, 1024) float (the HubertASR windows) or None when audio16 is already resident."""
        self._launch([(self.avatar, index, audio_feats)])

    def infer(self, index: int, audio_feats: Optional[np.ndarray] = None, want_pred: bool = True):
        with self.ctx.lock:
            self.infer_async(index, audio_feats)
            if want_pred:
                return self.ctx.download(self.pred)              # float32 (B,160,160,3) = pred * 255, as the reference returns
            self.ctx.sync()
            return None

    # ---- LightReal.paste_back_frame (ultralight_avatar.py:171-184)
    def paste_batch_async(self, index: int):
        self.paste_async([(self.avatar, index, None)])

    def paste_batch(self, index: int, out: Optional[np.ndarray] = None) -> np.ndarray:
        with self.ctx.lock:
            self.paste_batch_async(index)
            return self.ctx.download(self.frames_out, out)

    def infer_paste(self, index: int, audio_feats: Optional[np.ndarray] = None, out: Optional[np.ndarray] = None) -> np.ndarray:
        """inference_batch + B x paste_back_frame as one engine round: (B, H, W, 3) uint8 composited frames."""
        with self.ctx.lock:
            self.infer_async(index, audio_feats)
            self.paste_batch_async(index)
            return self.ctx.download(self.frames_out, out)

    def paste_pred(self, pred_frame: np.ndarray, idx: int) -> np.ndarray:
        """paste_back_frame for a host prediction (160,160,3) — the reference's exact argument, on the session's paste ctx."""
        a = self.avatar
        p = np.ascontiguousarray(pred_frame, np.float32)
        if p.shape != (FACE, FACE, 3):
            raise ValueError(f"paste_pred: prediction must be ({FACE},{FACE},3), got {p.shape}")
        if not 0 <= idx < a.n:
            raise ValueError("paste_pred: idx out of range")
        pc, pred, out = self.paste_ctx((1, FACE, FACE, 3), np.float32, (a.H, a.W, 3))
        with pc.lock:
            pc.h2d(pred, p, sync=False)
            pc.ul_paste(a.frames, a.faces, a.coords, pred, out, a.n, a.H, a.W, 0, idx, 0, 1)
            return pc.download(out)

    def step_async(self, index: int):
        self.infer_async(index, None)
        self.paste_batch_async(index)


def unet_gflop_per_frame() -> float:
    """Algorithmic GFLOP (2 x MAC) of one Model(6,'hubert') forward at 160x160 (real channel counts, no padding)."""
    fl = 0.0

    def ir(inp, oup, H, s=1):
        nonlocal fl
        hid, O = 2 * inp, H // s
        fl += 2.0 * H * H * inp * hid + 2.0 * O * O * 9 * hid + 2.0 * O * O * hid * oup
        return O

    def dc(inp, oup, H, s):
        O = ir(inp, oup, H, s)
        return ir(oup, oup, O)

    ir(6, CH[0], 160)
    H = 160
    for i in range(4):
        H = dc(CH[i], CH[i + 1], H, 2)
    ir(16, CH[1], 32), ir(CH[1], CH[2], 32)
    fl += 2.0 * 16 * 16 * 9 * CH[2] * CH[3]
    ir(CH[3], CH[3], 16)
    fl += 2.0 * 10 * 10 * 9 * CH[3] * CH[4]
    ir(CH[4], CH[4], 10), ir(CH[4], CH[4], 10)
    dc(2 * CH[4], CH[4], 10, 1), dc(CH[4], CH[3], 10, 1)
    for i, (ci, co) in enumerate(((CH[4], CH[3] // 2), (CH[3], CH[2] // 2), (CH[2], CH[1] // 2), (CH[1], CH[0]))):
        dc(ci, co, 20 << i, 1)
    fl += 2.0 * 160 * 160 * CH[0] * 3
    return fl / 1e9
