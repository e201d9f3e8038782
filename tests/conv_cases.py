"""Fixtures and helpers shared by the GPU tests of the individual conv kernels: one context per module, fp16 bit views, channel
slices of wider sentinel-filled buffers, and seeded 3x3 weights with their tap-major copy."""
import types

import numpy as np
import pytest
import torch


@pytest.fixture(scope="module")
def ctx():
    from livetalking_b200 import engine
    from livetalking_b200.ops import Ctx
    engine.set_device(0)
    c = Ctx()
    yield c
    c.close()


def bits(a):
    return np.ascontiguousarray(a).view(np.uint16)


def slice_buf(ctx, dense, pitch, off, fill):
    """dense [..., C] uploaded into channels [off, off + C) of a buffer with pixel pitch `pitch` whose other channels hold `fill`:
    (DevTensor view of the slice, the upload, the host buffer)."""
    from livetalking_b200.ops import DevTensor
    buf = np.full(dense.shape[:-1] + (pitch,), fill, np.float16)
    buf[..., off:off + dense.shape[-1]] = dense
    t = ctx.upload(buf)
    return DevTensor(t.ptr, dense.shape, pitch=pitch, c_off=off), t, buf


def weights(ctx, g, cin, cout):
    """Seeded 3x3 conv weights (He-scaled fp16) and bias: (w, b, conv weight namespace with the tap-major copy, device buffers)."""
    w = (torch.randn(cout, cin, 3, 3, generator=g) * (2.0 / (cin * 9)) ** 0.5).half()
    b = torch.randn(cout, generator=g) * 0.2
    wt = ctx.upload(w.permute(0, 2, 3, 1).reshape(cout, 9 * cin).numpy())
    bt = ctx.upload(b.numpy().astype(np.float32))
    wtap = ctx.alloc((9, cout, cin))
    ctx.w_tap_major(wt, wtap, cout, cin)
    cw = types.SimpleNamespace(cout=cout, cin=cin, kh=3, kw=3, ktot=9 * cin, w=wt, w_tap=wtap, bias=bt)
    return w, b, cw, [wt, bt, wtap]
