"""CPU test of parallel.download_band, the D2H step of ShardedSsgiChain.submit_host: a rank's band of the compose stage's image (output 9,
RGBA16F) and of `composed` (RGBA32F) lands tightly packed at the start of the host tensors, from pitched planes, through
rfx_plane_download_rows' contract (here a host stand-in that copies the rows the call names)."""
import ctypes as C

import numpy as np
import torch

from realism_effects_b200 import abi, parallel


class _Ctx:
    """the context surface download_band uses; rfx_plane_download_rows copies rows [row0, row1) of a pitched plane, tightly packed"""

    def __init__(self):
        self.h, self.calls = object(), []
        ctx = self

        class Lib:
            @staticmethod
            def rfx_plane_download_rows(h, stream, plane_ref, host, row0, row1):
                p = plane_ref._obj
                ctx.calls.append((p.ptr, row0, row1))
                row = p.width * abi.FMT_BYTES[p.format]
                for i, y in enumerate(range(row0, row1)):
                    C.memmove(host + i * row, p.ptr + y * p.pitch, row)
                return 0

        self.lib = Lib()

    def _chk(self, st):
        assert st == 0


def _plane(a: np.ndarray, width: int, fmt: int) -> abi.Plane:
    p = abi.Plane()
    p.ptr, p.width, p.height, p.pitch, p.format = a.ctypes.data, width, a.shape[0], a.strides[0], fmt
    return p


def test_band_download_of_the_image_matches_the_band_rows():
    W, H, pad = 40, 96, 24  # pitched planes: rows padded beyond the texels
    rng = np.random.default_rng(3)
    image = rng.standard_normal((H, W + pad, 4)).astype(np.float16)
    composed = rng.standard_normal((H, W + pad, 4)).astype(np.float32)
    for b0, b1 in ((0, 96), (0, 17), (17, 64), (64, 96)):
        ctx = _Ctx()
        out_c = torch.zeros((H, W, 4), dtype=torch.float32)
        out_i = torch.zeros((H, W, 4), dtype=torch.float16)
        pi, pc = _plane(image, W, abi.FMT_RGBA16F), _plane(composed, W, abi.FMT_RGBA32F)
        n = parallel.download_band(ctx, None, [(pc, out_c), (pi, out_i), (None, None)], b0, b1)
        assert n == (b1 - b0) * W * (16 + 8)
        assert ctx.calls == [(pc.ptr, b0, b1), (pi.ptr, b0, b1)]
        assert np.array_equal(out_i.numpy()[: b1 - b0].view(np.uint16), image[b0:b1, :W].view(np.uint16))
        assert np.array_equal(out_c.numpy()[: b1 - b0], composed[b0:b1, :W])
        assert not out_i.numpy()[b1 - b0:].any() and not out_c.numpy()[b1 - b0:].any()  # nothing beyond the band's rows
    # the image alone (out_host None): one download
    ctx = _Ctx()
    out_i = torch.zeros((H, W, 4), dtype=torch.float16)
    assert parallel.download_band(ctx, None, [(_plane(composed, W, abi.FMT_RGBA32F), None), (_plane(image, W, abi.FMT_RGBA16F), out_i)], 8, 40) == 32 * W * 8
    assert len(ctx.calls) == 1
