"""Clips for the H.264 tests (tests/test_h264_host.py, tests/test_gpu_h264.py): seeded uint8 frames of the kinds a
talking-head encoder meets and the kinds that stress it, and the case matrix both files run."""
from __future__ import annotations

import numpy as np


def _smooth(h, w, seed):
    """A smooth RGB picture (blobs of colour over a soft background, like a rendered portrait)."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    img = np.zeros((h, w, 3))
    for _ in range(6):
        cy, cx, r = rng.uniform(0, h), rng.uniform(0, w), rng.uniform(0.1, 0.4) * max(h, w)
        img += rng.uniform(-90, 90, 3) * np.exp(-((yy - cy) ** 2 + (xx - cx) ** 2) / (2 * r * r))[..., None]
    img += 128 + 20 * np.sin(xx / 9.0)[..., None] * np.cos(yy / 13.0)[..., None]
    return np.clip(img, 0, 255).astype(np.uint8)


def clip(kind: str, n: int, h: int, w: int, seed: int = 0) -> np.ndarray:
    """``n`` frames ``[n, h, w, 3]`` (``[n, h, w]`` for ``"masks"``) of one kind:
    noise, gradient, saturated, translate (known offsets, odd ones included), far (offsets beyond any search range),
    static (one frame repeated: every P macroblock skips), smooth (a portrait-like picture that sways), masks (grey
    0 / 255 shapes that move, like the rasterised feature maps)."""
    rng = np.random.default_rng(seed)
    if kind == "noise":
        return rng.integers(0, 256, (n, h, w, 3), dtype=np.uint8)
    yy, xx = np.mgrid[0:h, 0:w]
    if kind == "gradient":
        return np.stack([np.stack([(xx * 3 + yy + 5 * i) % 256, (yy * 2 + 7 * i) % 256, (xx + yy * 4) % 256], -1)
                         for i in range(n)]).astype(np.uint8)
    if kind == "saturated":
        out = np.zeros((n, h, w, 3), np.uint8)
        for i in range(n):
            out[i] = (rng.integers(0, 2, (h // 8 + 1, w // 8 + 1, 3))[yy // 8, xx // 8] * 255).astype(np.uint8)
            out[i, : h // 2] = 255 - out[i, : h // 2] if i % 2 else out[i, : h // 2]
        return out
    base = _smooth(h, w, seed)
    if kind == "translate":
        offs = [(0, 0), (1, 0), (0, -3), (2, 5), (-7, 3), (3, -1), (-5, -9), (11, 7)]
        return np.stack([np.roll(base, offs[i % len(offs)], (0, 1)) for i in range(n)])
    if kind == "far":
        return np.stack([np.roll(base, (23 * i, -37 * i), (0, 1)) for i in range(n)])
    if kind == "static":
        return np.repeat(base[None], n, axis=0)
    if kind == "smooth":
        return np.stack([np.roll(base, (int(round(2 * np.sin(i / 3.0))), i // 2), (0, 1)) for i in range(n)])
    if kind == "masks":
        out = np.zeros((n, h, w), np.uint8)
        for i in range(n):
            cy, cx = h / 2 + 3 * np.sin(i / 2.0), w / 2 + i
            out[i][((yy - cy) / (0.3 * h)) ** 2 + ((xx - cx) / (0.25 * w)) ** 2 <= 1] = 255
            out[i][np.abs(yy - (h * 0.7 + i)) < 1.5] = 255
        return out
    raise ValueError(kind)


# (content, height, width, qp, gop, search, frames): every content, QP 0 / 1 / 10 / 26 / 40 / 51, sizes 16x16, 48x32,
# 512x512 and 1024x512 (height x width 512 x 1024 too), gop 1 / 2 / 60
CASES = [
    ("noise", 48, 32, 26, 60, 4, 3),
    ("noise", 16, 16, 0, 2, 2, 4),
    ("gradient", 48, 32, 1, 60, 3, 3),
    ("gradient", 16, 16, 51, 1, 1, 3),
    ("saturated", 48, 32, 0, 2, 2, 4),
    ("saturated", 32, 48, 10, 60, 4, 3),
    ("translate", 64, 64, 26, 60, 8, 8),
    ("translate", 48, 32, 40, 60, 4, 6),
    ("far", 64, 80, 26, 60, 4, 3),
    ("static", 48, 32, 26, 60, 4, 5),
    ("smooth", 64, 64, 10, 2, 6, 5),
    ("smooth", 64, 48, 51, 60, 16, 4),
    ("masks", 48, 64, 26, 60, 4, 4),
    ("masks", 32, 32, 0, 1, 2, 3),
    ("smooth", 512, 512, 26, 60, 16, 2),
    ("masks", 512, 512, 40, 60, 16, 2),
    ("translate", 512, 1024, 26, 60, 16, 2),
]


def case_id(c) -> str:
    return "{}-{}x{}-qp{}-gop{}-s{}-n{}".format(*c)
