"""The image matrix of the JPEG encoder tests: sizes that put dummy blocks on the right, at the
bottom and in the corner and give an odd chroma width in blocks (1 x 1, 1 x W, H x 1, 15/17/31/33
on each axis, widths = 1 and 9 mod 16), and constant, noise, full-swing checkerboard, lone
high-frequency (ZRL), synthetic and overlay content, with one 1024 x 1024 and one 2160 x 3840
overlay; the qualities at every branch of jpeg_quality_scaling and both optimize settings."""
import numpy as np

import png_inputs
from matterport_maskrcnn_with_tensorflow_serving_b200 import synth

QUALITIES = (0, 1, 10, 49, 50, 51, 75, 95, 100)
OPTIMIZE = (False, True)
SIZES = [(1, 1), (1, 40), (40, 1), (8, 8), (16, 16), (15, 17), (17, 15), (31, 33), (33, 31),
         (17, 33), (37, 53), (20, 33), (24, 41), (9, 57)]


def checkerboard(h, w, cell=1):
    """Full swing: 0 and 255 in every channel, cells of `cell` pixels."""
    yy, xx = np.mgrid[:h, :w]
    return np.repeat((((yy // cell + xx // cell) & 1) * 255).astype(np.uint8)[..., None], 3, 2)


def lone_frequency(h, w, u, v, amp=100.0):
    """A gray image whose every 8 x 8 block is one DCT basis pattern (vertical frequency u,
    horizontal v): a block of one coefficient after many zeros (ZRL runs before it)."""
    yy, xx = np.mgrid[:h, :w]
    p = np.cos((2 * (yy % 8) + 1) * u * np.pi / 16) * np.cos((2 * (xx % 8) + 1) * v * np.pi / 16)
    g = np.clip(np.rint(128 + amp * p), 0, 255).astype(np.uint8)
    return np.repeat(g[..., None], 3, 2)


def matrix(big=True):
    """[(name, uint8 [H, W, 3] RGB image)]."""
    rng = np.random.default_rng(2025)
    out = []
    for h, w in SIZES:
        out.append((f"noise{h}x{w}", rng.integers(0, 256, (h, w, 3), dtype=np.uint8)))
        out.append((f"const{h}x{w}", np.full((h, w, 3), (200, 30, 90), np.uint8)))
    out.append(("checker40x56", checkerboard(40, 56)))
    out.append(("checker4_33x47", checkerboard(33, 47, 4)))
    out.append(("zrl_7_7", lone_frequency(32, 48, 7, 7)))
    out.append(("zrl_6_5", lone_frequency(24, 40, 6, 5, 60.0)))
    out.append(("noise97x130", rng.integers(0, 256, (97, 130, 3), dtype=np.uint8)))
    out.append(("synth120x161", synth.synth_rgb_image(rng, 120, 161)))
    out.append(("overlay250x371", png_inputs.overlay(rng, 250, 371)))
    out.append(("overlay480x640", png_inputs.overlay(rng, 480, 640)))
    if big:
        out.append(("overlay1024x1024", png_inputs.overlay(rng, 1024, 1024, 10)))
        out.append(("overlay2160x3840", png_inputs.overlay(rng, 2160, 3840, 12)))
    return out
