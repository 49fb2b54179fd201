"""Numpy restatement of the reference's flow colour coding, `flow_to_image` (core/utils/flow_viz.py:240-275) with
`compute_color` (:196-237) and `make_color_wheel` (:134-193), step by step in the dtypes numpy 2.x (NEP 50) gives them for a
float32 flow, so that each rounding is visible.  The radius and its maximum are float32; `np.finfo(float).eps` is a numpy
float64 scalar, so the normalisation and everything after it are float64.

The one deliberate difference: the arc tangent is the C library's, correctly rounded in practice.  numpy's `arctan2` may
dispatch to a SIMD routine whose last bit depends on the CPU, so the reference itself is not reproducible across machines;
this oracle is.
The reference also zeroes the unknown entries of its argument in place; this function does not modify its argument.
"""
import math

import numpy as np

UNKNOWN = np.float32(1e7)                          # flow_viz.py:141 UNKNOWN_FLOW_THRESH, compared in float32
EPS = np.finfo(np.float64).eps                     # flow_viz.py:268: a numpy float64 scalar, so it promotes what it meets


def color_wheel():
    """[55, 3] float64 Middlebury wheel (flow_viz.py:134-193): per segment one channel held at 255 and one ramping
    floor(255 * j / n) up or down."""
    segs = [(15, 1, True, 0), (6, 0, False, 1), (4, 2, True, 1), (11, 1, False, 2), (13, 0, True, 2), (6, 2, False, 0)]
    rows = []
    for n, ramp_ch, rising, full_ch in segs:
        ramp = np.floor(255 * np.arange(n) / n)
        seg = np.zeros((n, 3))
        seg[:, ramp_ch] = ramp if rising else 255 - ramp
        seg[:, full_ch] = 255
        rows.append(seg)
    return np.concatenate(rows)


def flow_to_image(flow):
    """flow: float32 [H, W, 2].  Returns uint8 [H, W, 3] in the reference's RGB order."""
    img, _ = _flow_to_image(flow)
    return img


def branch_mask(flow):
    """bool [H, W]: the known, non-NaN pixels whose normalised radius exceeds 1 (compute_color's `notidx`, :230-232)."""
    return _flow_to_image(flow)[1]


def _atan2(y, x):
    """float64 arc tangent through the C library's atan2, elementwise: correctly rounded in practice and the same on every
    CPU, where numpy's own float64 arctan2 may dispatch to a SIMD routine that is not."""
    return np.frompyfunc(math.atan2, 2, 1)(y, x).astype(np.float64)


def _flow_to_image(flow):
    flow = np.asarray(flow, np.float32)
    u, v = flow[..., 0].copy(), flow[..., 1].copy()
    unknown = (np.abs(u) > UNKNOWN) | (np.abs(v) > UNKNOWN)              # :254, inf included, NaN not
    u[unknown] = 0
    v[unknown] = 0
    rad = np.sqrt(u * u + v * v)                                         # :265, float32
    m = rad.max()
    maxrad = np.float64(-1.0) if np.isnan(m) else np.float64(m)          # :266 Python max(-1, nan) keeps -1
    den = maxrad + EPS                                                   # :268, eps is a float64 scalar: float64 from here
    u = u / den                                                          # :268-269, float32 / float64 -> float64
    v = v / den
    nan = np.isnan(u) | np.isnan(v)                                      # :207-209
    u[nan] = 0
    v[nan] = 0
    rad = np.sqrt(u * u + v * v)                                         # :214
    a = _atan2(-v, -u) / np.pi                                           # :216
    fk = (a + 1) / 2 * 54 + 1                                            # :218
    k0 = np.floor(fk).astype(np.int64)                                   # :220
    k1 = k0 + 1
    k1[k1 == 56] = 1                                                     # :222-223
    f = fk - k0                                                          # :224
    wheel = color_wheel()
    img = np.zeros(flow.shape[:2] + (3,), np.uint8)
    small = rad <= 1
    for c in range(3):
        col0 = wheel[k0 - 1, c] / 255
        col1 = wheel[k1 - 1, c] / 255
        col = (1 - f) * col0 + f * col1                                  # :229
        col = np.where(small, 1 - rad * (1 - col), col * 0.75)           # :231-235
        img[..., c] = np.floor(255 * col * (1 - nan))                    # :236
    img[unknown] = 0                                                     # :272-273
    return img, ~small & ~nan & ~unknown
