"""Flow colour coding (TEST INFRASTRUCTURE — the definition that fgt_b200/flowviz.py / csrc/flowviz.cu are checked
against; nothing under fgt_b200/ imports it).

Restates, in numpy with every dtype written out, the reference's RAFT/utils/flow_viz.py as numpy 2 (NEP 50) evaluates
it on the float32 flows the driver hands it:
    make_colorwheel  :20-67    the 55 x 3 Middlebury wheel (RY 15, YG 6, GC 4, CB 11, BM 13, MR 6 entries), float64
    flow_to_image    :109-132  r = sqrt(u^2 + v^2) and its maximum in float32; u, v divided by (max + 1e-5), float32
    flow_uv_to_colors :70-106  rad = sqrt(u^2 + v^2) and a = arctan2(-v, -u) / pi in float32 (:88-89); fk = (a + 1) / 2
                               * 54 in float32 (:90); k0 = floor(fk) as int32, k1 = k0 + 1 wrapped from 55 to 0
                               (:91-93); f = fk - k0 in float64 (float32 minus int32 promotes, :94); per channel
                               col = (1 - f) * w[k0] / 255 + f * w[k1] / 255 in float64 (:96-99); 1 - rad * (1 - col)
                               where rad <= 1, col * 0.75 elsewhere (:100-102); floor(255 * col) into uint8 (:105),
                               channel i at 2 - i for BGR (:104)
One deliberate difference: a NaN or Inf in a flow raises ValueError here, where the reference indexes the wheel with
floor(NaN) and raises IndexError.
"""
import numpy as np

NCOLS = 55


# (entries, channel held at 255, channel that ramps, +1 rising / -1 falling): RY, YG, GC, CB, BM, MR
SEGMENTS = ((15, 0, 1, +1), (6, 1, 0, -1), (4, 1, 2, +1), (11, 2, 1, -1), (13, 2, 0, +1), (6, 0, 2, -1))


def make_colorwheel():
    w = np.zeros((NCOLS, 3))
    k = 0
    for n, full, ramp, sign in SEGMENTS:
        step = np.floor(255 * np.arange(n) / n)
        w[k:k + n, full] = 255
        w[k:k + n, ramp] = step if sign > 0 else 255 - step
        k += n
    return w


def _wheel_check():
    w = make_colorwheel()
    assert (w[0] == [255, 0, 0]).all() and (w[15] == [255, 255, 0]).all() and (w[21] == [0, 255, 0]).all()
    assert (w[25] == [0, 255, 255]).all() and (w[36] == [0, 0, 255]).all() and (w[49] == [255, 0, 255]).all()
    return w


WHEEL = _wheel_check()


def flow_uv_to_colors(u, v, convert_to_bgr=False):
    """u, v: float32 [H,W], already normalised."""
    u, v = np.asarray(u, np.float32), np.asarray(v, np.float32)
    img = np.zeros(u.shape + (3,), np.uint8)
    rad = np.sqrt(np.square(u) + np.square(v))                                     # float32
    a = np.arctan2(-v, -u) / np.float32(np.pi)                                      # float32
    fk = (a + np.float32(1)) / np.float32(2) * np.float32(NCOLS - 1)                # float32
    k0 = np.floor(fk).astype(np.int32)
    k1 = k0 + 1
    k1[k1 == NCOLS] = 0
    f = fk.astype(np.float64) - k0.astype(np.float64)                               # float64
    small = rad <= 1
    r64 = rad.astype(np.float64)
    for i in range(3):
        col = (1 - f) * (WHEEL[k0, i] / 255.0) + f * (WHEEL[k1, i] / 255.0)
        col = np.where(small, 1 - r64 * (1 - col), col * 0.75)
        img[:, :, 2 - i if convert_to_bgr else i] = np.floor(255 * col)
    return img


def flow_to_image(flow_uv, convert_to_bgr=False):
    """flow_uv: [H,W,2] -> uint8 [H,W,3] (RGB, or BGR)."""
    flow_uv = np.asarray(flow_uv, np.float32)
    if flow_uv.ndim != 3 or flow_uv.shape[2] != 2:
        raise ValueError(f"flow_to_image: flow {flow_uv.shape} must be [H,W,2]")
    if not np.isfinite(flow_uv).all():
        raise ValueError("flow_to_image: the flow holds NaN or Inf")
    u, v = flow_uv[:, :, 0], flow_uv[:, :, 1]
    with np.errstate(over="ignore"):
        rad_max = np.max(np.sqrt(np.square(u) + np.square(v)))                      # float32, inf past 1.8e19
    d = rad_max + np.float32(1e-5)
    return flow_uv_to_colors(u / d, v / d, convert_to_bgr)


def flow_images(flows, convert_to_bgr=False):
    """[B,H,W,2] or [H,W,2] -> uint8 of the same leading shape, each image normalised by its own maximum."""
    flows = np.asarray(flows, np.float32)
    if flows.ndim == 3:
        return flow_to_image(flows, convert_to_bgr)
    return np.stack([flow_to_image(f, convert_to_bgr) for f in flows], 0)
