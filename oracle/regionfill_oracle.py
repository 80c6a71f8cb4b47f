"""CPU oracle for flow diffusion / region fill (TEST INFRASTRUCTURE — see oracle/fgt_oracle.py).

Restates /root/reference/tool/utils/region_fill.py:7-138 (regionfill with factor=1.0, the driver's call at
tool/video_inpainting.py:44-52) without the index bookkeeping: inside the mask the result is the discrete
harmonic function  sum over the in-image 4-neighbours q of (u_p - v_q) = 0,  v_q = u_q inside the mask and
the given image value outside (formRightSide :69-112 sums the perimeter values, computeNumberOfNeighbors
:115-127 puts 4 / 3 / 2 on the diagonal = the number of in-image neighbours, i.e. a zero-flux condition at
the image border); outside the mask the image is returned unchanged (:16). Solved with scipy's sparse
direct solver like the reference (third-party: scipy 1.18.1 in this image). Pinned against the unmodified
reference by tests/golden/regionfill_*.npz.
"""
import numpy as np
from scipy import sparse
from scipy.sparse.linalg import spsolve


def system(mask):
    """The operator of regionfill for mask [H,W] bool: (A [n,n] csr, R [n,H*W] csr) over the n mask pixels in raster
    order, so that the hole values solve A u = R I.ravel(). A's diagonal holds the number of in-image 4-neighbours,
    -1 couples in-mask neighbours; R sums the image values of the in-image neighbours outside the mask."""
    mask = np.asarray(mask).astype(bool)
    H, W = mask.shape
    idx = -np.ones((H, W), dtype=np.int64)
    idx[mask] = np.arange(int(mask.sum()))
    ys, xs = np.nonzero(mask)
    n = ys.size
    diag = np.zeros(n)
    rows, cols, vals, brow, bcol = [], [], [], [], []
    for dy, dx in ((-1, 0), (0, 1), (1, 0), (0, -1)):
        yy, xx = ys + dy, xs + dx
        ok = (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
        diag += ok
        yc, xc = np.clip(yy, 0, H - 1), np.clip(xx, 0, W - 1)
        inside = ok & mask[yc, xc]
        rows.append(np.arange(n)[inside])
        cols.append(idx[yc, xc][inside])
        vals.append(-np.ones(int(inside.sum())))
        out = ok & ~inside
        brow.append(np.arange(n)[out])
        bcol.append((yc * W + xc)[out])
    rows.append(np.arange(n)); cols.append(np.arange(n)); vals.append(diag)
    A = sparse.coo_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(n, n)).tocsr()
    br = np.concatenate(brow)
    R = sparse.coo_matrix((np.ones(br.size), (br, np.concatenate(bcol))), shape=(n, H * W)).tocsr()
    return A, R


def regionfill(I, mask):
    """I [H,W] float, mask [H,W] bool -> float64 [H,W]."""
    I = np.asarray(I, dtype=np.float64)
    mask = np.asarray(mask).astype(bool)
    if not mask.any():
        return I.copy()
    A, R = system(mask)
    out = I.copy()
    out[mask] = spsolve(A, R @ I.ravel())
    return out


def diffusion(flows, masks):
    """tool/video_inpainting.py:44-52: flows [N,H,W,2], masks [N,H,W,1] -> list of float64 [H,W,2]."""
    out = []
    for i in range(flows.shape[0]):
        f = np.zeros(flows[i].shape)
        f[:, :, 0] = regionfill(flows[i][:, :, 0], masks[i][:, :, 0])
        f[:, :, 1] = regionfill(flows[i][:, :, 1], masks[i][:, :, 0])
        out.append(f)
    return out
