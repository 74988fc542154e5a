"""Float64 restatement of region-edit detail (contextual residual aggregation on netG's attention weights, DESIGN.md 7b),
written from its definition: exact integer geometry, then float64 sums."""
import numpy as np
from PIL import Image


def work_of(x, b, n):
    """u(x) = ((2x + 1) n) // (2 b): the working pixel holding box pixel x's centre."""
    return ((2 * np.asarray(x, np.int64) + 1) * n) // (2 * b)


def anchors(b, n):
    """a(p) = min {x : u(x) >= 8 p} for the n // 8 - 1 patch positions, by search."""
    u = work_of(np.arange(b), b, n)
    return np.array([int(np.nonzero(u >= 8 * p)[0][0]) for p in range(n // 8 - 1)], np.int64)


def footprint(b, n):
    return -(-16 * b // n) + 2


def covering(w, n):
    """Patch positions whose footprint [8p, 8p + 16) holds working pixel w."""
    return [p for p in (w // 8 - 1, w // 8) if 0 <= p < n // 8 - 1]


def low_of(crop, Hn, Wn):
    bh, bw = crop.shape[:2]
    return np.asarray(Image.fromarray(crop).resize((Wn, Hn)).resize((bw, bh)))


def residual(crop, low, hole):
    """R at box resolution: crop - low, 0 where the working pixel under the box pixel is in the hole."""
    bh, bw = crop.shape[:2]
    Hn, Wn = hole.shape
    h = hole[work_of(np.arange(bh), bh, Hn)][:, work_of(np.arange(bw), bw, Wn)] != 0
    R = crop.astype(np.int64) - low.astype(np.int64)
    R[h] = 0
    return R, h


def aggregate(crop, low, hole, P):
    """(A float64 [bh,bw,3] (0 outside the hole), D int64 [bh,bw,3], in-hole bool [bh,bw]). P[k, q]: [L, L]."""
    bh, bw = crop.shape[:2]
    Hn, Wn = hole.shape
    hs, ws = Hn // 8 - 1, Wn // 8 - 1
    ax, ay = anchors(bw, Wn), anchors(bh, Hn)
    fw, fh = footprint(bw, Wn), footprint(bh, Hn)
    R, inh = residual(crop, low, hole)
    ky, kx = np.divmod(np.arange(hs * ws), ws)
    sy = np.minimum(ay[ky][:, None] + np.arange(fh)[None], bh - 1)           # [L, fh]
    sx = np.minimum(ax[kx][:, None] + np.arange(fw)[None], bw - 1)           # [L, fw]
    Rp = R[sy[:, :, None], sx[:, None, :]].reshape(hs * ws, -1).astype(np.float64)   # [L keys, fh fw 3]
    C = (P.astype(np.float64).T @ Rp).reshape(hs * ws, fh, fw, 3)            # C[q, y - ay(q), x - ax(q), c]
    A = np.zeros((bh, bw, 3))
    u, v = work_of(np.arange(bw), bw, Wn), work_of(np.arange(bh), bh, Hn)
    for y in np.nonzero(inh.any(1))[0]:
        for x in np.nonzero(inh[y])[0]:
            qs = [(py, px) for py in covering(v[y], Hn) for px in covering(u[x], Wn)]
            A[y, x] = sum(C[py * ws + px, y - ay[py], x - ax[px]] for py, px in qs) / len(qs)
    D = np.where(inh[..., None], np.sign(A) * np.floor(np.abs(A) + 0.5), 0).astype(np.int64)
    return A, D, inh


def _covering_pair(w, n):
    """Per working pixel w the two candidate patch positions w // 8 - 1 and w // 8 of `covering` (clamped into the grid) and
    whether each is one: [len(w), 2] each."""
    p = np.stack([w // 8 - 1, w // 8], 1)
    ok = (p >= 0) & (p < n // 8 - 1)
    return np.clip(p, 0, n // 8 - 2), ok


def aggregate_vec(crop, low, hole, P, device="cpu"):
    """aggregate() for boxes too large for its loop: the same definition with the fold vectorised, and the float64 sums in
    torch on `device`. Takes P as a torch tensor or an array; returns numpy (A, D, in-hole) like aggregate."""
    import torch
    bh, bw = crop.shape[:2]
    Hn, Wn = hole.shape
    hs, ws = Hn // 8 - 1, Wn // 8 - 1
    ax, ay = anchors(bw, Wn), anchors(bh, Hn)
    fw, fh = footprint(bw, Wn), footprint(bh, Hn)
    R, inh = residual(crop, low, hole)
    t = lambda a: torch.as_tensor(a, device=device)
    ky, kx = np.divmod(np.arange(hs * ws), ws)
    sy = t(np.minimum(ay[ky][:, None] + np.arange(fh)[None], bh - 1))
    sx = t(np.minimum(ax[kx][:, None] + np.arange(fw)[None], bw - 1))
    Rp = t(R).double()[sy[:, :, None], sx[:, None, :]].reshape(hs * ws, -1)       # [L keys, fh fw 3]
    C = (t(P).double().T @ Rp).reshape(hs * ws, fh, fw, 3)
    del Rp
    u, v = work_of(np.arange(bw), bw, Wn), work_of(np.arange(bh), bh, Hn)
    py, oky = _covering_pair(v, Hn)                                                 # [bh, 2]
    px, okx = _covering_pair(u, Wn)                                                 # [bw, 2]
    A = torch.zeros(bh, bw, 3, dtype=torch.float64, device=device)
    for a in (0, 1):                                                                # (py, px) order, as the loop sums
        for b in (0, 1):
            q = t(py[:, a] * ws)[:, None] + t(px[:, b])[None, :]
            dy = t(np.clip(np.arange(bh) - ay[py[:, a]], 0, fh - 1))[:, None]
            dx = t(np.clip(np.arange(bw) - ax[px[:, b]], 0, fw - 1))[None, :]
            ok = t(oky[:, a])[:, None] & t(okx[:, b])[None, :]
            A += torch.where(ok[..., None], C[q, dy, dx], torch.zeros((), dtype=torch.float64, device=device))
    del C
    nq = t(oky.sum(1))[:, None] * t(okx.sum(1))[None, :]
    inh_t = t(inh)
    A = torch.where(inh_t[..., None], A / nq.clamp(min=1)[..., None], torch.zeros((), dtype=torch.float64, device=device))
    A = A.cpu().numpy()
    D = np.where(inh[..., None], np.sign(A) * np.floor(np.abs(A) + 0.5), 0).astype(np.int64)
    return A, D, inh


def bound(L):
    """The fp32 bound of the device's A against float64 (include/sketchedit_b200.h, se_detail_u8)."""
    return 255.0 * (L + 8) * 2.0 ** -22


def near_boundary(A64, L):
    """Where A64 lies within bound(L) of a rounding boundary (x.5): there the device's D may be one off."""
    return np.abs(np.abs(A64 - np.floor(A64)) - 0.5) <= bound(L)


def violations(A, D, A64, D64, inh, L, exact=False):
    """The checks of a device plane (A, D) against float64's (A64, D64): the ones it fails, by name. exact: A and D must
    equal float64's with no boundary exemption (weights whose products and sums are exact in fp32)."""
    out = []
    if exact:
        if not np.array_equal(A, A64):
            out.append("A != A64")
        if not np.array_equal(D, D64):
            out.append("D != D64")
    else:
        if np.abs(A - A64).max(initial=0.0) > bound(L):
            out.append("|A - A64| > bound")
        near = near_boundary(A64, L)
        if not np.array_equal(D[~near], D64[~near]):
            out.append("D != D64 away from a rounding boundary")
    if np.abs(D - D64).max(initial=0) > 1:
        out.append("|D - D64| > 1")
    if D[~inh].any():
        out.append("D != 0 outside the hole")
    return out
