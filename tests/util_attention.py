"""Pointwise fp64 reference of the contextual attention (test infrastructure, like oracle/sketchedit_oracle.py).

``contextual_attention_at`` evaluates ``oracle.sketchedit_oracle.contextual_attention`` exactly (fp64) at listed output
pixels only. The full oracle keeps L x L tensors (hundreds of GB at 12 MP); this one keeps the plane norms, the key validity
and, for the at most four queries each output pixel reads, their softmax over all L keys, streamed over bands of key rows
with a running maximum. Its memory grows linearly with the map.
"""
import torch
import torch.nn.functional as F


def contextual_attention_at(feat, mask_s, pixels, patch=4, stride=2, th=0.1, scale=10.0, key_rows=32, err=None):
    """feat [B, C, h, w], mask_s [B, 1, h, w] (as contextual_attention); pixels: iterable of (b, y, x).
    Returns fp64 [len(pixels), C]: out[b, :, y, x] of contextual_attention(feat, mask_s).

    With err = dict(logit_rel, logit_abs, rel, abs) it also returns an error bound of an implementation whose logits are
    good to delta_n = logit_rel * max_l |scale m_l q_n| . |k_l| + logit_abs (query n; masked keys have the exact logit 0) and
    whose softmax-weighted sums are good to rel * sum_l P_l |V_l| + abs: a softmax whose logits move by at most delta moves
    each P_l by at most P_l (exp(2 delta) - 1), so query n's output element d is off by at most
    (exp(2 delta_n) - 1 + rel) * sum_l P_l |V_ld| + abs. Returns (out, dict(bound [npix, C] summed over the <= 4 queries a
    pixel reads))."""
    f = feat.detach().to("cpu", torch.float64)
    ms = mask_s.detach().to("cpu", torch.float64)
    B, C, h, w = f.shape
    hs, ws = (h - patch) // stride + 1, (w - patch) // stride + 1
    rnorm = 1.0 / torch.sqrt((f ** 2).sum(3).sum(2) + 1e-8)                                 # [B, C]
    valid = (F.avg_pool2d(1.0 - ms, patch, stride)[:, 0] > th).to(torch.float64)           # [B, hs, ws]
    pixels = [tuple(int(v) for v in p) for p in pixels]
    out = torch.zeros(len(pixels), C, dtype=torch.float64)
    bound = torch.zeros(len(pixels), C, dtype=torch.float64)
    for b in sorted({p[0] for p in pixels}):
        # queries read by the pixels of this image: pixel (y, x) += O[n][(c, u, v)] for 2 ny + u = y, 2 nx + v = x
        uses = []
        for i, (pb, y, x) in enumerate(pixels):
            if pb != b:
                continue
            for u in range(y % stride, patch, stride):
                for v in range(x % stride, patch, stride):
                    ny, nx = (y - u) // stride, (x - v) // stride
                    if 0 <= ny < hs and 0 <= nx < ws:
                        uses.append((i, (ny, nx), u, v))
        queries = sorted({q for _, q, _, _ in uses})
        if not queries:
            continue
        qi = {q: k for k, q in enumerate(queries)}
        Q = torch.stack([f[b, :, stride * ny:stride * ny + patch, stride * nx:stride * nx + patch].reshape(-1) for ny, nx in queries])
        m_run = torch.full((len(queries), 1), -float("inf"), dtype=torch.float64)
        s_run = torch.zeros(len(queries), 1, dtype=torch.float64)
        acc = torch.zeros(len(queries), Q.shape[1], dtype=torch.float64)
        acc_abs = torch.zeros_like(acc)
        qk_max = torch.zeros(len(queries), dtype=torch.float64)
        for k0 in range(0, hs, key_rows):
            k1 = min(k0 + key_rows, hs)
            rows = f[b:b + 1, :, stride * k0:stride * (k1 - 1) + patch]
            V = F.unfold(rows, kernel_size=patch, stride=stride)[0]                       # [(c, u, v), keys of rows k0..k1)
            K = (V.view(C, patch * patch, -1) * rnorm[b][:, None, None]).view(V.shape)
            s = (Q @ K) * valid[b, k0:k1].reshape(1, -1) * scale                          # masked keys keep logit 0
            m_new = torch.maximum(m_run, s.max(1, keepdim=True).values)
            e = torch.exp(s - m_new)
            corr = torch.exp(m_run - m_new)
            s_run = s_run * corr + e.sum(1, keepdim=True)
            acc = acc * corr + e @ V.T
            m_run = m_new
            if err is not None:
                acc_abs = acc_abs * corr + e @ V.abs().T
                qk_max = torch.maximum(qk_max, ((Q.abs() @ K.abs()) * valid[b, k0:k1].reshape(1, -1) * scale).max(1).values)
        O = acc / s_run                                                                   # [queries, (c, u, v)]
        if err is not None:
            PV = acc_abs / s_run
            d_n = err["logit_rel"] * qk_max + err["logit_abs"]
            Bq = (torch.expm1(2 * d_n)[:, None] + err["rel"]) * PV + err["abs"]
        for i, q, u, v in uses:
            out[i] += O[qi[q]].view(C, patch, patch)[:, u, v]
            if err is not None:
                bound[i] += Bq[qi[q]].view(C, patch, patch)[:, u, v]
    if err is not None:
        return out, dict(bound=bound)
    return out


def sample_pixels(B, h, w, n_blocks, seed, extra=()):
    """(b, y, x) for the four corners of every image, the listed extra pixels and n_blocks random 2 x 2 pixel blocks (a block
    reads the same four queries, which keeps contextual_attention_at cheap)."""
    g = torch.Generator().manual_seed(seed)
    px = []
    for b in range(B):
        px += [(b, 0, 0), (b, 0, w - 1), (b, h - 1, 0), (b, h - 1, w - 1)]
    px += list(extra)
    for _ in range(n_blocks):
        b = int(torch.randint(B, (1,), generator=g))
        y = 2 * int(torch.randint(h // 2, (1,), generator=g))
        x = 2 * int(torch.randint(w // 2, (1,), generator=g))
        px += [(b, y, x), (b, y, x + 1), (b, y + 1, x), (b, y + 1, x + 1)]
    return px
