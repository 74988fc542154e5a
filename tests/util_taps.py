"""Decoding of the engine's activation taps (Engine.taps(), se_taps_enable) to fp32 NCHW, from the layouts of DESIGN.md
section 4 (test infrastructure).

This is a second statement of the layout contract, written from the documentation rather than from the kernels: a
layout bug in the engine or here shows up as a failed stage check.

  NHWC              [B][H][W][ld], channels [8 cb_off, 8 cb_off + C)
  channel-blocked   [B][ld][H][W][8], channel block k at block cb_off + k
  space-to-depth    [B][ld][H/2][W/2][8]: pixel (y, x) of channel block k in parity group p = (y & 1) * 2 + (x & 1), at
                    block cb_off + p * CB + k (CB = C / 8 blocks per group)
  packed stem rows  [B][H][Wp][8], image pixel x at row position x + padl, zero pixels around it
Storage: fp32, bf16, or split-half fp16 pairs holding 64 v = hi + lo, so v = (hi + lo) / 64 (exact in fp32). The lo
blocks follow the hi blocks: ld / 2 blocks further on (channel-blocked), CB blocks further on inside each parity group
(space-to-depth: 2 CB blocks per group), one [H][Wp][8] plane further on (packed rows).
"""
import torch

NHWC, C8, S2D, PACKED = 0, 1, 2, 3
F32, BF16, SPLIT = 0, 1, 2
ACT_SCALE = 64.0


def _values(raw, dtype):
    """the stored numbers as fp32 (split-half: hi and lo fp16 halves, each as fp32)."""
    raw = raw.contiguous()
    if dtype == F32:
        return raw.view(torch.float32).float()
    if dtype == BF16:
        return raw.view(torch.bfloat16).float()
    return raw.view(torch.float16).float()


def decode(desc, raw):
    """(x, pad): x the tap as fp32 NCHW [B, C, H, W] (packed rows: all 8 channels), pad the stored values DESIGN promises
    are zero (the pad pixels of packed rows, both halves in split-half; empty otherwise)."""
    lay, dt = desc["layout"], desc["dtype"]
    B, C, H, W, ld, cb0 = desc["B"], desc["C"], desc["H"], desc["W"], desc["ld"], desc["cb_off"]
    v = _values(raw.cpu(), dt)
    empty = torch.zeros(0)
    if lay == NHWC:
        assert dt != SPLIT
        return v.view(B, H, W, ld)[..., 8 * cb0:8 * cb0 + C].permute(0, 3, 1, 2).contiguous(), empty
    if lay == PACKED:
        Wp, padl = desc["Wp"], desc["padl"]
        rows = v.view(B, 2, H, Wp, 8) if dt == SPLIT else v.view(B, 1, H, Wp, 8)
        inside = torch.zeros(Wp, dtype=torch.bool)
        inside[padl:padl + W] = True
        pad = rows[:, :, :, ~inside, :].reshape(-1)
        img = rows[:, :, :, padl:padl + W, :]
        x = (img[:, 0] + img[:, 1]) / ACT_SCALE if dt == SPLIT else img[:, 0]
        return x.permute(0, 3, 1, 2).contiguous(), pad
    CB = (C + 7) // 8
    if lay == C8:
        blocks = v.view(B, ld, H, W, 8)

        def take(k0):
            return blocks[:, k0:k0 + CB].permute(0, 1, 4, 2, 3).reshape(B, CB * 8, H, W)[:, :C]
        x = (take(cb0) + take(cb0 + ld // 2)) / ACT_SCALE if dt == SPLIT else take(cb0)
        return x.contiguous(), empty
    assert lay == S2D and C % 8 == 0
    blocks = v.view(B, ld, H // 2, W // 2, 8)
    x = torch.zeros(B, C, H, W)
    group = 2 * CB if dt == SPLIT else CB
    for p in range(4):
        k0 = cb0 + p * group
        part = blocks[:, k0:k0 + CB]
        if dt == SPLIT:
            part = (part + blocks[:, k0 + CB:k0 + 2 * CB]) / ACT_SCALE
        x[:, :, p // 2::2, p % 2::2] = part.permute(0, 1, 4, 2, 3).reshape(B, C, H // 2, W // 2)
    return x, empty


def decode_all(taps):
    """{name: (x, pad, desc)} of Engine.taps()."""
    return {k: decode(d, raw) + (d,) for k, (d, raw) in taps.items()}
