"""Pillow-exact bicubic resize (se_resize.cu, engine.resize_u8, DemoProcessor(resize='device')).

CPU: the coefficient tables of se_resize_coeffs, run through the fixed-point passes in numpy, reproduce PIL.Image.resize bit
for bit. GPU: the kernels reproduce Pillow in ragged batches, write nothing outside their destination slices, and the device
resize flow of the demo returns exactly what the Pillow flow returns."""
import ctypes
import os
import re
import shutil
import subprocess
import threading

import numpy as np
import PIL
import pytest
from PIL import Image

from sketchedit_b200 import _lib, build

# (src (h, w), dst (h, w)): each axis alone and both, upscales up to x5.7, downscales down to 1/11.8, the demo's floor-to-8
# sizes, and an 80-to-1 downscale on each axis (ksize 321)
CASES = [
    ((75, 100), (72, 96)), ((64, 90), (64, 88)), ((2667, 40), (2664, 40)), ((481, 641), (480, 640)), ((667, 1000), (664, 1000)),
    ((97, 131), (96, 128)), ((30, 40), (171, 40)), ((40, 30), (40, 171)), ((33, 21), (188, 120)), ((236, 50), (20, 50)),
    ((50, 236), (50, 20)), ((472, 354), (40, 30)), ((100, 100), (37, 251)), ((17, 300), (95, 23)), ((1, 50), (7, 9)),
    ((5, 5), (1, 1)), ((64, 64), (63, 65)), ((123, 457), (200, 200)), ((8, 8), (16, 16)), ((300, 200), (150, 100)),
    ((160, 8), (2, 8)), ((8, 1600), (8, 20)),
]
SAME = [((40, 56), (40, 56)), ((13, 7), (13, 7))]       # Pillow returns a copy; so must the kernels


@pytest.fixture(scope="module")
def lib():
    build.build(verbose=False)
    return _lib.load()


def _image(hw, channels, seed):
    rs = np.random.RandomState(seed)
    a = rs.randint(0, 256, hw + ((3,) if channels == 3 else ()), dtype=np.uint8)
    # smooth regions and hard edges next to the noise: both signs of every tap and the clamp at 0 and 255 are reached
    a[: hw[0] // 3] = 255
    a[hw[0] // 3: hw[0] // 2] = 0
    return a


def _pillow(a, dst):
    return np.array(Image.fromarray(a).resize((dst[1], dst[0])))


def _coeffs(lib, n_in, n_out):
    ksize = lib.se_resize_coeffs(n_in, n_out, None, None, 0)
    assert ksize > 0
    bounds = np.zeros((n_out, 2), np.int32)
    coeffs = np.zeros((n_out, ksize), np.int32)
    assert lib.se_resize_coeffs(n_in, n_out, bounds.ctypes.data, coeffs.ctypes.data, coeffs.size) == ksize
    return bounds, coeffs


def _pass(lib, a, axis, n_out):
    """One fixed-point pass of Pillow's resampler along `axis` (0 rows, 1 columns) of a uint8 [h, w, c] array."""
    n_in = a.shape[axis]
    bounds, coeffs = _coeffs(lib, n_in, n_out)
    ksize = coeffs.shape[1]
    taps = np.arange(ksize)
    assert (coeffs[taps[None, :] >= bounds[:, 1:2]] == 0).all()
    idx = np.minimum(bounds[:, :1] + taps[None, :], n_in - 1)          # [n_out, ksize]; taps beyond n carry weight 0
    src = np.moveaxis(a, axis, 0).astype(np.int64)                      # [n_in, other, c]
    acc = (1 << 21) + np.einsum("okxc,ok->oxc", src[idx], coeffs.astype(np.int64))
    assert np.abs(acc).max() < 2 ** 31                                  # the kernels accumulate in int32
    return np.moveaxis(np.clip(acc >> 22, 0, 255).astype(np.uint8), 0, axis)


def _numpy_resize(lib, a, dst):
    a3 = a if a.ndim == 3 else a[..., None]
    if a3.shape[1] != dst[1]:
        a3 = _pass(lib, a3, 1, dst[1])
    if a3.shape[0] != dst[0]:
        a3 = _pass(lib, a3, 0, dst[0])
    return a3 if a.ndim == 3 else a3[..., 0]


@pytest.mark.parametrize("channels", [1, 3])
def test_coefficients_reproduce_pillow(lib, channels):
    for i, (src, dst) in enumerate(CASES):
        a = _image(src, channels, seed=i)
        got, want = _numpy_resize(lib, a, dst), _pillow(a, dst)
        assert got.shape == want.shape and np.array_equal(got, want), \
            "%s -> %s, %d channels: %d bytes differ from Pillow %s" % (src, dst, channels, int((got != want).sum()), PIL.__version__)


def test_coefficient_table_shape_and_errors(lib):
    assert lib.se_resize_coeffs(160, 2, None, None, 0) == 321            # 80-to-1: support 160, ksize 2 * 160 + 1
    assert lib.se_resize_coeffs(40, 171, None, None, 0) == 5             # upscale: support 2
    bounds, coeffs = _coeffs(lib, 100, 37)
    assert np.abs(coeffs.sum(axis=1) - (1 << 22)).max() <= coeffs.shape[1]     # each row sums to 1.0 up to rounding
    assert (bounds[:, 0] >= 0).all() and (bounds.sum(axis=1) <= 100).all()
    assert lib.se_resize_coeffs(0, 5, None, None, 0) == -1
    b = np.zeros(2 * 37, np.int32)
    assert lib.se_resize_coeffs(100, 37, b.ctypes.data, b.ctypes.data, 10) == -1
    assert b"ksize" in lib.se_last_error()


def test_resize_call_validates_on_the_host(lib):
    need = ctypes.c_longlong(0)
    L = ctypes.c_longlong
    hw = (ctypes.c_int * 66)(*([10] * 66))
    off, pitch = (L * 33)(*([0] * 33)), lambda c: (L * 33)(*([10 * c] * 33))       # packed rows: pitch w * channels
    assert lib.se_resize_window_u8(None, pitch(2), hw, None, off, hw, 1, 2, 0, None, ctypes.byref(need), None) != 0      # channels
    assert lib.se_resize_window_u8(None, pitch(1), hw, None, off, hw, 1, 1, 1, None, ctypes.byref(need), None) != 0      # swap_rb, 1 ch
    assert lib.se_resize_window_u8(None, pitch(3), hw, None, off, hw, 33, 3, 0, None, ctypes.byref(need), None) != 0     # batch bound
    src_hw, dst_hw = (ctypes.c_int * 2)(75, 100), (ctypes.c_int * 2)(72, 96)
    src_pitch = (L * 1)(300)
    assert lib.se_resize_window_u8(None, src_pitch, src_hw, None, off, dst_hw, 1, 3, 0, None, ctypes.byref(need), None) == 0
    assert need.value >= 75 * 96 * 3                                                                          # the intermediate
    assert lib.se_resize_window_u8(None, src_pitch, src_hw, None, off, (ctypes.c_int * 2)(75, 96), 1, 3, 0, None, ctypes.byref(need),
                                   None) == 0
    assert need.value == 0                                                                                    # one axis: no scratch
    assert lib.se_resize_set_table_cache_limit(-1) != 0 and lib.se_resize_set_table_cache_limit(0) == 0


def test_resize_kernels_do_not_spill(tmp_path):
    """Every kernel of se_resize.cu, compiled for sm_90a with the library's flags, keeps everything in registers: the two
    horizontal passes, the vertical pass, feather_kernel, and one paste_v_kernel taking PasteList that runs every paste,
    feathered or not."""
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not available")
    if not (os.path.isabs(nvcc) and os.path.exists(nvcc)) and not shutil.which(nvcc):
        pytest.skip("nvcc not available")
    flags = [f for f in build.NVCC_FLAGS if not f.startswith("--use_fast_math")]   # as build.build() compiles
    cmd = [nvcc] + flags + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "se_resize.cu"), "-o", str(tmp_path / "r.o")]
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert out.returncode == 0, out.stdout[-3000:]
    lines = out.stdout.splitlines()
    entries = [i for i, ln in enumerate(lines) if re.search(r"Compiling entry function '\w+'", ln)]
    names = [re.search(r"'(\w+)'", lines[i]).group(1) for i in entries]
    count = lambda k: sum(k in n for n in names)
    assert len(names) == 5 and count("resize_h_kernel") == 2 and count("resize_v_kernel") == 1, names
    assert count("feather_kernel") == 1 and count("paste_v_kernel") == 1, names
    regs = {}
    for i, name in zip(entries, names):
        m = next(s for s in (re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", ln)
                             for ln in lines[i:]) if s)
        assert m.groups() == ("0", "0", "0"), lines[i:i + 4]
        regs[name] = int(next(s for s in (re.search(r"Used (\d+) registers", ln) for ln in lines[i:]) if s).group(1))
    paste = next(n for n in names if "paste_v_kernel" in n)
    assert "PasteList" in paste, names
    # 256 threads per block: up to 80 registers keeps paste_v_kernel at 3 blocks per SM, as with the 77 it used before feathering
    assert regs[paste] <= 80, regs


# ---------------------------------------------------------------------------------------------------------------- GPU
def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("channels", [1, 3])
@pytest.mark.parametrize("swap_rb", [False, True])
def test_ragged_batch_matches_pillow(lib, channels, swap_rb):
    """One call over every case of the matrix (mixed source sizes, copies, single-axis resizes, up- and downscales)."""
    if swap_rb and channels == 1:
        pytest.skip("swap_rb needs 3 channels")
    from sketchedit_b200.engine import resize_u8
    cases = CASES + SAME
    imgs = [_image(src, channels, seed=100 + i) for i, (src, _) in enumerate(cases)]
    got = resize_u8([_cuda(a) for a in imgs], [dst for _, dst in cases], swap_rb=swap_rb)
    for a, (src, dst), g in zip(imgs, cases, got):
        want = _pillow(a, dst) if src != dst else a
        if swap_rb:
            want = want[..., ::-1]
        g = g.cpu().numpy()
        assert g.shape == want.shape and np.array_equal(g, want), \
            "%s -> %s: %d bytes differ (Pillow %s)" % (src, dst, int((g != want).sum()), PIL.__version__)


@pytest.mark.gpu
def test_photo_sized_image(lib):
    from sketchedit_b200.engine import resize_u8
    a = _image((2667, 4000), 3, seed=7)
    (g,) = resize_u8([_cuda(a)], [(2664, 4000)])
    assert np.array_equal(g.cpu().numpy(), _pillow(a, (2664, 4000))), PIL.__version__


@pytest.mark.gpu
def test_table_cache_eviction_keeps_the_tables_a_call_launches_with(lib):
    """Past the cache limit the cached tables are dropped before a call looks any up: an image whose tables were cached and
    a later image of the same call whose tables are new both come out right, and the cache then holds this call's tables."""
    import torch

    from sketchedit_b200.engine import resize_table_cache_bytes, resize_u8, set_resize_table_cache_limit
    table = lambda n_in, n_out: n_out * (2 + lib.se_resize_coeffs(n_in, n_out, None, None, 0)) * 4
    a, b = _image((75, 100), 3, seed=300), _image((83, 139), 3, seed=301)      # b: lengths no other test resizes
    resize_u8([_cuda(a)], [(72, 96)])                       # caches the tables 100 -> 96 and 75 -> 72
    torch.cuda.synchronize()
    set_resize_table_cache_limit(1)
    try:
        got = resize_u8([_cuda(a), _cuda(b)], [(72, 96), (80, 136)])
        torch.cuda.synchronize()
        held = table(100, 96) + table(75, 72) + table(139, 136) + table(83, 80)
        assert resize_table_cache_bytes() == held
        for g, x, d in zip(got, (a, b), ((72, 96), (80, 136))):
            assert np.array_equal(g.cpu().numpy(), _pillow(x, d)), d
        (g,) = resize_u8([_cuda(b)], [(80, 136)])           # every table cached: nothing is dropped
        assert resize_table_cache_bytes() == held and np.array_equal(g.cpu().numpy(), _pillow(b, (80, 136)))
    finally:
        set_resize_table_cache_limit(0)


@pytest.mark.gpu
@pytest.mark.parametrize("channels", [1, 3])
def test_writes_stay_inside_the_destination_slices(lib, channels):
    """Canary bytes before, between and after the destination slices (odd offsets included) are left untouched."""
    import torch

    from sketchedit_b200.engine import resize_u8_packed
    cases = CASES + SAME
    imgs = [_image(src, channels, seed=200 + i) for i, (src, _) in enumerate(cases)]
    src_offs, total = [], 0
    for a in imgs:
        src_offs.append(total)
        total += a.nbytes + 3
    src = np.zeros(total, np.uint8)
    for a, o in zip(imgs, src_offs):
        src[o:o + a.nbytes] = a.reshape(-1)
    dst_offs, pos = [], 37
    for _, dst in cases:
        dst_offs.append(pos)
        pos += dst[0] * dst[1] * channels + 5 + pos % 3
    out = torch.full((pos + 41,), 0xA5, dtype=torch.uint8, device="cuda")
    src_dev = _cuda(src)
    resize_u8_packed(src_dev, src_offs, [s for s, _ in cases], [d for _, d in cases], channels, swap_rb=channels == 3, out=out,
                     dst_offsets=dst_offs)
    o = out.cpu().numpy()
    inside = np.zeros(o.size, bool)
    for (s, d), a, off in zip(cases, imgs, dst_offs):
        n = d[0] * d[1] * channels
        inside[off:off + n] = True
        want = (_pillow(a, d) if s != d else a)
        want = want[..., ::-1] if channels == 3 else want
        assert np.array_equal(o[off:off + n], np.ascontiguousarray(want).reshape(-1)), (s, d)
    assert (o[~inside] == 0xA5).all()
    assert np.array_equal(src_dev.cpu().numpy(), src)


def _requests():
    """The eight requests of the serving test, a 4000x2667 photo, and a mask of another size than its photo."""
    rs = np.random.RandomState(11)
    reqs = []
    for i in range(8):
        h, w = ((75, 100), (64, 90))[i % 2]
        m = np.zeros((h, w), np.uint8)
        m[10 + i:40, 20:22 + i] = 255
        reqs.append((Image.fromarray(rs.randint(0, 256, (h, w, 3), dtype=np.uint8)), Image.fromarray(m)))
    big = rs.randint(0, 256, (2667, 4000, 3), dtype=np.uint8)
    big[:, :1500] = 255 - big[:, :1500] // 4
    m = np.zeros((2667, 4000), np.uint8)
    m[900:1300, 1500:2600] = 255
    reqs.append((Image.fromarray(big), Image.fromarray(m)))
    m = np.zeros((150, 200), np.uint8)            # the canvas sent a mask at twice the photo's size
    m[30:90, 40:46] = 255
    reqs.append((Image.fromarray(rs.randint(0, 256, (75, 100, 3), dtype=np.uint8)), Image.fromarray(m)))
    return reqs


def _serve(model, reqs, resize):
    from sketchedit_b200.serving import DemoProcessor
    proc = DemoProcessor(model, max_batch=4, max_wait_ms=50.0, resize=resize)
    got = [None] * len(reqs)

    def worker(i):
        got[i] = proc.process_image(*reqs[i])

    ts = [threading.Thread(target=worker, args=(i,)) for i in range(len(reqs))]
    try:
        [t.start() for t in ts]
        [t.join() for t in ts]
    finally:
        proc.close()
    return got, proc.batcher.batches


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["bf16", "fp32_direct"])
def test_device_resize_flow_equals_the_pillow_flow(lib, precision):
    """The forward is batch-independent bit for bit, so any difference between the two flows is a resize difference."""
    from tests.test_gpu_configs import _model
    model = _model(precision)
    reqs = _requests()
    host, _ = _serve(model, reqs, "host")
    dev, batches = _serve(model, reqs, "device")
    assert sum(n for _, n in batches) == len(reqs) and len(batches) < len(reqs)     # concurrent requests still share forwards
    for (img, _), h, d in zip(reqs, host, dev):
        assert d.size == img.size and d.mode == h.mode == "RGB"
        hd, dd = np.array(h), np.array(d)
        assert np.array_equal(hd, dd), (img.size, int((hd != dd).sum()))
