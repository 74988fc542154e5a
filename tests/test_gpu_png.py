"""PNG encoding on the GPU: se_png_encode_u8 (engine.png_encode_u8 / png_encode_u8_packed) writes cv2.imencode's bytes over the
CPU matrix of sizes, contents and channel counts, in mixed batches longer than one call of windows with odd pitches that overlap,
from BGR and RGB sources, and nothing past each file; EditSession.png() is the cv2 statement on the session's photo after
chains of edits and undos, and a session gives its device memory back on close()."""
import gc

import cv2
import numpy as np
import pytest

from sketchedit_b200 import _lib, build
from tests import util_png as P
from tests.test_png import CONTENTS, SIZES, content, cv2_png, window_steps


@pytest.fixture(scope="module")
def lib():
    build.build(verbose=False)
    return _lib.load()


def _cases(rs):
    """(image, channels) over the CPU matrix: every size, content and channel count, the window steps and a 2667x4000 photo."""
    out = []
    for c in (1, 3):
        for hw in SIZES:
            out += [(content(kind, *hw, c, rs), c) for kind in CONTENTS]
    out += [(content(kind, h, w, c, rs), c) for h, w, c in window_steps() for kind in ("noise", "gradient")]
    out += [(content("places_11_512x408.npz", 2667, 4000, 3, rs), 3), (content("flat", 2667, 4000, 1, rs), 1)]
    return out


@pytest.mark.gpu
def test_kernels_are_cv2(lib):
    """The whole matrix, BGR sources for colour, in batches of up to 45 images (past one call's 32) per channel count."""
    import torch

    from sketchedit_b200.engine import png_encode_u8
    rs = np.random.RandomState(21)
    cases = _cases(rs)
    for c in (1, 3):
        imgs = [a for a, k in cases if k == c]
        for b0 in range(0, len(imgs), 45):
            batch = imgs[b0:b0 + 45]
            got = png_encode_u8([torch.from_numpy(a).cuda() for a in batch], swap_rb=True)
            for a, g in zip(batch, got):
                want = cv2_png(a)
                assert g == want, (a.shape, len(g), len(want))


@pytest.mark.gpu
@pytest.mark.parametrize("channels", [1, 3])
def test_mixed_batches_overlapping_windows_and_guard_bytes(lib, channels):
    """40 windows of two sources with odd pitches, overlapping and repeated, at mixed sizes, into one buffer with odd gaps:
    each file is cv2's of the crop (RGB sources read with swap_rb=False), and every byte past a file is untouched."""
    import torch

    from sketchedit_b200.engine import png_encode_u8_packed
    rs = np.random.RandomState(3 + channels)
    sources, bufs, pitches = [], [], []
    for h, w, extra in ((301, 403, 5), (64, 33, 1)):
        a = content("places_11_512x408.npz", h, w, channels, rs)
        if channels == 3:
            a[h // 2:, w // 2:] = rs.randint(0, 256, (h - h // 2, w - w // 2, 3))
        else:
            a[h // 2:, w // 2:] = rs.randint(0, 256, (h - h // 2, w - w // 2))
        p = channels * w + extra
        buf = np.full(h * p + 7, 0x5A, np.uint8)
        rgb = a[:, :, ::-1] if channels == 3 else a          # the device holds RGB
        buf[:h * p].reshape(h, p)[:, :channels * w] = rgb.reshape(h, -1)
        sources.append(a)
        bufs.append(torch.from_numpy(buf).cuda())
        pitches.append(p)
    wins = [(0, (0, 0, 403, 301)), (0, (0, 0, 403, 301)), (1, (0, 0, 33, 64)), (0, (400, 298, 403, 301)), (0, (5, 7, 6, 8))]
    for _ in range(35):
        s = int(rs.randint(0, 2))
        h, w = sources[s].shape[:2]
        bh, bw = int(rs.randint(1, h + 1)), int(rs.randint(1, w + 1))
        y, x = int(rs.randint(0, h - bh + 1)), int(rs.randint(0, w - bw + 1))
        wins.append((s, (x, y, x + bw, y + bh)))
    offs, pos = [], 3
    for s, b in wins:
        offs.append(pos)
        pos += P.max_bytes(b[3] - b[1], b[2] - b[0], channels) + 5
    out = torch.full((pos + 11,), 0xA5, dtype=torch.uint8, device="cuda")
    _, _, nbytes = png_encode_u8_packed([bufs[s] for s, _ in wins], [b[1] * pitches[s] + channels * b[0] for s, b in wins],
                                        [pitches[s] for s, _ in wins], [(b[3] - b[1], b[2] - b[0]) for _, b in wins], channels,
                                        swap_rb=False, out=out, out_offsets=offs)
    got, lens = out.cpu().numpy(), nbytes.cpu().tolist()
    written = np.zeros(got.size, bool)
    for (s, b), o, n in zip(wins, offs, lens):
        want = cv2_png(np.ascontiguousarray(sources[s][b[1]:b[3], b[0]:b[2]]))
        assert got[o:o + n].tobytes() == want, (b, n, len(want))
        written[o:o + n] = True
    assert (got[~written] == 0xA5).all()
    for buf, a, p in zip(bufs, sources, pitches):              # the sources are only read
        h, w = a.shape[:2]
        assert (buf.cpu().numpy()[:h * p].reshape(h, p)[:, channels * w:] == 0x5A).all()


@pytest.mark.gpu
def test_max_bytes_and_checks(lib):
    import torch

    from sketchedit_b200.engine import png_encode_u8, png_encode_u8_packed, png_max_bytes
    for h, w, c in ((1, 1, 1), (256, 256, 3), (2667, 4000, 3), (65535, 65535, 1)):
        assert png_max_bytes(h, w, c) == P.max_bytes(h, w, c)
    for bad in ((0, 5, 3), (5, 65536, 3), (5, 5, 2)):
        with pytest.raises(ValueError):
            png_max_bytes(*bad)
    t = torch.zeros(10, 10, 3, dtype=torch.uint8, device="cuda")
    with pytest.raises(_lib.SketchEditB200Error):
        png_encode_u8([t, t[:, :, 0]])
    with pytest.raises(_lib.SketchEditB200Error, match="pitch"):
        png_encode_u8_packed(t.view(-1), [0], [29], [(10, 10)], 3)
    with pytest.raises(_lib.SketchEditB200Error, match="outside"):
        png_encode_u8_packed(t.view(-1), [3], [30], [(10, 10)], 3)
    with pytest.raises(ValueError):
        png_encode_u8_packed(t.view(-1), [0], [30], [(10, 10)], 2)


@pytest.mark.gpu
def test_strided_views_are_encoded_where_they_lie(lib):
    import torch

    from sketchedit_b200.engine import png_encode_u8
    rs = np.random.RandomState(9)
    a = content("face_602_256x256.npz", 300, 401, 3, rs)     # BGR
    t = torch.from_numpy(np.ascontiguousarray(a[:, :, ::-1])).cuda()
    boxes = [(0, 0, 401, 300), (17, 3, 250, 77), (400, 0, 401, 300), (0, 299, 401, 300), (100, 100, 116, 116)]
    got = png_encode_u8([t[b[1]:b[3], b[0]:b[2]] for b in boxes])
    for b, g in zip(boxes, got):
        assert g == cv2_png(np.ascontiguousarray(a[b[1]:b[3], b[0]:b[2]])), b
    g = t[:, :, 1].contiguous()
    got = png_encode_u8([g[b[1]:b[3], b[0]:b[2]] for b in boxes])
    for b, p in zip(boxes, got):
        assert p == cv2_png(np.ascontiguousarray(a[b[1]:b[3], b[0]:b[2], 1])), b


@pytest.mark.gpu
def test_stream_png_is_cv2_of_the_uint8_results(lib):
    """inference_stream(png=...) yields cv2's files of the arrays uint8 mode yields for the same batches: a ragged last batch,
    batches with and without an edit mask, with and without mask files."""
    import torch

    from sketchedit_b200 import synth
    from tests.test_gpu_configs import _model
    model = _model("bf16")
    rs = np.random.RandomState(16)
    batches = []
    for i, (b, h, w) in enumerate(((3, 64, 64), (3, 64, 64), (3, 64, 64), (2, 64, 64), (1, 96, 64))):
        _, sk = synth.synth_inputs(b, h, w, seed=90 + i)
        d = {"image_u8": torch.from_numpy(rs.randint(0, 256, (b, h, w, 3), dtype=np.uint8)).pin_memory(),
             "mask_u8": (sk[:, 0] * 255).to(torch.uint8).pin_memory(), "tag": i}
        if i in (1, 3):
            d["edit_mask_u8"] = torch.from_numpy((rs.rand(b, h, w) > 0.6).astype(np.uint8) * rs.randint(1, 256)).pin_memory()
        batches.append(d)
    with torch.no_grad():
        want = [(a.clone().numpy(), m.clone().numpy(), d["tag"])
                for a, m, d in model.inference_stream(iter(batches), uint8=True, with_data=True)]
        for png in (("image", "mask"), ("image",)):
            got = list(model.inference_stream(iter(batches), uint8=True, with_data=True, png=png))
            assert [d["tag"] for _, _, d in got] == [t for _, _, t in want]
            for (files, mfiles, _), (a, m, _) in zip(got, want):
                assert files == [cv2_png(x) for x in a]
                assert mfiles == ([cv2_png(x) for x in m] if len(png) == 2 else None)
    with pytest.raises(ValueError):
        next(model.inference_stream(iter(batches), png=("image",)))


@pytest.mark.gpu
def test_test_py_writes_cv2_files(lib, tmp_path):
    """test.py with the test_celeb.sh flags on a list file and checkpoints, with --output_mask_dir and then --edit_mask_dir on
    those masks (some of them changed): every file is what cv2.imwrite writes for the arrays of the uint8 stream."""
    import torch
    from PIL import Image

    import data
    import models
    import test as test_entry
    from options.test_options import TestOptions
    from sketchedit_b200 import synth
    from tests.test_host_surface import _script_args
    from tests.util_parity import weights
    idir, mdir, odir, omdir, cdir = (tmp_path / n for n in ("images", "edges", "out", "out_mask", "ckpt"))
    idir.mkdir(); mdir.mkdir(); (cdir / "celeb").mkdir(parents=True)
    WM, WG = weights()
    torch.save(WM, cdir / "celeb" / "latest_net_M.pth")
    torch.save(WG, cdir / "celeb" / "latest_net_G.pth")
    names = []
    for j, (H, W) in enumerate(((64, 64), (64, 64), (64, 64), (96, 64))):
        img, sk = synth.synth_inputs(1, H, W, seed=50 + j)
        Image.fromarray(((img[0].permute(1, 2, 0) + 1) / 2 * 255).round().clamp(0, 255).to(torch.uint8).numpy()).save(idir / ("im_%02d.png" % j))
        Image.fromarray((sk[0, 0] * 255).to(torch.uint8).numpy()).save(mdir / ("im_%02d.png" % j))
        names.append("im_%02d" % j)
    (tmp_path / "list.txt").write_text("".join(n + ".png\n" for n in names))
    base = _script_args("test_celeb.sh") + ["--image_dirs", str(idir), "--mask_dirs", str(mdir), "--image_lists",
                                            str(tmp_path / "list.txt"), "--checkpoints_dir", str(cdir), "--nThreads", "0",
                                            "--batchSize", "3"]

    def arrays(argv):
        opt = TestOptions().parse(argv)
        model = models.create_model(opt).eval()
        out = {}
        with torch.no_grad():
            for bgr, mk, batch in model.inference_stream(data.create_dataloader(opt), uint8=True, with_data=True):
                for b, p in enumerate(batch["path"]):
                    out[p] = (bgr[b].numpy().copy(), mk[b].numpy().copy())
        return out

    argv = base + ["--output_dir", str(odir), "--output_mask_dir", str(omdir)]
    test_entry.main(argv)
    want = arrays(argv)
    for n in names:
        bgr, mk = want[n + ".png"]
        assert (odir / (n + ".png")).read_bytes() == cv2_png(bgr), n
        assert (omdir / (n + ".png")).read_bytes() == cv2_png(mk), n
    m = cv2.imread(str(omdir / "im_01.png"), cv2.IMREAD_GRAYSCALE)
    m[:, :20] = 255 - m[:, :20]
    assert cv2.imwrite(str(omdir / "im_01.png"), m)
    odir2 = tmp_path / "out2"
    argv = base + ["--output_dir", str(odir2), "--edit_mask_dir", str(omdir)]
    test_entry.main(argv)
    want = arrays(argv)
    for n in names:
        assert (odir2 / (n + ".png")).read_bytes() == cv2_png(want[n + ".png"][0]), n


def _cv2_of(img, box=None):
    a = np.asarray(img if box is None else img.crop(box))
    return cv2_png(np.ascontiguousarray(a[:, :, ::-1]))


@pytest.mark.gpu
def test_session_png_is_cv2_after_edits_and_undo(lib):
    from sketchedit_b200.serving import DemoProcessor
    from tests.test_gpu_configs import _model
    from tests.test_gpu_edit_session import _photo, _steps
    model = _model("bf16")
    rs = np.random.RandomState(29)
    for w, h in ((1000, 667), (4000, 2667)):
        img = _photo(w, h, rs)
        steps = _steps(w, h, rs)
        for resize in ("device", "host"):
            proc = DemoProcessor(model, max_batch=4, resize=resize, region_size=(256, 256))
            try:
                s = proc.open_session(img)
                assert s.png() == _cv2_of(s.image())
                for k, (mask, em, region, off) in enumerate(steps):
                    r = s.edit(mask, em, region=region, offset=off)
                    cur = s.image()
                    assert s.png() == _cv2_of(cur), (w, h, resize, k)
                    for b in r.boxes[:2]:
                        assert s.png(box=b) == _cv2_of(cur, b), (w, h, resize, k, b)
                for k in range(3):
                    boxes, _ = s.undo()
                    assert s.png(box=boxes[0]) == _cv2_of(s.image(), boxes[0]), (w, h, resize, k)
            finally:
                proc.close()


@pytest.mark.gpu
def test_session_png_checks_and_releases_memory(lib):
    import torch

    from sketchedit_b200.serving import DemoProcessor
    from tests.test_gpu_configs import _model
    from tests.test_gpu_edit_session import _photo
    rs = np.random.RandomState(7)
    img = _photo(4000, 2667, rs)
    proc = DemoProcessor(_model("bf16"), region_size=(256, 256))

    def allocated():
        gc.collect()
        torch.cuda.synchronize()
        return torch.cuda.memory_allocated()

    try:
        warm = proc.open_session(img)
        warm.png()
        warm.close()
        start = allocated()
        s = proc.open_session(img)
        assert s.png() == _cv2_of(img.convert("RGB"))
        box = tuple(np.int64(v) for v in (5, 7, 1001, 667))
        assert s.png(box=box) == _cv2_of(img.convert("RGB"), (5, 7, 1001, 667))
        for bad in [(0, 0, 4001, 10), (5, 5, 5, 10), (0, 0, 10), (False, 0, 10, 10)]:
            with pytest.raises(ValueError):
                s.png(box=bad)
        s.close()
        assert allocated() == start
        with pytest.raises(RuntimeError, match="closed"):
            s.png()
    finally:
        proc.close()
