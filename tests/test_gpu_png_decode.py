"""PNG decoding on the GPU: se_png_decode_u8 (engine.png_decode_u8 / png_decode_u8_packed) gives Pillow's pixels, byte for
byte, over the corpus of tests/util_png_decode.py (every encoder setting, hand-built streams, colour type and depth, size up
to 4000x2667) in mixed batches longer than one call (256 files), with the files the parser routes to Pillow among them; malformed files
each get a nonzero status and Pillow's result."""
import io
import zlib

import numpy as np
import pytest
from PIL import Image

from sketchedit_b200 import _lib, build, pngfile
from tests import util_png_decode as U


@pytest.fixture(scope="module")
def lib():
    build.build(verbose=False)
    return _lib.load()


def pillow(f, mode):
    try:
        return np.asarray(Image.open(io.BytesIO(f)).convert(mode))
    except Exception as e:   # noqa: BLE001  (Pillow's exception is the expected result)
        return e


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["RGB", "L"])
def test_mixed_batch_is_pillow(lib, mode):
    from sketchedit_b200 import engine as E
    small = U.corpus()
    files = U.corpus(big=True) + [(n, f) for n, f, _ in U.fallbacks()] + U.malformed() + small + small   # past one call
    files = [(n, f) for n, f in files if not isinstance(pillow(f, mode), Exception)]
    assert len(files) > E.PNG_DECODE_MAX_BATCH
    rng = np.random.default_rng(5)
    order = rng.permutation(len(files))
    got = E.png_decode_u8([files[i][1] for i in order], mode)
    for i, g in zip(order, got):
        name, f = files[i]
        want = pillow(f, mode)
        g = g.cpu().numpy()
        assert g.shape == want.shape and np.array_equal(g, want), name


@pytest.mark.gpu
def test_malformed_status_and_fallback(lib):
    import torch

    from sketchedit_b200 import engine as E
    for name, f in U.malformed():
        hd = pngfile.parse(f)
        staging, offs, lens = E.png_stage([hd])
        _, _, status = E.png_decode_u8_packed(staging.cuda(), offs, lens, [hd], "RGB")
        assert int(status.item()) != 0, name
        want = pillow(f, "RGB")
        if isinstance(want, Exception):
            with pytest.raises(type(want)):
                E.png_decode_u8([f], "RGB")
        else:
            assert np.array_equal(E.png_decode_u8([f], "RGB")[0].cpu().numpy(), want), name


@pytest.mark.gpu
def test_packed_offsets_and_guard_bytes(lib):
    """Files decoded into one buffer at odd offsets, RGB and L mixed: each file's pixels, and every byte between untouched."""
    import torch

    from sketchedit_b200 import engine as E
    files = [f for _, f in U.corpus()[:40]]
    heads = [pngfile.parse(f) for f in files]
    modes = ["RGB" if k % 3 else "L" for k in range(len(files))]
    staging, offs, lens = E.png_stage(heads)
    src = staging.cuda()
    sizes = [hd.h * hd.w * (3 if m == "RGB" else 1) for hd, m in zip(heads, modes)]
    out_offs, at = [], 5
    for s in sizes:
        out_offs.append(at)
        at += s + 7
    out = torch.full((at,), 0xA5, dtype=torch.uint8, device="cuda")
    _, _, status = E.png_decode_u8_packed(src, offs, lens, heads, modes, out=out, out_offsets=out_offs)
    assert status.cpu().tolist() == [0] * len(files)
    host = out.cpu().numpy()
    mask = np.ones(at, bool)
    for f, m, o, s in zip(files, modes, out_offs, sizes):
        assert np.array_equal(host[o:o + s], pillow(f, m).reshape(-1))
        mask[o:o + s] = False
    assert (host[mask] == 0xA5).all()


@pytest.mark.gpu
@pytest.mark.parametrize("batch", [1, 3])
def test_test_py_png_inputs_match_the_host_loader(lib, tmp_path, monkeypatch, batch):
    """test.py with the test_celeb.sh flags on PNG inputs, with --output_mask_dir and then --edit_mask_dir: every file equals
    what the run on the host loader's items writes. Among the inputs are sketches and edit masks of another size than their
    photo, and files Pillow decodes: an interlaced photo, a 16-bit sketch, JPEG bytes named .PNG (of another size) and a
    sketch the device decoder refuses."""
    import cv2
    import torch

    import data
    import test as test_entry
    from sketchedit_b200 import synth
    from tests.test_host_surface import _script_args
    from tests.util_parity import weights
    idir, mdir, cdir = (tmp_path / n for n in ("images", "edges", "ckpt"))
    idir.mkdir(); mdir.mkdir(); (cdir / "celeb").mkdir(parents=True)
    WM, WG = weights()
    torch.save(WM, cdir / "celeb" / "latest_net_M.pth")
    torch.save(WG, cdir / "celeb" / "latest_net_G.pth")
    names = []
    for j in range(5):
        img, sk = synth.synth_inputs(1, 64, 64, seed=70 + j)
        photo = ((img[0].permute(1, 2, 0) + 1) / 2 * 255).round().clamp(0, 255).to(torch.uint8).numpy()
        sketch = (sk[0, 0] * 255).to(torch.uint8).numpy()
        name = "im_%02d" % j
        if j == 0:   # Pillow decodes: an interlaced photo and a 16-bit sketch
            (idir / (name + ".png")).write_bytes(U.adam7(photo))
            Image.fromarray(sketch.astype(np.uint16) * 257).save(mdir / (name + ".PNG"))
        elif j == 2:   # Pillow decodes: JPEG bytes named .PNG, of another size than the photo
            Image.fromarray(photo).save(idir / (name + ".png"), compress_level=5)
            Image.fromarray(sketch).resize((80, 48)).save(mdir / (name + ".PNG"), "JPEG")
        elif j == 3:   # the device refuses it (too many bytes), Pillow decodes it; plus a device-decoded sketch of another size
            Image.fromarray(photo).save(idir / (name + ".png"), compress_level=6)
            (mdir / (name + ".PNG")).write_bytes(U.make_png(sketch[..., None], 8, 0, stream=lambda r: zlib.compress(r + b"\0" * 5)))
        else:
            Image.fromarray(photo).save(idir / (name + ".png"), compress_level=j + 3)
            s = Image.fromarray(sketch)
            (s.resize((72, 56)) if j == 4 else s).save(mdir / (name + ".PNG"))
        names.append(name)
    (tmp_path / "list.txt").write_text("".join(n + ".png\n" for n in names))
    base = _script_args("test_celeb.sh") + ["--image_dirs", str(idir), "--mask_dirs", str(mdir), "--image_lists",
                                            str(tmp_path / "list.txt"), "--checkpoints_dir", str(cdir), "--nThreads", "0",
                                            "--batchSize", str(batch), "--mask_postfix", ".PNG"]
    used = []
    loader_of = data.loader_of
    monkeypatch.setattr(data, "loader_of", lambda *a, **k: used.append(k.get("files")) or loader_of(*a, **k))

    def run(tag, extra, device):
        monkeypatch.setattr(test_entry, "PNG_DECODE_MIN_BATCH", 1 if device else 1 << 30)
        out = {d: tmp_path / (tag + d + ("_dev" if device else "_host")) for d in ("out", "mask")}
        argv = base + ["--output_dir", str(out["out"])] + (["--output_mask_dir", str(out["mask"])] if extra is None else extra)
        used.clear()
        test_entry.main(argv)
        assert (True in used) == device
        return out

    for device in (False, True):
        run("a", None, device)
    for n in names:
        for d in ("out", "mask"):
            assert (tmp_path / ("a" + d + "_dev") / (n + ".png")).read_bytes() == \
                (tmp_path / ("a" + d + "_host") / (n + ".png")).read_bytes(), (n, d)
    emdir = tmp_path / "amask_host"
    m = cv2.imread(str(emdir / "im_01.png"), cv2.IMREAD_GRAYSCALE)
    m[:, :20] = 255 - m[:, :20]
    assert cv2.imwrite(str(emdir / "im_01.png"), m)
    assert cv2.imwrite(str(emdir / "im_03.png"), cv2.resize(cv2.imread(str(emdir / "im_03.png"), cv2.IMREAD_GRAYSCALE), (50, 70)))
    for device in (False, True):
        run("b", ["--edit_mask_dir", str(emdir)], device)
    for n in names:
        assert (tmp_path / "bout_dev" / (n + ".png")).read_bytes() == (tmp_path / "bout_host" / (n + ".png")).read_bytes(), n
