"""EvaluateSet's page preparation against the golden fixture (tests/golden/evaluate_set.npz) recorded from the reference's own
EvaluateSet.resize_pad_tensor: the numpy restatement of Pillow's bicubic resampler (tests/evaluate_set_ref.py) bit for bit,
the Normalize and pad, and ops.evaluate_set_geometry on every recorded size.  A last test re-runs the reference from the
staged Dataloader.py (oracle/_ref) when that copy and the packages it imports (cv2, PIL, torchvision) are there."""
import importlib.util
import os

import numpy as np
import pytest

import evaluate_set_ref as R
from conftest import GOLDEN, ROOT
from text_segmentation_image_inpainting_b200 import ops

MEAN_STD = ((0.4935, 0.4563, 0.4544), (0.3769, 0.3615, 0.3566))


def _golden():
    return np.load(os.path.join(GOLDEN, "evaluate_set.npz"))


def _names(g):
    return sorted({k.split(".")[0] for k in g.files if "." in k})


def _case(g, k):
    page = g[k + ".page"]
    H, W = page.shape[:2]
    return page, H, W, int(g[k + ".resize"]), tuple(int(v) for v in g[k + ".pad"])


def test_fixture_covers_the_cases():
    g = _golden()
    names = _names(g)
    cases = [_case(g, k) + (g[k + ".resized"].shape[:2],) for k in names]
    # the 592 quirk in both orientations: a landscape page gets 8 columns on the right and no bottom padding
    assert any(r == 600 and (rh, rw) == (432, 592) and pad == (0, 8, 0, 0) for _, H, W, r, pad, (rh, rw) in cases)
    assert any(r == 600 and rh == 592 and pad[1] > 0 for _, H, W, r, pad, (rh, rw) in cases)
    # reductions of about 16 on both axes at small resizes, upscaling, a square page, a short side off the multiple of 8
    small = [(H / rh, W / rw) for _, H, W, r, pad, (rh, rw) in cases if r < 600]
    assert len(small) >= 3 and all(15.9 <= a <= 16 and 15.9 <= b <= 16 for a, b in small)
    assert any(rh > H and rw > W for _, H, W, r, pad, (rh, rw) in cases)
    assert any(H == W for _, H, W, *_ in cases)
    assert any(min(H, W) % 8 for _, H, W, *_ in cases)
    geo = g["geometry"]
    quirks = [L for L in range(281, 8001) if int(L * (600 / L)) < 600]
    assert len(quirks) == 39
    for L in quirks:                                                    # both orientations of every quirk long side
        assert ((geo[:, 0] == L) & (geo[:, 2] == 600) & (geo[:, 4] == 592)).any(), L
        assert ((geo[:, 1] == L) & (geo[:, 2] == 600) & (geo[:, 3] == 592)).any(), L


def test_restatement_matches_golden():
    g = _golden()
    for k in _names(g):
        page, H, W, resize, pad = _case(g, k)
        want = g[k + ".resized"]
        rh, rw = want.shape[:2]
        chw = np.ascontiguousarray(page.transpose(2, 0, 1))
        assert np.array_equal(R.page_bytes(R.to_tensor(chw)), chw), k             # to_pil_image gives to_tensor's bytes back
        got = R.resize_bytes(chw, rh, rw)
        assert np.array_equal(got.transpose(1, 2, 0), want), k
        x = g[k + ".input"]
        assert x.shape == (1, 3, rh + pad[3], rw + pad[1]), k
        assert np.array_equal(R.normalize_pad(R.to_tensor(got)[None], *MEAN_STD, *x.shape[2:]), x), k
        assert np.array_equal(R.page_resize(R.to_tensor(chw)[None], rh, rw)[0], R.to_tensor(got)), k


def test_page_bytes_clamps_and_truncates():
    v = np.array([np.nan, -np.inf, -1.0, 0.0, 0.5 / 255, 1.0 / 255, 0.99999, 1.0, 1.5, np.inf], np.float32)
    assert R.page_bytes(v).tolist() == [0, 0, 0, 0, 0, 1, 254, 255, 255, 255]


def test_geometry_matches_golden():
    g = _golden()
    rows = [tuple(int(v) for v in r) for r in g["geometry"]]
    for k in _names(g):
        page, H, W, resize, pad = _case(g, k)
        rh, rw = g[k + ".resized"].shape[:2]
        rows.append((W, H, resize, rh, rw, *pad))
    refused = 0
    for W, H, resize, rh, rw, *pad in rows:
        if H > ops.PAGE_RESIZE_MAX_REDUCTION * rh or W > ops.PAGE_RESIZE_MAX_REDUCTION * rw:
            with pytest.raises(ValueError, match="reduction"):
                ops.evaluate_set_geometry(H, W, resize)
            refused += 1
            continue
        assert ops.evaluate_set_geometry(H, W, resize) == ((rh, rw), tuple(pad)), (W, H, resize)
    assert refused >= 1


def test_geometry_refuses():
    for resize in (0, -8, 4, 601):
        with pytest.raises(ValueError, match="multiple of 8"):
            ops.evaluate_set_geometry(800, 600, resize)
    with pytest.raises(ValueError, match="resizes to"):
        ops.evaluate_set_geometry(2000, 10, 600)                    # the short side rounds to 0
    with pytest.raises(ValueError, match="reduction"):
        ops.evaluate_set_geometry(3508, 2480, 128)
    with pytest.raises(ValueError):
        ops.evaluate_set_geometry(0, 100, 600)


def test_golden_matches_reference_dataloader():
    for pkg in ("cv2", "PIL", "torchvision"):
        pytest.importorskip(pkg)
    if not os.path.exists(os.path.join(ROOT, "oracle", "_ref", "Dataloader.py")):
        pytest.skip("the reference is not staged at oracle/_ref")
    spec = importlib.util.spec_from_file_location("make_golden_evaluate_set", os.path.join(GOLDEN, "make_golden_evaluate_set.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    dl = gen.load_dataloader()
    g = _golden()
    assert sorted(gen.CASES) == _names(g)
    for name, (W, H, resize) in gen.CASES.items():
        page = gen.case_page(name, W, H)
        assert np.array_equal(page, g[name + ".page"]) and int(g[name + ".resize"]) == resize, name
        resized, x, pad = gen.reference_prepare(dl, page, resize)
        assert np.array_equal(resized, g[name + ".resized"]), name
        assert np.array_equal(x, g[name + ".input"]), name
        assert np.array_equal(pad, g[name + ".pad"]), name
    rows = []
    for W, H, resize in gen.geometry_sizes():
        resized, _, pad = gen.reference_prepare(dl, np.zeros((H, W, 3), np.uint8), resize)
        rows.append((W, H, resize, resized.shape[0], resized.shape[1], *pad))
    assert np.array_equal(np.asarray(rows, np.int32), g["geometry"])
