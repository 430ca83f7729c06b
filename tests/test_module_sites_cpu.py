"""The per-module fp64 suite (tests/test_gpu_module_sites.py) checks the modules of a fixed type table.  Build the five
networks on the CPU and assert that every module in them is of a table type, a pure container, or a part owned by a table
leaf -- so a new module type cannot go unchecked without this test saying so."""
import pytest

from module_sites import CONTAINERS, LEAF_PARTS, NOT_CALLED, TABLE
from text_segmentation_image_inpainting_b200.models import image_inpainting as MI
from text_segmentation_image_inpainting_b200.models import text_segmentation as MT


@pytest.mark.parametrize("name", ["ImageFillOrigin", "ImageFillOriginV2", "ImageFill", "TextSegament", "XceptionTextSegment"])
def test_every_module_type_is_checked_or_a_container(name):
    net = getattr(MI if hasattr(MI, name) else MT, name)()
    assert type(net) in TABLE, f"{name} itself (its head) must be in the table"
    leaves = [n for n, m in net.named_modules() if type(m) in TABLE and not any(type(c) in TABLE for c in m.children())]
    unknown, orphans = [], []
    for n, m in net.named_modules():
        if type(m) in TABLE or type(m) in CONTAINERS:
            continue
        if isinstance(m, LEAF_PARTS):
            # a part (BatchNorm, activation, the frozen mask kernel) belongs to a table leaf -- under any of its names: one
            # activation instance may be shared by the network and its blocks -- or to a module the forward never calls
            names = [a for a, b in net.named_modules(remove_duplicate=False) if b is m]
            if not any(a.startswith(lf + ".") or any(p in NOT_CALLED for p in a.split(".")) for a in names for lf in leaves):
                orphans.append(n)
            continue
        unknown.append(f"{n}: {type(m).__name__}")
    assert not unknown, f"{name}: module types neither checked nor declared a container: {unknown[:8]}"
    assert not orphans, f"{name}: leaf parts outside every table leaf: {orphans[:8]}"
