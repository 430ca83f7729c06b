"""Import the reference's OWN network files (unmodified) on top of this repo's layer library -- INTEGRATION.md section 1.

`reference_dir()` is `oracle/_ref` (a verbatim, git-ignored staging copy made by oracle/stage_reference.py at build time).
Only the L2 file itself comes from the reference; every `models.*` module it imports resolves to
`text_segmentation_image_inpainting_b200.models.*`."""
import contextlib
import importlib.util
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.stage_reference import reference_dir  # noqa: E402

L1_MODULES = ("BaseModels", "MobileNetV2", "partial_convolution", "Xception", "common")


@contextlib.contextmanager
def reference_l2(filename):
    """`with reference_l2("image_inpainting.py") as mod:` -> the reference's module object, executed with the aliased L1."""
    ref = reference_dir()
    if ref is None:
        raise FileNotFoundError("the reference is not staged at oracle/_ref (run __graft_entry__.build())")
    import text_segmentation_image_inpainting_b200.models as mine
    saved = {k: v for k, v in sys.modules.items() if k == "models" or k.startswith("models.")}
    for k in saved:
        del sys.modules[k]
    try:
        pkg = types.ModuleType("models")
        pkg.__path__ = []
        sys.modules["models"] = pkg
        for name in L1_MODULES:
            mod = importlib.import_module(f"{mine.__name__}.{name}")
            sys.modules["models." + name] = mod
            setattr(pkg, name, mod)
        modname = "models." + filename[:-3]
        path = os.path.join(ref, "models", filename)
        spec = importlib.util.spec_from_file_location(modname, path)
        mod = importlib.util.module_from_spec(spec)
        sys.modules[modname] = mod
        spec.loader.exec_module(mod)
        mod.__reference_file__ = path
        yield mod
    finally:
        for k in [k for k in sys.modules if k == "models" or k.startswith("models.")]:
            del sys.modules[k]
        sys.modules.update(saved)
