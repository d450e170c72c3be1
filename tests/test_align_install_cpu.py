"""install(face_align=True) rebinds utils.shape_predictor.align_face and hair_swap's imported name to
hairfastgan_b200.face_align.align_face, the other options leave both alone, and uninstall() restores them.  Runs on a
stand-in reference tree (no device, no dlib)."""
from __future__ import annotations

import importlib
import sys

import pytest

_MODULES = ("utils", "utils.shape_predictor", "hair_swap")


def _fake_reference(root):
    (root / "utils").mkdir()
    (root / "utils" / "__init__.py").write_text("")
    (root / "utils" / "shape_predictor.py").write_text(
        "def align_face(data, predictor=None, is_filepath=False, return_tensors=True):\n    return 'reference'\n")
    (root / "hair_swap.py").write_text("from utils.shape_predictor import align_face\n")


@pytest.mark.parametrize("flags", [{"face_align": True}, {"face_align": True, "sean": True, "shape_adaptor": True},
                                   {}, {"sean": True, "sean_encode": True, "shape_adaptor": True,
                                        "modulation": True}])
@pytest.mark.parametrize("order", ["defining_first", "importer_first"])
def test_install_binds_align_face(tmp_path, flags, order):
    import hairfastgan_b200.install as inst
    import hairfastgan_b200.face_align as FA
    _fake_reference(tmp_path)
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k in _MODULES}
    sys.path.insert(0, str(tmp_path))
    try:
        inst.install(**flags)
        names = ["utils.shape_predictor", "hair_swap"]
        for n in (names if order == "defining_first" else names[::-1]):
            importlib.import_module(n)
        sp, hs = sys.modules[names[0]], sys.modules[names[1]]
        on = flags.get("face_align", False)
        for m in (sp, hs):
            assert (m.align_face is FA.align_face) == on, m.__name__
        inst.uninstall()
        for m in (sp, hs):
            assert m.align_face(None) == "reference", m.__name__
    finally:
        inst.uninstall()
        sys.path.remove(str(tmp_path))
        for k in [k for k in sys.modules if k in _MODULES]:
            del sys.modules[k]
        sys.modules.update(saved)


def test_install_after_import_rebinds_and_restores(tmp_path):
    """Modules imported before install() are rebound on the spot."""
    import hairfastgan_b200.install as inst
    import hairfastgan_b200.face_align as FA
    _fake_reference(tmp_path)
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k in _MODULES}
    sys.path.insert(0, str(tmp_path))
    try:
        import hair_swap
        sp = sys.modules["utils.shape_predictor"]
        inst.install(face_align=True)
        assert sp.align_face is FA.align_face and hair_swap.align_face is FA.align_face
        inst.uninstall()
        assert sp.align_face(None) == "reference" and hair_swap.align_face(None) == "reference"
    finally:
        inst.uninstall()
        sys.path.remove(str(tmp_path))
        for k in [k for k in sys.modules if k in _MODULES]:
            del sys.modules[k]
        sys.modules.update(saved)


def test_signature_matches_reference():
    import inspect
    import hairfastgan_b200.face_align as FA
    sig = inspect.signature(FA.align_face)
    assert list(sig.parameters) == ["data", "predictor", "is_filepath", "return_tensors"]
    assert [p.default for p in sig.parameters.values()][1:] == [None, False, True]
