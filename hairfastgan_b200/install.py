"""Make an unmodified HairFastGAN checkout use this implementation.

    import hairfastgan_b200.install as hfi
    hfi.install()                       # before `import hair_swap`
    from hair_swap import HairFast, get_parser

After ``install()`` the import statements of the reference resolve to this package:

* ``from models.stylegan2.op import FusedLeakyReLU, fused_leaky_relu, upfirdn2d`` (models/stylegan2/model.py:11,
  models/encoder4editing/models/stylegan2/model.py:7,
  models/FeatureStyleEncoder/pixel2style2pixel/models/stylegan2/model.py:7)      -> ``hairfastgan_b200.op``
* ``from models.stylegan2.model import Generator`` (models/Net.py:9), ``PixelNorm`` (models/Encoders.py:10)
                                                                                    -> ``hairfastgan_b200.model``
* ``from pixel2style2pixel.models.stylegan2.model import Generator, get_keys`` (FeatureStyleEncoder/trainer.py:18)
                                                                                    -> ``hairfastgan_b200.fse_model``
* ``from models.encoder4editing.models.encoders import psp_encoders`` (encoder4editing/models/psp.py:6;
  ``psp_encoders.Encoder4Editing(50, 'ir_se', opts)`` :34) and ``from nets.feature_style_encoder import *``
  (FeatureStyleEncoder/trainer.py:20; ``fs_encoder_v2(...)`` :168)                  -> ``hairfastgan_b200.encoders``

* ``FeatureEncoderMult`` / ``FeatureiResnet`` as ``PostProcessModel`` builds them (models/Encoders.py:106-113): the
  names are rebound inside ``models.Net`` / ``models.Encoders`` when those modules are imported
                                                                                    -> ``hairfastgan_b200.postprocess``

* ``from models.CtrlHair.external_code.face_parsing.model import BiSeNet`` (face_parsing/my_parsing_util.py:15)
                                                                                    -> ``hairfastgan_b200.bisenet``

* ``from utils.bicubic import BicubicDownSample`` (models/Embedding.py:13, models/Blending.py:6)
                                                                                    -> ``hairfastgan_b200.bicubic``
* ``from utils.image_utils import DilateErosion`` (models/Alignment.py:11, models/Blending.py:7): the name is rebound
  inside ``utils.image_utils`` after import                                         -> ``hairfastgan_b200.masks``

* ``FaceParsing_tensor.parsing_img`` (face_parsing/my_parsing_util.py:70-89) is wrapped after import: same labels from
  ``BiSeNet.parse_labels`` without the full-resolution logits (``install(fuse_face_parsing=False)`` to keep it)
                                                                                    -> ``hairfastgan_b200.parsing_fast``

* opt-in, ``install(sean=True)``: ``decode_sean`` (models/sean_codes/models/pix2pix_model.py:309-325) is rebound inside
  ``models.sean_codes.models.pix2pix_model`` and ``models.Alignment`` (which imports the name, Alignment.py:10)
                                                                                    -> ``hairfastgan_b200.sean``
* opt-in, ``install(sean_encode=True)``: ``encode_sean`` (pix2pix_model.py:299-306) is rebound in the same two modules
                                                                                    -> ``hairfastgan_b200.sean``
* opt-in, ``install(shape_adaptor=True)``: CtrlHair's ``get_hair_face_code`` and ``get_new_shape``
  (models/CtrlHair/shape_branch/solver.py:248-262) are rebound inside that module and ``models.Alignment`` (which
  imports both names, Alignment.py:7)                                               -> ``hairfastgan_b200.shape_adaptor``
* opt-in, ``install(face_align=True)``: ``align_face`` (utils/shape_predictor.py:80-194) is rebound inside
  ``utils.shape_predictor`` and ``hair_swap`` (which imports the name, hair_swap.py:19); the landmarks stay on dlib
                                                                                    -> ``hairfastgan_b200.face_align``
* opt-in, ``install(modulation=True)``: ``RotateModel.forward``, ``ClipBlendingModel.forward`` and
  ``PostProcessModel.forward`` (models/Encoders.py:66-137) are wrapped inside ``models.Encoders`` after import; the
  classes, their submodules and state-dict keys stay the reference's             -> ``hairfastgan_b200.modulation``

Nothing in the reference tree is edited and its JIT build of the two 2019 CUDA extensions
(op/fused_act.py:10-16, op/upfirdn2d.py:10-16) never runs.
"""
from __future__ import annotations

import importlib
import importlib.abc
import importlib.util
import sys
import types

_OPS = {
    "models.stylegan2.op": "hairfastgan_b200.op",
    "models.stylegan2.op.fused_act": "hairfastgan_b200.op.fused_act",
    "models.stylegan2.op.upfirdn2d": "hairfastgan_b200.op.upfirdn2d",
}
_GENERATORS = {
    "models.stylegan2.model": "hairfastgan_b200.model",
    # FeatureStyleEncoder puts its own directory on sys.path (FSencoder.py:12-13) and imports by these names
    "pixel2style2pixel.models.stylegan2.model": "hairfastgan_b200.fse_model",
    "models.FeatureStyleEncoder.pixel2style2pixel.models.stylegan2.model": "hairfastgan_b200.fse_model",
}
_ENCODERS = {
    "models.encoder4editing.models.encoders.psp_encoders": "hairfastgan_b200.encoders",
    "nets.feature_style_encoder": "hairfastgan_b200.encoders",
}
# BiSeNet face parsing: `from models.CtrlHair.external_code.face_parsing.model import BiSeNet`
# (models/CtrlHair/external_code/face_parsing/my_parsing_util.py:15)
_SEGMENTATION = {
    "models.CtrlHair.external_code.face_parsing.model": "hairfastgan_b200.bisenet",
}
# stage glue: `from utils.bicubic import BicubicDownSample` (models/Embedding.py:13, models/Blending.py:6)
_GLUE = {
    "utils.bicubic": "hairfastgan_b200.bicubic",
}
_created_stubs = []

# PostProcess conv stack (SURVEY 8f-1).  models/Net.py and models/Encoders.py hold much more than these classes
# (BiSeNet glue, CLIP models, ...), so the modules stay the reference's and only these names are rebound right after
# the module body has run -- PostProcessModel.__init__ (models/Encoders.py:106-113) looks them up at call time.
_POSTPROCESS = {
    "models.Net": ("FeatureEncoder", "FeatureEncoderMult"),
    "models.Encoders": ("FeatureEncoderMult", "FeatureiResnet"),
}
# stage glue living in a module with unrelated content: utils/image_utils.py also holds the Poisson-blending helpers
_GLUE_ATTRS = {
    "utils.image_utils": (("DilateErosion", "hairfastgan_b200.masks"),),
}
_saved_attrs = []
# FeatureStyleEncoder/FSencoder.py:12-19 puts its directory on sys.path and does `from trainer import *`; with
# install(skip_fse_reconstruction=True) Trainer.test gets the fast path of hairfastgan_b200/fse_fast.py (SURVEY 8f-2)
_FSE_TRAINER = "trainer"
# face parsing: FaceParsing_tensor.parsing_img (my_parsing_util.py:70-89) -> label-only path of hairfastgan_b200/parsing_fast.py
_PARSING_UTIL = "models.CtrlHair.external_code.face_parsing.my_parsing_util"
_patched_parsing = []
# SEAN and the shape adaptor (opt-in): function name -> (our module, the modules that hold the name; the first defines
# it), the names chosen by install(), and (module, name) -> the reference function it held
_SEAN_MODULES = ("models.sean_codes.models.pix2pix_model", "models.Alignment")
_SHAPE_MODULES = ("models.CtrlHair.shape_branch.solver", "models.Alignment")
_ALIGN_MODULES = ("utils.shape_predictor", "hair_swap")
_FUNCTIONS = {"decode_sean": ("hairfastgan_b200.sean", _SEAN_MODULES),
              "encode_sean": ("hairfastgan_b200.sean", _SEAN_MODULES),
              "get_hair_face_code": ("hairfastgan_b200.shape_adaptor", _SHAPE_MODULES),
              "get_new_shape": ("hairfastgan_b200.shape_adaptor", _SHAPE_MODULES),
              "align_face": ("hairfastgan_b200.face_align", _ALIGN_MODULES)}
_sean_names = set()
_sean_saved = {}
_post_import = set()          # module names the meta-path hook currently patches
_patched_trainers = []
# HairFast's modulation nets (opt-in): the forwards of three classes in models/Encoders.py are wrapped after import
_MODULATION_MODULE = "models.Encoders"
_options = {"postprocess": False, "modulation": False}
_patched_modulation = []


def _patch_sean(module, name: str) -> None:
    ours_module, modules = _FUNCTIONS[name]
    ours = getattr(importlib.import_module(ours_module), name)
    current = getattr(module, name, None)
    if current is None or current is ours:
        # models.Alignment imported the name after the defining module was rebound: restore it to the reference's
        ref = sys.modules.get(modules[0])
        if current is ours and ref is not None and (ref, name) in _sean_saved and (module, name) not in _sean_saved:
            _sean_saved[(module, name)] = _sean_saved[(ref, name)]
        return
    _sean_saved[(module, name)] = current
    setattr(module, name, ours)


def _patch_postprocess(module) -> None:
    if module.__name__ in _SEAN_MODULES + _SHAPE_MODULES + _ALIGN_MODULES:
        for name in sorted(_sean_names):
            if module.__name__ in _FUNCTIONS[name][1]:
                _patch_sean(module, name)
        return
    if module.__name__ == _PARSING_UTIL:
        fast = importlib.import_module("hairfastgan_b200.parsing_fast")
        if fast.patch_parsing_module(module):
            _patched_parsing.append(module)
        return
    if module.__name__ == _FSE_TRAINER:
        fast = importlib.import_module("hairfastgan_b200.fse_fast")
        if fast.patch_trainer_module(module):
            _patched_trainers.append(module)
        return
    if module.__name__ == _MODULATION_MODULE and _options["modulation"]:
        mod = importlib.import_module("hairfastgan_b200.modulation")
        if mod.patch_encoders_module(module):
            _patched_modulation.append(module)
    rebind = [(attr, "hairfastgan_b200.postprocess") for attr in _POSTPROCESS.get(module.__name__, ())
              if _options["postprocess"]]
    rebind += list(_GLUE_ATTRS.get(module.__name__, ()))
    for attr, ours_name in rebind:
        ours = importlib.import_module(ours_name)
        if hasattr(module, attr) and getattr(module, attr) is not getattr(ours, attr):
            _saved_attrs.append((module, attr, getattr(module, attr)))
            setattr(module, attr, getattr(ours, attr))


class _PatchingLoader(importlib.abc.Loader):
    def __init__(self, inner):
        self.inner = inner

    def create_module(self, spec):
        return self.inner.create_module(spec)

    def exec_module(self, module):
        self.inner.exec_module(module)
        _patch_postprocess(module)
        for name in list(_post_import):          # targets pulled in as a side effect while the hook was re-entrant
            other = sys.modules.get(name)
            if other is not None and other is not module:
                _patch_postprocess(other)


class _PostImportPatcher(importlib.abc.MetaPathFinder):
    """Meta-path finder that lets the normal machinery locate models.Net / models.Encoders and wraps their loader."""
    _busy = False

    def find_spec(self, fullname, path=None, target=None):
        if fullname not in _post_import or _PostImportPatcher._busy:
            return None
        _PostImportPatcher._busy = True
        try:
            spec = importlib.util.find_spec(fullname)
        finally:
            _PostImportPatcher._busy = False
        if spec is None or spec.loader is None:
            return None
        spec.loader = _PatchingLoader(spec.loader)
        return spec


_patcher = _PostImportPatcher()


def _register(ref_name: str, ours: str) -> None:
    top = ref_name.split(".")[0]
    if top in ("pixel2style2pixel", "nets"):
        # parents of these names only exist once FSencoder.py has extended sys.path; register stub packages
        # so the absolute import resolves without executing the reference copy
        parts = ref_name.split(".")
        for i in range(1, len(parts)):
            name = ".".join(parts[:i])
            if name not in sys.modules:
                sys.modules[name] = types.ModuleType(name)
                _created_stubs.append(name)
    sys.modules[ref_name] = importlib.import_module(ours)


def install(generator: bool = True, encoders: bool = True, postprocess: bool = True, segmentation: bool = True,
            glue: bool = True, skip_fse_reconstruction: bool = False, fuse_face_parsing: bool = True,
            sean: bool = False, sean_encode: bool = False, shape_adaptor: bool = False,
            modulation: bool = False, face_align: bool = False) -> None:
    """Register the overlay.  ``generator=False`` swaps only the operator package (L1 boundary) and leaves the
    reference's own ``models/stylegan2/model.py`` classes in place on top of our ops; ``encoders=False`` keeps
    the reference's PyTorch encoders; ``postprocess=False`` keeps its PostProcess conv stack; ``segmentation=False``
    its BiSeNet.  ``sean=True`` (off by default) runs SEAN's ``decode_sean`` on our kernels; ``sean_encode=True`` (off
    by default, independent of ``sean``) runs its ``encode_sean`` (the Zencoder) on them; ``shape_adaptor=True`` (off by
    default) runs CtrlHair's shape adaptor (``get_hair_face_code`` / ``get_new_shape``) on them; ``modulation=True``
    (off by default, independent of ``postprocess``) runs HairFast's latent modulation stacks of ``RotateModel``,
    ``ClipBlendingModel`` and ``PostProcessModel`` on them; ``face_align=True`` (off by default) runs the warp of
    ``align_face`` -- what ``swap(..., align=True)`` and scripts/align_face.py call -- on them."""
    if segmentation:
        for ref_name, ours in _SEGMENTATION.items():
            _register(ref_name, ours)
    if glue:
        for ref_name, ours in _GLUE.items():
            _register(ref_name, ours)
    for ref_name, ours in _OPS.items():
        _register(ref_name, ours)
    if generator:
        for ref_name, ours in _GENERATORS.items():
            _register(ref_name, ours)
    if encoders:
        for ref_name, ours in _ENCODERS.items():
            _register(ref_name, ours)
    if postprocess:
        _options["postprocess"] = True
        _post_import.update(_POSTPROCESS)
    if modulation:
        _options["modulation"] = True
        _post_import.add(_MODULATION_MODULE)
    if glue:
        _post_import.update(_GLUE_ATTRS)
    if segmentation and fuse_face_parsing:
        # label-only face parsing (bit-identical labels, no full-resolution logits): hairfastgan_b200/parsing_fast.py
        _post_import.add(_PARSING_UTIL)
    if skip_fse_reconstruction:
        # opt-in: Trainer.test(img=..., return_latent=True) skips the StyleGAN reconstruction whose image swap() never
        # reads (x_1_recon comes back as None) and draws the same noise, so later random numbers are unchanged
        _post_import.add(_FSE_TRAINER)
    if sean:
        _sean_names.add("decode_sean")
    if sean_encode:
        _sean_names.add("encode_sean")
    if shape_adaptor:
        _sean_names.update(("get_hair_face_code", "get_new_shape"))
    if face_align:
        _sean_names.add("align_face")
    for name in _sean_names:
        _post_import.update(_FUNCTIONS[name][1])
    if _post_import:
        if _patcher not in sys.meta_path:
            sys.meta_path.insert(0, _patcher)
        for name in list(_post_import):              # already imported: rebind now
            if name in sys.modules:
                _patch_postprocess(sys.modules[name])


def uninstall() -> None:
    for ref_name in list(_OPS) + list(_GENERATORS) + list(_ENCODERS) + list(_SEGMENTATION) + list(_GLUE) + _created_stubs:
        sys.modules.pop(ref_name, None)
    _created_stubs.clear()
    if _patcher in sys.meta_path:
        sys.meta_path.remove(_patcher)
    for module, attr, value in reversed(_saved_attrs):
        setattr(module, attr, value)
    _saved_attrs.clear()
    for module in _patched_trainers:
        importlib.import_module("hairfastgan_b200.fse_fast").unpatch_trainer_module(module)
    _patched_trainers.clear()
    for module in _patched_parsing:
        importlib.import_module("hairfastgan_b200.parsing_fast").unpatch_parsing_module(module)
    _patched_parsing.clear()
    for module in _patched_modulation:
        importlib.import_module("hairfastgan_b200.modulation").unpatch_encoders_module(module)
    _patched_modulation.clear()
    _options.update(postprocess=False, modulation=False)
    for (module, name), ref in _sean_saved.items():
        setattr(module, name, ref)
    _sean_saved.clear()
    _sean_names.clear()
    _post_import.clear()
