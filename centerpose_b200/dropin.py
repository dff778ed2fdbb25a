"""Make the UNMODIFIED reference entry points (src/demo.py, src/test.py) run on
the H100-native hot path without editing a reference file.

    import centerpose_b200.dropin as dropin
    dropin.install()          # before `from lib.detectors.detector_factory import ...`

`install()` pre-registers three modules in `sys.modules`, which Python's import
system consults before it looks at the reference's files:

  lib.models.model               -> create_model / load_model / save_model of this package
                                    (reference: src/lib/models/model.py:16-105)
  lib.detectors.detector_factory -> detector_factory = {'object_pose': ObjectPoseDetector}
                                    (reference: src/lib/detectors/detector_factory.py:7-9)
  _ext                           -> dcn_v2_forward / dcn_v2_backward backed by cp_dcn_v2_forward /
                                    cp_dcn_v2_backward, so that even the reference's own DLASeg graph and its
                                    autograd Function (DCNv2/dcn_v2.py:13-76) run our deformable kernels;
                                    PSROI pooling (unused by CenterPose) raises NotImplementedError
"""
import sys
import types


def install(model=True, detector=True, ext=True):
    from . import model as _model
    from . import detector as _detector
    from . import engine as _engine
    if model:
        m = types.ModuleType("lib.models.model")
        m.create_model = _model.create_model
        m.load_model = _model.load_model
        m.save_model = _model.save_model
        m._model_factory = _model._model_factory
        m.__doc__ = "centerpose_b200 drop-in for lib.models.model"
        sys.modules["lib.models.model"] = m
    if detector:
        d = types.ModuleType("lib.detectors.detector_factory")
        d.detector_factory = _detector.detector_factory
        sys.modules["lib.detectors.detector_factory"] = d
    if ext:
        e = types.ModuleType("_ext")
        e.dcn_v2_forward = _engine.dcn_v2_forward

        def _no(*a, **k):
            raise NotImplementedError("centerpose_b200 `_ext`: deformable PSROI pooling is not used by CenterPose and not provided")
        e.dcn_v2_backward = _engine.dcn_v2_backward
        e.dcn_v2_psroi_pooling_forward = _no
        e.dcn_v2_psroi_pooling_backward = _no
        sys.modules["_ext"] = e


def uninstall():
    for k in ("lib.models.model", "lib.detectors.detector_factory", "_ext"):
        m = sys.modules.get(k)
        if m is not None and (getattr(m, "__doc__", "") or "").startswith("centerpose_b200") or k == "_ext":
            sys.modules.pop(k, None)
