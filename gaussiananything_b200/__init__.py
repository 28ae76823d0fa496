"""gaussiananything_b200 -- H100 (sm_90a) kernels for GaussianAnything's two hot paths
(surfel rasteriser; DiT denoiser + flow-matching sampler) behind the reference's own Python API.
See INTEGRATION.md.  Nothing here falls back to CPU or to a library path."""
import sys

__all__ = ["install_shims"]


def install_shims(replace_classes: bool = True):
    """Registers this package under the module names the reference imports (INTEGRATION.md section 1)."""
    from . import diff_surfel_rasterization as _dsr
    from . import transport as _tr
    sys.modules["diff_surfel_rasterization"] = _dsr
    sys.modules["transport"] = _tr
    sys.modules["transport.transport"] = _tr.transport
    sys.modules["transport.path"] = _tr.path
    sys.modules["transport.integrators"] = _tr.integrators
    if replace_classes:
        from . import dit as _dit
        from . import gs_surfel as _gs
        for name, attr, obj in (("nsr.gs_surfel", "GaussianRenderer2DGS", _gs.GaussianRenderer2DGS),):
            m = sys.modules.get(name)
            if m is not None:
                setattr(m, attr, obj)
        m = sys.modules.get("dit.dit_i23d")
        if m is not None and hasattr(m, "DiT_models"):
            m.DiT_models.update(_dit.DiT_models)
        from . import dino as _dino
        for name in ("sgm.modules.encoders.modules", "sgm.modules"):
            m = sys.modules.get(name)
            if m is not None:
                for attr in ("FrozenDinov2ImageEmbedder", "PCD_Scaler", "GeneralConditioner"):
                    setattr(m, attr, getattr(_dino, attr))
        m = sys.modules.get("nsr.lsgm.flow_matching_trainer")
        if m is not None and hasattr(m, "FlowMatchingEngine"):
            from . import mesh as _mesh
            m.FlowMatchingEngine.extract_mesh_bounded = _mesh._engine_extract_mesh_bounded
            m.FlowMatchingEngine.export_mesh_from_2dgs = _mesh._engine_export_mesh_from_2dgs
