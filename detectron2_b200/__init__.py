"""detectron2_b200 -- Hopper-native (sm_90a) implementation of Detectron2's per-image detection hot path
behind the `detectron2.layers` operator surface.  See DESIGN.md / INTEGRATION.md."""
__version__ = "0.1.0"
