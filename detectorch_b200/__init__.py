"""detectorch_b200 -- H100-native (sm_90a) two-stage detector inference hot path behind the
reference's own operator / model interface (ignacio-rocco/detectorch lib/model, lib/utils)."""
__version__ = "0.1"
