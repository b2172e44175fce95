"""H100-native (sm_90a) inverted-residual training path behind the module surface of
meijieru/yet_another_mobilenet_series (models/mobilenet_base.py)."""
__version__ = "0.1.0"
