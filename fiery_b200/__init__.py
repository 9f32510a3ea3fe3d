"""fiery_b200: Hopper-native (sm_90a, H100) camera->BEV lift, a drop-in for the Lift-Splat hot path of
wayveai/fiery (``fiery/models/fiery.py:193-286``, ``fiery/models/encoder.py:96-104``,
``fiery/utils/geometry.py:283-314``).  See DESIGN.md.

Importing this package does not need a GPU; every compute entry point loads ``libfiery_b200.so`` (built
in-tree by ``python -m fiery_b200.build``) and raises if it is missing -- there is no CPU fallback.
"""
__version__ = "0.1.0"
