"""fruitnerf_b200 -- H100-native (sm_90a) implementation of FruitNeRF's per-ray hot path behind the
reference's Nerfstudio plugin surface.  See DESIGN.md / INTEGRATION.md."""
from .compat import FieldHeadNames, Frustums, RayBundle, RaySamples, SceneBox, Semantics  # noqa: F401
from .fruit_field import FruitField, SceneContraction  # noqa: F401

__version__ = "0.1.0"
