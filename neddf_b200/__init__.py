"""neddf_b200: H100-native (sm_90a) implementation of the NeDDF volumetric-rendering hot path
behind the reference's NeRFRender / NeDDF Python API.  See DESIGN.md."""
from .camera import Camera, PinholeCalib  # noqa: F401
from .network import BaseNeuralField, LinearGradLayer, NeDDF  # noqa: F401
from .nerf import NeRF  # noqa: F401
from .neus import NeuS  # noqa: F401
from .ray import CONE_RAY_RADIUS, Ray, Sampling  # noqa: F401
from .render import BaseNeuralRender, NeRFRender  # noqa: F401
from . import losses, optim  # noqa: F401

__all__ = ["NeRFRender", "NeDDF", "NeRF", "NeuS", "BaseNeuralRender", "BaseNeuralField", "LinearGradLayer", "Ray", "Sampling",
           "Camera", "PinholeCalib", "CONE_RAY_RADIUS"]
