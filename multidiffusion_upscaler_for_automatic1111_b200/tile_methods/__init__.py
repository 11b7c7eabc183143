from .abstractdiffusion import AbstractDiffusion
from .multidiffusion import MultiDiffusion
from .mixtureofdiffusers import MixtureOfDiffusers
from .demofusion import DemoFusion
from .spotdiffusion import SpotDiffusion

__all__ = ["AbstractDiffusion", "MultiDiffusion", "MixtureOfDiffusers", "DemoFusion", "SpotDiffusion"]
