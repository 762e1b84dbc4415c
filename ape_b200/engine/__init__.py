"""Predictor / input pipeline in front of the model (reference: ape/engine/defaults.py)."""
from .defaults import DefaultPredictor, NoOpTransform, ResizeShortestEdge, ResizeTransform  # noqa: F401
from .read import read_image  # noqa: F401
