"""Drop-in for the reference's `models` package (models/__init__.py:16-17): `build_model(args)` returns
(model, criterion, postprocessors) where `model` is the CUDA-native LWDETR module."""
from .lwdetr import build


def build_model(args):
    return build(args)
