"""H100-native OpenFlamingo hot path.  Public surface mirrors `open_flamingo/__init__.py:1-2`."""
from .src.flamingo import Flamingo
from .src.factory import create_model_and_transforms

__all__ = ["Flamingo", "create_model_and_transforms"]
