from . import swa_utils
from .adam import Adam, AdamW
from .sgd import SGD

__all__ = ["Adam", "AdamW", "SGD", "swa_utils"]
