from . import swa_utils
from .adagrad import Adagrad
from .adam import Adam, AdamW
from .rmsprop import RMSprop
from .sgd import SGD

__all__ = ["Adagrad", "Adam", "AdamW", "RMSprop", "SGD", "swa_utils"]
