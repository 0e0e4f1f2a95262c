from . import swa_utils
from .adagrad import Adagrad
from .adam import Adam, AdamW
from .nadam import NAdam
from .radam import RAdam
from .rmsprop import RMSprop
from .sgd import SGD

__all__ = ["Adagrad", "Adam", "AdamW", "NAdam", "RAdam", "RMSprop", "SGD", "swa_utils"]
