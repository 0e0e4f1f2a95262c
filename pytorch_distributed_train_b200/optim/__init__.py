from . import swa_utils
from .adadelta import Adadelta
from .adagrad import Adagrad
from .adam import Adam, AdamW
from .adamax import Adamax
from .asgd import ASGD
from .nadam import NAdam
from .radam import RAdam
from .rmsprop import RMSprop
from .rprop import Rprop
from .sgd import SGD

__all__ = ["ASGD", "Adadelta", "Adagrad", "Adam", "AdamW", "Adamax", "NAdam", "RAdam", "RMSprop", "Rprop", "SGD", "swa_utils"]
