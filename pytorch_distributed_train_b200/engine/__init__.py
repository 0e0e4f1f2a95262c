from .evaluate import evaluate
from .graphed_step import GraphedTrainStep

__all__ = ["GraphedTrainStep", "evaluate"]
