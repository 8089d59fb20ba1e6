from .astar import NeuralAstar, VanillaAstar  # noqa: F401  (same exports as the reference's planner/__init__.py:1)
from .astar import BBAstar  # noqa: F401  (Neural A* trained through the black-box gradient of BB-A*)
