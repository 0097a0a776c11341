"""Plugin package `fasttd3.b200`: importing it registers the algorithm (the reference's registration contract, rl_x/algorithms/algorithm_manager.py)."""
from rl_x_b200.algorithms.algorithm_manager import register_algorithm_package

NAME = register_algorithm_package(__file__, "fasttd3", "FastTD3")
