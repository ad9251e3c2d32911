"""
Differentiable robot model on the H100
======================================
Batched forward kinematics, end-effector Jacobian and inverse dynamics as hand-written sm_90a CUDA
kernels behind the API of facebookresearch/differentiable-robot-model (package exports of the
reference: ``differentiable_robot_model/__init__.py:7-12``).
"""
from .robot_model import (
    DifferentiableRobotModel,
    DifferentiableKUKAiiwa,
    DifferentiableFrankaPanda,
    DifferentiableTwoLinkRobot,
    DifferentiableTrifingerEdu,
)

__all__ = [
    "DifferentiableRobotModel",
    "DifferentiableKUKAiiwa",
    "DifferentiableFrankaPanda",
    "DifferentiableTwoLinkRobot",
    "DifferentiableTrifingerEdu",
]
