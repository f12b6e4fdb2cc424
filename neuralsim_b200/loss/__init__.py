"""Training losses whose inputs are the renderer's own per-sample buffers (the other losses stay the trainer's, in PyTorch)."""
from .lidar import DepthLoss, LidarLoss, LineOfSightLoss  # noqa: F401
