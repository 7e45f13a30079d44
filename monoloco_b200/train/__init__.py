from .losses import LaplacianLoss, MultiTaskLoss, AutoTuneMultiTaskLoss, CompositeLoss, l1_loss_from_laplace, angle_loss
from .fused import train_step, fused_train_forward
from .optim import FusedClipAdam
from .datasets import KeypointsDataset, DeviceLoader
from .stats import task_stats
from .trainer import Trainer
