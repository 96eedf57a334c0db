from .data_parallel import DataParallelWrapper
from .losses import PanopticLoss, panoptic_losses
from .mlp_backward import network_backward, network_forward_autograd, network_forward_rays_autograd, training_step
from .network_wrapper import NetworkWrapper, make_network_wrapper
from .optim import FusedAdam

__all__ = ["PanopticLoss", "panoptic_losses", "network_backward", "network_forward_autograd",
           "network_forward_rays_autograd", "training_step", "NetworkWrapper", "make_network_wrapper", "FusedAdam",
           "DataParallelWrapper"]
