"""``select_device``, ``time_synchronized``, ``TracedModel`` as imported by tracker/track.py:31."""
import time

import torch


def select_device(device='', batch_size=None):
    if str(device).lower() == 'cpu' or not torch.cuda.is_available():
        raise RuntimeError("the GPU detector path has no CPU fallback: a CUDA device is required")
    idx = 0 if device in ('', None) else int(str(device).split(',')[0])
    return torch.device('cuda:%d' % idx)


def time_synchronized():
    if torch.cuda.is_available():
        torch.cuda.synchronize()
    return time.time()


class TracedModel(torch.nn.Module):
    """The reference wraps the model in a torch.jit trace (utils/torch_utils.py:343-373); the GPU forward is a fixed
    launch sequence already, so the wrapper only forwards."""

    def __init__(self, model=None, device=None, img_size=(640, 640)):
        super().__init__()
        self.model = model
        self.stride = model.stride
        self.names = model.names

    def forward(self, x, augment=False, profile=False):
        return self.model(x)
