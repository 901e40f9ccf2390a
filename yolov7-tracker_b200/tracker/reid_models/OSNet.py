"""Drop-in for the reference's ``tracker/reid_models/OSNet.py``, imported by ``strongsort.py`` as
``from reid_models.OSNet import osnet_x0_25``.

``osnet_x0_25(num_classes, pretrained=False)`` returns an ``nn.Module`` whose parameters and buffers carry the reference's names and
shapes, so ``state_dict()``, ``load_state_dict()`` and the reference's ``load_model_tools.load_pretrained_weights`` work unchanged.
In eval mode its forward runs on the GPU kernels of csrc/b2t_osnet.cu through ``b200track.osnet.OsnetExtractor``: (n, 3, H, W) CUDA
float32 (H, W multiples of 16; StrongSORT feeds 128 x 256) -> (n, 512) CUDA float32, the features after fc's ReLU, not normalised.
The folded weights are rebuilt whenever a parameter or buffer changed since the last forward (``load_state_dict``, ``.cuda()``).
Training mode is not supported.  The other widths and ``osnet_ibn_x1_0`` (InstanceNorm) are not built and raise."""
import os
import sys

import torch
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import _b2t_path  # noqa: F401,E402
from b200track.osnet import OsnetExtractor  # noqa: E402

__all__ = ['osnet_x1_0', 'osnet_x0_75', 'osnet_x0_5', 'osnet_x0_25', 'osnet_ibn_x1_0']


class _ConvBN(nn.Module):
    """conv (no bias) + BatchNorm2d, named ``conv`` / ``bn`` like the reference's ConvLayer, Conv1x1 and Conv1x1Linear"""

    def __init__(self, cin, cout, k=1, stride=1, padding=0):
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, k, stride=stride, padding=padding, bias=False)
        self.bn = nn.BatchNorm2d(cout)


class _LightConv3x3(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.conv1 = nn.Conv2d(c, c, 1, bias=False)
        self.conv2 = nn.Conv2d(c, c, 3, padding=1, bias=False, groups=c)
        self.bn = nn.BatchNorm2d(c)


class _ChannelGate(nn.Module):
    def __init__(self, c, reduction=16):
        super().__init__()
        self.fc1 = nn.Conv2d(c, c // reduction, 1, bias=True)
        self.fc2 = nn.Conv2d(c // reduction, c, 1, bias=True)


class _OSBlock(nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        mid = cout // 4
        self.conv1 = _ConvBN(cin, mid)
        self.conv2a = _LightConv3x3(mid)
        self.conv2b = nn.Sequential(*[_LightConv3x3(mid) for _ in range(2)])
        self.conv2c = nn.Sequential(*[_LightConv3x3(mid) for _ in range(3)])
        self.conv2d = nn.Sequential(*[_LightConv3x3(mid) for _ in range(4)])
        self.gate = _ChannelGate(mid)
        self.conv3 = _ConvBN(mid, cout)
        self.downsample = _ConvBN(cin, cout) if cin != cout else None


class OSNet(nn.Module):
    """osnet_x0_25's module tree (channels 16, 64, 96, 128; feature_dim 512) with the GPU forward."""

    def __init__(self, num_classes, channels=(16, 64, 96, 128), feature_dim=512, loss='softmax', **kwargs):
        super().__init__()
        c = list(channels)
        self.loss = loss
        self.feature_dim = feature_dim
        self.conv1 = _ConvBN(3, c[0], 7, stride=2, padding=3)
        self.maxpool = nn.MaxPool2d(3, stride=2, padding=1)
        self.conv2 = nn.Sequential(_OSBlock(c[0], c[1]), _OSBlock(c[1], c[1]), nn.Sequential(_ConvBN(c[1], c[1]), nn.AvgPool2d(2, stride=2)))
        self.conv3 = nn.Sequential(_OSBlock(c[1], c[2]), _OSBlock(c[2], c[2]), nn.Sequential(_ConvBN(c[2], c[2]), nn.AvgPool2d(2, stride=2)))
        self.conv4 = nn.Sequential(_OSBlock(c[2], c[3]), _OSBlock(c[3], c[3]))
        self.conv5 = _ConvBN(c[3], c[3])
        self.global_avgpool = nn.AdaptiveAvgPool2d(1)
        self.fc = nn.Sequential(nn.Linear(c[3], feature_dim), nn.BatchNorm1d(feature_dim), nn.ReLU(inplace=True))
        self.classifier = nn.Linear(feature_dim, num_classes)
        self._ext = {}
        self._stamp = None

    def _fingerprint(self):
        return tuple((t.data_ptr(), t._version) for t in list(self.parameters()) + list(self.buffers()))

    def extractor(self, device, size):
        """The OsnetExtractor of the current weights for inputs of `size` (rows, columns) on `device`."""
        stamp = self._fingerprint()
        if stamp != self._stamp:
            self._ext, self._stamp = {}, stamp
        key = (str(device), tuple(size))
        if key not in self._ext:
            self._ext[key] = OsnetExtractor(self.state_dict(), device=device, size=size)
        return self._ext[key]

    def forward(self, x, return_featuremaps=False):
        if self.training:
            raise RuntimeError("reid_models.OSNet runs in eval mode only (call .eval(); StrongSORT does, strongsort.py:28)")
        if return_featuremaps:
            raise NotImplementedError("reid_models.OSNet: return_featuremaps is not supported")
        if not isinstance(x, torch.Tensor) or not x.is_cuda or x.dtype != torch.float32 or x.dim() != 4:
            raise RuntimeError("reid_models.OSNet: expected a CUDA float32 (n, 3, H, W) tensor (there is no CPU fallback)")
        return self.extractor(x.device, tuple(x.shape[2:])).forward_nchw(x).clone()


def _not_built(name):
    raise NotImplementedError("reid_models.OSNet.%s is not built on the GPU kernels; osnet_x0_25 is (StrongSORT's network)" % name)


def osnet_x0_25(num_classes=1000, pretrained=True, loss='softmax', **kwargs):
    if pretrained:
        raise RuntimeError("osnet_x0_25(pretrained=True) would download ImageNet weights; build with pretrained=False and load a checkpoint "
                           "with reid_models.load_model_tools.load_pretrained_weights(model, path), as StrongSORT does")
    return OSNet(num_classes, loss=loss, **kwargs)


def osnet_x1_0(num_classes=1000, pretrained=True, loss='softmax', **kwargs):
    _not_built("osnet_x1_0")


def osnet_x0_75(num_classes=1000, pretrained=True, loss='softmax', **kwargs):
    _not_built("osnet_x0_75")


def osnet_x0_5(num_classes=1000, pretrained=True, loss='softmax', **kwargs):
    _not_built("osnet_x0_5")


def osnet_ibn_x1_0(num_classes=1000, pretrained=True, loss='softmax', **kwargs):
    raise NotImplementedError("reid_models.OSNet.osnet_ibn_x1_0 (InstanceNorm) is not built on the GPU kernels")
