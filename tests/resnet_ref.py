"""ORACLE for the ResNet-50 trunk (test infrastructure, never on the product path).

The reference contains no ResNet trunk, so this restates the one netspec.build_acr_spec(backbone="resnet50") defines,
independently of netspec: a plain ``nn.Module`` tree built from the reference's Bottleneck / _make_layer recipe
(/root/reference/acr/model.py:501-539, :738-752) whose module names ARE the state-dict keys, so a strict
``load_state_dict`` pins the parameter registry.  Plus the per-op restatements the teacher-forced sweep needs for the
kinds the ResNet plan adds (7x7 stem, max-pool, ConvTranspose2d + BN + ReLU)."""
import torch
import torch.nn as nn
import torch.nn.functional as Fn

EPS = 1e-5


class Bottleneck(nn.Module):
    expansion = 4

    def __init__(self, inplanes, planes, stride=1, downsample=None):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = nn.Conv2d(planes, planes, 3, stride, 1, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.conv3 = nn.Conv2d(planes, planes * 4, 1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes * 4)
        self.downsample = downsample

    def forward(self, x):
        y = torch.relu(self.bn1(self.conv1(x)))
        y = torch.relu(self.bn2(self.conv2(y)))
        y = self.bn3(self.conv3(y))
        return torch.relu(y + (self.downsample(x) if self.downsample is not None else x))


class ResNet50Trunk(nn.Module):
    """x/255*2-1 -> conv1 7x7 s2 + bn1 + ReLU -> MaxPool 3x3 s2 p1 -> layer1..4 -> 3 x (ConvT k4 s2 p1, BN, ReLU)."""

    def __init__(self):
        super().__init__()
        self.conv1 = nn.Conv2d(3, 64, 7, 2, 3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        self.inplanes = 64
        self.layer1 = self._make_layer(64, 3, 1)
        self.layer2 = self._make_layer(128, 4, 2)
        self.layer3 = self._make_layer(256, 6, 2)
        self.layer4 = self._make_layer(512, 3, 2)
        layers, cin = [], 2048
        for cout in (256, 128, 32):
            layers += [nn.ConvTranspose2d(cin, cout, 4, 2, 1, bias=False), nn.BatchNorm2d(cout), nn.ReLU()]
            cin = cout
        self.deconv_layers = nn.Sequential(*layers)

    def _make_layer(self, planes, blocks, stride):
        down = None
        if stride != 1 or self.inplanes != planes * 4:
            down = nn.Sequential(nn.Conv2d(self.inplanes, planes * 4, 1, stride, bias=False), nn.BatchNorm2d(planes * 4))
        layers = [Bottleneck(self.inplanes, planes, stride, down)]
        self.inplanes = planes * 4
        layers += [Bottleneck(self.inplanes, planes) for _ in range(1, blocks)]
        return nn.Sequential(*layers)

    def forward(self, image_bhwc):
        x = image_bhwc.float().permute(0, 3, 1, 2) / 255.0 * 2.0 - 1.0
        x = torch.relu(self.bn1(self.conv1(x)))
        x = Fn.max_pool2d(x, 3, 2, 1)
        x = self.layer4(self.layer3(self.layer2(self.layer1(x))))
        return self.deconv_layers(x)


def trunk_state(sd):
    """The trunk's entries of a full ACR state dict, without the ``backbone.`` prefix (hand_segm belongs to the heads)."""
    return {k[len("backbone."):]: v for k, v in sd.items()
            if k.startswith("backbone.") and not k.startswith("backbone.hand_segm.")}


def _bn(y, sd, bnkey):
    g, be = sd[bnkey + ".weight"].float(), sd[bnkey + ".bias"].float()
    m, v = sd[bnkey + ".running_mean"].float(), sd[bnkey + ".running_var"].float()
    s = g / torch.sqrt(v + EPS)
    return y * s.view(1, -1, 1, 1) + (be - m * s).view(1, -1, 1, 1)


def stem7(image_bhwc, sd):
    """x/255*2-1 (as acr/model.py:832), conv1 7x7 s2 p3 + bn1 + ReLU."""
    x = image_bhwc.float().permute(0, 3, 1, 2) / 255.0 * 2.0 - 1.0
    return torch.relu(_bn(Fn.conv2d(x, sd["backbone.conv1.weight"].float(), None, 2, 3), sd, "backbone.bn1"))


def maxpool(x):
    return Fn.max_pool2d(x, 3, 2, 1)


def deconv_bn_relu(x, sd, wkey, bnkey):
    """nn.ConvTranspose2d(k4, s2, p1, no bias) (weight (cin, cout, 4, 4)) + BN + ReLU."""
    return torch.relu(_bn(Fn.conv_transpose2d(x, sd[wkey + ".weight"].float(), None, 2, 1), sd, bnkey))
