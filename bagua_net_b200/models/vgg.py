"""VGG family (the reference's headline benchmark model is VGG16: reference README.md:52-84)."""
from __future__ import annotations

import torch
from torch import nn

CFGS = {
    "vgg11": [64, "M", 128, "M", 256, 256, "M", 512, 512, "M", 512, 512, "M"],
    "vgg13": [64, 64, "M", 128, 128, "M", 256, 256, "M", 512, 512, "M", 512, 512, "M"],
    "vgg16": [64, 64, "M", 128, 128, "M", 256, 256, 256, "M", 512, 512, 512, "M", 512, 512, 512, "M"],
    "vgg19": [64, 64, "M", 128, 128, "M", 256, 256, 256, 256, "M", 512, 512, 512, 512, "M", 512, 512, 512, 512, "M"],
}


class VGG(nn.Module):
    def __init__(self, cfg="vgg16", num_classes: int = 1000, batch_norm: bool = False, dropout: float = 0.5,
                 width_div: int = 1, fc_dim: int = 4096, image_size: int = 224, fused: bool = False):
        """fused=True builds the feature extractor from bagua_net_b200.ops.ConvBiasReLU blocks: bias, ReLU,
        2x2 max-pool, their backward and the bias-gradient reduction run as one sm_90a pass each."""
        super().__init__()
        layers, cin = [], 3
        spec = list(CFGS[cfg] if isinstance(cfg, str) else cfg)
        if fused and not batch_norm:
            from ..ops.fused_nn import ConvBiasReLU

            i = 0
            while i < len(spec):
                v = spec[i]
                if v == "M":            # a pool that does not directly follow a convolution
                    layers.append(nn.MaxPool2d(2, 2))
                    i += 1
                    continue
                cout = max(8, v // width_div)
                pool = i + 1 < len(spec) and spec[i + 1] == "M"
                layers.append(ConvBiasReLU(cin, cout, 3, 1, 1, pool=pool))
                cin = cout
                i += 2 if pool else 1
        else:
            for v in spec:
                if v == "M":
                    layers.append(nn.MaxPool2d(2, 2))
                else:
                    cout = max(8, v // width_div)
                    layers.append(nn.Conv2d(cin, cout, 3, padding=1))
                    if batch_norm:
                        layers.append(nn.BatchNorm2d(cout))
                    layers.append(nn.ReLU(inplace=True))
                    cin = cout
        self.features = nn.Sequential(*layers)
        side = image_size // 32
        self.avgpool = nn.AdaptiveAvgPool2d((side, side)) if image_size % 32 else nn.Identity()
        from ..ops import tc_linear

        if fused and tc_linear.enabled():
            # opt-in (BNET_TC=1): Linear + bias + ReLU as one wgmma kernel; Identity keeps the Sequential indices —
            # and so the state_dict keys — of the stock layout
            self.classifier = nn.Sequential(
                tc_linear.TCLinear(cin * side * side, fc_dim, relu=True), nn.Identity(), nn.Dropout(dropout),
                tc_linear.TCLinear(fc_dim, fc_dim, relu=True), nn.Identity(), nn.Dropout(dropout),
                tc_linear.TCLinear(fc_dim, num_classes),
            )
        else:
            self.classifier = nn.Sequential(
                nn.Linear(cin * side * side, fc_dim), nn.ReLU(True), nn.Dropout(dropout),
                nn.Linear(fc_dim, fc_dim), nn.ReLU(True), nn.Dropout(dropout),
                nn.Linear(fc_dim, num_classes),
            )
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
                nn.init.zeros_(m.bias)
            elif isinstance(m, nn.Linear):
                nn.init.normal_(m.weight, 0, 0.01)
                nn.init.zeros_(m.bias)

    def forward(self, x):
        x = self.features(x)
        x = self.avgpool(x)
        return self.classifier(torch.flatten(x, 1))


def vgg11(**kw) -> VGG:
    return VGG("vgg11", **kw)


def vgg13(**kw) -> VGG:
    return VGG("vgg13", **kw)


def vgg16(**kw) -> VGG:
    return VGG("vgg16", **kw)


def vgg19(**kw) -> VGG:
    return VGG("vgg19", **kw)
