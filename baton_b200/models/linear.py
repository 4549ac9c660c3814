"""The demo regression model and the 2-layer MLP of BASELINE config #1.

Parity target: demo ``Model`` = ``nn.Linear(10, 1)`` named "lineartest"
(reference demo.py:15-24).  ``MLP2`` is the "2-layer MLP FedAvg, 2 workers on
CPU/gloo via demo.py" plumbing model of the benchmark configurations.
"""
from __future__ import annotations

import torch
from torch import nn

from .base import FederatedModule


class LinearModel(FederatedModule):
    name = "lineartest"
    loss_kind = "mse"
    head = "fc1"                   # the whole model: it cannot be kept local

    def __init__(self, in_features: int = 10, out_features: int = 1):
        super().__init__()
        self.fc1 = nn.Linear(in_features, out_features)

    def forward(self, X):
        return self.fc1(X)


class MLP2(FederatedModule):
    name = "mlp2"
    loss_kind = "mse"
    head = "fc2"
    default_lr = 0.01

    def __init__(self, in_features: int = 10, hidden: int = 64, out_features: int = 1):
        super().__init__()
        self.fc1 = nn.Linear(in_features, hidden)
        self.fc2 = nn.Linear(hidden, out_features)

    def forward(self, X):
        return self.fc2(torch.relu(self.fc1(X)))
