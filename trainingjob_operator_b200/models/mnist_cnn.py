"""MNIST CNN (the PyTorch ``examples/mnist`` network) -- BASELINE.json config "torch DDP MNIST CNN
AITrainingJob on 8xH100", and the stand-in for the reference's only example workload
(/root/reference/example/paddle-mnist.yaml:20-21 runs Paddle's recognize_digits).  Synthetic 1x28x28
images, random-init weights; trained through ``parallel.flat_ddp`` with bf16 autocast on CUDA."""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as TF


class MnistCNN(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv1 = nn.Conv2d(1, 32, 3, 1)
        self.conv2 = nn.Conv2d(32, 64, 3, 1)
        self.fc1 = nn.Linear(9216, 128)
        self.fc2 = nn.Linear(128, 10)

    def forward(self, x):
        x = TF.relu(self.conv1(x))
        x = TF.max_pool2d(TF.relu(self.conv2(x)), 2)
        x = torch.flatten(x, 1)
        x = TF.relu(self.fc1(x))
        return self.fc2(x)


class MLP(nn.Module):
    """Tiny CPU-friendly model used by the gloo plumbing tests (world_size=2 on CPU)."""

    def __init__(self, d_in: int = 64, d_hidden: int = 128, n_cls: int = 10):
        super().__init__()
        self.fc1 = nn.Linear(d_in, d_hidden)
        self.fc2 = nn.Linear(d_hidden, n_cls)

    def forward(self, x):
        return self.fc2(TF.relu(self.fc1(x)))
