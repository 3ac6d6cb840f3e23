"""Stand-in for the part of torchmetrics that models/faed/FAED.py uses: `Metric` with `add_state` (states are plain
attributes; the distributed reduction is not restated)."""
import torch


class Metric(torch.nn.Module):
    def __init__(self, **kwargs):
        super().__init__()
        self._defaults = {}

    def add_state(self, name, default, dist_reduce_fx=None, persistent=False):
        self._defaults[name] = default.clone()
        setattr(self, name, default.clone())

    def reset(self):
        for name, default in self._defaults.items():
            setattr(self, name, default.clone())
