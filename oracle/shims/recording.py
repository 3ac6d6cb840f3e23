"""A metric stand-in that only records its update calls (oracle/eval_pano.py runs the reference's
EvalPanoGen.test_step against these, so the call sequence, the images and the flags are pinned; the oracle's own
networks turn the recorded images into features afterwards)."""
import torch


class RecordingMetric(torch.nn.Module):
    def __init__(self, *args, **kwargs):
        super().__init__()
        self.init_args, self.init_kwargs = args, kwargs
        self.calls = []

    @property
    def _update_called(self):
        return bool(self.calls)

    def update(self, *args, **kwargs):
        self.calls.append((tuple(a.detach().clone() if torch.is_tensor(a) else a for a in args), dict(kwargs)))
