"""Stand-in for torchmetrics.image.inception: InceptionScore records its update calls."""
from oracle.shims.recording import RecordingMetric


class InceptionScore(RecordingMetric):
    pass
