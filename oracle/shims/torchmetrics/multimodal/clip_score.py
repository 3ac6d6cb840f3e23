"""Stand-in for torchmetrics.multimodal.clip_score: CLIPScore records its update calls."""
from oracle.shims.recording import RecordingMetric


class CLIPScore(RecordingMetric):
    pass
