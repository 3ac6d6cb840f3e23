"""Stand-in for the reference's models/faed/FAED.py as EvalPanoGen imports it: the metric records its update calls."""
from oracle.shims.recording import RecordingMetric


class FrechetAutoEncoderDistance(RecordingMetric):
    pass
