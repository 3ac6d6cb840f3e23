"""Stand-in for the reference's models/horizonnet/HorizonNet.py as EvalPanoGen imports it: LayoutConsistency records
its update calls (the layout metric is not computed by the driver)."""
from oracle.shims.recording import RecordingMetric


class LayoutConsistency(RecordingMetric):
    pass
