"""Stand-in for lightning.pytorch.utilities.rank_zero_only (a single process is rank zero)."""


def rank_zero_only(fn):
    return fn
