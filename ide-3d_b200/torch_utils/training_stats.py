"""The one call of the reference's torch_utils/training_stats.py its calc_metrics.py makes (:44).  The metrics here report through
their return values, so there are no statistics to synchronise; the call only checks and records its arguments."""

_rank = 0
_sync_device = None


def init_multiprocessing(rank, sync_device):
    global _rank, _sync_device
    assert not _sync_device or rank >= 0
    _rank = rank
    _sync_device = sync_device
