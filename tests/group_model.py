"""The layout of hqs_tick_fetch_grouped (include/hqsched.h) as a few lines of numpy: a stable sort of the flat record stream
by key = kind == 2 ? 2W : 2 * worker + (kind == 0), and the offsets of the keys."""
import numpy as np


def group_keys(flat: np.ndarray, n_workers: int) -> np.ndarray:
    kind = flat["kind"].astype(np.int64)
    return np.where(kind == 2, 2 * n_workers, 2 * flat["worker"].astype(np.int64) + (kind == 0))


def group_model(flat: np.ndarray, n_workers: int):
    """(grouped records, worker_off [2W + 2] u32) of the flat stream `flat` over n_workers workers."""
    key = group_keys(flat, n_workers)
    grouped = flat[np.argsort(key, kind="stable")]
    off = np.zeros(2 * n_workers + 2, dtype=np.uint32)
    off[1:] = np.cumsum(np.bincount(key, minlength=2 * n_workers + 1))
    return grouped, off
