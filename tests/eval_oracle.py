"""The evaluater's bookkeeping (evaluater/evaluater.py:45-49, 94-119) restated in float64 numpy: the oracle of
mr_eval_accumulate and SequenceEvaluater.log()."""
import numpy as np


def accumulate(rows, sizes, state=None):
    """Folds the fp32 metric rows [G,M] of G batches of `sizes` images into state = (total, valid, running_avg,
    num_samples), in the evaluater's operation order.  Returns the new state (float64 arrays and an int)."""
    rows = np.asarray(rows, np.float32)
    m = rows.shape[1]
    total, valid, avg, n = (np.zeros(m), np.zeros(m), np.zeros(m), 0) if state is None else \
        (state[0].copy(), state[1].copy(), state[2].copy(), state[3])
    for row, b in zip(rows, sizes):
        metrics = np.zeros(m)
        metrics += row.astype(np.float64)                    # acc_metrics[i] += metric(...)
        if np.any(np.isnan(metrics)):
            metrics, ok = np.zeros(m), np.zeros(m)
        else:
            ok = np.ones(m)
        total += metrics
        valid += ok
        if n == 0:
            avg += metrics
        else:
            avg = avg * (n / (n + b)) + metrics * (b / (n + b))
        n += b
    return total, valid, avg, n


def log(state):
    total, valid, avg, _ = state
    with np.errstate(divide="ignore", invalid="ignore"):
        metrics = total / valid
    return {"loss": 0.0, "metrics": metrics.tolist(), "metrics_correct": avg.tolist(), "valid_batches": valid[0],
            "loss_loss": 0.0}


def batch_sizes(n, batch_size):
    """The DataLoader's batch sizes over n key frames (shuffle=False, drop_last=False)."""
    return [min(batch_size, n - b) for b in range(0, n, batch_size)]
