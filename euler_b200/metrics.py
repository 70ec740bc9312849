"""The streaming metrics of tf_euler/python/utils/metrics.py (acc_score, auc_score, f1_score) on the device, with TF 1.x
tf.metrics semantics: each call adds the batch's counts to the metric's state and returns the value over every batch seen
since construction or the last reset(), as the metric's update op does.

Each metric is a torch module whose state lives in non-persistent buffers: it moves with the module (.to, .cuda) and
follows the inputs' device, and it never enters a state_dict, so a model holding one keeps its checkpoint keys.
    m(labels, predict)   adds the batch and returns the value (a 0-d float32 device tensor of its own)
    m.result()           the value of the current state
    m.reset()            zeroes the state (and StreamingAuc's refused count)
The update is one device op (ops.metric_auc_update, ops.metric_count_update) that never synchronises with the host, so a
training step that reports a metric stays capturable in a CUDA graph.  Labels and predictions are float32 of one numel.

Per-batch counts are exact integers rounded once to float32 and added with one float32 add; TF's float reduce_sum gives the
same counts for batches below 2^24 elements.  StreamingAuc departs from TF in one way: a batch with a sigmoid outside [0, 1]
or NaN is skipped and counted in `refused` (TF raises), and the value reads NaN until reset().
"""
import torch

from . import ops


class _Streaming(torch.nn.Module):
    def _state(self, name, shape, dtype, device):
        self.register_buffer(name, torch.zeros(shape, dtype=dtype, device=device), persistent=False)

    def _follow(self, device):
        if self.value.device != device:
            self.to(device)

    def result(self):
        """the value of the current state (NaN while a StreamingAuc has refused a batch)"""
        return self.value.clone()

    def reset(self):
        """zero the state: the next value counts the batches after this call only"""
        for b in self.buffers():
            b.zero_()


class StreamingAuc(_Streaming):
    """auc_score(labels, predict, num_thresholds=5000): tf.metrics.auc(labels, sigmoid(predict), num_thresholds), the
    trapezoidal ROC over the thresholds -1e-7, i / (T - 1) for 0 < i < T - 1, and 1 + 1e-7 (2 <= T <= 16384).  State: tp,
    fn, tn, fp f32[T] and refused (the batches skipped for a sigmoid outside [0, 1] or NaN)."""

    def __init__(self, num_thresholds=5000, device=None):
        super().__init__()
        T = int(num_thresholds)
        if not 2 <= T <= 16384:
            raise ValueError("num_thresholds must lie in [2, 16384], got %r" % (num_thresholds,))
        self.num_thresholds = T
        for name in ('tp', 'fn', 'tn', 'fp'):
            self._state(name, (T,), torch.float32, device)
        self._state('refused', (), torch.int64, device)
        self._state('value', (), torch.float32, device)

    def forward(self, labels, predict):
        self._follow(predict.device)
        predictions = torch.sigmoid(predict.detach())
        ops.metric_auc_update(labels, predictions, self.tp, self.fn, self.tn, self.fp, self.refused, self.value)
        return self.value.clone()


class StreamingF1(_Streaming):
    """f1_score(labels, predict): predictions floor(predict + 0.5), state tp, fn, fp (f32[3], tf.metrics.true_positives,
    false_negatives, false_positives), value 2 p r / (p + r + 1e-7) with p = tp / (1e-7 + tp + fp), r = tp / (1e-7 + tp + fn)."""

    def __init__(self, device=None):
        super().__init__()
        self._state('state', (3,), torch.float32, device)
        self._state('value', (), torch.float32, device)

    def forward(self, labels, predict):
        self._follow(predict.device)
        ops.metric_count_update('f1', self.state, self.value, labels, predict)
        return self.value.clone()


class StreamingAccuracy(_Streaming):
    """acc_score(labels, predict): tf.metrics.accuracy(labels, floor(predict + 0.5)), state total and count (f32[2]), value
    total / count (0 before any element)."""

    def __init__(self, device=None):
        super().__init__()
        self._state('state', (2,), torch.float32, device)
        self._state('value', (), torch.float32, device)

    def forward(self, labels, predict):
        self._follow(predict.device)
        ops.metric_count_update('acc', self.state, self.value, labels, predict)
        return self.value.clone()

    def add_counts(self, correct, total):
        """add a batch already counted: correct (an int64 device scalar, e.g. ops.gae_loss's) of total (a host int)
        predictions; the same state as the (labels, predict) form over that batch"""
        self._follow(correct.device)
        ops.metric_count_update('acc', self.state, self.value, correct=correct, total=total)
        return self.value.clone()


METRICS = {'acc': StreamingAccuracy, 'auc': StreamingAuc, 'f1': StreamingF1}


def get(name, device=None):
    """metrics.get: a new streaming metric of `name`, one of 'acc', 'auc' and 'f1' (auc at upstream's 5000 thresholds), its
    state on `device`"""
    if name not in METRICS:
        raise ValueError("streaming metric_name must be one of %s, got %r" % (sorted(METRICS), name))
    return METRICS[name](device=device)
