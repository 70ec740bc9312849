"""numpy float32 restatements of TF 1.x tf.metrics.auc, true_positives / false_negatives / false_positives and accuracy as
tf_euler/python/utils/metrics.py uses them, and of the fixed order the device sums the AUC in (include/euler_b200.h,
eu_metric_auc_update).  The reference of tests/test_streaming_metrics_cpu.py and _gpu.py."""
import numpy as np

F32 = np.float32
LANES = 1024   # the lanes of the AUC value's fixed-order sum


def thresholds(T):
    """metrics_impl.auc's thresholds, computed in Python doubles and rounded once to float32"""
    kepsilon = 1e-7
    t = [0.0 - kepsilon] + [(i + 1) * 1.0 / (T - 1) for i in range(T - 2)] + [1.0 + kepsilon]
    return np.asarray(t, dtype=np.float64).astype(F32)


def literal_counts(labels, predictions, T, tile=1 << 16):
    """metrics_impl._confusion_matrix_at_thresholds literally: the [T, N] comparison predictions > thresholds (tiled over N),
    labels cast to bool; (tp, fn, tn, fp) int64[T]"""
    thr = thresholds(T)[:, None]
    lab = np.asarray(labels, F32).reshape(-1) != 0
    pred = np.asarray(predictions, F32).reshape(-1)
    out = np.zeros((4, T), np.int64)
    for s in range(0, pred.size, tile):
        above = pred[None, s:s + tile] > thr
        pos = lab[None, s:s + tile]
        out[0] += (above & pos).sum(1)
        out[1] += (~above & pos).sum(1)
        out[2] += (~above & ~pos).sum(1)
        out[3] += (above & ~pos).sum(1)
    return out


def bucket_counts(labels, predictions, T):
    """the same counts by bucket and suffix sum: bucket b(p) = #{i : t[i] < p}, positive at threshold i iff i < b(p)"""
    lab = np.asarray(labels, F32).reshape(-1) != 0
    b = np.searchsorted(thresholds(T), np.asarray(predictions, F32).reshape(-1), side='left')
    hp = np.bincount(b[lab], minlength=T + 1)
    hn = np.bincount(b[~lab], minlength=T + 1)
    cp, cn = np.cumsum(hp)[:T], np.cumsum(hn)[:T]   # at or below threshold i
    return np.stack([hp.sum() - cp, cp, cn, hn.sum() - cn]).astype(np.int64)


def auc_value(tp, fn, tn, fp):
    """the trapezoidal AUC of the float32 state, each op in float32, summed in the device's fixed order"""
    eps = F32(1e-6)
    tp, fn, tn, fp = [np.asarray(v, F32) for v in (tp, fn, tn, fp)]
    rec = (tp + eps) / ((tp + fn) + eps)
    fpr = fp / ((fp + tn) + eps)
    terms = (fpr[:-1] - fpr[1:]) * ((rec[:-1] + rec[1:]) / F32(2))
    part = np.zeros(LANES, F32)
    for r in range(0, terms.size, LANES):
        chunk = terms[r:r + LANES]
        part[:chunk.size] = part[:chunk.size] + chunk
    s = LANES // 2
    while s:
        part[:s] = part[:s] + part[s:2 * s]
        s //= 2
    return part[0]


def auc_value_f64(tp, fn, tn, fp):
    """the same AUC in float64 from the same state"""
    tp, fn, tn, fp = [np.asarray(v, np.float64) for v in (tp, fn, tn, fp)]
    rec = (tp + 1e-6) / (tp + fn + 1e-6)
    fpr = fp / (fp + tn + 1e-6)
    return float(np.sum((fpr[:-1] - fpr[1:]) * (rec[:-1] + rec[1:]) / 2))


class Auc(object):
    """tf.metrics.auc's state over batches: counts added as float32, a batch with a prediction outside [0, 1] or NaN is
    skipped and counted in refused, and the value reads NaN while refused > 0"""

    def __init__(self, T, counts=literal_counts):
        self.T, self.counts = T, counts
        self.state = np.zeros((4, T), F32)   # tp, fn, tn, fp
        self.refused = 0

    def update(self, labels, predictions):
        p = np.asarray(predictions, F32).reshape(-1)
        if not np.all((p >= 0) & (p <= 1)):
            self.refused += 1
        else:
            self.state = self.state + self.counts(labels, p, self.T).astype(F32)
        return self.value()

    def value(self):
        return F32(np.nan) if self.refused else auc_value(*self.state)


def rounded(predict):
    """tf.floor(predict + 0.5) in float32"""
    return np.floor(np.asarray(predict, F32) + F32(0.5))


class F1(object):
    """metrics.f1_score's streaming state (tp, fn, fp) and value, in float32"""

    def __init__(self):
        self.state = np.zeros(3, F32)

    def update(self, labels, predict):
        lab = np.asarray(labels, F32).reshape(-1) != 0
        pred = rounded(predict).reshape(-1) != 0   # NaN casts to True
        counts = np.array([(lab & pred).sum(), (lab & ~pred).sum(), (~lab & pred).sum()], np.int64)
        self.state = self.state + counts.astype(F32)
        return self.value()

    def value(self):
        eps = F32(1e-7)
        tp, fn, fp = self.state
        p = tp / ((eps + tp) + fp)
        r = tp / ((eps + tp) + fn)
        return ((F32(2) * p) * r) / ((p + r) + eps)


class Accuracy(object):
    """metrics.acc_score's streaming state (total, count) and value, in float32"""

    def __init__(self):
        self.state = np.zeros(2, F32)

    def add_counts(self, correct, total):
        self.state = self.state + np.array([correct, total], np.int64).astype(F32)
        return self.value()

    def update(self, labels, predict):
        lab = np.asarray(labels, F32).reshape(-1)
        return self.add_counts(int((rounded(predict).reshape(-1) == lab).sum()), lab.size)

    def value(self):
        total, count = self.state
        return total / count if count > 0 else F32(0)
