"""Evaluation nodes of the reference (keystoneml.evaluation) on top of the device path.

EXPERIMENTAL -- the "next" row after the solver (SURVEY.md section 8(f)): the confusion matrix is counted on the GPU
(`ks_model_confusion_matrix`: apply -> MaxClassifier -> counts, summed over the ranks); the metrics are closed-form
functions of the k x k matrix evaluated on the host, as the reference does on the Spark driver
(K/evaluation/MulticlassClassifierEvaluator.scala:23-54, K/evaluation/BinaryClassifierEvaluator.scala:16-41).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import List

import numpy as np

from ._capi import check, lib
from .context import feature_source_args
from .nodes import BlockLinearMapper, _as_dataset, _device_matrix


@dataclass(frozen=True)
class BinaryClassificationMetrics:
    tp: float
    fp: float
    tn: float
    fn: float

    def merge(self, o: "BinaryClassificationMetrics") -> "BinaryClassificationMetrics":
        return BinaryClassificationMetrics(self.tp + o.tp, self.fp + o.fp, self.tn + o.tn, self.fn + o.fn)

    @property
    def accuracy(self) -> float:
        return (self.tp + self.tn) / (self.tp + self.fp + self.tn + self.fn)

    @property
    def error(self) -> float:
        return (self.fp + self.fn) / (self.tp + self.fp + self.tn + self.fn)

    @property
    def recall(self) -> float:
        return self.tp / (self.tp + self.fn)

    @property
    def precision(self) -> float:
        return self.tp / (self.tp + self.fp)

    @property
    def specificity(self) -> float:
        return self.tn / (self.fp + self.tn)

    def fScore(self, beta: float = 1.0) -> float:
        b2 = beta * beta
        return (1.0 + b2) * self.tp / ((1.0 + b2) * self.tp + b2 * self.fn + self.fp)


class MulticlassMetrics:
    """confusionMatrix: rows are the true labels, columns the predicted labels (MulticlassClassifierEvaluator.scala:21-24)."""

    def __init__(self, confusion_matrix: np.ndarray):
        cm = np.asarray(confusion_matrix, dtype=np.float64)
        if cm.ndim != 2 or cm.shape[0] != cm.shape[1]:
            raise ValueError("Confusion matrix must be square")
        self.confusionMatrix = cm
        total, actual, predicted = cm.sum(), cm.sum(axis=1), cm.sum(axis=0)
        self.classMetrics: List[BinaryClassificationMetrics] = []
        for c in range(cm.shape[0]):
            tp = cm[c, c]
            fp = predicted[c] - tp
            tn = total - actual[c] - fp
            self.classMetrics.append(BinaryClassificationMetrics(tp, fp, tn, total - tp - fp - tn))

    def _avg(self, f) -> float:
        return sum(f(m) for m in self.classMetrics) / len(self.classMetrics)

    def _micro(self, f) -> float:
        merged = self.classMetrics[0]
        for m in self.classMetrics[1:]:
            merged = merged.merge(m)
        return f(merged)

    avgAccuracy = property(lambda self: self._avg(lambda m: m.accuracy))
    avgError = property(lambda self: self._avg(lambda m: m.error))
    macroPrecision = property(lambda self: self._avg(lambda m: m.precision))
    macroRecall = property(lambda self: self._avg(lambda m: m.recall))
    totalAccuracy = property(lambda self: self._micro(lambda m: m.precision))
    totalError = property(lambda self: self._micro(lambda m: m.fn / (m.fn + m.tp)))
    microPrecision = property(lambda self: self._micro(lambda m: m.precision))
    microRecall = property(lambda self: self._micro(lambda m: m.recall))

    def macroFScore(self, beta: float = 1.0) -> float:
        return self._avg(lambda m: m.fScore(beta))

    def microFScore(self, beta: float = 1.0) -> float:
        return self._micro(lambda m: m.fScore(beta))


class BinaryClassifierEvaluator:
    """BinaryClassifierEvaluator (K/evaluation/BinaryClassifierEvaluator.scala): the contingency table of boolean predictions
    against boolean actuals."""

    @staticmethod
    def evaluate(predictions, actuals) -> BinaryClassificationMetrics:
        p = np.asarray(predictions).astype(bool).ravel()
        a = np.asarray(actuals).astype(bool).ravel()
        if p.shape != a.shape:
            raise ValueError("predictions and actuals differ in length")
        return BinaryClassificationMetrics(float(np.sum(p & a)), float(np.sum(p & ~a)), float(np.sum(~p & ~a)), float(np.sum(~p & a)))


class MulticlassClassifierEvaluator:
    """MulticlassClassifierEvaluator(numClasses).  `evaluate_model` runs model -> MaxClassifier -> confusion matrix on the device
    for a fitted BlockLinearMapper and +-1 indicator labels; `from_confusion_matrix` wraps counts obtained elsewhere."""

    def __init__(self, num_classes: int):
        self.num_classes = int(num_classes)

    def evaluate_model(self, model: BlockLinearMapper, data, labels) -> MulticlassMetrics:
        ds = _as_dataset(model.ctx, data)
        lb = _as_dataset(model.ctx, labels)
        if model.k != self.num_classes:
            raise ValueError("model output width and numClasses differ")
        f, x, rfs, n = feature_source_args(ds)
        out = np.zeros((self.num_classes, self.num_classes), dtype=np.float64)
        check(model.ctx.handle, lib().ks_model_confusion_matrix(model.ctx.handle, model.handle, f, x, rfs, n, lb.handle,
                                                                out.ctypes.data_as(C.c_void_p)))
        return MulticlassMetrics(out)

    @staticmethod
    def from_confusion_matrix(cm: np.ndarray) -> MulticlassMetrics:
        return MulticlassMetrics(cm)


AVERAGE, BORDA = "average", "borda"   # AggregationPolicyType (K/evaluation/AugmentedExamplesEvaluator.scala)


class AugmentedExamplesEvaluator:
    """``new AugmentedExamplesEvaluator(names, numClasses, policy)`` (K/evaluation/AugmentedExamplesEvaluator.scala): the views that
    share a name are one example.  ``average`` adds their scores and divides by the count; ``borda`` adds each class's rank in the
    view's ascending stable sort (ties go by class index).  The first maximum is the prediction.  Grouping the names is host
    bookkeeping (a permutation and group offsets); the pass over the (n_views x k) scores and the counts run on the device
    (``ks_grouped_confusion_matrix``).  Every view of a name must carry the same label, as the reference asserts.  One rank only:
    the groups must not span ranks."""

    def __init__(self, names, numClasses: int, policy: str = AVERAGE):
        if policy not in (AVERAGE, BORDA):
            raise ValueError("policy must be 'average' or 'borda'")
        self.names, self.num_classes, self.policy = np.asarray(names), int(numClasses), policy

    def groups(self):
        """(rows, offsets): the view rows of each name, names in order of first appearance, views in their order."""
        _, first, inv = np.unique(self.names, return_index=True, return_inverse=True)
        rank = np.empty(first.size, dtype=np.int64)
        rank[np.argsort(first, kind="stable")] = np.arange(first.size)
        g = rank[inv.reshape(-1)]
        rows = np.argsort(g, kind="stable").astype(np.int64)
        offsets = np.concatenate([[0], np.cumsum(np.bincount(g, minlength=first.size))]).astype(np.int64)
        return rows, offsets

    def evaluate(self, predicted, actual_labels, ctx=None) -> MulticlassMetrics:
        scores = _device_matrix(ctx, predicted)
        labels = np.ascontiguousarray(actual_labels, dtype=np.int32).reshape(-1)
        if labels.size != scores.rows or self.names.size != scores.rows:
            raise ValueError("names, scores and labels need one entry per view")
        rows, offsets = self.groups()
        out = np.zeros((self.num_classes, self.num_classes), dtype=np.float64)
        check(scores.ctx.handle, lib().ks_grouped_confusion_matrix(scores.ctx.handle, scores.handle, rows.ctypes.data_as(C.c_void_p),
                                                                   offsets.ctypes.data_as(C.c_void_p), offsets.size - 1,
                                                                   labels.ctypes.data_as(C.c_void_p), self.num_classes,
                                                                   0 if self.policy == AVERAGE else 1, out.ctypes.data_as(C.c_void_p)))
        return MulticlassMetrics(out)
