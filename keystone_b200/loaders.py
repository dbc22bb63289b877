"""Loaders for the file formats the reference's hot-path pipelines read, and model persistence (SURVEY 8f next-4).

Reference (K/ = src/main/scala/keystoneml/):
  CsvDataLoader             K/loaders/CsvDataLoader.scala:28-30       headerless CSV of doubles, one row per line
  LabeledData               K/loaders/LabeledData.scala               (labels, data) pair
  TimitFeaturesDataLoader   K/loaders/TimitFeaturesDataLoader.scala:22-83  feature CSVs + sparse "row label" files (both 1-based)
  CifarLoader               K/loaders/CifarLoader.scala:30-45         records of 1 label byte + 3072 image bytes
  MNIST CSV layout          K/pipelines/images/mnist/MnistRandomFFT.scala:34-36  column 0 = 1-based label, rest = pixels
  AmazonReviewsDataLoader   K/loaders/AmazonReviewsDataLoader.scala   JSON lines: label = overall >= threshold, data = reviewText
  NewsgroupsDataLoader      K/loaders/NewsgroupsDataLoader.scala      one directory per class, one document per file
Parsing happens in the native library (keystone_b200/csrc/io.cu); the arrays returned here are host buffers ready for
``Context.matrix`` / ``Context.labels_from_classes``.
"""
from __future__ import annotations

import ctypes as C
import json
import os
from dataclasses import dataclass
from typing import List, Tuple

import numpy as np

from ._capi import KeystoneError, lib


def _io_check(rc: int) -> None:
    if rc != 0:
        msg = lib().ks_io_last_error()
        raise KeystoneError(rc, msg.decode("utf-8", "replace") if msg else "i/o error")


@dataclass
class LabeledData:
    """K/loaders/LabeledData.scala: ``labels`` (int class ids) and ``data`` (one row per item)."""
    labels: np.ndarray
    data: np.ndarray


def CsvDataLoader(path: str, dtype=np.float32) -> np.ndarray:
    """All rows of a headerless CSV of numbers as an (n_rows x n_cols) array (CsvDataLoader.scala:28-30)."""
    rows, cols = C.c_int64(0), C.c_int64(0)
    _io_check(lib().ks_csv_dims(path.encode(), C.byref(rows), C.byref(cols)))
    out = np.empty((rows.value, cols.value), dtype=dtype)
    if rows.value == 0:
        return out
    fn = lib().ks_csv_read_f64 if dtype == np.float64 else lib().ks_csv_read_f32
    _io_check(fn(path.encode(), out.ctypes.data_as(C.c_void_p), rows.value, cols.value, cols.value))
    return out


def MnistCsvLoader(path: str) -> LabeledData:
    """MNIST CSV as the reference's pipeline reads it: label = int(column 0) - 1, data = columns 1.. (MnistRandomFFT.scala:34-36)."""
    m = CsvDataLoader(path, np.float32)
    return LabeledData(labels=m[:, 0].astype(np.int32) - 1, data=np.ascontiguousarray(m[:, 1:]))


def TimitLabelsLoader(path: str, n_rows: int) -> np.ndarray:
    """Sparse "row label" file (both 1-based) -> zero-based int32 labels per data row (TimitFeaturesDataLoader.scala:26-42)."""
    out = np.empty(n_rows, dtype=np.int32)
    _io_check(lib().ks_timit_labels_read(path.encode(), out.ctypes.data_as(C.c_void_p), n_rows))
    if (out < 0).any():
        raise KeystoneError(-1, f"{path}: no label for data row {int(np.argmax(out < 0)) + 1}")
    return out


def TimitFeaturesDataLoader(train_data: str, train_labels: str, test_data: str, test_labels: str) -> Tuple[LabeledData, LabeledData]:
    """TimitFeaturesDataLoader.apply (:59-83): (train, test) LabeledData; 440 features, 147 classes in the real data set."""
    tr = CsvDataLoader(train_data, np.float32)
    te = CsvDataLoader(test_data, np.float32)
    return (LabeledData(TimitLabelsLoader(train_labels, tr.shape[0]), tr), LabeledData(TimitLabelsLoader(test_labels, te.shape[0]), te))


def CifarLoader(path: str) -> LabeledData:
    """CIFAR-10 binary file -> labels (int32) and images as uint8 [n][3][32][32] (channel planes as stored; CifarLoader.scala:20-45)."""
    n = C.c_int64(0)
    _io_check(lib().ks_cifar_read(path.encode(), None, None, 0, C.byref(n)))
    images = np.empty((n.value, 3072), dtype=np.uint8)
    labels = np.empty(n.value, dtype=np.int32)
    _io_check(lib().ks_cifar_read(path.encode(), images.ctypes.data_as(C.c_void_p), labels.ctypes.data_as(C.c_void_p), n.value,
                                  C.byref(n)))
    return LabeledData(labels=labels, data=images.reshape(n.value, 3, 32, 32))


def _json_files(path: str) -> List[str]:
    if os.path.isdir(path):
        return [os.path.join(path, f) for f in sorted(os.listdir(path)) if os.path.isfile(os.path.join(path, f)) and not f.startswith((".", "_"))]
    return [path]


def AmazonReviewsDataLoader(path: str, threshold: float) -> LabeledData:
    """The Amazon product reviews (AmazonReviewsDataLoader.scala): JSON records, one per line, from one file or from every file of a
    directory in sorted name order.  ``labels[i]`` is 1 when record i's ``overall`` is >= ``threshold``, else 0; ``data`` is the list
    of its ``reviewText`` strings.  A record without either field raises ``ValueError`` naming the file and line."""
    labels: List[int] = []
    docs: List[str] = []
    for f in _json_files(path):
        with open(f, encoding="utf-8") as fh:
            for ln, line in enumerate(fh, 1):
                if not line.strip():
                    continue
                rec = json.loads(line)
                if not isinstance(rec, dict) or "overall" not in rec or "reviewText" not in rec:
                    raise ValueError(f"{f}:{ln}: a review needs the fields overall and reviewText")
                labels.append(1 if float(rec["overall"]) >= threshold else 0)
                docs.append(str(rec["reviewText"]))
    return LabeledData(np.asarray(labels, dtype=np.int32), docs)


class NewsgroupsDataLoader:
    """The 20 Newsgroups documents (NewsgroupsDataLoader.scala): ``NewsgroupsDataLoader(path)`` returns ``LabeledData`` whose data
    holds every file of ``path/<class>/`` for the classes below in order, files in sorted name order, decoded as UTF-8 with invalid
    bytes replaced by U+FFFD (as Hadoop's ``Text`` decodes them); the label is the class index.  A missing class directory raises
    ``FileNotFoundError``, as the reference's ``wholeTextFiles`` fails on a missing path."""

    classes = ["comp.graphics", "comp.os.ms-windows.misc", "comp.sys.ibm.pc.hardware", "comp.sys.mac.hardware", "comp.windows.x",
               "rec.autos", "rec.motorcycles", "rec.sport.baseball", "rec.sport.hockey", "sci.crypt", "sci.electronics", "sci.med",
               "sci.space", "misc.forsale", "talk.politics.misc", "talk.politics.guns", "talk.politics.mideast", "talk.religion.misc",
               "alt.atheism", "soc.religion.christian"]

    def __new__(cls, path: str) -> LabeledData:
        labels: List[int] = []
        docs: List[str] = []
        for k, name in enumerate(cls.classes):
            d = os.path.join(path, name)
            if not os.path.isdir(d):
                raise FileNotFoundError(f"{d}: the class directory {name!r} is missing")
            for f in sorted(os.listdir(d)):
                fp = os.path.join(d, f)
                if os.path.isfile(fp):
                    with open(fp, "rb") as fh:
                        docs.append(fh.read().decode("utf-8", "replace"))
                    labels.append(k)
        return LabeledData(np.asarray(labels, dtype=np.int32), docs)
