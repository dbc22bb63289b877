"""AmazonReviewsDataLoader, NewsgroupsDataLoader and BinaryClassifierEvaluator on the host (no GPU needed)."""
import json

import numpy as np
import pytest

import keystone_b200 as ks


def test_amazon_loader_threshold_and_sorted_files(tmp_path):
    d = tmp_path / "amazon"
    d.mkdir()
    (d / "b.json").write_text(json.dumps({"overall": 3.5, "reviewText": "at the threshold"}) + "\n")
    (d / "a.json").write_text(json.dumps({"overall": 3.4, "reviewText": "just below", "asin": "x"}) + "\n\n" +
                              json.dumps({"overall": 5, "reviewText": "Great!"}) + "\n")
    ld = ks.AmazonReviewsDataLoader(str(d), 3.5)
    assert ld.data == ["just below", "Great!", "at the threshold"]
    assert ld.labels.tolist() == [0, 1, 1]
    one = ks.AmazonReviewsDataLoader(str(d / "b.json"), 4.0)
    assert one.labels.tolist() == [0]


def test_amazon_loader_missing_field_names_file_and_line(tmp_path):
    f = tmp_path / "r.json"
    f.write_text(json.dumps({"overall": 1.0, "reviewText": "ok"}) + "\n" + json.dumps({"overall": 2.0}) + "\n")
    with pytest.raises(ValueError, match=r"r\.json:2"):
        ks.AmazonReviewsDataLoader(str(f), 3.5)


def test_newsgroups_loader_classes_order_and_replacement(tmp_path):
    assert len(ks.NewsgroupsDataLoader.classes) == 20 and ks.NewsgroupsDataLoader.classes[0] == "comp.graphics"
    for name in ks.NewsgroupsDataLoader.classes:
        (tmp_path / name).mkdir()
    (tmp_path / "sci.med" / "2").write_bytes(b"caf\xe9 latin-1")
    (tmp_path / "sci.med" / "1").write_bytes("naïve".encode())
    (tmp_path / "comp.graphics" / "9").write_bytes(b"pixels")
    ld = ks.NewsgroupsDataLoader(str(tmp_path))
    assert ld.data == ["pixels", "naïve", "caf� latin-1"]
    assert ld.labels.tolist() == [0, 11, 11]


def test_binary_classifier_evaluator():
    m = ks.BinaryClassifierEvaluator.evaluate(np.array([1, 1, 0, 0, 1]) > 0, np.array([1, 0, 0, 1, 1]) > 0)
    assert (m.tp, m.fp, m.tn, m.fn) == (2.0, 1.0, 1.0, 1.0)
    assert abs(m.accuracy - 0.6) < 1e-15


def test_newsgroups_loader_missing_class_directory_raises(tmp_path):
    for name in ks.NewsgroupsDataLoader.classes[:-1]:
        (tmp_path / name).mkdir()
    with pytest.raises(FileNotFoundError, match="soc.religion.christian"):
        ks.NewsgroupsDataLoader(str(tmp_path))
