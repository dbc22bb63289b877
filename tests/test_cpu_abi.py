"""CPU-side checks (no GPU needed): the C-ABI library loads, exports every symbol the header declares,
refuses to run without a device (no CPU fallback), and the host-side workflow mirror keeps the
reference's andThen / gather / fit-once semantics."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import keystone_b200 as ks
from keystone_b200 import _capi
from keystone_b200.workflow import Estimator, LabelEstimator, Pipeline, Transformer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", autouse=True)
def built():
    if not os.path.exists(_capi.LIB_PATH):
        from keystone_b200 import build
        build.build(verbose=False)


def test_library_exports_every_declared_symbol():
    syms = _capi.declared_symbols()
    assert len(syms) >= 30
    out = subprocess.check_output(["nm", "-D", "--defined-only", _capi.LIB_PATH], text=True)
    exported = {line.split()[-1] for line in out.splitlines() if " T " in line}
    missing = [s for s in syms if s not in exported]
    assert not missing, missing
    lib = _capi.lib()
    for s in syms:
        assert hasattr(lib, s)
    assert lib.ks_version() >= 100


def test_library_has_hopper_tensor_core_code():
    """The shipped binary must contain sm_90a wgmma / TMA instructions (SASS mnemonics HGMMA, UTMALDG, UTMASTG)."""
    try:
        sass = subprocess.check_output(["cuobjdump", "-sass", _capi.LIB_PATH], text=True, stderr=subprocess.DEVNULL)
    except (OSError, subprocess.CalledProcessError):
        pytest.skip("cuobjdump not available")
    assert "HGMMA" in sass and "UTMALDG" in sass and "UTMASTG" in sass
    assert "sm_90a" in sass


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(ks.KeystoneError) as ei:
        ks.Context(0)
    assert ei.value.code == -5 and "no CPU fallback" in str(ei.value)
    # unknown context handles are reported, not dereferenced
    assert _capi.lib().ks_ctx_synchronize(12345) == -6


def test_product_does_not_import_oracle():
    for root, _, files in os.walk(os.path.join(ROOT, "keystone_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(root, f)).read()
                assert "import oracle" not in src and "from oracle" not in src, f


def test_shard_range_partitions_rows():
    for n in (0, 1, 7, 1000, 1_000_000):
        for w in (1, 2, 3, 8):
            r = [ks.shard_range(n, i, w) for i in range(w)]
            assert r[0][0] == 0 and r[-1][1] == n
            assert all(r[i][1] == r[i + 1][0] for i in range(w - 1))
            sizes = [b - a for a, b in r]
            assert max(sizes) - min(sizes) <= 1


# ---- workflow semantics (T/workflow/PipelineSuite.scala, EstimatorSuite, LabelEstimatorSuite) ----
class _Plus(Transformer):
    def __init__(self, c):
        self.c = c

    def apply(self, x):
        return x + self.c


class _MeanEst(Estimator):
    def __init__(self):
        self.n_fit = 0

    def fit(self, data):
        self.n_fit += 1
        return _Plus(-float(np.mean(data)))


class _LabelEst(LabelEstimator):
    def __init__(self):
        self.n_fit = 0

    def fit(self, data, labels):
        self.n_fit += 1
        return _Plus(float(np.mean(labels) - np.mean(data)))


def test_and_then_chains_transformers():
    p = _Plus(1).andThen(_Plus(2)).andThen(_Plus(3))
    assert isinstance(p, Pipeline) and p(np.array([0.0]))[0] == 6.0


def test_and_then_estimator_fits_once_on_prefix_output():
    est = _MeanEst()
    data = np.array([1.0, 2.0, 3.0])
    p = _Plus(10).andThen(est, data)           # Chainable.scala:44-50
    assert est.n_fit == 0                       # lazy
    assert np.allclose(p(data), [-1, 0, 1])
    p(data); p.fit()
    assert est.n_fit == 1                       # PipelineSuite.scala:28


def test_and_then_label_estimator():
    est = _LabelEst()
    data, labels = np.array([1.0, 3.0]), np.array([10.0, 20.0])
    p = _Plus(0).andThen(est, data, labels)    # Chainable.scala:67-73
    assert np.allclose(p(data).mean(), 15.0) and est.n_fit == 1
    with pytest.raises(TypeError):
        _Plus(0).andThen(est, data)


def test_gather_applies_branches_to_same_input():
    g = Pipeline.gather([_Plus(1), _Plus(2).andThen(_Plus(3))])
    out = g(np.array([0.0]))
    assert [o[0] for o in out] == [1.0, 5.0]


def test_estimator_constants_match_reference():
    e = ks.BlockLeastSquaresEstimator(1000, 3)
    assert e.weight == 10                                            # BlockLinearMapper.scala:204
    # cost formula, BlockLinearMapper.scala:268-282
    c = e.cost(1_000_000, 10000, 1000, 1.0, 16, 3.8e-4, 2.9e-1, 1.32)
    flops = 1e6 * 10000 * 2000 / 16; byt = 1e6 * 10000 / 16 + 1e7; net = 2.0 * 10000 * 2000 * 4
    assert np.isclose(c, 3 * (max(3.8e-4 * flops, 2.9e-1 * byt) + 1.32 * net))
    assert ks.VectorSplitter(5).bounds(12) == [(0, 5), (5, 10), (10, 12)]
    assert ks.VectorSplitter(8, 12).bounds(20) == [(0, 8), (8, 12)]


def test_multiclass_metrics_host_formulas_match_the_reference_suite():
    """T/evaluation/MulticlassClassifierEvaluatorSuite.scala:9-68 through the product's host-side metric formulas, and the
    same numbers from the oracle restatement (the device part, the counting, is exercised by the GPU tests)."""
    import numpy as np
    import keystone_b200 as ks
    from oracle import keystone_oracle as ko
    cm = np.array([[2, 1, 1], [1, 3, 0], [0, 0, 1]], dtype=float)
    m = ks.MulticlassClassifierEvaluator.from_confusion_matrix(cm)
    o = ko.multiclass_metrics(cm)
    assert abs(m.classMetrics[0].precision - 2.0 / 3) < 1e-12 and abs(m.classMetrics[2].recall - 1.0) < 1e-12
    assert abs(m.microRecall - 6.0 / 9) < 1e-12 and abs(m.microPrecision - m.microRecall) < 1e-12
    for mine, theirs in [(m.macroPrecision, o["macro_precision"]), (m.macroRecall, o["macro_recall"]),
                         (m.macroFScore(), o["macro_fscore"]), (m.microFScore(), o["micro_fscore"]),
                         (m.totalAccuracy, o["total_accuracy"]), (m.totalError, o["total_error"]),
                         (m.avgAccuracy, o["avg_accuracy"]), (m.avgError, o["avg_error"])]:
        assert abs(mine - theirs) < 1e-12
    assert abs(m.macroFScore(2.0) - ko.multiclass_metrics(cm, beta=2.0)["macro_fscore"]) < 1e-12


def test_least_squares_estimator_cost_model_selection():
    """T/nodes/learning/LeastSquaresEstimatorSuite.scala:11-102: with the reference's weights and 16 machines the cost model picks
    the exact solver for (n=1e6, d=1000, k=1000), the block solver for (n=1e6, d=10000, k=1000) and sparse L-BFGS for
    (n=1e6, d=10000, k=2, sparsity 0.01)."""
    import keystone_b200 as ks
    est = ks.LeastSquaresEstimator(num_machines=16)
    assert est.optimize(1_000_000, 1000, 1000, 1.0) == "exact"
    assert est.optimize(1_000_000, 10000, 1000, 1.0) == "block"
    assert est.optimize(1_000_000, 10000, 2, 0.01) == "sparse_lbfgs"
    c = est.costs(1_000_000, 10000, 1000, 1.0, 16)
    # BlockLinearMapper.scala:268-282 with blockSize 1000, 3 iterations
    flops = 1e6 * 10000 * (1000 + 1000) / 16
    bytes_scanned = 1e6 * 10000 / 16 + 10000.0 * 1000
    network = 2.0 * 10000 * (1000 + 1000) * 4.0
    assert abs(c["block"] - 3 * (max(3.8e-4 * flops, 2.9e-1 * bytes_scanned) + 1.32 * network)) < 1e-6 * c["block"]
