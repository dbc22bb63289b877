"""Multi-GPU parity (needs >= 2 visible GPUs; skipped otherwise): rows sharded over 2 ranks, NCCL all-reduce of the Gram
inside ks_blockls_fit, every rank solves redundantly -> all ranks hold the same model and it matches the fp64 oracle."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, world, id_holder, ret, custom_solve, precision):
    sys.path.insert(0, ROOT)
    import keystone_b200 as ks
    from oracle import keystone_oracle as ko
    rng = np.random.default_rng(21)
    n, d_in, n_out, k = 6001, 40, 256, 6
    X = rng.standard_normal((n, d_in)).astype(np.float32)
    cls = rng.integers(0, k, n)
    X[: n // 2] *= 4.0   # the two ranks see inputs of different magnitude: their fp16 operand scales differ
    params = [ko.cosine_random_features_params(d_in, n_out, 0.2 / 2, rng) for _ in range(2)]
    lo, hi = ks.shard_range(n, rank, world)
    ctx = ks.Context(device=rank, rank=rank, world_size=world, nccl_id=id_holder["id"])
    ctx.set_option("custom_solve", custom_solve)   # 0: cuSOLVER potrs, -1: automatic (the DMMA kernel at this k)
    x = ctx.matrix(X[lo:hi]); y = ctx.labels_from_classes(cls[lo:hi], k)
    rfs = [ks.CosineRandomFeatures(ctx, W, b) for W, b in params]
    feats = ks.Pipeline.gather(rfs).andThen(ks.VectorCombiner())(x)
    model = ks.BlockLeastSquaresEstimator(n_out, 2, 0.5, precision=precision).fit(feats, y)
    assert ctx.last_fit_stats()["mma"] == {"f16": "f16", "tf32": "tf32x1", "default": "f16x2"}[precision]
    assert ctx.last_fit_stats()["lookahead"] == 2
    assert ctx.last_fit_stats()["solve"] == ("potrs-column-sharded" if custom_solve == 0 else "dmma-kernel-column-sharded")
    W = np.concatenate(model.xs, 0)
    cost = model.compute_cost(feats, y, 0.5)
    if rank == 0:
        F = np.concatenate([ko.cosine_random_features(X.astype(np.float64), Wm, b) for Wm, b in params], 1)
        Y = ko.class_label_indicators(cls, k)
        xs, b0, mus = ko.block_ls_fit(F, Y, n_out, 2, 0.5)
        Wr = np.concatenate(xs, 0)
        ret["rel"] = float(np.linalg.norm(W - Wr) / np.linalg.norm(Wr))
        ret["cost_rel"] = float(abs(cost - ko.compute_cost(F, Y, 0.5, xs, n_out, b0)) / cost)
        ret["b_err"] = float(np.abs(model.b_opt - b0).max())
    ret[f"W{rank}"] = W
    ctx.close()


@pytest.mark.parametrize("custom_solve,precision", [(-1, "default"), (-1, "f16"), (0, "tf32")],
                         ids=["parity-mode", "fp16-operands", "tf32-potrs-solve"])
def test_two_rank_fit_matches_oracle(custom_solve, precision):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import keystone_b200 as ks
    mgr = mp.Manager()
    id_holder = mgr.dict(); ret = mgr.dict()
    id_holder["id"] = ks.Context.new_nccl_id()
    mp.spawn(_worker, args=(2, id_holder, ret, custom_solve, precision), nprocs=2, join=True)
    assert ret["rel"] < (1e-4 if precision == "default" else 1.5e-3), ret["rel"]
    assert ret["cost_rel"] < 1e-4 and ret["b_err"] < 1e-6   # computeCost applies the model in the context's (parity) mode
    assert np.array_equal(ret["W0"], ret["W1"])      # redundant solves are bit-identical across ranks


def _bwls_worker(rank, world, id_holder, ret):
    sys.path.insert(0, ROOT)
    import keystone_b200 as ks
    A = np.loadtxt(os.path.join(ROOT, "tests", "golden", "aMat.csv"), delimiter=",")
    B = np.loadtxt(os.path.join(ROOT, "tests", "golden", "bMat.csv"), delimiter=",")
    rows = np.r_[0:10] if rank == 0 else np.r_[10:15]            # classes {0, 1} on rank 0, class 2 on rank 1
    ctx = ks.Context(device=rank, rank=rank, world_size=world, nccl_id=id_holder["id"])
    model = ks.BlockWeightedLeastSquaresEstimator(4, 10, 0.1, 0.3).fit(ctx.matrix(A[rows]), ctx.matrix(B[rows]))
    ret[f"W{rank}"] = np.concatenate(model.xs, 0)
    ret[f"b{rank}"] = model.b_opt
    # a class split over two ranks must be rejected on every rank
    bad = np.r_[0:8] if rank == 0 else np.r_[8:15]
    try:
        ks.BlockWeightedLeastSquaresEstimator(4, 1, 0.1, 0.3).fit(ctx.matrix(A[bad]), ctx.matrix(B[bad]))
        ret[f"rejected{rank}"] = False
    except ks.KeystoneError:
        ret[f"rejected{rank}"] = True
    ctx.close()


def test_two_rank_class_sharded_bwls_matches_oracle():
    """BlockWeightedLeastSquares with the rows sharded by class over 2 ranks (the reference's one-class-per-partition layout,
    T/nodes/learning/BlockWeightedLeastSquaresSuite.scala:67-68) equals the single-process fp64 oracle on the full fixture."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import keystone_b200 as ks
    from oracle import keystone_oracle as ko
    mgr = mp.Manager()
    id_holder = mgr.dict(); ret = mgr.dict()
    id_holder["id"] = ks.Context.new_nccl_id()
    mp.spawn(_bwls_worker, args=(2, id_holder, ret), nprocs=2, join=True)
    A = np.loadtxt(os.path.join(ROOT, "tests", "golden", "aMat.csv"), delimiter=",")
    B = np.loadtxt(os.path.join(ROOT, "tests", "golden", "bMat.csv"), delimiter=",")
    xs, fb = ko.bwls_fit(A, B, 4, 10, 0.1, 0.3)
    Wr = np.concatenate(xs, 0)
    assert np.linalg.norm(ret["W0"] - Wr) / np.linalg.norm(Wr) < 1e-4
    assert np.abs(ret["b0"] - fb).max() < 1e-4
    assert np.array_equal(ret["W0"], ret["W1"]) and np.array_equal(ret["b0"], ret["b1"])
    assert ret["rejected0"] and ret["rejected1"]
