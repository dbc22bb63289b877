"""CTA pairs of the split-operand kernels (parity mode, fp16 pairs).

The split Gram and the split residual update run as clusters of two CTAs whose tiles share one operand panel; each CTA fetches
half of that panel for both.  The Gram's tile list pairs tiles along a row (shared A panel), pairs the leftover last tiles of
odd-length rows across rows (shared B panel), and runs a final odd leftover beside an idle partner; the update pairs column tiles
(m, 2q) and (m, 2q + 1) and leaves the partner of an odd last column tile idle.  Every tile must be computed exactly once, so a
tile dropped or computed twice, a half panel missing or landing in the wrong CTA, moves entries by O(1).

The operands and bounds are those of test_gpu_split_gram.py and test_gpu_kmajor.py: every partial sum is exact in fp32."""
import numpy as np
import pytest

import keystone_b200 as ks
from test_gpu_kmajor import TILE, _check_update
from test_gpu_split_gram import _check, _debug_gram, _pair_operand, _split

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = ks.Context(0)
    c.set_option("precision", 2)  # KS_PRECISION_F16X2: ks_debug_gram runs the split kernel
    yield c
    c.close()


@pytest.fixture(scope="module")
def n_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _g_pairs(b):
    """(A-shared pairs, B-shared pairs, lone tiles) of the G triangle with b columns, as the host builds the list."""
    nb = -(-b // TILE)
    lens = [nb - i for i in range(nb)]
    left = sum(n % 2 for n in lens)
    return sum(n // 2 for n in lens), left // 2, left % 2


def _run(ctx, n, m, kc, chunk=0):
    rng = np.random.default_rng(n * 31 + m * 7 + kc)
    A = _pair_operand(rng, n, m)
    B = _pair_operand(rng, n, kc)
    ah, al = _split(A)
    bh, bl = _split(B)
    ctx.set_option("gram_chunk_rows", chunk)
    try:
        G, Cm = _debug_gram(ctx, A, B)
    finally:
        ctx.set_option("gram_chunk_rows", 0)
    n_chunks = -(-n // (chunk or 4096))
    g_ref = ah.T @ ah + al.T @ ah + ah.T @ al
    c_ref = ah.T @ bh + al.T @ bh + ah.T @ bl
    assert np.abs(g_ref - ah.T @ ah).max() > 1e-3 and np.abs(c_ref - ah.T @ bh).max() > 1e-3
    _check(G, g_ref, ah, ah, al, al, n_chunks)
    _check(Cm, c_ref, ah, bh, al, bl, n_chunks)


def test_g_at_the_fit_block_size(ctx):
    """b = 4096: 32 tile rows; the 16 odd-length rows leave tile (i, 31) over, and those 16 pair across rows on B_31.  k = 1000:
    8 column tiles of C, 4 A-shared pairs per row.  Two row chunks."""
    assert _g_pairs(4096) == (256, 8, 0)
    _run(ctx, 300, 4096, 1000, chunk=160)


# b with an odd number of column tiles: 5 tiles -> 6 A-shared pairs, the leftovers of rows 0, 2, 4 give one B-shared pair and a
# lone tile; 2 tiles -> one A-shared pair and a lone diagonal tile; 1 tile -> a lone tile only
@pytest.mark.parametrize("b", [5 * TILE - 3, 2 * TILE - 2, 64])
def test_g_leftovers(ctx, b):
    a_pairs, b_pairs, lone = _g_pairs(b)
    assert lone == 1 and (b < TILE or a_pairs > 0) and (b != 5 * TILE - 3 or b_pairs == 1)
    _run(ctx, 1000, b, 37, chunk=96)


# C with 1 column tile (every tile a leftover: B-shared pairs across the 3 rows of A and a lone one), 7 (three A-shared pairs per
# row, leftovers across rows) and 8 (A-shared pairs only)
@pytest.mark.parametrize("kc", [1, 7 * TILE - 5, 8 * TILE - 24])
def test_c_column_tiles(ctx, kc):
    _run(ctx, 777, 3 * TILE - 1, kc)


# odd column-tile counts of the update: the partner of the last column tile of each row of tiles is idle (1 tile: every pair)
@pytest.mark.parametrize("M,N,K", [(1000, 1, 64), (4097, 3 * TILE - 1, 65), (300, 5 * TILE, 200), (129, 7 * TILE - 3, 33)])
def test_update_odd_column_tiles(ctx, M, N, K):
    _check_update(ctx, M, N, K, "f16x2", seed=M + N + K, combos=((0, 0), (0, 1)))


def test_update_pairs_wrap_the_tile_ring(ctx, n_sms):
    """At least 9 pairs per cluster with an odd column-tile count: the 8-slot tile ring wraps while some pairs have an idle
    partner."""
    N, K = 3 * TILE - 7, 32
    pairs_per_row = 2
    m_tiles = -(-9 * (n_sms // 2) // pairs_per_row) + 1
    M = m_tiles * TILE - 5
    _check_update(ctx, M, N, K, "f16x2", seed=29, combos=((0, 1),))
