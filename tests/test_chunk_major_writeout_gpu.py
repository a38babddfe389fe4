"""GPU tests for the write-out and the chunk choice of the chunk-major score kernel (pecos_b200/csrc/xlinear_cm_kernel.cuh):
a slice's scores go out eight columns at a time through a shared-memory tile, four pairs per store instruction, and a CTA
whose chunk runs dry moves to the chunk with the most unclaimed work per CTA already on it.  The cases put the write-out at
chunk widths around multiples of 8, at candidate positions that are not multiples of 8, with both staging depths (chunks of
up to 16 columns stage four rounds, wider ones two), for queries of 0 to 40 features, and make the claims run dry exactly
at a slice boundary or find nothing at all.  Each must return the same ids, counts and score bits as the query-major
kernels (kernel mode 6), for a batch whose rows are shuffled between runs (a pair no warp scores would show another
query's scores), and match the oracles."""
import numpy as np
import pytest
import scipy.sparse as smat

from pecos_b200 import synth

from .test_chunk_major_claims_gpu import _check
from .util import random_tree

pytestmark = pytest.mark.gpu

D = 400


def _leaf_model(folder, seed, widths, upper):
    """Upper layers from random_tree(upper); the leaf gives layer-1 node j exactly widths[j] children (one chunk each)."""
    assert len(widths) == upper[-1]
    layers = random_tree(seed, upper, D, 24, bias=1.0)
    W_leaf, _ = synth.make_tree_model(seed + 1, [1, int(np.sum(widths))], D, 24, bias=1.0)[1]
    layers.append((smat.csc_matrix(W_leaf, dtype=np.float32), synth._contiguous_codes(widths)))
    synth.save_xlinear_model(folder, layers, bias=1.0, only_topk=8)


def _ragged_queries(seed, n):
    """n query rows of 0, 1, 3, 7, 8, 9, 17 or 40 features (the first eight rows: one of each)."""
    rng = np.random.default_rng(seed)
    choices = np.array([0, 1, 3, 7, 8, 9, 17, 40])
    lens = rng.choice(choices, size=n)
    lens[: choices.size] = choices
    indptr = np.r_[0, np.cumsum(lens)].astype(np.int64)
    indices = np.concatenate([np.sort(rng.choice(D, size=k, replace=False)) for k in lens]).astype(np.int64)
    data = rng.uniform(0.1, 1.0, size=indices.size).astype(np.float32)
    X = smat.csr_matrix((data, indices, indptr), shape=(n, D))
    X.has_sorted_indices = True
    return X


def _widths(case):
    rng = np.random.default_rng(903)
    return {
        "1": np.full(48, 1), "7": np.full(48, 7), "8": np.full(48, 8), "9": np.full(48, 9), "33": np.full(48, 33),
        "256": np.full(12, 256),                    # the widest chunk the kernel takes uncut
        "mixed": rng.integers(1, 41, 48),           # candidate positions at every residue mod 8
        "cut": rng.integers(257, 330, 12),          # cut into two column ranges each, of odd widths
    }[case]


@pytest.mark.parametrize("case", ["1", "7", "8", "9", "33", "256", "mixed", "cut"])
def test_writeout_widths_and_positions(tmp_path, gpu_clib, have_ref, case):
    """Leaf chunks of one width each (1, 7, 8, 9, 33, 256 columns), of mixed widths, and wider than 256 columns (cut into
    column ranges); queries of 0 to 40 features, forced onto the chunk-major kernel (mode 5)."""
    widths = _widths(case)
    folder = str(tmp_path / "m")
    _leaf_model(folder, 901, widths, [4, widths.size])
    X = _ragged_queries(902, 1500)
    _check(gpu_clib, have_ref, folder, X, 3, 5, f"width {case}", runs=2, oracle_rows=np.r_[0:64])


@pytest.mark.parametrize("queries", [96, 1024])
def test_buckets_of_whole_slices(tmp_path, gpu_clib, have_ref, queries):
    """Six leaf chunks, all in every beam: every bucket holds exactly `queries` = 32 x k pairs, so the claim after a
    chunk's last slice lands exactly on the bucket's end, and every slice is full."""
    folder = str(tmp_path / "m")
    _leaf_model(folder, 911, np.array([20, 5, 13, 20, 9, 31]), [2, 6])
    X = synth.make_queries(912, queries, D, 24)
    _check(gpu_clib, have_ref, folder, X, 3, 5, f"{queries} pairs per chunk", runs=3)


def test_fewer_slices_than_warps(tmp_path, gpu_clib, have_ref):
    """20 queries over three leaf chunks: three slices in the whole launch, fewer than the warps of one CTA; most CTAs
    find their chunk dry at once, and the last ones find every chunk claimed."""
    folder = str(tmp_path / "m")
    _leaf_model(folder, 921, np.array([9, 40, 17]), [2, 3])
    X = _ragged_queries(922, 20)
    _check(gpu_clib, have_ref, folder, X, 3, 5, "fewer slices than warps", runs=3)
