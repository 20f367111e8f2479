"""The motion matching oracle (oracle/feature_search_oracle.c) on the CPU: its cost against exact rational arithmetic, its pack against a
numpy float32 restatement with directions through the pinned rtm operation, and its selection rules on hand-built databases. The GPU tests
(tests/test_gpu_feature_search.py) compare the library with this oracle bit for bit."""
import numpy as np
import pytest

from acl_b200 import api
from oracle import feature_search as FS
from tests import feature_search_cases as cases

NO_ROW = cases.NO_ROW


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("dims", [1, 3, 23, 64])
def test_cost_is_one_rounding_per_subtract_and_per_fma(seed, dims):
    rng = np.random.default_rng(seed * 100 + dims)
    for _ in range(20):
        q = rng.normal(size=dims).astype(np.float32) * np.float32(rng.choice([1e-3, 1.0, 1e3]))
        x = rng.normal(size=dims).astype(np.float32)
        assert FS.cost(q, x).view(np.uint32) == cases.exact_cost(q, x).view(np.uint32)


def test_cost_is_fused_where_the_orders_differ():
    """Inputs on which acc + diff * diff (two roundings) and fmaf (one) give different bits: the oracle must give the fused bits"""
    rng = np.random.default_rng(7)
    found = 0
    for _ in range(400):
        q = rng.normal(size=5).astype(np.float32)
        x = rng.normal(size=5).astype(np.float32)
        fused, unfused = cases.exact_cost(q, x), cases.unfused_cost(q, x)
        if fused.view(np.uint32) != unfused.view(np.uint32):
            found += 1
            assert FS.cost(q, x).view(np.uint32) == fused.view(np.uint32)
    assert found >= 20, found


def test_cost_of_special_values():
    assert FS.cost([0.0], [0.0]).view(np.uint32) == 0                     # +0, never -0
    assert FS.cost([-0.0], [0.0]).view(np.uint32) == 0
    assert np.isinf(FS.cost([3e38, 0.0], [-3e38, 0.0]))                    # the difference overflows: +inf
    assert np.isinf(FS.cost([1e20], [0.0]))                                # the square overflows
    assert np.isnan(FS.cost([np.inf], [np.inf]))
    assert np.isnan(FS.cost([1.0, np.nan], [1.0, 0.0]))


def test_pack_every_kind_and_mask_against_numpy():
    rng = np.random.default_rng(1)
    S, K = 4, 4
    rows = cases.fabricated_rows(rng, 9, S, K)
    terms = cases.every_term(S, K)
    got = FS.pack(rows, 9, K, S * K * 48, terms)
    want = cases.numpy_pack(rows, K, terms)
    assert np.array_equal(_bits(got), _bits(want))


def test_pack_normalises_unfused_and_keeps_padding():
    rng = np.random.default_rng(2)
    S, K = 3, 2
    rows = cases.fabricated_rows(rng, 5, S, K)
    terms = api.make_feature_terms([api.FEATURE_POSITION, api.FEATURE_VELOCITY, api.FEATURE_DIRECTION], [0, 1, 2], [1, 0, 1], [7, 5, 3],
                                   s1=[0, 2, 0], axis=[0, 0, 2], inv_dt=[0.0, 7.5, 0.0])
    dims = api.feature_term_dims(terms)
    mean = rng.normal(size=dims).astype(np.float32)
    scale = rng.uniform(0.1, 3.0, dims).astype(np.float32)
    padding = np.full((5, 12), 1234.5, np.float32)
    got = FS.pack(rows, 5, K, S * K * 48, terms, mean, scale, out_stride=12, out=padding)
    want = cases.numpy_pack(rows, K, terms, mean, scale)
    assert np.array_equal(_bits(got[:, :dims]), _bits(want))
    assert np.all(got[:, dims:] == 1234.5)
    # identity statistics: the same as none
    assert np.array_equal(_bits(FS.pack(rows, 5, K, S * K * 48, terms, np.zeros(dims), np.ones(dims))),
                          _bits(FS.pack(rows, 5, K, S * K * 48, terms)))


def test_direction_is_the_rotated_unit_axis():
    for axis in range(3):
        assert np.array_equal(FS.direction([0, 0, 0, 1], axis), np.eye(3, dtype=np.float32)[axis])
    # a quarter turn about z takes x to y
    h = np.float32(np.sqrt(0.5))
    assert np.allclose(FS.direction([0, 0, h, h], 0), [0, 1, 0], atol=1e-6)
    rng = np.random.default_rng(3)
    for _ in range(50):
        q = rng.normal(size=4).astype(np.float32)
        q /= np.linalg.norm(q)
        for axis in range(3):
            assert np.array_equal(_bits(FS.direction(q, axis)), _bits(cases.pinned_direction(q, axis)))


def _database(costs_rows):
    """one dimension databases: row r = [value], the query = [0]: cost of row r = value^2"""
    return np.asarray(costs_rows, np.float32).reshape(-1, 1)


def _search(database, queries, tags=None, query_vectors=None, dims=1):
    query_vectors = np.zeros((len(queries), database.shape[1] if database.ndim == 2 else dims), np.float32) if query_vectors is None else query_vectors
    got = FS.search(database, query_vectors, queries, dims, tags)
    return [(int(r), np.float32(c)) for r, c in zip(got["row"], got["cost"])]


@pytest.mark.parametrize("best", [[31, 32, 255, 256, 257], [0, 299], [63, 64, 128], [299], [255, 256]])
def test_ties_go_to_the_lowest_row_anywhere(best):
    """equal costs on both sides of what would be tile boundaries (the rows -1 and +1 square to the same cost)"""
    v = np.full(300, 5.0, np.float32)
    v[best] = [(-1.0) ** i for i in range(len(best))]
    assert _search(_database(v), api.make_search_queries(1))[0] == (min(best), np.float32(1.0))


def test_exclusion_windows():
    db = _database(np.arange(10, dtype=np.float32))
    q = lambda b, e: _search(db, api.make_search_queries(1, b, e))[0][0]
    assert q(0, 0) == 0                # empty
    assert q(5, 3) == 0                # begin after end: empty
    assert q(0, 1) == 1                # begin is excluded, end is not
    assert q(0, 4) == 4
    assert q(1, 4) == 0                # partial
    assert q(0, 10) == NO_ROW          # whole
    assert q(0, 0xFFFFFFFF) == NO_ROW  # beyond the end
    assert q(0, 12) == NO_ROW
    assert q(10, 20) == 0              # entirely beyond the end


def test_tags():
    db = _database([3.0, 1.0, 2.0, 0.5])
    tags = np.array([1, 2, 4, 2], np.uint32)
    assert _search(db, api.make_search_queries(1), tags)[0][0] == 0
    assert _search(db, api.make_search_queries(4), tags)[0][0] == 2
    assert _search(db, api.make_search_queries(6), tags)[0][0] == 3
    assert _search(db, api.make_search_queries(8), tags)[0] == (NO_ROW, np.float32(np.inf))    # no tag allowed
    assert _search(db, api.make_search_queries(0), tags)[0] == (NO_ROW, np.float32(np.inf))


def test_nan_and_inf():
    db = _database([np.nan, 3e38, np.inf, 2.0])
    # a NaN row is never a candidate; +inf costs are
    assert _search(db, api.make_search_queries(1, 3, 4))[0] == (1, np.float32(np.inf))
    assert _search(db, api.make_search_queries(1))[0] == (3, np.float32(4.0))
    tags = np.array([1, 2, 2, 2], np.uint32)
    assert _search(db, api.make_search_queries(1), tags)[0] == (NO_ROW, np.float32(np.inf))     # only the NaN row is allowed
    # a NaN query has no candidate
    qv = np.array([[np.nan]], np.float32)
    assert _search(db, api.make_search_queries(0xFFFFFFFF), query_vectors=qv)[0] == (NO_ROW, np.float32(np.inf))
    # inf - inf is NaN, inf - finite is inf
    qv = np.array([[np.inf]], np.float32)
    assert _search(db, api.make_search_queries(1), query_vectors=qv)[0] == (1, np.float32(np.inf))


def test_empty_database():
    got = FS.search(np.zeros((0, 4), np.float32), np.zeros((3, 4), np.float32), api.make_search_queries([1, 2, 3]), 4)
    assert list(got["row"]) == [NO_ROW] * 3 and np.all(np.isinf(got["cost"]))


@pytest.mark.parametrize("seed", range(3))
def test_search_equals_the_written_rules(seed):
    """random databases with duplicates, tags, windows, a NaN row: the oracle against cases.reference_search with exact costs"""
    rng = np.random.default_rng(seed)
    n, dims, q = 97, 5, 13
    db = rng.integers(-3, 4, size=(n, 8)).astype(np.float32) * np.float32(0.5)
    db[rng.integers(0, n, 10)] = db[rng.integers(0, n, 10)]
    db[17, 2] = np.nan
    tags = rng.integers(0, 8, n).astype(np.uint32)
    qv = rng.integers(-3, 4, size=(q, 8)).astype(np.float32) * np.float32(0.5)
    begin = rng.integers(0, n + 5, q)
    queries = api.make_search_queries(rng.integers(0, 8, q), begin, begin + rng.integers(0, 30, q))
    got = FS.search(db, qv, queries, dims, tags)
    want = cases.reference_search(db, qv, queries, dims, tags, cost=lambda a, b: cases.exact_cost(a, b)
                                  if np.all(np.isfinite(a)) and np.all(np.isfinite(b)) else np.float32(np.nan))
    assert [(int(r), int(np.float32(c).view(np.uint32))) for r, c in zip(got["row"], got["cost"])] == \
           [(r, int(np.float32(c).view(np.uint32))) for r, c in want]
