"""aclb200_pack_pose_features and aclb200_search_pose_features against the C oracle (oracle/feature_search.py), bit for bit: every packed
float, and each result's row and the bits of its cost. The search is checked at every launch shape (one query, a few, many), across row
tile boundaries, with ties in different blocks, windows, tags, NaN and inf rows, on two streams, and end to end from
aclb200_extract_pose_features output."""
import numpy as np
import pytest

from acl_b200.api import make_search_queries
from oracle import feature_search as FS
from tests import bones_cases
from tests import clips
from tests import feature_search_cases as cases

pytestmark = pytest.mark.gpu
NO_ROW = cases.NO_ROW
OFFSETS = np.array([-1.0 / 30.0, 0.0, 1.0 / 3.0, 2.0 / 3.0], np.float32)


@pytest.fixture(scope="module")
def gpu():
    import torch
    import acl_b200 as ab
    return dict(torch=torch, ab=ab, ctx=ab.Context(0))


def _dev(gpu, array):
    return gpu["torch"].from_numpy(np.ascontiguousarray(array).reshape(-1).view(np.uint8)).cuda()


def _stride(dims, extra=4):
    return (dims + 3) // 4 * 4 + extra


def _search(gpu, database, query_vectors, queries, dims, tags=None, stream=None):
    """the library's results as SEARCH_RESULT_DTYPE [Q]; database and query_vectors are float32 [rows][stride] host arrays"""
    torch, ab = gpu["torch"], gpu["ab"]
    q = queries.size
    d_db = torch.from_numpy(np.ascontiguousarray(database, np.float32)).cuda() if database.shape[0] else None
    d_qv = torch.from_numpy(np.ascontiguousarray(query_vectors, np.float32)).cuda()
    d_results = torch.full((q * 2,), 0x55555555, dtype=torch.int32, device="cuda")
    gpu["ctx"].search_pose_features(d_db, database.shape[0], database.shape[1], d_qv, _dev(gpu, queries), q, query_vectors.shape[1], dims,
                                    d_results, d_row_tags=None if tags is None else _dev(gpu, tags), stream=stream)
    torch.cuda.synchronize()
    return d_results.cpu().numpy().view(ab.SEARCH_RESULT_DTYPE)


def _assert_oracle(got, database, query_vectors, queries, dims, tags=None):
    want = FS.search(database, query_vectors, queries, dims, tags)
    bad = np.nonzero(got.view(np.uint64) != want.view(np.uint64))[0]
    assert bad.size == 0, f"{bad.size} of {queries.size} differ, first {bad[0]}: got {got[bad[0]]}, want {want[bad[0]]}"
    return want


def _random(rng, rows, dims, stride, quantum=None):
    x = np.full((rows, stride), np.nan, np.float32)        # the padding floats are never read into a cost
    values = rng.normal(size=(rows, dims)).astype(np.float32)
    if quantum is not None:
        values = (np.round(values / quantum) * quantum).astype(np.float32)
    x[:, :dims] = values
    return x


def _queries(rng, q, n, tag_bits=3):
    begin = rng.integers(0, max(n, 1) + 3, q)
    return make_search_queries(rng.integers(1, 1 << tag_bits, q), begin, begin + rng.integers(0, 12, q))


@pytest.mark.parametrize("dims", [1, 3, 4, 5, 23, 63, 64])
@pytest.mark.parametrize("num_queries", [1, 9, 130])
def test_every_dimension_count(gpu, dims, num_queries):
    rng = np.random.default_rng(dims * 1000 + num_queries)
    n = 700
    db = _random(rng, n, dims, _stride(dims))
    qv = _random(rng, num_queries, dims, _stride(dims, 8))
    tags = rng.integers(0, 8, n).astype(np.uint32)
    queries = _queries(rng, num_queries, n)
    _assert_oracle(_search(gpu, db, qv, queries, dims, tags), db, qv, queries, dims, tags)


@pytest.mark.parametrize("num_rows", [1, 31, 32, 33, 63, 64, 65, 255, 256, 257, 513])
@pytest.mark.parametrize("num_queries", [1, 3, 100])
def test_row_counts_around_tiles(gpu, num_rows, num_queries):
    """64 rows per tile for many queries, 256 for one or a few"""
    rng = np.random.default_rng(num_rows * 7 + num_queries)
    dims = 5
    db = _random(rng, num_rows, dims, 8, quantum=0.5)       # coarse values: many equal costs
    qv = _random(rng, num_queries, dims, 8, quantum=0.5)
    queries = _queries(rng, num_queries, num_rows)
    _assert_oracle(_search(gpu, db, qv, queries, dims), db, qv, queries, dims)


@pytest.mark.parametrize("num_queries", [1, 3])
def test_a_large_database(gpu, num_queries):
    rng = np.random.default_rng(11)
    n, dims = 2_500_000, 23
    db = _random(rng, n, dims, 24)
    qv = _random(rng, num_queries, dims, 24)
    tags = (np.arange(n) % 2 + 1).astype(np.uint32)
    queries = make_search_queries([1, 3, 2][:num_queries], [0, n - 10, 123456][:num_queries], [0, n, 123466][:num_queries])
    _assert_oracle(_search(gpu, db, qv, queries, dims, tags), db, qv, queries, dims, tags)


@pytest.mark.parametrize("num_queries", [1, 7, 64, 65, 4097, 70000])
def test_query_counts(gpu, num_queries):
    rng = np.random.default_rng(num_queries)
    n, dims = 45, 7
    db = _random(rng, n, dims, 8)
    qv = _random(rng, num_queries, dims, 12)
    tags = rng.integers(0, 4, n).astype(np.uint32)
    queries = _queries(rng, num_queries, n, tag_bits=2)
    _assert_oracle(_search(gpu, db, qv, queries, dims, tags), db, qv, queries, dims, tags)


def test_many_queries_against_many_rows(gpu):
    rng = np.random.default_rng(1024)
    n, q, dims = 100_000, 1024, 23
    db = _random(rng, n, dims, 24)
    qv = _random(rng, q, dims, 24)
    tags = rng.integers(0, 4, n).astype(np.uint32)
    queries = _queries(rng, q, n, tag_bits=2)
    _assert_oracle(_search(gpu, db, qv, queries, dims, tags), db, qv, queries, dims, tags)


@pytest.mark.parametrize("num_queries", [1, 5, 200])
def test_duplicated_best_rows_in_different_blocks(gpu, num_queries):
    """every query's own vector sits at several rows far apart, so different blocks find the same cost: the lowest row must win"""
    rng = np.random.default_rng(3 + num_queries)
    n, dims = 300_000, 9
    db = _random(rng, n, dims, 12)
    qv = _random(rng, num_queries, dims, 12)
    copies = []
    for q in range(num_queries):
        at = np.sort(rng.choice(n, 4, replace=False))
        db[at] = qv[q]
        copies.append(at)
    queries = make_search_queries(np.full(num_queries, 1), 0, 0)
    got = _search(gpu, db, qv, queries, dims)
    want = _assert_oracle(got, db, qv, queries, dims)
    for q in range(num_queries):
        assert want["row"][q] == copies[q][0] and want["cost"][q] == 0.0


def test_windows_tags_nan_and_inf(gpu):
    rng = np.random.default_rng(5)
    n, dims = 1000, 4
    db = _random(rng, n, dims, 4)
    db[100] = np.nan
    db[101, 2] = np.inf
    db[102, 0] = 3e38
    db[103] = db[100]
    tags = np.ones(n, np.uint32)
    tags[500:600] = 0                                   # tagged out of every query
    tags[[100, 101, 102]] = 2
    qv = np.zeros((8, 4), np.float32)
    qv[[0, 1, 2, 6]] = db[[999, 600, 102, 300]]
    qv[3, 1] = np.nan                                   # a NaN query
    qv[4, 2] = np.inf
    queries = make_search_queries([1, 1, 3, 3, 2, 2, 1, 1],
                            [990, 599, 0, 0, 100, 101, 300, 500],
                            [n, n, 0, 0, 101, 103, 301, 0xFFFFFFFF])
    got = _search(gpu, db, qv, queries, dims, tags)
    want = _assert_oracle(got, db, qv, queries, dims, tags)
    assert want["row"][0] != 999 and want["row"][1] != 600                  # windows ending at N
    assert want["row"][3] == NO_ROW                                          # NaN query
    assert want["row"][5] == NO_ROW                                          # the window leaves only the NaN row of tag 2
    assert want["row"][6] != 300                                             # exclude_begin itself is excluded
    assert want["row"][7] < 500                                              # a window past the end


def test_only_nan_rows_allowed(gpu):
    db = np.full((70, 4), np.nan, np.float32)
    db[::2, 0] = 1.0                                    # rows with one NaN component: NaN costs
    db[69] = 0.0
    tags = np.ones(70, np.uint32)
    tags[69] = 2
    qv = np.zeros((3, 4), np.float32)
    queries = make_search_queries([1, 2, 3], 0, 0)
    got = _search(gpu, db, qv, queries, 4, tags)
    _assert_oracle(got, db, qv, queries, 4, tags)
    assert got["row"][0] == NO_ROW and np.isinf(got["cost"][0]) and got["row"][1] == 69 and got["row"][2] == 69


def test_empty_database(gpu):
    qv = np.zeros((5, 4), np.float32)
    launches = gpu["ctx"].launch_count
    got = _search(gpu, np.zeros((0, 4), np.float32), qv, make_search_queries(np.full(5, 1), 0, 0), 4)
    assert np.all(got.view(np.uint64) == 0x7F800000FFFFFFFF)
    assert gpu["ctx"].launch_count == launches + 1      # only the results' clear


def test_two_streams_and_repeated_launches(gpu):
    torch, ab = gpu["torch"], gpu["ab"]
    rng = np.random.default_rng(9)
    n, dims = 200_000, 23
    db = _random(rng, n, dims, 24)
    d_db = torch.from_numpy(db).cuda()
    launches = []
    for q in (1, 37, 3000):
        qv = _random(rng, q, dims, 24)
        queries = _queries(rng, q, n)
        launches.append((q, qv, queries, torch.from_numpy(qv).cuda(), _dev(gpu, queries)))
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    results = [[torch.zeros(q * 2, dtype=torch.int32, device="cuda") for q, *_ in launches] for _ in range(2)]
    torch.cuda.synchronize()
    for repeat in range(2):
        for i, (q, qv, queries, d_qv, d_queries) in enumerate(launches):
            gpu["ctx"].search_pose_features(d_db, n, 24, d_qv, d_queries, q, 24, dims, results[repeat][i], stream=streams[(i + repeat) % 2])
    torch.cuda.synchronize()
    for i, (q, qv, queries, *_) in enumerate(launches):
        first = results[0][i].cpu().numpy()
        assert np.array_equal(first, results[1][i].cpu().numpy())
        _assert_oracle(first.view(ab.SEARCH_RESULT_DTYPE), db, qv, queries, dims)


def _features(gpu, name, requests_time, looping):
    """extract_pose_features rows of clip `name` (S = 4 offsets, K = 4 bones of a binary tree skeleton) and the bone count"""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    blob = clips.load_blob(name)
    clipset = ctx.upload([blob])
    bones = clipset.max_tracks
    tree = bones_cases.tree(bones)
    bone_list = np.array([0, bones - 1, bones // 2, min(1, bones - 1)], np.uint32)
    n = requests_time.size
    requests = ab.make_feature_requests(np.zeros(n, np.uint32), requests_time, looping)
    d_out = torch.zeros((n, 4, 4, 12), dtype=torch.float32, device="cuda")
    ctx.extract_pose_features(clipset, _dev(gpu, requests), n, ab.Options(looping_policy=ab.LOOP_CLAMP), OFFSETS, _dev(gpu, bone_list), 4,
                              _dev(gpu, tree), d_out)
    torch.cuda.synchronize()
    return d_out, clipset


def _bench_terms(ab):
    """the D = 23 packing of tools/bench_feature_search.py"""
    P, V, Dn = ab.FEATURE_POSITION, ab.FEATURE_VELOCITY, ab.FEATURE_DIRECTION
    return ab.make_feature_terms([P, P, V, V, V, P, P, Dn, Dn], [1, 1, 0, 0, 0, 2, 3, 2, 3], [1, 2, 1, 2, 3, 0, 0, 0, 0],
                                 [7, 7, 7, 7, 7, 5, 5, 5, 5], s1=1, axis=2, inv_dt=30.0)


@pytest.mark.parametrize("name", ["c1_30bones", "mixed_scale", "looping", "one_bone"])
def test_pack_of_extracted_features(gpu, name):
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    rng = np.random.default_rng(4)
    n = 333
    d_rows, _ = _features(gpu, name, rng.uniform(-0.2, 3.0, n).astype(np.float32), (np.arange(n) % 2).astype(np.uint32))
    rows = d_rows.cpu().numpy()
    for terms in (_bench_terms(ab), cases.every_term(4, 4)):
        dims = ab.feature_term_dims(terms)
        stride = _stride(dims)
        mean = rng.normal(size=dims).astype(np.float32)
        scale = rng.uniform(0.5, 2.0, dims).astype(np.float32)
        for stats in ((None, None), (mean, scale)):
            d_out = torch.full((n, stride), 777.0, dtype=torch.float32, device="cuda")
            ctx.pack_pose_features(d_rows, n, 4, 4, terms, d_out, stride, *stats)
            torch.cuda.synchronize()
            got = d_out.cpu().numpy()
            want = FS.pack(rows, n, 4, 4 * 4 * 48, terms, *stats, out_stride=stride, out=np.full((n, stride), 777.0, np.float32))
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_pack_with_a_pose_stride(gpu):
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    rng = np.random.default_rng(8)
    S, K, n = 3, 5, 100
    pose = S * K * 48 + 32
    rows = np.zeros((n, pose // 4), np.float32)
    rows[:, : S * K * 12] = cases.fabricated_rows(rng, n, S, K).reshape(n, -1)
    terms = ab.make_feature_terms([ab.FEATURE_POSITION, ab.FEATURE_VELOCITY, ab.FEATURE_DIRECTION], [2, 0, 1], [4, 3, 0], [3, 6, 7], s1=2,
                                  axis=1, inv_dt=7.0)
    d_out = torch.zeros((n, 8), dtype=torch.float32, device="cuda")
    ctx.pack_pose_features(torch.from_numpy(rows).cuda(), n, S, K, terms, d_out, 8, pose_stride_bytes=pose)
    torch.cuda.synchronize()
    want = FS.pack(rows, n, K, pose, terms, out_stride=8)
    assert np.array_equal(d_out.cpu().numpy().view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("name", ["c1_30bones", "looping"])
def test_end_to_end_from_one_clip(gpu, name):
    """a database from every sample of the clip, queries packed from requests on the same clip: with a window around each query's own
    time, and without one (the query's own sample then costs 0)"""
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    info_clip = ctx.upload([clips.load_blob(name)]).clip_info(0)
    samples = info_clip.num_samples
    times = (np.arange(samples, dtype=np.float32) / np.float32(info_clip.sample_rate)).astype(np.float32)
    d_rows, _ = _features(gpu, name, times, np.ones(samples, np.uint32))
    terms = _bench_terms(ab)
    dims = ab.feature_term_dims(terms)
    d_database = torch.zeros((samples, 24), dtype=torch.float32, device="cuda")
    ctx.pack_pose_features(d_rows, samples, 4, 4, terms, d_database, 24)
    # normalisation as INTEGRATION describes: identity stats first, then per dimension mean and 1 / std
    mean = d_database[:, :dims].mean(0).cpu().numpy().astype(np.float32)
    std = d_database[:, :dims].std(0).cpu().numpy().astype(np.float32)
    scale = np.where(std > 0, 1.0 / np.maximum(std, 1e-6), 1.0).astype(np.float32)
    ctx.pack_pose_features(d_rows, samples, 4, 4, terms, d_database, 24, mean, scale)
    query_at = np.arange(0, samples, 3)
    d_query_rows, _ = _features(gpu, name, times[query_at] + np.float32(0.004), np.ones(query_at.size, np.uint32))
    d_queries = torch.zeros((query_at.size, 24), dtype=torch.float32, device="cuda")
    ctx.pack_pose_features(d_query_rows, query_at.size, 4, 4, terms, d_queries, 24, mean, scale)
    torch.cuda.synchronize()
    database, query_vectors = d_database.cpu().numpy(), d_queries.cpu().numpy()
    assert np.array_equal(database.view(np.uint32), FS.pack(d_rows.cpu().numpy(), samples, 4, 768, terms, mean, scale, 24).view(np.uint32))
    for window in (0, 5):
        queries = make_search_queries(1, np.maximum(query_at - window, 0), query_at + window + (1 if window else 0))
        got = _search(gpu, database, query_vectors, queries, dims)
        want = _assert_oracle(got, database, query_vectors, queries, dims)
        if window:
            assert np.all((want["row"] < queries["exclude_begin"]) | (want["row"] >= queries["exclude_end"]))


def test_refusals_launch_nothing(gpu):
    torch, ab, ctx = gpu["torch"], gpu["ab"], gpu["ctx"]
    n, dims = 50, 8
    d_db = torch.zeros((n, 8), dtype=torch.float32, device="cuda")
    d_qv = torch.zeros((4, 8), dtype=torch.float32, device="cuda")
    d_queries = _dev(gpu, make_search_queries(np.full(4, 1), 0, 0))
    d_results = torch.full((8,), 0x12345678, dtype=torch.int32, device="cuda")
    base = dict(d_database=d_db.data_ptr(), num_rows=n, db_stride=8, d_query_vectors=d_qv.data_ptr(), d_queries=d_queries, num_queries=4,
                q_stride=8, num_dims=dims, d_results=d_results.data_ptr())
    bad = [dict(num_dims=0), dict(num_dims=65), dict(db_stride=7), dict(q_stride=6), dict(db_stride=10), dict(num_dims=9),
           dict(d_database=d_db.data_ptr() + 4), dict(d_query_vectors=d_qv.data_ptr() + 8), dict(d_results=d_results.data_ptr() + 4),
           dict(num_rows=0xFFFFFFFF), dict(num_rows=1 << 33), dict(d_database=0), dict(d_query_vectors=0), dict(d_queries=0),
           dict(d_results=0)]
    launches = ctx.launch_count
    for change in bad:
        with pytest.raises(ab.AclB200Error):
            ctx.search_pose_features(**{**base, **change})
    torch.cuda.synchronize()
    assert np.all(d_results.cpu().numpy() == 0x12345678) and ctx.launch_count == launches
    ctx.search_pose_features(**base)         # the unchanged call is accepted: the results' clear and the search
    torch.cuda.synchronize()
    assert np.all(d_results.cpu().numpy().view(np.uint64) == 0)     # every query finds row 0 at cost 0
    assert ctx.launch_count == launches + 2

    rows = torch.zeros((10, 4, 4, 12), dtype=torch.float32, device="cuda")
    d_out = torch.full((10, 8), 5.0, dtype=torch.float32, device="cuda")
    good = ab.make_feature_terms([ab.FEATURE_POSITION], [0], [0], [7])
    P = dict(d_rows=rows, num_requests=10, num_offsets=4, bones_per_list=4, terms=good, d_out=d_out, out_stride=8)
    term = lambda **kw: ab.make_feature_terms(**{**dict(kinds=ab.FEATURE_POSITION, s0=0, k=0, components=7), **kw})
    bad = [dict(terms=term(kinds=3)), dict(terms=term(s0=4)), dict(terms=term(kinds=ab.FEATURE_VELOCITY, s1=4, inv_dt=1.0)),
           dict(terms=term(k=4)), dict(terms=term(kinds=ab.FEATURE_DIRECTION, axis=3)), dict(terms=term(components=0)),
           dict(terms=term(components=8)), dict(terms=term(kinds=ab.FEATURE_VELOCITY, s1=1, inv_dt=np.inf)),
           dict(mean=np.full(3, np.nan, np.float32)), dict(scale=np.array([1, np.inf, 1], np.float32)), dict(num_dims=2), dict(num_dims=4),
           dict(out_stride=2), dict(out_stride=6), dict(num_offsets=0), dict(num_offsets=9), dict(bones_per_list=33),
           dict(pose_stride_bytes=40), dict(pose_stride_bytes=4 * 4 * 48 + 8), dict(d_rows=rows.data_ptr() + 4), dict(d_out=d_out.data_ptr() + 4),
           dict(d_rows=0), dict(terms=ab.make_feature_terms([], [], [], [])),
           dict(terms=ab.make_feature_terms([ab.FEATURE_POSITION] * 22, 0, 0, 7))]
    launches = ctx.launch_count
    for change in bad:
        with pytest.raises(ab.AclB200Error):
            ctx.pack_pose_features(**{**P, **change})
    torch.cuda.synchronize()
    assert np.all(d_out.cpu().numpy() == 5.0) and ctx.launch_count == launches
