"""Genome browser tracks on the device (csrc/browser_tracks.cu): every golden case of
`tombo text_output browser_files` against the unmodified reference's files, slot means bit for
bit against the reference's slice-add loop on fresh seeds at scale, coverage runs against the
np.diff encoding for a million reads, and the error paths."""
import numpy as np
import pytest

import tracks_cases as tc

pytestmark = pytest.mark.gpu

GOLD = tc.load_golden()


@pytest.fixture
def ctx():
    from tombo_b200 import _lib
    c = _lib.Context(0)
    yield c
    c.close()


def _last_error(c):
    return c.lib.tb2_last_error(c.handle).decode()


@pytest.mark.parametrize('case', GOLD['cases'], ids=lambda c: c['name'])
def test_browser_files_match_reference(case, tmp_path, ctx):
    tc.same_files(tc.run_case(case, str(tmp_path), ctx), case['files'])


def _genome_reads(rng, n_reads, glen, mean_len):
    """reads of ~mean_len bases over both strands of a glen genome, in index order"""
    start = rng.randint(0, glen - 2 * mean_len, size=n_reads)
    nv = rng.randint(mean_len // 2, 3 * mean_len // 2, size=n_reads)
    rev = rng.rand(n_reads) < 0.5
    return start.astype(np.int64), nv.astype(np.int64), rev


@pytest.mark.parametrize('seed', [1001, 1002])
def test_slot_means_at_scale_bit_exact(ctx, seed):
    # 2e5 reads of ~450 values on a 1 Mb genome, one strand per accumulation, several adds
    rng = np.random.RandomState(seed)
    glen = 1000000
    start, nv, rev = _genome_reads(rng, 200000, glen, 450)
    for strand in (False, True):
        sel = rev == strand
        s, n = start[sel], nv[sel]
        off = np.concatenate([[0], np.cumsum(n)])
        vals = rng.normal(0, 1.5, size=off[-1]) * 10.0 ** rng.uniform(-3, 3, size=off[-1])
        vals[rng.rand(vals.shape[0]) < 1e-5] = np.nan
        cuts = [0] + sorted(rng.choice(np.arange(1, s.shape[0]), size=6, replace=False)) + [s.shape[0]]
        batches = [(s[a:b], off[a:b + 1] - off[a], vals[off[a]:off[b]], np.full(b - a, strand))
                   for a, b in zip(cuts[:-1], cuts[1:])]
        got = ctx.slot_means(glen, batches)
        # the reference's loop: base_sums[s:s + n] += values (reversed on -), in read order
        base_sums, base_cov = np.zeros(glen), np.zeros(glen, dtype=np.int64)
        for r in range(s.shape[0]):
            v = vals[off[r]:off[r + 1]]
            if strand:
                v = v[::-1]
            base_sums[s[r]:s[r] + n[r]] += v
            base_cov[s[r]:s[r] + n[r]] += 1
        with np.errstate(invalid='ignore', divide='ignore'):
            want = base_sums / base_cov
        assert got.tobytes() == want.tobytes()


def test_coverage_runs_million_reads(ctx):
    rng = np.random.RandomState(77)
    glens = [5000000, 5000000, 2000000, 2000000, 1000, 1]
    n_per = [400000, 400000, 100000, 100000, 300, 1]
    grp_off = np.concatenate([[0], np.cumsum(n_per)])
    start, end = [], []
    for gl, n in zip(glens, n_per):
        s = rng.randint(0, max(gl - 1, 1), size=n)
        start.append(s)
        end.append(np.minimum(s + rng.randint(1, 900, size=n), gl))
    start, end = np.concatenate(start), np.concatenate(end)
    end = np.maximum(end, start + 1)
    run_off, run_start, run_cov = ctx.coverage_runs(grp_off, start, end)
    assert grp_off[-1] >= 1000000
    for g in range(len(glens)):
        s, e = start[grp_off[g]:grp_off[g + 1]], end[grp_off[g]:grp_off[g + 1]]
        diff = np.zeros(e.max() + 1, dtype=np.int64)
        np.add.at(diff, s, 1)
        np.add.at(diff, e, -1)
        cov = np.cumsum(diff)[:-1]
        starts = np.concatenate([[0], np.where(np.diff(cov))[0] + 1])
        assert np.array_equal(run_start[run_off[g]:run_off[g + 1]], starts)
        assert np.array_equal(run_cov[run_off[g]:run_off[g + 1]], cov[starts])


def test_slot_sums_error_paths(ctx):
    from tombo_b200 import _lib
    one = (np.array([5]), np.array([0, 10]), np.ones(10), np.zeros(1, bool))
    # a read past chrm_len
    with pytest.raises(_lib.TomboB200Error, match='outside'):
        ctx.slot_means(12, [one])
    # means after that failed add: the accumulation is invalid
    assert ctx.lib.tb2_slot_sums_means(ctx.handle, _lib.ptr(np.empty(12), _lib.f64)) == _lib.TB2_ERR_INVALID_ARG
    assert 'failed' in _last_error(ctx)
    # bad offsets
    with pytest.raises(_lib.TomboB200Error, match='decreasing'):
        ctx.slot_means(100, [(np.array([0, 5]), np.array([0, 4, 2]), np.ones(4), np.zeros(2, bool))])
    # a clean message on the next call, and a good accumulation after a failed one
    assert ctx.slot_means(20, [one])[5:15].tolist() == [1.0] * 10
    assert _last_error(ctx) == ''


def test_slot_sums_means_without_begin():
    from tombo_b200 import _lib
    c = _lib.Context(0)
    try:
        assert c.lib.tb2_slot_sums_means(c.handle, _lib.ptr(np.empty(4), _lib.f64)) == _lib.TB2_ERR_INVALID_ARG
        assert 'begin' in _last_error(c)
    finally:
        c.close()


def test_coverage_runs_rejects_bad_reads(ctx):
    from tombo_b200 import _lib
    with pytest.raises(_lib.TomboB200Error, match='0 <= start < end'):
        ctx.coverage_runs(np.array([0, 2]), np.array([3, 7]), np.array([5, 7]))
    assert ctx.coverage_runs(np.array([0, 1]), np.array([3]), np.array([5]))[2].tolist() == [0, 1]
    assert _last_error(ctx) == ''
