"""Standard / motif model estimation host logic against the unmodified reference's goldens
(tests/golden/model_ref.npz), with the device calls restated in numpy in read order."""
import os

import numpy as np
import pytest

from tombo_b200 import _lib
from tombo_b200 import tombo_helper as th
from tombo_b200 import tombo_stats as ts

import model_ref_cases as mc

G = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'model_ref.npz'))


def run_case(name, kw, genome, reads, served):
    kw = dict(kw)
    motif = kw.pop('motif', None)
    if motif is not None:
        raw, pos = motif.split(':')
        motif = th.TomboMotif(raw, int(pos))
    if kw.pop('valid_poss', None):
        kw['valid_poss'] = mc.valid_poss_of(genome)
    np.random.seed(mc.CFG['shuffle_seed'])
    with mc.serve(served):
        regs = ts.extract_kmer_levels(mc.Index(reads), motif=motif, **kw)
    return regs, motif


@pytest.fixture
def restated(monkeypatch):
    monkeypatch.setattr(_lib, 'get_context', lambda device=0: mc.RestatedContext())


@pytest.mark.parametrize('name,kw', mc.extraction_cases(), ids=[c[0] for c in mc.extraction_cases()])
def test_extraction_matches_reference(restated, name, kw):
    _, genome, reads, served = mc.make_inputs()
    regs, motif = run_case(name, kw, genome, reads, served)
    counts, rows = mc.flatten(regs)
    # regions, keys and row counts are the reference's
    assert np.array_equal(counts, G[name + '_counts'])
    ref, order = G[name + '_rows'], G[name + '_order']
    tol = mc.order_tol(order, ref[:, 1])
    # exact where the reference summarised a position in read order, within the
    # summation-order bound elsewhere; a median does not depend on the order at all
    assert np.all(np.abs(rows[:, 1] - ref[:, 1]) <= tol)
    if kw['est_mean']:
        assert np.all(np.abs(rows[:, 0] - ref[:, 0]) <= tol)
    else:
        assert np.array_equal(rows[:, 0], ref[:, 0])
    assert (order[:, 0] > 0).any() or name == 'motif1'   # both kinds of position occur

    def tabulate(r):
        return (ts.tabulate_kmer_levels(r, mc.CFG['min_kmer_obs']) if motif is None else
                ts.tabulate_mod_kmer_levels(r, mc.CFG['min_kmer_obs'], motif))
    first = next(iter(regs[0]))
    gap = [dict((k, np.zeros((0, 2)) if k == first else v) for k, v in reg.items()) for reg in regs]
    with pytest.raises(th.TomboError) as e:
        tabulate(gap)
    assert str(e.value) == mc.message(G[name + '_gap_stderr'])
    tab = G[name + '_tab']
    if tab.shape[0] == 0:
        with pytest.raises(th.TomboError) as e:
            tabulate(regs)
        assert str(e.value) == mc.message(G[name + '_tab_stderr'])
        return
    got = np.array([t[-2:] for t in tabulate(regs)], dtype=np.float64)
    # a median moves by at most the largest change of the values it is taken over
    assert np.all(np.abs(got[:, 1] - tab[:, 1]) <= tol.max())
    if kw['est_mean']:
        assert np.all(np.abs(got[:, 0] - tab[:, 0]) <= tol.max())
    else:
        assert np.array_equal(got[:, 0], tab[:, 0])


def test_valid_poss_without_motif_gives_empty_regions(restated):
    """the reference's (kmer, offset) look-ups miss its k-mer keyed dicts: every row is
    skipped and each region gives empty lists"""
    _, genome, reads, served = mc.make_inputs()
    kw = dict(mc.extraction_cases()[0][1])
    with mc.serve(served):
        regs = ts.extract_kmer_levels(mc.Index(reads), valid_poss=mc.valid_poss_of(genome), **kw)
    assert len(regs) == G['median_counts'].shape[0]
    assert all(len(v) == 0 for reg in regs for v in reg.values())


def test_no_region_raises(restated):
    _, genome, reads, served = mc.make_inputs()
    with mc.serve(served), pytest.raises(th.TomboError, match='No genomic positions'):
        ts.extract_kmer_levels(mc.Index(reads), 200, 10 ** 6, 1, 1, None)


def test_zero_context_raises():
    with pytest.raises(th.TomboError, match='must be greater'):
        ts.estimate_kmer_model(mc.Index([]), 3, 0, 1, 1, False, None, False, 200)
    with pytest.raises(th.TomboError, match='Invalid motif'):
        ts.estimate_motif_alt_model(mc.Index([]), 'CG', 1, 1, None, 1, 3, None, 200)


@pytest.mark.parametrize('raw,pos', [('CG', 1), ('CCWGG', 2), ('GATC', 2), ('CHG', 1)])
def test_motif_mod_poss_match_reference_definition(raw, pos):
    """find_mod_poss / matches_seq on every 4-mer against a direct statement of the partial
    match rule: a k-mer holds the mod position where the motif, shifted anywhere over it,
    matches every base it overlaps and overlaps the mod position"""
    import itertools
    import re
    m = th.TomboMotif(raw, pos)
    for kmer in (''.join(k) for k in itertools.product('ACGT', repeat=4)):
        want = set()
        for shift in range(-len(raw) + 1, len(kmer)):
            mp = shift + pos - 1
            if not 0 <= mp < len(kmer):
                continue
            ok = all(re.match(th.SINGLE_LETTER_CODE[raw[j]], kmer[shift + j])
                     for j in range(len(raw)) if 0 <= shift + j < len(kmer))
            if ok:
                want.add(mp + 1)
        got = m.find_mod_poss(kmer)
        # full matches come from finditer (non-overlapping), as in the reference
        full = set(x.start() + pos for x in m.motif_pat.finditer(kmer)) if len(kmer) >= len(raw) else set()
        partial = set(p for p in want if p not in set(range(pos, len(kmer) - len(raw) + pos + 1)))
        assert set(got) == full | partial, (raw, kmer)
        assert m.matches_seq(kmer) == bool(got)


def test_parse_locs_file(tmp_path, capsys):
    fn = tmp_path / 'locs.bed'
    fn.write_text('chr\t5\t6\t.\t.\t+\nchr\t3\t4\t.\t.\t+\nbad line\nchr\t7\t8\t.\t.\t-\n')
    locs = th.parse_locs_file(str(fn))
    assert set(locs) == {('chr', '+'), ('chr', '-')}
    assert list(locs[('chr', '+')]) == [3, 5] and list(locs[('chr', '-')]) == [7]
    assert 'Some provided locations (1) were incorrectly formatted' in capsys.readouterr().err
