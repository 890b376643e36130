"""`tombo text_output browser_files` on the host: tombo_b200.text_output over the numpy
restatement of the device calls writes the files the unmodified reference writes (wiggles byte
for byte, bedgraphs group by group), the text formatting gives the characters of
'{:d} {:.4f}', and the argument checks raise where the reference exits."""
import argparse

import numpy as np
import pytest

import tracks_cases as tc
from tombo_b200 import formats, text_output, tombo_helper as th

GOLD = tc.load_golden()


@pytest.mark.parametrize('case', GOLD['cases'], ids=lambda c: c['name'])
def test_browser_files_match_reference(case, tmp_path):
    tc.same_files(tc.run_case(case, str(tmp_path), tc.HostContext()), case['files'])


def test_wig_formatting_matches_str_format():
    rng = np.random.RandomState(7)
    vals = np.concatenate([
        rng.normal(0, 2, 4000), rng.normal(0, 1e-4, 2000), rng.uniform(-1e8, 1e8, 500),
        np.round(rng.normal(0, 3, 2000), 4) + rng.choice([-5e-5, 5e-5, 0], 2000),
        [0.0, -0.0, 0.00005, -0.00005, 0.00015, 0.03125, -0.03125, 2.5e-5, 1e8, -1e8, 99999999.99995,
         1e300, -1e300, 5e-324, np.inf, -np.inf, np.nan]])
    poss = rng.randint(0, 1 << 40, size=vals.shape[0])
    want = '\n'.join('{:d} {:.4f}'.format(p + 1, v) for p, v in zip(poss, vals)) + '\n'
    assert text_output.format_wig_lines(poss, vals).decode() == want
    assert text_output.format_wig_lines(np.zeros(0, np.int64), np.zeros(0)) == b'\n'


def test_bedgraph_formatting():
    cov = np.array([0, 3, 12, 0, 1000000])
    starts = np.array([0, 9, 10, 99, 1000, 123456789012])
    want = '\n'.join('\t'.join(('chrX', '%d' % starts[i], '%d' % starts[i + 1], '%d' % cov[i]))
                     for i in range(cov.shape[0])) + '\n'
    assert text_output.format_bedgraph_lines('chrX', cov, starts).decode() == want


def test_slot_batches_split_at_read_boundaries(tmp_path):
    case = [c for c in GOLD['cases'] if c['name'] == 'minus_strand'][0]
    paths, store = tc.index_dirs(str(tmp_path), case['sample'])
    ri = formats.load_reads_index(paths, tc.CORR_GRP)
    sizes = th.get_chrm_sizes(ri)
    with tc.events_h5py(store):
        for cs, cs_reads in ri.items():
            whole = th.get_mean_slot_genome_centric(cs_reads, sizes[cs[0]], 'norm_mean', ctx=tc.HostContext())
            split = th.get_mean_slot_genome_centric(cs_reads, sizes[cs[0]], 'norm_mean', ctx=tc.HostContext(),
                                                    max_values=97)
            assert whole.tobytes() == split.tobytes()


def test_reads_index_needs_an_index(tmp_path):
    with pytest.raises(th.TomboError):
        formats.load_reads_index([str(tmp_path)], tc.CORR_GRP)


def _args(**kw):
    a = dict(fast5_basedirs=['x/'], control_fast5_basedirs=None, statistics_filename=None,
             corrected_group=tc.CORR_GRP, basecall_subgroups=None, browser_file_basename='t',
             file_types=['coverage'], genome_fasta=None, motif_descriptions=None)
    a.update(kw)
    return argparse.Namespace(**a)


@pytest.mark.parametrize('kw, text', [
    (dict(fast5_basedirs=None, file_types=['dwell']), 'Must provide a fast5 basedir'),
    (dict(file_types=['fraction']), 'Must provide a statistics filename'),
    (dict(file_types=['difference']), 'Must provide two sets of FAST5s'),
    (dict(fast5_basedirs=None, control_fast5_basedirs=['y/'], file_types=['fraction'],
          statistics_filename='s'), 'Cannot provide a control FAST5 set'),
    (dict(file_types=['coverage', 'statistic'], statistics_filename='s'), 'not supported yet'),
])
def test_argument_checks(kw, text):
    with pytest.raises(th.TomboError, match=text):
        text_output.browser_files_main(_args(**kw), ctx=tc.HostContext())
