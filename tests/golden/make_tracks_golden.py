#!/usr/bin/env python
"""Writes tests/golden/tracks.npz: `tombo text_output browser_files` for the read-derived file
types (coverage, signal, signal_sd, dwell, difference), run by the UNMODIFIED reference
in-process.

Each case (tests/tracks_cases.py) writes its directories' indexes to a temporary directory
and serves every read's Events table (norm_mean, norm_stdev, length) through the FakeFile
stand-in; the reference's write_all_browser_files then writes its files there, with the
relative basename tracks_cases.WIG_BASE (the track headers carry it).  _text_output_commands
is imported from the reference checkout (TOMBO_REFERENCE_ROOT) into the package oracle/_ref
provides.  The deep_order case is checked to pin the summation order: at its deepest position
the sequential sum of the values in read order differs from the sum in ascending order.

The inputs are not stored: tracks_cases.golden_cases() regenerates them from fixed seeds, and
each case keeps the sha256 of its inputs (tracks_cases.inputs_digest) so a test compares the
files only with the inputs they came from.  One JSON document under key 'json':
  cases: [{name, digest, files: {file name: text}}]

    python oracle/build_ref.py && python tests/golden/make_tracks_golden.py
"""
import importlib.util
import json
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
for p in (REPO, os.path.join(REPO, 'oracle'), os.path.dirname(HERE)):
    if p not in sys.path:
        sys.path.insert(0, p)
import ref_harness as rh                      # noqa: E402
import tracks_cases as tc                     # noqa: E402

REF_ROOT = os.environ.get('TOMBO_REFERENCE_ROOT', '/root/reference')


def load_text_output_module():
    m = rh.load_reference()
    spec = importlib.util.spec_from_file_location(
        'tombo._text_output_commands', os.path.join(REF_ROOT, 'tombo', '_text_output_commands.py'))
    to = importlib.util.module_from_spec(spec)
    sys.modules['tombo._text_output_commands'] = to
    spec.loader.exec_module(to)
    return m, to


def check_deep_order(groups, store):
    """the deepest position's read-order sum must differ from its ascending-order sum"""
    recs = groups[0][1]
    cov = {}
    for rec in recs:
        v = store[rec[0]]['events']['norm_mean']
        for k, x in enumerate(v):
            cov.setdefault(rec[1] + k, []).append(x)
    pos, vals = max(cov.items(), key=lambda kv: len(kv[1]))
    seq = 0.0
    for x in vals:
        seq += x
    alt = 0.0
    for x in sorted(vals):
        alt += x
    assert len(vals) >= 2000 and seq != alt, (len(vals), seq, alt)
    return pos, len(vals)


def main():
    m, to = load_text_output_module()
    out = []
    for case in tc.case_inputs():
        name, sample, control = case['name'], case['sample'], case['control']
        bc_subgrps, wig_types = case['bc_subgrps'], case['wig_types']
        if name == 'deep_order':
            print('deep_order position / depth', check_deep_order(sample[0][1], sample[0][2]))
        with tempfile.TemporaryDirectory() as tmp:
            s_dirs, store = tc.index_dirs(tmp, sample)
            c_dirs = None
            if control:
                c_dirs, c_store = tc.index_dirs(tmp, control)
                store.update(c_store)
            cwd = os.getcwd()
            os.chdir(tmp)
            try:
                with tc.events_h5py(store) as mod:
                    m['th'].h5py = mod
                    with rh.ref_errstate():
                        to.write_all_browser_files(s_dirs, c_dirs, tc.CORR_GRP, bc_subgrps, None,
                                                   tc.WIG_BASE, wig_types, None, None)
            finally:
                os.chdir(cwd)
            files = tc.output_files(tmp)
        out.append(dict(name=name, digest=tc.inputs_digest(case), files=files))
        print(name, len(files), 'files', sum(len(t) for t in files.values()), 'chars')
    np.savez_compressed(tc.GOLDEN, json=np.array(json.dumps(dict(cases=out))))
    print('wrote', tc.GOLDEN, len(out), 'cases')


if __name__ == '__main__':
    main()
