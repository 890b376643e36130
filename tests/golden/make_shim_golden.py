#!/usr/bin/env python
"""Goldens for tests/test_shim_cpu.py and tests/test_abi_cpu.py from the UNMODIFIED
reference (oracle/_ref): trim_seq_and_means and remove_stall_cpts on the tests' seeded
random inputs, and the reference's default parameters, namedtuple fields and
load_resquiggle_parameters tuples.  Results that are slices of the inputs are stored as
(start, length), the changepoints remove_stall_cpts drops as [start, end) index runs.

    python oracle/build_ref.py && python tests/golden/make_shim_golden.py
"""
import gzip
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tests'))
sys.path.insert(0, os.path.join(REPO, 'oracle'))

import ref_harness as rh  # noqa: E402
import test_abi_cpu as abi  # noqa: E402
import test_shim_cpu as shim  # noqa: E402


def main():
    m = rh.load_reference()
    import tombo._default_parameters as rdp

    def trim(seq, means, args):
        try:
            k, mm, r, ms = m['ts'].trim_seq_and_means(seq, means.copy(), *args)
        except m['th'].TomboError as e:
            return ['err', str(e)]
        K = args[4]
        k0 = next((i for i in range(len(seq) + 1)
                   if [seq[i + j:i + j + K] for j in range(len(k))] == list(k)), None)
        m0 = next((i for i in range(len(means) + 1)
                   if means[i:i + len(mm)].tolist() == mm.tolist()), None)
        s0 = seq.find(ms)
        g = ['ok', k0, len(k), m0, len(mm), int(r), [s0, len(ms)] if s0 >= 0 else ms]
        assert shim.decode_trim(seq, means, args, g) == ('ok', list(k), mm.tolist(), r, ms)
        return g

    def stall(ints, cp):
        out = m['ts'].remove_stall_cpts(ints, cp)
        kept = set(out.tolist())
        runs = []
        for i, c in enumerate(cp.tolist()):
            if c in kept:
                continue
            if runs and runs[-1][1] == i:
                runs[-1][1] = i + 1
            else:
                runs.append([i, i + 1])
        assert np.array_equal(shim.drop_runs(cp, runs), out)
        return runs
    out = {
        'trim_seq_and_means': [trim(seq, means, args) for seq, means, args in shim.trim_cases()],
        'remove_stall_cpts': [stall(ints, cp) for ints, cp in shim.stall_cases()],
        'default_parameters': {n: getattr(rdp, n) for n in dir(rdp) if n.isupper()},
        'namedtuple_fields': {nt: list(getattr(m['th'], nt)._fields) for nt in abi.NAMEDTUPLES},
        'resquiggle_parameters': {
            '%s_%d' % (kind, save): [float(v) if isinstance(v, np.floating) else v
                                     for v in m['ts'].load_resquiggle_parameters(
                                         m['th'].seqSampleType(kind, kind == 'RNA'),
                                         use_save_bandwidth=save)]
            for kind in ('DNA', 'RNA') for save in (False, True)},
        'HALF_NORM_EXPECTED_VAL': float(m['ts'].HALF_NORM_EXPECTED_VAL),
    }
    p = os.path.join(HERE, 'shim_reference.json.gz')
    with gzip.GzipFile(p, 'wb', mtime=0) as f:
        f.write(json.dumps(out, sort_keys=True).encode())
    print('wrote', p, os.path.getsize(p), 'bytes')


if __name__ == '__main__':
    main()
