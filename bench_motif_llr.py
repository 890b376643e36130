#!/usr/bin/env python
"""Motif alternative-model LLRs on one GPU: a configs[1]-shaped DNA batch (100 000 reads x 444
bases, strands alternating) is resquiggled once; then tb2_batch_alt_llr_motif runs for 5mC
(C:1), CpG (CG:1), dcm (CCWGG:2) and dam (GATC:2) on the resident batch, alternating with the
single-base tb2_batch_alt_llr (5mC, '+' only), each timed with CUDA events after warm-up.
The host-array entry tb2_alt_model_llr_motif_batch is timed end to end (upload, kernels,
download) on the downloaded means.  After the timed region a parity sample is checked
against tests/motif_cases.py.  If the reference oracle (oracle/_ref) is importable, its
per-read compute_alt_model_read_stats runs on a small sample as a CPU arm.

Prints one JSON line; nothing is written to the tree."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.abspath(__file__))
for p in (REPO, os.path.join(REPO, 'tests'), os.path.join(REPO, 'oracle')):
    if p not in sys.path:
        sys.path.insert(0, p)

MODELS = [('5mC', 'C', 1, 'C'), ('CpG', 'CG', 1, 'C'), ('dcm', 'CCWGG', 2, 'C'),
          ('dam', 'GATC', 2, 'A')]


def card_info(device):
    info = {}
    try:
        import torch
        info['name'] = torch.cuda.get_device_name(device)
    except Exception as e:                       # noqa: BLE001
        info['name_error'] = repr(e)
    try:
        o = subprocess.run(['nvidia-smi', '-i', str(device), '--query-gpu=name,power.limit',
                            '--format=csv,noheader'], capture_output=True, text=True, timeout=20)
        info['nvidia_smi'] = o.stdout.strip()
    except Exception as e:                       # noqa: BLE001
        info['nvidia_smi_error'] = repr(e)
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reads', type=int, default=100000)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--device', type=int, default=0)
    ap.add_argument('--parity', type=int, default=400)
    ap.add_argument('--cpu-reads', type=int, default=20)
    a = ap.parse_args()
    import bench
    import motif_cases as mc
    from tombo_b200 import _lib, synthetic as syn, tombo_helper as th
    cfg = bench.CONFIGS['c1']
    kmer_ref, cpos, raw, raw_off, seq, seq_off = bench.make_workload(cfg, a.reads, 1)
    K = len(kmer_ref[0][0])
    kmeans, ksds = syn.kmer_table(kmer_ref)
    ctx = _lib.Context(a.device)
    ctx.set_model(kmeans, ksds, K, cpos)
    rp, sp = bench.RP(cfg['aln'], cfg['seg']), bench.RP(cfg['aln'], cfg['seg'], save=True)
    pol = _lib.make_policy('DNA')
    ctx.batch_upload(raw, raw_off, seq, seq_off, rp, pol)
    ctx.batch_compute(rp, sp, pol)
    res = ctx.batch_download()
    n = raw_off.shape[0] - 1
    ok = res['status'] == 0
    start = (np.arange(n, dtype=np.int64) * 500) % 10 ** 7
    strand = (np.arange(n) % 2).astype(np.int8)
    bb, ab = mc.motif_bounds([(m, p) for _, m, p, _ in MODELS])
    reg = (-10 ** 12, 10 ** 12)
    tables = dict((b, mc.alt_table(kmer_ref, b)) for b in ('A', 'C'))
    motifs = dict((name, _lib.motif_struct(th.TomboMotif(m, p))) for name, m, p, _ in MODELS)

    def run(name):
        if name == 'single_base_5mC':
            return ctx.batch_alt_llr(start, 1)
        return ctx.batch_alt_llr_motif(start, strand, motifs[name], bb, ab, *reg)[0]

    names = ['single_base_5mC'] + [m[0] for m in MODELS]
    times = dict((nm, []) for nm in names)
    sites = {}
    for step in range(a.warmup + a.steps):
        for nm in names:                                  # alternating in one session
            base = 'C' if nm == 'single_base_5mC' else [m[3] for m in MODELS if m[0] == nm][0]
            ctx.set_alt_model(tables[base], K)
            ctx.timer_start()
            sites[nm] = int(run(nm))
            ms = ctx.timer_stop()
            if step >= a.warmup:
                times[nm].append(ms)
    out = dict(metric='motif_llr', reads=n, resquiggled=int(ok.sum()), steps=a.steps,
               warmup=a.warmup, card=card_info(a.device), resident={})
    for nm in names:
        t = np.array(times[nm]) / 1e3
        med = float(np.median(t))
        out['resident'][nm] = dict(sites=sites[nm], median_ms=med * 1e3,
                                   min_ms=float(t.min()) * 1e3, max_ms=float(t.max()) * 1e3,
                                   sites_per_s=sites[nm] / med, reads_per_s=n / med)
    # host-array entry, end to end
    nm_, mo = res['norm_mean'], res['base_off']
    st_h = np.where(ok, strand, -1).astype(np.int8)
    out['host_array'] = {}
    for name, m, p, base in MODELS:
        ctx.set_alt_model(tables[base], K)
        t = []
        for step in range(a.warmup + max(1, a.steps // 2)):
            t0 = time.perf_counter()
            llr, pos, off, st = ctx.alt_model_llr_motif_batch(nm_, mo, seq, seq_off, start, st_h,
                                                              motifs[name], bb, ab, *reg)
            if step >= a.warmup:
                t.append(time.perf_counter() - t0)
        med = float(np.median(t))
        out['host_array'][name] = dict(sites=int(off[-1]), median_ms=med * 1e3,
                                       reads_per_s=n / med, sites_per_s=int(off[-1]) / med)
    # parity after the timed region
    rs = np.random.RandomState(0)
    pick = np.sort(rs.choice(np.nonzero(ok)[0], min(a.parity, int(ok.sum())), replace=False))
    sub_mo = np.concatenate([[0], np.cumsum(np.diff(mo)[pick])]).astype(np.int64)
    sub_nm = np.concatenate([nm_[mo[r]:mo[r + 1]] for r in pick])
    sub_so = np.concatenate([[0], np.cumsum(np.diff(seq_off)[pick])]).astype(np.int64)
    sub_sq = np.concatenate([seq[seq_off[r]:seq_off[r + 1]] for r in pick])
    mism = {}
    for name, m, p, base in MODELS:
        ctx.set_alt_model(tables[base], K)
        ctx.batch_alt_llr_motif(start, strand, motifs[name], bb, ab, *reg, use_standard_llhr=True)
        llr, pos, off = ctx.batch_llr_download()
        want = mc.motif_llr_reads(sub_nm, sub_mo, sub_sq, sub_so, start[pick], strand[pick], m, p,
                                  bb, ab, *reg, kmeans, ksds, tables[base], K, cpos, 1)
        got_llr = np.concatenate([llr[off[r]:off[r + 1]] for r in pick])
        got_pos = np.concatenate([pos[off[r]:off[r + 1]] for r in pick])
        bad = int(got_pos.shape[0] != want[1].shape[0])
        if not bad:
            bad = int(np.sum(got_pos != want[1]) + np.sum(
                ~((got_llr == want[0]) | (np.isnan(got_llr) & np.isnan(want[0])))))
        mism[name] = bad
    out['parity'] = dict(reads=int(pick.shape[0]), mismatches=mism)
    # CPU arm: the reference's per-read function, if the oracle is built
    try:
        import ref_harness as rh
        if not rh.available():
            raise ImportError('oracle/_ref not built')
        from unittest import mock
        m_ = rh.load_reference()
        rth, rts = m_['th'], m_['ts']
        std_ref = rts.TomboModel(kmer_ref=kmer_ref, central_pos=cpos)
        alt_refs = [(name, rts.AltModel(kmer_ref=syn.make_alt_kmer_ref(kmer_ref, base, seed=1),
                                        central_pos=cpos, alt_base=base, name=name,
                                        motif=rth.TomboMotif(m, p))) for name, m, p, base in MODELS]
        orig = (rth.get_multiple_slots_read_centric, rth.get_raw_read_slot)
        cpu_pick = pick[:a.cpu_reads]
        t0 = time.perf_counter()
        try:
            for r in cpu_pick:
                nb = int(mo[r + 1] - mo[r])
                S = np.array(list(''.join('ACGT'[c] for c in seq[seq_off[r] + cpos:
                                                                 seq_off[r] + cpos + nb])), 'S1')
                vals = (nm_[mo[r]:mo[r + 1]], S)
                rth.get_multiple_slots_read_centric = lambda *x, **k: vals
                rth.get_raw_read_slot = lambda *x, **k: mock.MagicMock()
                rd = rth.readData(start=int(start[r]), end=int(start[r]) + nb, filtered=False,
                                  read_start_rel_to_raw=0, strand='+-'[strand[r]], fn='x',
                                  corr_group='g', rna=False)
                with rh.ref_errstate():
                    rts.compute_alt_model_read_stats(rd, std_ref, alt_refs)
        finally:
            rth.get_multiple_slots_read_centric, rth.get_raw_read_slot = orig
        dt = time.perf_counter() - t0
        out['cpu_reference'] = dict(reads=int(cpu_pick.shape[0]), models=len(MODELS),
                                    reads_per_s=cpu_pick.shape[0] / dt, threads=1)
    except ImportError as e:
        out['cpu_reference'] = dict(skipped=str(e))
    ctx.close()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
