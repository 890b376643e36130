"""helper (not a test): where the device time of one resquiggle step goes, kernel by kernel.

Runs a bench.py workload (default c1 = configs[1], 100k DNA reads of ~4k samples) with the
inputs resident on the device, then times `--steps` calls of Context.batch_compute under
torch.profiler with CUDA activities and writes, per kernel, its launches, total device time,
mean time per launch and share of the summed kernel time, plus the step's wall time on CUDA
events.  Nsight is not needed.  The profiled steps run apart from any end-to-end timing: the
tracer slows the host, not the kernels.

usage: python tools/kernel_shares.py [--workload c1] [--steps 3] [--warmup 2] [--out DIR]
writes DIR/kernel_shares.json and DIR/kernel_shares.txt (DIR defaults to ./kernel_shares)"""
import argparse
import json
import os
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)


def gpu_info():
    """card, power limit and SM clock ceiling: every time below is only meaningful with them"""
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                            '--format=csv,noheader'], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else None
    except (OSError, subprocess.SubprocessError):
        return None


def main():
    import bench
    ap = argparse.ArgumentParser()
    ap.add_argument('--workload', default='c1', choices=sorted(bench.CONFIGS))
    ap.add_argument('--reads', type=int, default=0, help='reads per step (0 = config default)')
    ap.add_argument('--steps', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--out', default='kernel_shares')
    args = ap.parse_args()

    import numpy as np
    import torch
    from torch.profiler import profile, ProfilerActivity
    from tombo_b200 import _lib, synthetic as syn
    if not torch.cuda.is_available():
        raise SystemExit('kernel_shares: no CUDA device')

    cfg = bench.CONFIGS[args.workload]
    n_reads = args.reads or cfg['reads']
    rna = cfg['kind'] == 'RNA'
    kmer_ref, cpos, raw, raw_off, seq, seq_off = bench.make_workload(cfg, n_reads, 1)
    means, sds = syn.kmer_table(kmer_ref)
    ctx = _lib.Context(0)
    ctx.set_model(means, sds, len(kmer_ref[0][0]), cpos)
    rp = bench.RP(cfg['aln'], cfg['seg'], rna=rna)
    sp = bench.RP(cfg['aln'], cfg['seg'], save=True, rna=rna)
    pol = _lib.make_policy(cfg['kind'], subsample_seed=0)
    ctx.batch_upload(raw, raw_off, seq, seq_off, rp, pol)
    for _ in range(max(0, args.warmup)):
        ctx.batch_compute(rp, sp, pol)

    # step time on CUDA events, profiler off
    step_ms = []
    for _ in range(args.steps):
        ctx.timer_start()
        ctx.batch_compute(rp, sp, pol)
        step_ms.append(ctx.timer_stop())

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            ctx.batch_compute(rp, sp, pol)
        torch.cuda.synchronize()
    ctx.close()

    kern = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = ev.name
        if name.startswith('Memcpy') or name.startswith('Memset'):
            continue
        k = kern.setdefault(name, {'launches': 0, 'total_us': 0.0})
        k['launches'] += 1
        k['total_us'] += ev.time_range.elapsed_us()
    total_us = sum(k['total_us'] for k in kern.values())
    rows = []
    for name, k in sorted(kern.items(), key=lambda kv: -kv[1]['total_us']):
        rows.append({'kernel': name, 'launches': k['launches'],
                     'ms_per_step': k['total_us'] / 1e3 / args.steps,
                     'us_per_launch': k['total_us'] / max(1, k['launches']),
                     'share': k['total_us'] / total_us if total_us > 0 else 0.0})
    res = {'gpu': gpu_info(), 'workload': cfg['label'] % n_reads, 'steps': args.steps,
           'step_ms_events': step_ms, 'step_ms_events_median': float(np.median(step_ms)),
           'kernel_ms_per_step': total_us / 1e3 / args.steps, 'kernels': rows,
           'time': time.strftime('%Y-%m-%d %H:%M:%S')}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, 'kernel_shares.json'), 'w') as f:
        json.dump(res, f, indent=1)
    lines = ['gpu (name, power limit, max SM clock): %s' % res['gpu'],
             'workload: %s' % res['workload'],
             'step on CUDA events (profiler off), ms: %s' % ' '.join('%.2f' % v for v in step_ms),
             'summed kernel time per step (profiler on), ms: %.2f' % res['kernel_ms_per_step'],
             '%8s %10s %10s %9s  %s' % ('share', 'ms/step', 'us/launch', 'launches', 'kernel')]
    for r in rows:
        lines.append('%7.2f%% %10.3f %10.1f %9d  %s' % (100 * r['share'], r['ms_per_step'],
                                                        r['us_per_launch'], r['launches'],
                                                        r['kernel'][:110]))
    txt = '\n'.join(lines) + '\n'
    with open(os.path.join(args.out, 'kernel_shares.txt'), 'w') as f:
        f.write(txt)
    print(txt, end='')


if __name__ == '__main__':
    main()
