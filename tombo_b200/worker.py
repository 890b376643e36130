"""Batch assembly between Tombo's mapping threads and the GPU (SURVEY.md 8(f)-4).

The reference hands reads over one at a time: every mapping thread sends
``[map_res, fast5_fn]`` through its own pipe and blocks until ``_resquiggle_worker``
answers with ``[read_failed, result]`` (resquiggle.py:1417-1421, 1558-1597).  One read per
call cannot feed a GPU, so the hand-off is replaced by an assembler that collects reads,
flushes them through :func:`tombo_b200.resquiggle.resquiggle_reads` in large batches
and returns the answers in submission order, in the reference's wire format:

    [False, resquiggleResults]                       success      (resquiggle.py:1597)
    [True, [message, fast5_fn, is_tombo_error]]      failure      (resquiggle.py:1591-1594)

:class:`FailureSummary` keeps the reference's "unsuccessful reads" bookkeeping
(resquiggle.py:1704-1826): message -> file names, the percentage table and the
``--failed-reads-filename`` output.  Nothing here touches the device itself; the resquiggle
function is injectable, which is how the CPU tests drive this module.
"""
from __future__ import unicode_literals

import io
import traceback
from collections import OrderedDict

from . import tombo_helper as th

UNEXPECTED_ERROR = 'Unexpected error'       # resquiggle.py:1762
MAX_NUM_UNEXP_ERRORS = 50                   # _MAX_NUM_UNEXP_ERRORS resquiggle.py:61
POOR_MATCH_MESSAGE = ('Poor raw to expected signal matching '
                      '(revert with `tombo filter clear_filters`)')      # resquiggle.py:1442
OBS_FILTER_MESSAGE = ('Read filtered by observation per base '
                      'thresholds (revert with `tombo filter clear_filters`)')   # :1451


class ReadBatcher(object):
    """Collects ``(map_res, fast5_fn)`` pairs and resquiggles them in batches.

    A batch is flushed when it holds ``max_reads`` reads or ``max_samples`` raw samples
    (the device buffers grow with the samples, not the reads), and by :meth:`flush`.
    ``add`` / ``flush`` return the finished ``(fast5_fn, message)`` pairs in submission
    order; ``message`` is what ``rsqgl_conn.send`` would have carried for that read."""

    def __init__(self, std_ref, rsqgl_params, save_params=None, max_reads=65536,
                 max_samples=1 << 30, resquiggle_fn=None, index=None, corr_grp=None,
                 bc_subgrp=None, index_sig_match_thresh=None, obs_filter=None,
                 **resquiggle_kwargs):
        if max_reads < 1 or max_samples < 1:
            raise ValueError('max_reads and max_samples must be positive')
        self.std_ref, self.rsqgl_params, self.save_params = std_ref, rsqgl_params, save_params
        self.max_reads, self.max_samples = int(max_reads), int(max_samples)
        self.kwargs = resquiggle_kwargs
        # index opt-in (_io_and_map_read, resquiggle.py:1425-1465): every successful read
        # goes into ``index`` (a formats.ReadsIndex) with its filter flag, and the messages
        # the reference queues on failed_reads_q collect in ``failed_reads``
        self.index, self.corr_grp, self.bc_subgrp = index, corr_grp, bc_subgrp
        self.failed_reads = []
        if index is not None:
            if corr_grp is None or bc_subgrp is None:
                raise ValueError('the index needs corr_grp and bc_subgrp')
            self.kwargs = dict(resquiggle_kwargs, index_sig_match_thresh=index_sig_match_thresh,
                               obs_filter=obs_filter)
        self.obs_filter = obs_filter
        if resquiggle_fn is None:
            from . import resquiggle as rsqgl        # needs the CUDA library: fail loudly
            resquiggle_fn = rsqgl.resquiggle_reads_for_index if index is not None else \
                rsqgl.resquiggle_reads
        self.resquiggle_fn = resquiggle_fn
        self._pending, self._samples = [], 0
        self.n_batches = 0

    def __len__(self):
        return len(self._pending)

    def add(self, map_res, fast5_fn):
        n_raw = 0 if map_res.raw_signal is None else len(map_res.raw_signal)
        out = []
        # a read that would overflow the sample budget goes into the next batch
        if self._pending and self._samples + n_raw > self.max_samples:
            out = self.flush()
        self._pending.append((map_res, fast5_fn))
        self._samples += n_raw
        if len(self._pending) >= self.max_reads or self._samples >= self.max_samples:
            out = out + self.flush()
        return out

    def flush(self):
        if not self._pending:
            return []
        pending, self._pending, self._samples = self._pending, [], 0
        self.n_batches += 1
        fns = [fn for _, fn in pending]
        try:
            results = self.resquiggle_fn([m for m, _ in pending], self.std_ref, self.rsqgl_params,
                                         self.save_params, **self.kwargs)
            if len(results) != len(pending):
                raise RuntimeError('resquiggle returned %d results for %d reads'
                                   % (len(results), len(pending)))
        except th.TomboError as e:
            # the batch call itself refused the input: every read reports that message
            return [self._failed(fn, str(e), True) for fn in fns]
        except Exception:
            tb = traceback.format_exc()
            return [self._failed(fn, tb, False) for fn in fns]
        if self.index is not None:
            return [self._index_read(fn, res, code) for fn, (res, code) in zip(fns, results)]
        out = []
        for fn, res in zip(fns, results):
            if isinstance(res, th.TomboError):
                out.append((fn, [True, [str(res), fn, True]]))
            elif isinstance(res, Exception):
                out.append((fn, [True, [repr(res), fn, False]]))
            else:
                out.append((fn, [False, res]))
        return out


    def _failed(self, fn, message, is_tombo_error):
        if self.index is not None:
            self.failed_reads.append((message, self.bc_subgrp + ':::' + fn, is_tombo_error))
        return (fn, [True, [message, fn, is_tombo_error]])

    def _index_read(self, fn, res, code):
        """one read of an index batch, as _io_and_map_read records it"""
        if isinstance(res, Exception):
            return self._failed(fn, str(res) if isinstance(res, th.TomboError) else repr(res),
                                isinstance(res, th.TomboError))
        key = self.bc_subgrp + ':::' + fn
        if code == 1:
            self.failed_reads.append((POOR_MATCH_MESSAGE, key, True))
        elif self.obs_filter is not None:
            # queued for every read tested, filtered or not (resquiggle.py:1446-1453)
            self.failed_reads.append((OBS_FILTER_MESSAGE, key, True))
        loc = res.genome_loc
        rna = bool(self.kwargs.get('seq_samp_type', th.seqSampleType('DNA', False)).rev_sig)
        self.index.add_read_data(loc.Chrom, loc.Strand, th.readData(
            loc.Start, loc.Start + len(res.segs) - 1, code != 0, res.read_start_rel_to_raw,
            loc.Strand, fn, self.corr_grp + '/' + self.bc_subgrp, rna, res.sig_match_score,
            res.mean_q_score, res.align_info.ID))
        return (fn, [False, res])


def resquiggle_stream(reads, std_ref, rsqgl_params, save_params=None, **kwargs):
    """Generator form: ``reads`` yields ``(map_res, fast5_fn)``; yields
    ``(fast5_fn, message)`` in the same order, batching underneath."""
    batcher = ReadBatcher(std_ref, rsqgl_params, save_params, **kwargs)
    for map_res, fast5_fn in reads:
        for item in batcher.add(map_res, fast5_fn):
            yield item
    for item in batcher.flush():
        yield item


class FailureSummary(object):
    """Unsuccessful-read bookkeeping of ``_get_progress_fail_queues``
    (resquiggle.py:1748-1826)."""

    def __init__(self):
        self.failed_reads = OrderedDict()      # message -> [fast5_fn]
        self.non_tombo_errors = []
        self.num_processed = 0

    def record(self, message):
        """feed one ``[read_failed, payload]`` message of the worker"""
        self.num_processed += 1
        read_failed, payload = message
        if read_failed:
            error_type, fn, is_tombo_error = payload
            self.add(error_type, fn, is_tombo_error)

    def add(self, error_type, fn, is_tombo_error):
        if is_tombo_error:
            self.failed_reads.setdefault(error_type, []).append(fn)
        else:
            self.failed_reads.setdefault(UNEXPECTED_ERROR, []).append(fn)
            if len(self.non_tombo_errors) < MAX_NUM_UNEXP_ERRORS:
                self.non_tombo_errors.append(fn + '\n:::\n' + error_type)

    def counts(self):
        return [(len(fns), err) for err, fns in self.failed_reads.items()]

    @staticmethod
    def format(header, fail_summ=(), num_proc=0, num_errs=None):
        """the percentage table (format_fail_summ, resquiggle.py:1707-1722): most frequent
        message first, padded with dashes to ``num_errs`` lines"""
        rows = sorted(fail_summ, reverse=True)
        if num_errs is not None:
            rows = rows[:num_errs]
            rows = rows + [(None, '')] * (num_errs - len(rows))
        lines = [header]
        for n_fns, err in rows:
            if n_fns is None or num_proc <= 0:
                lines.append('     -----')
            else:
                lines.append('{:8.1f}% ({:>7} reads) : {:<80}'.format(
                    100 * n_fns / float(num_proc), n_fns, err))
        return '\n'.join(lines)

    def final_message(self, num_reads):
        counts = self.counts()
        if not counts:
            return 'All reads successfully re-squiggled!'
        total = sum(n for n, _ in counts)
        header = ('Final unsuccessful reads summary '
                  '({:.1%} reads unsuccessfully processed; {} total reads):'.format(
                      float(total) / num_reads, total))
        return self.format(header, counts, num_reads)

    def write(self, failed_reads_fn):
        """``--failed-reads-filename``: message TAB comma separated file names"""
        lines = []
        for err, fns in self.failed_reads.items():
            lines.append('%s\t%s' % (err, ', '.join(fns)))
        with io.open(failed_reads_fn, 'wt') as fp:
            fp.write('\n'.join(lines))
            fp.write('\n')
