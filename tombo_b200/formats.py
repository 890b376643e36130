"""On-disk formats either side of the hot path (SURVEY.md 8(f)-3), host only:

* the resquiggled-reads index the reference pickles next to a FAST5 directory
  (``TomboReads.write_index_file`` / ``_load_index_data``, tombo_helper.py:1068-1104,
  1235-1290): what ``tombo resquiggle`` leaves behind for every later command;
* the per-read statistics blocks of a ``PerReadStats`` file (tombo_stats.py:3335-3366) and
  the (pos, stat, read_id) table ``collate_reg_stats`` builds for them (:4136-4154);
* the statistics file of ``ModelStats`` / ``LevelStats`` (:2594-2636, 3064-3099): its block
  tables and its most-significant table, which the device keeps (tb2_most_signif_*).

The FAST5 ``Events`` group writer is in :mod:`tombo_b200.tombo_helper`.  HDF5 objects are
duck-typed (anything with ``create_group`` / ``create_dataset`` / ``attrs``), h5py itself is
not a requirement of this package."""
import io
import os
import pickle
import re
from collections import OrderedDict, defaultdict

import numpy as np

from . import _lib
from . import tombo_helper as th

INDEX_SUFFIX = '.tombo.index'
PER_READ_BLOCKS_NAME = 'Statistic_Blocks'          # tombo_stats.py:114 STAT_BLOCKS_H5_NAME
PER_READ_DTYPE = [(str('pos'), 'u4'), (str('stat'), 'f8'), (str('read_id'), 'u4')]
MOST_SIGNIF_NAME = 'Most_Significant_Stats'         # tombo_stats.py:115-117
COV_DAMP_COUNTS_NAME = 'Cov_Damp_Counts'
COV_THRESH_NAME = 'Cov_Threshold'
MODEL_STATS_DTYPE = [(str('damp_frac'), 'f8'), (str('frac'), 'f8'), (str('pos'), 'u4'),
                     (str('cov'), 'u4'), (str('control_cov'), 'u4'), (str('valid_cov'), 'u4')]
LEVEL_STATS_DTYPE = [(str('stat'), 'f8'), (str('pos'), 'u4'), (str('cov'), 'u4'),
                     (str('control_cov'), 'u4')]
MOST_SIGNIF_EXTRA = [(str('chrm'), 'u4'), (str('strand'), 'S1')]


def index_filename(fast5s_dir, corr_grp='RawGenomeCorrected_000'):
    """``.<fast5s_dir>.<corr_grp>.tombo.index`` next to the directory (tombo_helper.py:1099-1108)"""
    if fast5s_dir.endswith('/'):
        fast5s_dir = fast5s_dir[:-1]
    head, tail = os.path.split(fast5s_dir)
    return os.path.join(head, '.' + tail + '.' + corr_grp + INDEX_SUFFIX)


class ReadsIndex(object):
    """The write side of ``TomboReads`` (``for_writing=True``): collect
    :class:`tombo_helper.readData` per (chrm, strand) and pickle them in the reference's
    record layout, so the reference (or this class) can load the index back."""

    def __init__(self, fast5s_dir, corr_grp='RawGenomeCorrected_000'):
        self.basedir = fast5s_dir if fast5s_dir.endswith('/') else fast5s_dir + '/'
        self.corr_grp = corr_grp
        self.index_fn = index_filename(self.basedir, corr_grp)
        self.reads_index = defaultdict(list)

    def add_read_data(self, chrm, strand, read_data):
        self.reads_index[(chrm, strand)].append(read_data)

    def records(self):
        """{(chrm, strand): [11-tuples]} exactly as write_index_file builds them (:1086-1096)"""
        out = defaultdict(list)
        for chrm_strand, cs_reads in self.reads_index.items():
            for rd in cs_reads:
                grp = rd.corr_group.split('/')
                out[chrm_strand].append((
                    re.sub(self.basedir, '', rd.fn, 1), rd.start, rd.end, rd.read_start_rel_to_raw,
                    grp[0], grp[-1], rd.filtered, rd.rna, rd.sig_match_score, rd.mean_q_score,
                    rd.read_id))
        return dict(out)

    def dumps(self):
        return pickle.dumps(self.records(), protocol=2)      # protocol 2: py2 / py3 readable

    def write_index_file(self):
        with io.open(self.index_fn, 'wb') as fp:
            fp.write(self.dumps())
        return self.index_fn


def load_index(index_fn, fast5s_dir, corr_grp='RawGenomeCorrected_000', remove_filtered=False):
    """{(chrm, strand): [readData]} from an index file (``_load_index_data``: 8-, 10- and
    11-field records of the successive Tombo versions).  ``remove_filtered`` drops the reads
    whose filtered flag is set, and then any (chrm, strand) left without reads, as
    ``TomboReads(remove_filtered=True)`` does (tombo_helper.py:1296-1310)."""
    with io.open(index_fn, 'rb') as fp:
        raw = pickle.load(fp)
    if not raw:
        raise th.TomboError('Tombo index file appears to be empty')
    n = len(next(iter(raw.values()))[0])
    if n not in (8, 10, 11):
        raise th.TomboError('Invalid Tombo index file.')
    out = {}
    for (chrm, strand), recs in raw.items():
        rds = []
        for rec in recs:
            fn, start, end, rsrtr, c_grp, s_grp, filtered, rna = rec[:8]
            extra = tuple(rec[8:])
            rds.append(th.readData(start, end, filtered, rsrtr, strand,
                                   os.path.join(fast5s_dir, fn), corr_grp + '/' + s_grp, rna,
                                   *extra))
        if remove_filtered:
            rds = [rd for rd in rds if not rd.filtered]
            if not rds:
                continue
        out[(chrm, strand)] = rds
    return out


def load_reads_index(fast5s_dirs, corr_grp='RawGenomeCorrected_000', bc_subgrps=None):
    """{(chrm, strand): [readData]} of ``TomboReads(fast5s_dirs, corr_grp, bc_subgrps)``
    (tombo_helper.py:1292-1348) from the directories' Tombo indexes: filtered reads removed,
    reads outside ``bc_subgrps`` (when given) dropped, a (chrm, strand) left without reads
    dropped, and each (chrm, strand) concatenating its reads in directory order.  Groups come
    in order of first appearance (the reference's follow a set).  A directory without an index
    raises TomboError: building one from the FAST5 files is not done here."""
    merged = OrderedDict()
    for fast5s_dir in fast5s_dirs:
        fast5s_dir = fast5s_dir if fast5s_dir.endswith('/') else fast5s_dir + '/'
        index_fn = index_filename(fast5s_dir, corr_grp)
        if not os.path.exists(index_fn):
            raise th.TomboError('Tombo index file does not exist for ' + fast5s_dir)
        for cs, rds in load_index(index_fn, fast5s_dir, corr_grp, remove_filtered=True).items():
            if bc_subgrps is not None:
                rds = [rd for rd in rds if rd.corr_group.split('/')[-1] in bc_subgrps]
            if rds:
                merged.setdefault(cs, []).extend(rds)
    return dict(merged)


# ---------------------------------------------------------------------------
# per-read statistics blocks
# ---------------------------------------------------------------------------
def per_read_block(stats, stat_locs, read_ids):
    """The table ``collate_reg_stats`` queues for the per-read statistics file
    (tombo_stats.py:4136-4154): ``stats`` / ``stat_locs`` are the per-read arrays of one
    region, ``read_ids`` the ``(read_id, n_stats)`` pairs.  Returns ``(block, lookup)``:
    a structured array (pos u4, stat f8, read_id u4) without the NaN statistics and the
    read_id -> integer lookup that keeps strings out of the table."""
    stats = np.concatenate(stats)
    stat_locs = np.concatenate(stat_locs)
    valid = ~np.isnan(stats)
    rep_ids = []
    for r_id, r_len in read_ids:
        rep_ids.extend([r_id.decode() if isinstance(r_id, bytes) else r_id] * int(r_len))
    if len(rep_ids) != stats.shape[0]:
        raise th.TomboError('read id counts do not match the statistics')
    valid_ids = [rid for rid, ok in zip(rep_ids, valid) if ok]
    lookup = OrderedDict()
    for rid in valid_ids:                      # first-seen order (the reference: set order)
        if rid not in lookup:
            lookup[rid] = len(lookup)
    block = np.empty(int(valid.sum()), dtype=PER_READ_DTYPE)
    block['pos'] = stat_locs[valid]
    block['stat'] = stats[valid]
    block['read_id'] = [lookup[rid] for rid in valid_ids]
    return block, lookup


class PerReadStatsWriter(object):
    """``PerReadStats._write_per_read_block`` (tombo_stats.py:3335-3366) over an h5py-like
    file object: one ``Block_<n>`` group per region with its chrm / strand / start attributes,
    the ``block_stats`` table and the read-id lookup as two parallel datasets."""

    def __init__(self, h5_file, stat_type, region_size):
        self._fp = h5_file
        h5_file.attrs['stat_type'] = stat_type
        h5_file.attrs['block_size'] = region_size
        self.per_read_blocks = h5_file.create_group(PER_READ_BLOCKS_NAME)
        self.curr_block_num = 0

    def write_block(self, block, read_id_lookup, chrm, strand, start):
        grp = self.per_read_blocks.create_group('Block_' + str(self.curr_block_num))
        self.curr_block_num += 1
        grp.attrs['chrm'] = chrm
        grp.attrs['strand'] = strand
        grp.attrs['start'] = start
        grp.create_dataset('block_stats', data=block, compression='gzip')
        ids = np.array(list(read_id_lookup.keys()), dtype=object)
        ds = grp.create_dataset('read_ids', data=ids, compression='gzip')
        grp.create_dataset('read_id_vals', data=np.array(list(read_id_lookup.values())),
                           compression='gzip')
        if hasattr(self._fp, 'flush'):
            self._fp.flush()
        return ds


# ---------------------------------------------------------------------------
# statistics files
# ---------------------------------------------------------------------------
def _strand_byte(strand):
    """the byte the most-significant table's S1 column stores for a strand"""
    b = strand if isinstance(strand, bytes) else str(strand).encode()
    return b[:1] if b else b'\0'


class _StatsWriter(object):
    _level = False
    _dtype = MODEL_STATS_DTYPE

    def __init__(self, h5_file, stat_type, region_size, cov_thresh, num_most_signif, ctx=None,
                 device=0):
        self._fp = h5_file
        self.region_size = region_size
        h5_file.attrs['stat_type'] = stat_type
        h5_file.attrs['block_size'] = region_size
        self.stat_blocks = h5_file.create_group(PER_READ_BLOCKS_NAME)
        h5_file.attrs[COV_THRESH_NAME] = cov_thresh
        self._init_extra()
        self.most_signif_sites = h5_file.create_group(MOST_SIGNIF_NAME)
        self.chrm_names = OrderedDict()
        self.chrm_id_grp = self.most_signif_sites.create_group('chrm_ids')
        self.curr_block_num = 0
        self.is_empty = True
        # the device table lives on the context, one per context: a writer owns a context
        # unless given one, so writers open at once never share a table
        self._own_ctx = ctx is None
        self.ctx = _lib.Context(device) if ctx is None else ctx
        self.ctx.most_signif_begin(self._level, num_most_signif)

    def _init_extra(self):
        pass

    def _chrm_id(self, chrm):
        if chrm not in self.chrm_names:
            self.chrm_names[chrm] = len(self.chrm_names)
        return self.chrm_names[chrm]

    def write_block_table(self, table, chrm, strand, start):
        """one ``Block_<n>`` group: its chrm / strand / start attributes and the table"""
        grp = self.stat_blocks.create_group('Block_' + str(self.curr_block_num))
        self.curr_block_num += 1
        grp.attrs['chrm'] = chrm
        grp.attrs['strand'] = strand
        grp.attrs['start'] = start
        grp.create_dataset('block_stats', data=table, compression='gzip')
        self.is_empty = False

    def _write_rows(self, table, chrm, strand, start):
        self.write_block_table(table, chrm, strand, start)
        cid = self._chrm_id(chrm)
        key = table[self._dtype[0][0]]
        self.ctx.most_signif_add_rows(
            key, table['pos'], table['cov'], table['control_cov'], cid, _strand_byte(strand),
            frac=None if self._level else table['frac'],
            valid_cov=None if self._level else table['valid_cov'])

    def most_signif_table(self):
        """the most-significant table as ``_close_write`` stores it (trimmed when fewer rows
        than requested exist)"""
        c = self.ctx.most_signif_get()
        out = np.empty(c['key'].shape[0], dtype=self._dtype + MOST_SIGNIF_EXTRA)
        out[self._dtype[0][0]] = c['key']
        for name, _ in self._dtype[1:] + MOST_SIGNIF_EXTRA:
            out[name] = c[name]
        return out

    def close(self):
        """``_close_write``: the most-significant dataset and the chromosome ids"""
        self.most_signif_sites.create_dataset(MOST_SIGNIF_NAME, data=self.most_signif_table(),
                                              compression='gzip')
        for chrm_name, chrm_id in self.chrm_names.items():
            self.chrm_id_grp.attrs[chrm_name] = chrm_id
        self.discard()

    def discard(self):
        """close the device table (and the writer's own context) without writing it"""
        self.ctx.most_signif_end()
        if self._own_ctx:
            self.ctx.close()


class ModelStatsWriter(_StatsWriter):
    """``ModelStats`` opened for writing (tombo_stats.py:2594-2636, 2737-2795) over an
    h5py-like file: the reference's layout, with the running most-significant table on the
    device.  ``cov_damp_counts`` is (unmod, mod).  Without ``ctx`` the writer opens a context
    of its own on ``device`` (the table belongs to the context) and closes it in close()."""

    def __init__(self, h5_file, stat_type, region_size, cov_damp_counts, cov_thresh,
                 num_most_signif, ctx=None, device=0):
        self.cov_damp_counts = dict(zip(('unmod', 'mod'), cov_damp_counts))
        super(ModelStatsWriter, self).__init__(h5_file, stat_type, region_size, cov_thresh,
                                               num_most_signif, ctx, device)

    def _init_extra(self):
        grp = self._fp.create_group(COV_DAMP_COUNTS_NAME)
        grp.attrs['unmod'] = self.cov_damp_counts['unmod']
        grp.attrs['mod'] = self.cov_damp_counts['mod']

    def _write_stat_block(self, reg_stats):
        """one ``regionStats`` (:2737-2773): the block table without NaN damp_frac rows; the
        fields are zipped, so the shortest one sets the row count"""
        fracs = np.asarray(reg_stats.reg_frac_standard_base, dtype=np.float64)
        valid_cov = np.asarray(reg_stats.valid_cov)
        damp = (np.round(fracs * valid_cov) + self.cov_damp_counts['unmod']) / (
            valid_cov + sum(list(self.cov_damp_counts.values())))
        cols = (damp, fracs, reg_stats.reg_poss, reg_stats.reg_cov, reg_stats.ctrl_cov, valid_cov)
        n = min(len(c) for c in cols)
        keep = ~np.isnan(damp[:n])
        table = np.empty(int(keep.sum()), dtype=MODEL_STATS_DTYPE)
        for (name, _), c in zip(MODEL_STATS_DTYPE, cols):
            table[name] = np.asarray(c)[:n][keep]
        self._write_rows(table, reg_stats.chrm, reg_stats.strand, reg_stats.start)

    def write_aggregated(self, blocks, row_off, cols):
        """the block tables of one tb2_stats_file_aggregate call: ``blocks`` (chrm, strand,
        start) in order, ``cols`` its downloaded (pos, damp_frac, frac, cov, valid_cov); the
        rows join the most-significant table without leaving the device"""
        pos, damp, frac, cov, valid = cols
        for b, (chrm, strand, start) in enumerate(blocks):
            lo, hi = row_off[b], row_off[b + 1]
            table = np.zeros(hi - lo, dtype=MODEL_STATS_DTYPE)
            table['damp_frac'], table['frac'], table['pos'] = damp[lo:hi], frac[lo:hi], pos[lo:hi]
            table['cov'], table['valid_cov'] = cov[lo:hi], valid[lo:hi]
            self.write_block_table(table, chrm, strand, start)
        self.ctx.most_signif_add_aggregate()


class LevelStatsWriter(_StatsWriter):
    """``LevelStats`` opened for writing (tombo_stats.py:3064-3099, 3194-3224)"""
    _level = True
    _dtype = LEVEL_STATS_DTYPE

    def _write_stat_block(self, grp_stats):
        """one ``groupStats``: the block table without NaN stat rows (zip semantics)"""
        cols = (grp_stats.reg_stats, grp_stats.reg_poss, grp_stats.reg_cov, grp_stats.ctrl_cov)
        n = min(len(c) for c in cols)
        stat = np.asarray(grp_stats.reg_stats, dtype=np.float64)[:n]
        keep = ~np.isnan(stat)
        table = np.empty(int(keep.sum()), dtype=LEVEL_STATS_DTYPE)
        for (name, _), c in zip(LEVEL_STATS_DTYPE, cols):
            table[name] = np.asarray(c)[:n][keep]
        self._write_rows(table, grp_stats.chrm, grp_stats.strand, grp_stats.start)
