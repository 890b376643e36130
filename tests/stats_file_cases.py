"""Statistics-file cases shared by tests/golden/make_stats_file_golden.py, the tests and
bench_stats_file.py: an in-memory h5py-like file, a PerReadStats-like iterable, and the numpy
restatements of aggregate_per_read_stats' block tables (_agg_stats_worker +
ModelStats._write_stat_block) and of the most-significant table.

The table restatement is one stable sort of every row in arrival order, by the structured
array's fields in dtype order (numpy's tie rule for ``sort(order=key)``), cut to N rows."""
from collections import OrderedDict

import numpy as np

from tombo_b200 import formats

MODEL_MS_DTYPE = formats.MODEL_STATS_DTYPE + formats.MOST_SIGNIF_EXTRA
LEVEL_MS_DTYPE = formats.LEVEL_STATS_DTYPE + formats.MOST_SIGNIF_EXTRA


class FakeGroup(object):
    """the h5py surface the writers use: attrs, create_group, create_dataset, item access"""

    def __init__(self):
        self.attrs = OrderedDict()
        self.children = OrderedDict()

    def create_group(self, name):
        if name in self.children:
            raise ValueError('name already exists: ' + name)
        g = self.children[name] = FakeGroup()
        return g

    def create_dataset(self, name, shape=None, dtype=None, data=None, compression=None):
        if name in self.children:
            raise ValueError('name already exists: ' + name)
        arr = np.array(data) if data is not None else np.empty(shape, dtype=object)
        self.children[name] = arr
        return arr

    def __getitem__(self, name):
        return self.children[name]

    def __contains__(self, name):
        return name in self.children

    def items(self):
        return self.children.items()

    def flush(self):
        pass

    def close(self):
        pass


def layout(grp, prefix=''):
    """[(path, kind, attrs or (dtype, array))] of a FakeGroup tree in creation order"""
    out = [(prefix or '/', 'group', dict(grp.attrs))]
    for name, c in grp.children.items():
        path = prefix + '/' + name
        if isinstance(c, FakeGroup):
            out.extend(layout(c, path))
        else:
            out.append((path, 'dataset', c))
    return out


class PerReadBlocks(object):
    """PerReadStats' iteration surface over in-memory blocks (chrm, strand, start, table)"""

    def __init__(self, stat_type, region_size, blocks):
        self.stat_type, self.region_size, self.blocks = stat_type, region_size, blocks

    def __iter__(self):
        for chrm, strand, start, table in self.blocks:
            yield chrm, strand, start, start + self.region_size, table.copy()


def per_read_table(pos, stat):
    t = np.empty(len(pos), dtype=formats.PER_READ_DTYPE)
    t['pos'], t['stat'], t['read_id'] = pos, stat, np.arange(len(pos)) % 7
    return t


def restate_block(pos, stat, thresh, lower, llr, unmod, mod):
    """one block's table: covered positions ascending, NaN damp_frac rows dropped"""
    pos = np.asarray(pos, dtype=np.int64)
    stat = np.asarray(stat, dtype=np.float64)
    out = np.zeros(0, dtype=formats.MODEL_STATS_DTYPE)
    if pos.shape[0] == 0:
        return out
    o = np.argsort(pos, kind='stable')
    p, s = pos[o], stat[o]
    us, first, cov = np.unique(p, return_index=True, return_counts=True)
    with np.errstate(invalid='ignore', divide='ignore'):
        if lower is not None:
            valid = (s <= lower) | (s >= thresh)
        elif llr:
            valid = np.abs(s) >= thresh
        else:
            valid = np.ones(s.shape[0], dtype=bool)
        ge = valid & (s >= thresh)
        v = np.add.reduceat(valid.astype(np.int64), first)
        g = np.add.reduceat(ge.astype(np.int64), first)
        frac = np.where(v > 0, g / np.maximum(v, 1), np.nan)
        damp = (np.round(frac * v) + unmod) / (v + (0 + unmod + mod))
    keep = ~np.isnan(damp)
    out = np.zeros(int(keep.sum()), dtype=formats.MODEL_STATS_DTYPE)
    out['damp_frac'], out['frac'], out['pos'] = damp[keep], frac[keep], us[keep]
    out['cov'], out['valid_cov'] = cov[keep], v[keep]
    return out


def with_chrm_strand(table, chrm_id, strand, level=False):
    out = np.zeros(table.shape[0], dtype=LEVEL_MS_DTYPE if level else MODEL_MS_DTYPE)
    for name in table.dtype.names:
        out[name] = table[name]
    out['chrm'] = chrm_id
    out['strand'] = strand
    return out


def restate_most_signif(rows, n_keep):
    """first n_keep rows of one stable sort by every field in dtype order"""
    names = rows.dtype.names
    keys = []
    for name in reversed(names):                       # np.lexsort: last key is primary
        col = rows[name]
        if col.dtype.kind == 'S':
            col = col.view(np.uint8)
        keys.append(col)
    idx = np.lexsort(keys)
    return rows[idx[:n_keep]]


def random_blocks(rng, n_blocks, region_size, reads_per_pos, chrms=('chr1', 'chr2'),
                  quantum=None, nan_frac=0.0, llr=False):
    """(chrm, strand, start, per-read table) blocks over (chrm, strand) groups; statistics
    rounded to multiples of ``quantum`` make damp_frac ties common"""
    blocks = []
    groups = [(c, s) for c in chrms for s in ('+', '-')]
    for b in range(n_blocks):
        chrm, strand = groups[b % len(groups)]
        start = (b // len(groups)) * region_size
        n_pos = int(rng.integers(max(1, region_size // 4), region_size + 1))
        cov_pos = np.sort(rng.choice(region_size, size=n_pos, replace=False))
        reps = rng.poisson(reads_per_pos, size=n_pos) + 1
        pos = np.repeat(cov_pos, reps) + start
        n = pos.shape[0]
        stat = rng.normal(0, 3, n) if llr else rng.uniform(0, 1, n)
        if quantum:
            stat = np.round(stat / quantum) * quantum
        if nan_frac:
            stat[rng.random(n) < nan_frac] = np.nan
        o = rng.permutation(n)
        blocks.append((chrm, strand, start, per_read_table(pos[o], stat[o])))
    return blocks


class RestatedContext(object):
    """the tb2_stats_file_* / tb2_most_signif_* surface of _lib.Context computed by the numpy
    restatements: lets the writers' file layout be checked without a device"""

    def stats_file_aggregate(self, blocks, region_size, pos, stat, thresh, lower, stat_type,
                             unmod, mod):
        self._agg, off = [], [0]
        for start, s0, n, chrm, strand in np.asarray(blocks).reshape(-1, 5):
            p = np.asarray(pos[s0:s0 + n], dtype=np.int64)
            if ((p < start) | (p >= start + region_size)).any():
                raise ValueError('position outside its block')
            t = restate_block(p, stat[s0:s0 + n], thresh, lower, stat_type == 0, unmod, mod)
            self._agg.append(with_chrm_strand(t, chrm, bytes([strand])))
            off.append(off[-1] + t.shape[0])
        return np.array(off, dtype=np.int64)

    def stats_file_download(self, n_rows):
        t = np.concatenate(self._agg) if self._agg else np.zeros(0, MODEL_MS_DTYPE)
        return t['pos'], t['damp_frac'], t['frac'], t['cov'], t['valid_cov']

    def most_signif_begin(self, level, n):
        self._level, self._n, self._rows = level, n, []

    def most_signif_end(self):
        self._rows = None

    def most_signif_add_rows(self, key, pos, cov, control_cov, chrm, strand, frac=None,
                             valid_cov=None):
        t = np.zeros(len(key), dtype=LEVEL_MS_DTYPE if self._level else MODEL_MS_DTYPE)
        t[t.dtype.names[0]] = key
        t['pos'], t['cov'], t['control_cov'], t['chrm'], t['strand'] = pos, cov, control_cov, chrm, strand
        if not self._level:
            t['frac'], t['valid_cov'] = frac, valid_cov
        self._rows.append(t)

    def most_signif_add_aggregate(self):
        self._rows.extend(self._agg)

    def most_signif_get(self):
        dt = LEVEL_MS_DTYPE if self._level else MODEL_MS_DTYPE
        t = restate_most_signif(np.concatenate(self._rows) if self._rows else np.zeros(0, dt), self._n)
        c = dict((name, t[name]) for name in t.dtype.names)
        c['key'] = t[t.dtype.names[0]]
        return c


# ---------------------------------------------------------------------------
# goldens (tests/golden/stats_file.npz)
# ---------------------------------------------------------------------------
def golden_cases(g, prefix):
    return sorted((k[:-4] for k in g.files if k.startswith(prefix) and k.endswith('_par')),
                  key=lambda q: int(q[1:]))


def golden_model_input(g, q):
    """(PerReadBlocks, thresh, lower, (unmod, mod), N, min_test_reads)"""
    par = g[q + '_par']
    chrms, blk, off = list(g[q + '_chrms']), g[q + '_blk'], g[q + '_off']
    blocks = []
    for b, (c, s, start) in enumerate(blk):
        lo, hi = off[b], off[b + 1]
        blocks.append((str(chrms[c]), '-' if s else '+', int(start),
                       per_read_table(g[q + '_pos'][lo:hi], g[q + '_stat'][lo:hi])))
    lower = None if np.isnan(par[1]) else float(par[1])
    return (PerReadBlocks(str(g[q + '_stype']), int(par[6]), blocks), float(par[0]), lower,
            (par[3].item(), par[4].item()), int(par[5]), int(par[8]))


def golden_level_input(g, q):
    """[(chrm, strand, start, stat, poss, cov, ctrl)], N"""
    chrms, blk, off = list(g[q + '_chrms']), g[q + '_blk'], g[q + '_off']
    out = []
    for b, (c, s, start) in enumerate(blk):
        lo, hi = off[b], off[b + 1]
        out.append((str(chrms[c]), '-' if s else '+', int(start), g[q + '_lstat'][lo:hi],
                    g[q + '_lpos'][lo:hi], g[q + '_lcov'][lo:hi], g[q + '_lctrl'][lo:hi]))
    return out, int(g[q + '_par'][5])


def file_layout(root):
    """the golden's ``_layout`` form of a FakeGroup tree"""
    out = []
    for path, kind, val in layout(root):
        if kind == 'group':
            out.append([path, kind, [[k, v.decode() if isinstance(v, bytes) else
                                      (v.item() if isinstance(v, np.generic) else v)]
                                     for k, v in val.items()]])
        else:
            out.append([path, kind, str(val.dtype)])
    return out


def file_tables(root):
    blocks = root['Statistic_Blocks']
    return [blocks['Block_%d' % i]['block_stats'] for i in range(len(blocks.children))]
