"""tombo_b200 -- a CUDA (H100, sm_90a) implementation of the Tombo resquiggle hot
path behind the ``tombo.resquiggle`` / ``tombo.tombo_stats`` / ``tombo.tombo_helper``
Python API.  Host code is Python calling hand-written CUDA through a C ABI
(include/tombo_b200.h, tombo_b200/libtombo_b200.so); there is no CPU fallback.

    from tombo_b200 import tombo_helper, tombo_stats, resquiggle
    std_ref = tombo_stats.TomboModel(kmer_ref=..., central_pos=2)
    params = tombo_stats.load_resquiggle_parameters(seq_samp_type)
    res = resquiggle.resquiggle_read(map_res, std_ref, params, outlier_thresh=5.0)
    many = resquiggle.resquiggle_reads(list_of_map_res, std_ref, params, save_params)

Sub-modules are imported lazily so that the package (and the ABI) can be inspected
on machines without a GPU."""
__version__ = '0.1.0'
__all__ = ['tombo_helper', 'tombo_stats', 'resquiggle', 'synthetic', '_lib']


def __getattr__(name):
    if name in __all__:
        import importlib
        return importlib.import_module('.' + name, __name__)
    raise AttributeError(name)
