"""Tuning constants of the resquiggle hot path.

Values mirror the reference tables in tombo/_default_parameters.py (line numbers in
comments); they are data the algorithm is defined by, and tests/ check them against
the reference build when it is available."""

RNA_SAMP_TYPE = 'RNA'                      # :8
DNA_SAMP_TYPE = 'DNA'                      # :9

# (running_stat_width, min_obs_per_base, raw_min_obs_per_base, mean_obs_per_event)
SEG_PARAMS_TABLE = {                       # :34-37
    RNA_SAMP_TYPE: (12, 6, 2, 15),
    DNA_SAMP_TYPE: (5, 3, 1, 5),
}
# (match_evalue, skip_pen, bandwidth, save_bandwidth, max_half_z_score,
#  band_bound_thresh, start_bw, start_save_bw, start_n_bases)
ALGN_PARAMS_TABLE = {                      # :50-53
    RNA_SAMP_TYPE: (6, 4, 500, 1500, 20.0, 50, 1000, 3000, 250),
    DNA_SAMP_TYPE: (4.2, 4.2, 300, 1500, 20.0, 40, 750, 2500, 250),
}
SIG_MATCH_THRESH = {RNA_SAMP_TYPE: 2, DNA_SAMP_TYPE: 1.1}      # :57-60
OUTLIER_THRESH = 5.0                       # :63
EXTRA_SIG_FACTOR = 1.1                     # :67
MASK_BASES = 50                            # :69
MASK_FILL_Z_SCORE = -15                    # :70
DEL_FIX_WINDOW = 2                         # :72
MAX_DEL_FIX_WINDOW = 10                    # :73
MAX_RAW_CPTS = 200                         # :74
MIN_EVENT_TO_SEQ_RATIO = 1.1               # :75
USE_RNA_EVENT_SCALE = True                 # :78
RNA_SCALE_NUM_EVENTS = 10000               # :79
RNA_SCALE_MAX_FRAC_EVENTS = 0.75           # :80
COLLAPSE_RNA_STALLS = True                 # :84
COLLAPSE_DNA_STALLS = False                # :85
MEAN_STALL_PARAMS = dict((                 # :93-96
    ('window_size', 7 * 50), ('threshold', 40), ('edge_buffer', 100),
    ('min_consecutive_obs', 200), ('n_windows', 7), ('mini_window_size', 50)))
STALL_PARAMS = MEAN_STALL_PARAMS           # :97
START_CLIP_PARAMS = (1000, 200)            # :100
LLR_THRESH = {DNA_SAMP_TYPE: (-1.5, 2.5), RNA_SAMP_TYPE: (-2.5, 2.5)}   # :107-110
OCLLHR_SCALE = 4.0                         # :132
OCLLHR_HEIGHT = 1.0                        # :133
OCLLHR_POWER = 0.2                         # :134
SHIFT_CHANGE_THRESH = 0.1                  # :169
SCALE_CHANGE_THRESH = 0.1                  # :170
MAX_SCALING_ITERS = 3                      # :171
MAX_POINTS_FOR_THEIL_SEN = 1000            # :178
FM_OFFSET_DEFAULT = 1                      # :136
SMALLEST_PVAL = 1e-50                      # :158
MEAN_PRIOR_CONST = 5                       # :139
SD_PRIOR_CONST = 40                        # :140
COV_DAMP_COUNTS = [2, 0]                   # (unmodified, modified pseudo counts)
ALT_EST_BATCH = 1000                       # :147
MAX_KMER_OBS = 10000                       # :148
MIN_KMER_OBS_TO_EST = 50                   # :149
KERNEL_DENSITY_RANGE = (-5, 5)             # :150
ALT_EST_PCTL = 5                           # :151
NUM_DENS_POINTS = 500                      # :164
NUM_READS_TO_ADJUST_MODEL = 5000           # :174
ROC_PLOT_POINTS = 1000                     # :181
