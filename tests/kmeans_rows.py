"""The rows of the native k-means initialisation's stage tests (test_gpu_kmeans_init.py), shared with the CPU test that
pins the kernels each row reaches (test_kmeans_cpu.py)."""
from collections import namedtuple

from stages import HB_KS_FFMA_CONTRACTIONS, HB_KS_WIDE, M_FFMA, M_LOGITS, M_TC, M_WIDE

Row = namedtuple("Row", "K d N J kind launches")
ROWS = {
    "tc_K12": Row(12, 12, 3000, 3, "blobs", 1),
    "tc_K64": Row(64, 50, 20000, 5, "blobs", 1),
    "tc_K65": Row(65, 50, 20000, 5, "blobs", 2),
    "tc_K128": Row(128, 64, 20000, 5, "blobs", 2),
    "tc_K129": Row(129, 64, 20000, 5, "blobs", 3),
    "tc_K256_d120": Row(256, 120, 20000, 5, "blobs", 4),
    "ffma_K257_d120": Row(257, 120, 20000, 5, "blobs", None),
    "ffma_d121": Row(100, 121, 20000, 5, "blobs", None),
    "ffma_at_limit": Row(400, 128, 20000, 5, "blobs", None),
    "wide_past_limit": Row(401, 128, 20000, 5, "blobs", None),
    "tc_K450_d120": Row(450, 120, 20000, 5, "blobs", 8),
    "tc_K1024_d64": Row(1024, 64, 19000, 3, "blobs", 16),      # N: enough blobs that few cells are ambiguous
    "wide_K200_d512": Row(200, 512, 20000, 3, "blobs", None),
    "c3like": Row(100, 50, 200000, 20, "blobs", 2),
    "wide_forced_K705_d8": Row(705, 8, 20000, 5, "blobs", None),
    "d1": Row(5, 1, 2000, 2, "d1", 1),
    "antipodal": Row(64, 16, 1500, 3, "antipodal", 1),
    "special_rows_J1": Row(100, 50, 20000, 1, "special", 2),
    "special_rows_J100": Row(100, 50, 20000, 100, "special", 2),
    "N_equals_K": Row(40, 16, 40, 1, "n_equals_k", 1),
}
# (row, kernel set, k-means path, NV of the race and pick kernels: sp_nv(KS), None on the FFMA path)
CASES = [
    ("tc_K12", 0, M_TC, 1),
    ("tc_K64", 0, M_TC, 1),
    ("tc_K65", 0, M_TC, 1),
    ("tc_K128", 0, M_TC, 1),
    ("tc_K129", 0, M_TC, 2),
    ("tc_K256_d120", 0, M_TC, 2),                 # KS = 256 and d = 120: both limits of the LogitsTc choice
    ("ffma_K257_d120", 0, M_FFMA, None),          # KS = 260 > 256
    ("ffma_d121", 0, M_FFMA, None),               # d = 121: no k_logits_tc
    ("ffma_at_limit", 0, M_FFMA, None),           # 4 K d = 200 KB exactly
    ("wide_past_limit", 0, M_WIDE, 4),            # 4 K d = 200 KB + 512 B, d = 128: k_logits_wide
    ("tc_K450_d120", 0, M_LOGITS, 4),             # past the FFMA limit, KS = 452 > 256
    ("tc_K1024_d64", 0, M_LOGITS, 8),
    ("wide_K200_d512", 0, M_WIDE, 2),
    ("c3like", 0, M_TC, 1),
    ("c3like", HB_KS_FFMA_CONTRACTIONS, M_FFMA, None),
    ("c3like", HB_KS_WIDE, M_WIDE, 1),
    ("wide_forced_K705_d8", HB_KS_WIDE, M_WIDE, 8),
    ("d1", 0, M_TC, 1),
    ("d1", HB_KS_FFMA_CONTRACTIONS, M_FFMA, None),
    ("antipodal", 0, M_TC, 1),
    ("antipodal", HB_KS_FFMA_CONTRACTIONS, M_FFMA, None),
    ("special_rows_J1", 0, M_TC, 1),
    ("special_rows_J1", HB_KS_FFMA_CONTRACTIONS, M_FFMA, None),
    ("special_rows_J100", 0, M_TC, 1),
    ("special_rows_J100", HB_KS_FFMA_CONTRACTIONS, M_FFMA, None),
    ("N_equals_K", 0, M_TC, 1),
    ("N_equals_K", HB_KS_FFMA_CONTRACTIONS, M_FFMA, None),
]
