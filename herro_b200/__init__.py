"""herro_b200 — H100-native (sm_90a) implementation of HERRO's features -> inference -> consensus
hot path behind the C ABI of include/herro_b200.h.  See DESIGN.md."""
from .api import Context, Corrected, HerroError, fasta_records, load_library, pack_2bit  # noqa: F401
from .weights import NetConfig, load_blob, random_weights, save_blob  # noqa: F401

__version__ = "0.1.0"
