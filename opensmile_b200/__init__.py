"""opensmile_b200 -- H100 (sm_90a) back end for openSMILE's per-frame LLD extraction path.

The compute path is the in-tree CUDA library libosm_b200.so behind the C ABI in
include/osm_b200.h; importing this package does not load it, the first use of
`opensmile_b200.plan.Plan` does (and fails loudly if it has not been built).
"""
from . import capi  # noqa: F401
from .plan import (Plan, comp, components_frontend, components_mfcc12_0_d_a,  # noqa: F401
                   components_plp_0_d_a, pack_utterances)

from .session import Session, SessionError, write_arff, write_csv, write_htk  # noqa: F401

__all__ = ["Session", "SessionError", "Plan", "components_mfcc12_0_d_a", "components_plp_0_d_a", "pack_utterances", "capi"]
