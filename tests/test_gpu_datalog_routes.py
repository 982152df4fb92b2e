"""GPU (-m gpu): what every Datalog entry point costs, pinned for each shape it takes.

Every case runs twice, each time on a context of its own, and checks, for each call, the result against the oracle and the
*fingerprint* against a literal. A fingerprint is the change of every integer counter of kb_stats across the call (launches per
family, kernel launches, rows, bytes copied, index joins; counters that did not move are left out) and every field of the stats the
call returns, except device time. d2h_bytes counts whole control-arena reads, so it also pins the number of host synchronisations.
Results are compared as multisets; where the layout is defined (kb_datalog_fixpoint, kb_datalog_fixpoint_seed) the predicate blocks of
the `p` column are checked too: accepted seed facts first, then inferred facts, each in ascending predicate order.

The shapes:
  kb_datalog_fixpoint        the reference's fc_* fixtures and a taxonomy slice under all four strategies; a known-fact set that grows
                             in the middle of a derive launch; the radix-partitioned dedup forced onto a small store
  kb_datalog_fixpoint_seed   two seeded calls in a row after a fixpoint, with the kept state (KOLIBRIE_FIX_STATE=1) and without
  kb_datalog_query           a variable-predicate query, an open subject, a ground query that stops early, a depth bound below the
                             fixpoint
  kb_datalog_maintain        no-op, evict only, add only, add a fact that was inferred, a diamond over-deleted and rederived; each after
                             a first maintenance call, with its kept state and without
  kb_datalog_query_repairs   one inconsistent store
and the status code of a refused call at each entry point.
"""
import numpy as np
import pytest

import tests.bc_reference as B
import tests.repairs_reference as R
from kolibrie_b200 import capi as c
from kolibrie_b200 import datagen
from kolibrie_b200.engine import Constant, Variable, compile_rule
from tests import helpers as H
from tests import oracle_api as O
from tests import sharded_cases as SC
from tests.test_gpu_backward import to_kb as bc_to_kb
from tests.test_gpu_repairs import to_kb as repairs_to_kb
from tests.window_oracle import as_rows, rows_set

pytestmark = pytest.mark.gpu

FIELDS = ("scan_launches", "build_launches", "probe_launches", "filter_launches", "group_launches", "other_launches", "kernel_launches",
          "rows_scanned", "rows_built", "rows_probed", "rows_out", "h2d_bytes", "d2h_bytes", "fused_scan_builds", "index_joins")
# switches that select routes: pinned to their defaults, so that the literals hold whatever the caller's environment says
DEFAULT_ENV = {"KOLIBRIE_ORDERED": "0", "KOLIBRIE_USE_INDEX": "1", "KOLIBRIE_INDEX_MAINTAIN": "1", "KOLIBRIE_FIX_STATE": "1",
               "KOLIBRIE_DERIVE_PART": "1", "KOLIBRIE_DERIVE_SLICE": str(32 << 20), "KOLIBRIE_DERIVE_MIN_ROWS": str(1 << 20),
               "KOLIBRIE_DERIVE_SLACK": "8192"}
STRATEGIES = {"semi_naive": c.SEMI_NAIVE, "naive": c.NAIVE, "parallel": c.SEMI_NAIVE_PARALLEL, "old_delta": c.SEMI_NAIVE_OLD_DELTA}
FC = H.load("datalog_fc.json")["cases"]

# name -> the fingerprints of one run's calls, in call order (recorded on an H100; both runs must give them)
ROUTES = {
    "fc_1hop_base_semi_naive": [
        ({'scan_launches': 1, 'build_launches': 1, 'other_launches': 1, 'kernel_launches': 3, 'rows_scanned': 1, 'rows_out': 1, 'd2h_bytes': 65536}, {'rounds': 1, 'inferred': 1, 'derivations': 1, 'round_new': [1]}),
    ],
    "fc_1hop_base_naive": [
        ({'scan_launches': 1, 'build_launches': 1, 'other_launches': 2, 'kernel_launches': 4, 'rows_scanned': 1, 'rows_out': 1, 'd2h_bytes': 98304}, {'rounds': 1, 'inferred': 1, 'derivations': 2, 'round_new': [1]}),
    ],
    "fc_1hop_base_parallel": [
        ({'scan_launches': 1, 'build_launches': 1, 'other_launches': 1, 'kernel_launches': 3, 'rows_scanned': 1, 'rows_out': 1, 'd2h_bytes': 65536}, {'rounds': 1, 'inferred': 1, 'derivations': 1, 'round_new': [1]}),
    ],
    "fc_1hop_base_old_delta": [
        ({'scan_launches': 1, 'build_launches': 1, 'other_launches': 1, 'kernel_launches': 3, 'rows_scanned': 1, 'rows_out': 1, 'd2h_bytes': 65536}, {'rounds': 1, 'inferred': 1, 'derivations': 1, 'round_new': [1]}),
    ],
    "fc_2hop_transitive_semi_naive": [
        ({'scan_launches': 1, 'build_launches': 9, 'probe_launches': 6, 'other_launches': 3, 'kernel_launches': 35, 'rows_scanned': 2, 'rows_built': 6, 'rows_probed': 10, 'rows_out': 3, 'd2h_bytes': 393216}, {'rounds': 2, 'inferred': 3, 'derivations': 4, 'round_new': [2, 1]}),
    ],
    "fc_2hop_transitive_naive": [
        ({'scan_launches': 1, 'build_launches': 5, 'probe_launches': 4, 'other_launches': 5, 'kernel_launches': 23, 'rows_scanned': 2, 'rows_built': 5, 'rows_probed': 5, 'rows_out': 3, 'd2h_bytes': 327680}, {'rounds': 2, 'inferred': 3, 'derivations': 8, 'round_new': [2, 1]}),
    ],
    "fc_2hop_transitive_parallel": [
        ({'scan_launches': 1, 'build_launches': 9, 'probe_launches': 6, 'other_launches': 3, 'kernel_launches': 35, 'rows_scanned': 2, 'rows_built': 6, 'rows_probed': 10, 'rows_out': 3, 'd2h_bytes': 393216}, {'rounds': 2, 'inferred': 3, 'derivations': 4, 'round_new': [2, 1]}),
    ],
    "fc_2hop_transitive_old_delta": [
        ({'scan_launches': 1, 'build_launches': 7, 'probe_launches': 4, 'other_launches': 2, 'kernel_launches': 26, 'rows_scanned': 2, 'rows_built': 4, 'rows_probed': 7, 'rows_out': 3, 'd2h_bytes': 294912}, {'rounds': 2, 'inferred': 3, 'derivations': 3, 'round_new': [2, 1]}),
    ],
    "fc_3hop_transitive_semi_naive": [
        ({'scan_launches': 1, 'build_launches': 13, 'probe_launches': 10, 'other_launches': 5, 'kernel_launches': 53, 'rows_scanned': 3, 'rows_built': 12, 'rows_probed': 28, 'rows_out': 6, 'd2h_bytes': 589824}, {'rounds': 3, 'inferred': 6, 'derivations': 9, 'round_new': [3, 2, 1]}),
    ],
    "fc_3hop_transitive_naive": [
        ({'scan_launches': 1, 'build_launches': 7, 'probe_launches': 6, 'other_launches': 7, 'kernel_launches': 33, 'rows_scanned': 3, 'rows_built': 14, 'rows_probed': 14, 'rows_out': 6, 'd2h_bytes': 458752}, {'rounds': 3, 'inferred': 6, 'derivations': 22, 'round_new': [3, 2, 1]}),
    ],
    "fc_3hop_transitive_parallel": [
        ({'scan_launches': 1, 'build_launches': 13, 'probe_launches': 10, 'other_launches': 5, 'kernel_launches': 53, 'rows_scanned': 3, 'rows_built': 12, 'rows_probed': 28, 'rows_out': 6, 'd2h_bytes': 589824}, {'rounds': 3, 'inferred': 6, 'derivations': 9, 'round_new': [3, 2, 1]}),
    ],
    "fc_3hop_transitive_old_delta": [
        ({'scan_launches': 1, 'build_launches': 11, 'probe_launches': 8, 'other_launches': 4, 'kernel_launches': 44, 'rows_scanned': 3, 'rows_built': 9, 'rows_probed': 22, 'rows_out': 6, 'd2h_bytes': 491520}, {'rounds': 3, 'inferred': 6, 'derivations': 7, 'round_new': [3, 2, 1]}),
    ],
    "fc_join_sibling_semi_naive": [
        ({'scan_launches': 1, 'build_launches': 5, 'probe_launches': 4, 'other_launches': 2, 'kernel_launches': 20, 'rows_scanned': 2, 'rows_built': 4, 'rows_probed': 4, 'rows_out': 2, 'd2h_bytes': 229376}, {'rounds': 1, 'inferred': 2, 'derivations': 4, 'round_new': [2]}),
    ],
    "fc_join_sibling_naive": [
        ({'scan_launches': 1, 'build_launches': 5, 'probe_launches': 4, 'other_launches': 2, 'kernel_launches': 20, 'rows_scanned': 2, 'rows_built': 4, 'rows_probed': 4, 'rows_out': 2, 'd2h_bytes': 229376}, {'rounds': 1, 'inferred': 2, 'derivations': 4, 'round_new': [2]}),
    ],
    "fc_join_sibling_parallel": [
        ({'scan_launches': 1, 'build_launches': 5, 'probe_launches': 4, 'other_launches': 2, 'kernel_launches': 20, 'rows_scanned': 2, 'rows_built': 4, 'rows_probed': 4, 'rows_out': 4, 'd2h_bytes': 229376}, {'rounds': 1, 'inferred': 4, 'derivations': 8, 'round_new': [4]}),
    ],
    "fc_join_sibling_old_delta": [
        ({'scan_launches': 1, 'build_launches': 3, 'probe_launches': 2, 'other_launches': 1, 'kernel_launches': 11, 'rows_scanned': 2, 'rows_built': 2, 'rows_probed': 2, 'rows_out': 2, 'd2h_bytes': 131072}, {'rounds': 1, 'inferred': 2, 'derivations': 2, 'round_new': [2]}),
    ],
    "fc_multi_rule_cascade_semi_naive": [
        ({'scan_launches': 1, 'build_launches': 2, 'other_launches': 2, 'kernel_launches': 5, 'rows_scanned': 1, 'rows_out': 2, 'd2h_bytes': 98304}, {'rounds': 2, 'inferred': 2, 'derivations': 2, 'round_new': [1, 1]}),
    ],
    "fc_multi_rule_cascade_naive": [
        ({'scan_launches': 1, 'build_launches': 2, 'other_launches': 5, 'kernel_launches': 8, 'rows_scanned': 1, 'rows_out': 2, 'd2h_bytes': 196608}, {'rounds': 2, 'inferred': 2, 'derivations': 5, 'round_new': [1, 1]}),
    ],
    "fc_multi_rule_cascade_parallel": [
        ({'scan_launches': 1, 'build_launches': 2, 'other_launches': 2, 'kernel_launches': 5, 'rows_scanned': 1, 'rows_out': 2, 'd2h_bytes': 98304}, {'rounds': 2, 'inferred': 2, 'derivations': 2, 'round_new': [1, 1]}),
    ],
    "fc_multi_rule_cascade_old_delta": [
        ({'scan_launches': 1, 'build_launches': 2, 'other_launches': 2, 'kernel_launches': 5, 'rows_scanned': 1, 'rows_out': 2, 'd2h_bytes': 98304}, {'rounds': 2, 'inferred': 2, 'derivations': 2, 'round_new': [1, 1]}),
    ],
    "fc_three_premise_rule_semi_naive": [
        ({'scan_launches': 1, 'build_launches': 10, 'probe_launches': 10, 'other_launches': 3, 'kernel_launches': 40, 'rows_scanned': 3, 'rows_built': 5, 'rows_probed': 5, 'rows_out': 1, 'd2h_bytes': 425984}, {'rounds': 1, 'inferred': 1, 'derivations': 3, 'round_new': [1]}),
    ],
    "fc_three_premise_rule_naive": [
        ({'scan_launches': 1, 'build_launches': 9, 'probe_launches': 8, 'other_launches': 2, 'kernel_launches': 36, 'rows_scanned': 3, 'rows_built': 4, 'rows_probed': 4, 'rows_out': 1, 'd2h_bytes': 360448}, {'rounds': 1, 'inferred': 1, 'derivations': 2, 'round_new': [1]}),
    ],
    "fc_three_premise_rule_parallel": [
        ({'scan_launches': 1, 'build_launches': 1, 'kernel_launches': 2, 'rows_scanned': 3, 'd2h_bytes': 32768}, {'rounds': 0, 'inferred': 0, 'derivations': 0, 'round_new': []}),
    ],
    "fc_three_premise_rule_old_delta": [
        ({'scan_launches': 1, 'build_launches': 5, 'probe_launches': 4, 'other_launches': 1, 'kernel_launches': 19, 'rows_scanned': 3, 'rows_built': 2, 'rows_probed': 2, 'rows_out': 1, 'd2h_bytes': 196608}, {'rounds': 1, 'inferred': 1, 'derivations': 1, 'round_new': [1]}),
    ],
    "fc_no_spurious_semi_naive": [
        ({'scan_launches': 1, 'build_launches': 1, 'other_launches': 1, 'kernel_launches': 3, 'rows_scanned': 2, 'rows_out': 1, 'd2h_bytes': 65536}, {'rounds': 1, 'inferred': 1, 'derivations': 1, 'round_new': [1]}),
    ],
    "fc_no_spurious_naive": [
        ({'scan_launches': 1, 'build_launches': 1, 'other_launches': 2, 'kernel_launches': 4, 'rows_scanned': 2, 'rows_out': 1, 'd2h_bytes': 98304}, {'rounds': 1, 'inferred': 1, 'derivations': 2, 'round_new': [1]}),
    ],
    "fc_no_spurious_parallel": [
        ({'scan_launches': 1, 'build_launches': 1, 'other_launches': 1, 'kernel_launches': 3, 'rows_scanned': 2, 'rows_out': 1, 'd2h_bytes': 65536}, {'rounds': 1, 'inferred': 1, 'derivations': 1, 'round_new': [1]}),
    ],
    "fc_no_spurious_old_delta": [
        ({'scan_launches': 1, 'build_launches': 1, 'other_launches': 1, 'kernel_launches': 3, 'rows_scanned': 2, 'rows_out': 1, 'd2h_bytes': 65536}, {'rounds': 1, 'inferred': 1, 'derivations': 1, 'round_new': [1]}),
    ],
    "fc_sibling_three_children_semi_naive": [
        ({'scan_launches': 1, 'build_launches': 5, 'probe_launches': 4, 'other_launches': 2, 'kernel_launches': 20, 'rows_scanned': 3, 'rows_built': 6, 'rows_probed': 6, 'rows_out': 6, 'd2h_bytes': 229376}, {'rounds': 1, 'inferred': 6, 'derivations': 12, 'round_new': [6]}),
    ],
    "fc_sibling_three_children_naive": [
        ({'scan_launches': 1, 'build_launches': 5, 'probe_launches': 4, 'other_launches': 2, 'kernel_launches': 20, 'rows_scanned': 3, 'rows_built': 6, 'rows_probed': 6, 'rows_out': 6, 'd2h_bytes': 229376}, {'rounds': 1, 'inferred': 6, 'derivations': 12, 'round_new': [6]}),
    ],
    "fc_sibling_three_children_parallel": [
        ({'scan_launches': 1, 'build_launches': 5, 'probe_launches': 4, 'other_launches': 2, 'kernel_launches': 20, 'rows_scanned': 3, 'rows_built': 6, 'rows_probed': 6, 'rows_out': 9, 'd2h_bytes': 229376}, {'rounds': 1, 'inferred': 9, 'derivations': 18, 'round_new': [9]}),
    ],
    "fc_sibling_three_children_old_delta": [
        ({'scan_launches': 1, 'build_launches': 3, 'probe_launches': 2, 'other_launches': 1, 'kernel_launches': 11, 'rows_scanned': 3, 'rows_built': 3, 'rows_probed': 3, 'rows_out': 6, 'd2h_bytes': 131072}, {'rounds': 1, 'inferred': 6, 'derivations': 6, 'round_new': [6]}),
    ],
    "fc_multi_conclusion_semi_naive": [
        ({'scan_launches': 1, 'build_launches': 2, 'other_launches': 2, 'kernel_launches': 5, 'rows_scanned': 1, 'rows_out': 2, 'd2h_bytes': 98304}, {'rounds': 1, 'inferred': 2, 'derivations': 2, 'round_new': [2]}),
    ],
    "fc_multi_conclusion_naive": [
        ({'scan_launches': 1, 'build_launches': 2, 'other_launches': 4, 'kernel_launches': 7, 'rows_scanned': 1, 'rows_out': 2, 'd2h_bytes': 163840}, {'rounds': 1, 'inferred': 2, 'derivations': 4, 'round_new': [2]}),
    ],
    "fc_multi_conclusion_parallel": [
        ({'scan_launches': 1, 'build_launches': 2, 'other_launches': 2, 'kernel_launches': 5, 'rows_scanned': 1, 'rows_out': 2, 'd2h_bytes': 98304}, {'rounds': 1, 'inferred': 2, 'derivations': 2, 'round_new': [2]}),
    ],
    "fc_multi_conclusion_old_delta": [
        ({'scan_launches': 1, 'build_launches': 2, 'other_launches': 2, 'kernel_launches': 5, 'rows_scanned': 1, 'rows_out': 2, 'd2h_bytes': 98304}, {'rounds': 1, 'inferred': 2, 'derivations': 2, 'round_new': [2]}),
    ],
    "fc_diamond_ancestor_semi_naive": [
        ({'scan_launches': 1, 'build_launches': 9, 'probe_launches': 6, 'other_launches': 3, 'kernel_launches': 35, 'rows_scanned': 4, 'rows_built': 10, 'rows_probed': 18, 'rows_out': 5, 'd2h_bytes': 393216}, {'rounds': 2, 'inferred': 5, 'derivations': 8, 'round_new': [4, 1]}),
    ],
    "fc_diamond_ancestor_naive": [
        ({'scan_launches': 1, 'build_launches': 5, 'probe_launches': 4, 'other_launches': 5, 'kernel_launches': 23, 'rows_scanned': 4, 'rows_built': 9, 'rows_probed': 9, 'rows_out': 5, 'd2h_bytes': 327680}, {'rounds': 2, 'inferred': 5, 'derivations': 16, 'round_new': [4, 1]}),
    ],
    "fc_diamond_ancestor_parallel": [
        ({'scan_launches': 1, 'build_launches': 9, 'probe_launches': 6, 'other_launches': 3, 'kernel_launches': 35, 'rows_scanned': 4, 'rows_built': 10, 'rows_probed': 18, 'rows_out': 5, 'd2h_bytes': 393216}, {'rounds': 2, 'inferred': 5, 'derivations': 8, 'round_new': [4, 1]}),
    ],
    "fc_diamond_ancestor_old_delta": [
        ({'scan_launches': 1, 'build_launches': 7, 'probe_launches': 4, 'other_launches': 2, 'kernel_launches': 26, 'rows_scanned': 4, 'rows_built': 6, 'rows_probed': 13, 'rows_out': 5, 'd2h_bytes': 294912}, {'rounds': 2, 'inferred': 5, 'derivations': 6, 'round_new': [4, 1]}),
    ],
    "fc_disconnected_graphs_semi_naive": [
        ({'scan_launches': 1, 'build_launches': 1, 'other_launches': 1, 'kernel_launches': 3, 'rows_scanned': 2, 'rows_out': 2, 'd2h_bytes': 65536}, {'rounds': 1, 'inferred': 2, 'derivations': 2, 'round_new': [2]}),
    ],
    "fc_disconnected_graphs_naive": [
        ({'scan_launches': 1, 'build_launches': 1, 'other_launches': 2, 'kernel_launches': 4, 'rows_scanned': 2, 'rows_out': 2, 'd2h_bytes': 98304}, {'rounds': 1, 'inferred': 2, 'derivations': 4, 'round_new': [2]}),
    ],
    "fc_disconnected_graphs_parallel": [
        ({'scan_launches': 1, 'build_launches': 1, 'other_launches': 1, 'kernel_launches': 3, 'rows_scanned': 2, 'rows_out': 2, 'd2h_bytes': 65536}, {'rounds': 1, 'inferred': 2, 'derivations': 2, 'round_new': [2]}),
    ],
    "fc_disconnected_graphs_old_delta": [
        ({'scan_launches': 1, 'build_launches': 1, 'other_launches': 1, 'kernel_launches': 3, 'rows_scanned': 2, 'rows_out': 2, 'd2h_bytes': 65536}, {'rounds': 1, 'inferred': 2, 'derivations': 2, 'round_new': [2]}),
    ],
    "fc_no_matching_facts_semi_naive": [
        ({'scan_launches': 1, 'build_launches': 1, 'kernel_launches': 2, 'rows_scanned': 1, 'd2h_bytes': 32768}, {'rounds': 0, 'inferred': 0, 'derivations': 0, 'round_new': []}),
    ],
    "fc_no_matching_facts_naive": [
        ({'scan_launches': 1, 'build_launches': 1, 'kernel_launches': 2, 'rows_scanned': 1, 'd2h_bytes': 32768}, {'rounds': 0, 'inferred': 0, 'derivations': 0, 'round_new': []}),
    ],
    "fc_no_matching_facts_parallel": [
        ({'scan_launches': 1, 'build_launches': 1, 'kernel_launches': 2, 'rows_scanned': 1, 'd2h_bytes': 32768}, {'rounds': 0, 'inferred': 0, 'derivations': 0, 'round_new': []}),
    ],
    "fc_no_matching_facts_old_delta": [
        ({'scan_launches': 1, 'build_launches': 1, 'kernel_launches': 2, 'rows_scanned': 1, 'd2h_bytes': 32768}, {'rounds': 0, 'inferred': 0, 'derivations': 0, 'round_new': []}),
    ],
    "fc_idempotent_semi_naive": [
        ({'scan_launches': 1, 'build_launches': 1, 'other_launches': 1, 'kernel_launches': 3, 'rows_scanned': 1, 'rows_out': 1, 'd2h_bytes': 65536}, {'rounds': 1, 'inferred': 1, 'derivations': 1, 'round_new': [1]}),
    ],
    "fc_idempotent_naive": [
        ({'scan_launches': 1, 'build_launches': 1, 'other_launches': 2, 'kernel_launches': 4, 'rows_scanned': 1, 'rows_out': 1, 'd2h_bytes': 98304}, {'rounds': 1, 'inferred': 1, 'derivations': 2, 'round_new': [1]}),
    ],
    "fc_idempotent_parallel": [
        ({'scan_launches': 1, 'build_launches': 1, 'other_launches': 1, 'kernel_launches': 3, 'rows_scanned': 1, 'rows_out': 1, 'd2h_bytes': 65536}, {'rounds': 1, 'inferred': 1, 'derivations': 1, 'round_new': [1]}),
    ],
    "fc_idempotent_old_delta": [
        ({'scan_launches': 1, 'build_launches': 1, 'other_launches': 1, 'kernel_launches': 3, 'rows_scanned': 1, 'rows_out': 1, 'd2h_bytes': 65536}, {'rounds': 1, 'inferred': 1, 'derivations': 1, 'round_new': [1]}),
    ],
    "fc_uncle_derived_semi_naive": [
        ({'scan_launches': 1, 'build_launches': 8, 'probe_launches': 6, 'other_launches': 3, 'kernel_launches': 30, 'rows_scanned': 3, 'rows_built': 8, 'rows_probed': 9, 'rows_out': 3, 'd2h_bytes': 327680}, {'rounds': 2, 'inferred': 3, 'derivations': 5, 'round_new': [2, 1]}),
    ],
    "fc_uncle_derived_naive": [
        ({'scan_launches': 1, 'build_launches': 12, 'probe_launches': 10, 'other_launches': 5, 'kernel_launches': 48, 'rows_scanned': 3, 'rows_built': 13, 'rows_probed': 15, 'rows_out': 3, 'd2h_bytes': 524288}, {'rounds': 2, 'inferred': 3, 'derivations': 8, 'round_new': [2, 1]}),
    ],
    "fc_uncle_derived_parallel": [
        ({'scan_launches': 1, 'build_launches': 8, 'probe_launches': 6, 'other_launches': 3, 'kernel_launches': 30, 'rows_scanned': 3, 'rows_built': 9, 'rows_probed': 11, 'rows_out': 7, 'd2h_bytes': 327680}, {'rounds': 2, 'inferred': 7, 'derivations': 12, 'round_new': [5, 2]}),
    ],
    "fc_uncle_derived_old_delta": [
        ({'scan_launches': 1, 'build_launches': 6, 'probe_launches': 4, 'other_launches': 2, 'kernel_launches': 21, 'rows_scanned': 3, 'rows_built': 5, 'rows_probed': 6, 'rows_out': 3, 'd2h_bytes': 229376}, {'rounds': 2, 'inferred': 3, 'derivations': 3, 'round_new': [2, 1]}),
    ],
    "taxonomy_semi_naive": [
        ({'scan_launches': 1, 'build_launches': 29, 'probe_launches': 25, 'other_launches': 12, 'kernel_launches': 119, 'rows_scanned': 5340, 'rows_built': 7276, 'rows_probed': 62501, 'rows_out': 19295, 'd2h_bytes': 1277952}, {'rounds': 3, 'inferred': 19295, 'derivations': 56052, 'round_new': [5323, 10184, 3788]}),
    ],
    "taxonomy_naive": [
        ({'scan_launches': 1, 'build_launches': 20, 'probe_launches': 16, 'other_launches': 8, 'kernel_launches': 79, 'rows_scanned': 5340, 'rows_built': 7040, 'rows_probed': 61485, 'rows_out': 19295, 'd2h_bytes': 819200}, {'rounds': 3, 'inferred': 19295, 'derivations': 117643, 'round_new': [5323, 10184, 3788]}),
    ],
    "taxonomy_parallel": [
        ({'scan_launches': 1, 'build_launches': 29, 'probe_launches': 25, 'other_launches': 12, 'kernel_launches': 119, 'rows_scanned': 5340, 'rows_built': 7276, 'rows_probed': 62501, 'rows_out': 19295, 'd2h_bytes': 1277952}, {'rounds': 3, 'inferred': 19295, 'derivations': 56052, 'round_new': [5323, 10184, 3788]}),
    ],
    "taxonomy_old_delta": [
        ({'scan_launches': 1, 'build_launches': 25, 'probe_launches': 21, 'other_launches': 10, 'kernel_launches': 101, 'rows_scanned': 5340, 'rows_built': 6596, 'rows_probed': 41654, 'rows_out': 19295, 'd2h_bytes': 1081344}, {'rounds': 3, 'inferred': 19295, 'derivations': 45786, 'round_new': [5323, 10184, 3788]}),
    ],
    "grows_mid_launch": [
        ({'scan_launches': 1, 'build_launches': 3, 'other_launches': 2, 'kernel_launches': 8, 'rows_scanned': 4000000, 'rows_built': 4000000, 'rows_out': 4000000, 'd2h_bytes': 98304}, {'rounds': 1, 'inferred': 4000000, 'derivations': 4000000, 'round_new': [4000000]}),
    ],
    "partitioned_semi_naive": [
        ({'scan_launches': 1, 'build_launches': 35, 'probe_launches': 30, 'other_launches': 14, 'kernel_launches': 172, 'rows_scanned': 5363, 'rows_built': 89180, 'rows_probed': 97838, 'rows_out': 23713, 'd2h_bytes': 1540096}, {'rounds': 3, 'inferred': 23713, 'derivations': 80132, 'round_new': [5344, 10425, 7944]}),
    ],
    "partitioned_naive": [
        ({'scan_launches': 1, 'build_launches': 21, 'probe_launches': 16, 'other_launches': 8, 'kernel_launches': 96, 'rows_scanned': 5363, 'rows_built': 160868, 'rows_probed': 66278, 'rows_out': 23713, 'd2h_bytes': 819200}, {'rounds': 3, 'inferred': 23713, 'derivations': 152618, 'round_new': [5344, 10425, 7944]}),
    ],
    "seed_state1": [
        ({'scan_launches': 1, 'build_launches': 29, 'probe_launches': 25, 'other_launches': 12, 'kernel_launches': 119, 'rows_scanned': 3120, 'rows_built': 2487, 'rows_probed': 35640, 'rows_out': 10856, 'd2h_bytes': 1277952}, {'rounds': 3, 'inferred': 10856, 'derivations': 31220, 'round_new': [3096, 5755, 2005]}),
        ({'scan_launches': 1, 'build_launches': 6, 'probe_launches': 4, 'filter_launches': 2, 'other_launches': 4, 'kernel_launches': 25, 'rows_scanned': 13976, 'rows_built': 726, 'rows_probed': 1188, 'rows_out': -10094, 'd2h_bytes': 360448}, {'rounds': 1, 'inferred': 762, 'derivations': 1441, 'round_new': [762]}),
        ({'build_launches': 4, 'probe_launches': 4, 'filter_launches': 2, 'other_launches': 3, 'kernel_launches': 21, 'rows_built': 726, 'rows_probed': 1184, 'rows_out': -4, 'd2h_bytes': 294912}, {'rounds': 1, 'inferred': 758, 'derivations': 1423, 'round_new': [758]}),
    ],
    "seed_state0": [
        ({'scan_launches': 1, 'build_launches': 29, 'probe_launches': 25, 'other_launches': 12, 'kernel_launches': 119, 'rows_scanned': 3120, 'rows_built': 2487, 'rows_probed': 35640, 'rows_out': 10856, 'd2h_bytes': 1277952}, {'rounds': 3, 'inferred': 10856, 'derivations': 31220, 'round_new': [3096, 5755, 2005]}),
        ({'scan_launches': 1, 'build_launches': 6, 'probe_launches': 4, 'filter_launches': 2, 'other_launches': 4, 'kernel_launches': 25, 'rows_scanned': 13976, 'rows_built': 726, 'rows_probed': 1188, 'rows_out': -10094, 'd2h_bytes': 360448}, {'rounds': 1, 'inferred': 762, 'derivations': 1441, 'round_new': [762]}),
        ({'scan_launches': 1, 'build_launches': 6, 'probe_launches': 4, 'filter_launches': 2, 'other_launches': 3, 'kernel_launches': 24, 'rows_scanned': 15038, 'rows_built': 726, 'rows_probed': 1184, 'rows_out': -4, 'd2h_bytes': 327680}, {'rounds': 1, 'inferred': 758, 'derivations': 1423, 'round_new': [758]}),
    ],
    "query_variable_predicate": [
        ({'scan_launches': 1, 'build_launches': 20, 'probe_launches': 18, 'other_launches': 10, 'kernel_launches': 87, 'rows_scanned': 28, 'rows_built': 73, 'rows_probed': 234, 'rows_out': 90, 'd2h_bytes': 983040}, {'rounds': 10, 'reached_fixpoint': 0, 'stopped_early': 0, 'relevant_rules': 2, 'demand_patterns': 2, 'restricted_predicates': 0, 'base_facts': 26, 'derived': 76, 'derivations': 152, 'answers': 90}),
    ],
    "query_open_subject": [
        ({'scan_launches': 1, 'build_launches': 16, 'probe_launches': 13, 'filter_launches': 1, 'other_launches': 7, 'kernel_launches': 66, 'rows_scanned': 28, 'rows_built': 7, 'rows_probed': 182, 'rows_out': 7, 'd2h_bytes': 786432}, {'rounds': 8, 'reached_fixpoint': 1, 'stopped_early': 0, 'relevant_rules': 2, 'demand_patterns': 2, 'restricted_predicates': 1, 'base_facts': 26, 'derived': 7, 'derivations': 38, 'answers': 7}),
    ],
    "query_ground_stops_early": [
        ({'scan_launches': 1, 'build_launches': 6, 'probe_launches': 4, 'filter_launches': 1, 'other_launches': 3, 'kernel_launches': 23, 'rows_scanned': 28, 'rows_built': 2, 'rows_probed': 52, 'rows_out': 1, 'd2h_bytes': 327680}, {'rounds': 3, 'reached_fixpoint': 0, 'stopped_early': 1, 'relevant_rules': 2, 'demand_patterns': 2, 'restricted_predicates': 1, 'base_facts': 26, 'derived': 3, 'derivations': 30, 'answers': 1}),
    ],
    "query_depth_bound": [
        ({'scan_launches': 1, 'build_launches': 6, 'probe_launches': 4, 'other_launches': 3, 'kernel_launches': 22, 'rows_scanned': 28, 'rows_built': 24, 'rows_probed': 52, 'rows_out': 3, 'd2h_bytes': 294912}, {'rounds': 3, 'reached_fixpoint': 0, 'stopped_early': 0, 'relevant_rules': 2, 'demand_patterns': 2, 'restricted_predicates': 0, 'base_facts': 26, 'derived': 34, 'derivations': 68, 'answers': 3}),
    ],
    "maintain_no_op_state1": [
        ({'scan_launches': 1, 'build_launches': 5, 'probe_launches': 3, 'other_launches': 2, 'kernel_launches': 19, 'rows_scanned': 2, 'rows_built': 3, 'rows_probed': 4, 'rows_out': 3, 'd2h_bytes': 229376}, {'rounds': 2, 'inferred': 3, 'derivations': 3, 'round_new': [2, 1]}),
        ({'scan_launches': 2, 'build_launches': 12, 'probe_launches': 4, 'filter_launches': 4, 'other_launches': 5, 'kernel_launches': 39, 'rows_scanned': 5, 'rows_built': 5, 'rows_probed': 11, 'h2d_bytes': 24, 'd2h_bytes': 622592}, {'base_removed': 0, 'base_added': 2, 'overdeleted': 0, 'rederived': 0, 'inferred_removed': 0, 'inferred_added': 3, 'derivations': 3, 'overdelete_rounds': 0, 'insert_rounds': 2}),
        ({}, {'base_removed': 0, 'base_added': 0, 'overdeleted': 0, 'rederived': 0, 'inferred_removed': 0, 'inferred_added': 0, 'derivations': 0, 'overdelete_rounds': 0, 'insert_rounds': 0}),
    ],
    "maintain_no_op_state0": [
        ({'scan_launches': 1, 'build_launches': 5, 'probe_launches': 3, 'other_launches': 2, 'kernel_launches': 19, 'rows_scanned': 2, 'rows_built': 3, 'rows_probed': 4, 'rows_out': 3, 'd2h_bytes': 229376}, {'rounds': 2, 'inferred': 3, 'derivations': 3, 'round_new': [2, 1]}),
        ({'scan_launches': 2, 'build_launches': 12, 'probe_launches': 4, 'filter_launches': 4, 'other_launches': 5, 'kernel_launches': 39, 'rows_scanned': 5, 'rows_built': 5, 'rows_probed': 11, 'h2d_bytes': 24, 'd2h_bytes': 622592}, {'base_removed': 0, 'base_added': 2, 'overdeleted': 0, 'rederived': 0, 'inferred_removed': 0, 'inferred_added': 3, 'derivations': 3, 'overdelete_rounds': 0, 'insert_rounds': 2}),
        ({}, {'base_removed': 0, 'base_added': 0, 'overdeleted': 0, 'rederived': 0, 'inferred_removed': 0, 'inferred_added': 0, 'derivations': 0, 'overdelete_rounds': 0, 'insert_rounds': 0}),
    ],
    "maintain_evict_only_state1": [
        ({'scan_launches': 1, 'build_launches': 7, 'probe_launches': 5, 'other_launches': 3, 'kernel_launches': 28, 'rows_scanned': 3, 'rows_built': 6, 'rows_probed': 9, 'rows_out': 6, 'd2h_bytes': 327680}, {'rounds': 3, 'inferred': 6, 'derivations': 6, 'round_new': [3, 2, 1]}),
        ({'scan_launches': 2, 'build_launches': 12, 'probe_launches': 4, 'filter_launches': 4, 'other_launches': 5, 'kernel_launches': 39, 'rows_scanned': 9, 'rows_built': 5, 'rows_probed': 16, 'rows_out': -3, 'h2d_bytes': 24, 'd2h_bytes': 622592}, {'base_removed': 0, 'base_added': 2, 'overdeleted': 0, 'rederived': 0, 'inferred_removed': 0, 'inferred_added': 3, 'derivations': 3, 'overdelete_rounds': 0, 'insert_rounds': 2}),
        ({'scan_launches': 1, 'build_launches': 10, 'probe_launches': 5, 'filter_launches': 4, 'other_launches': 3, 'kernel_launches': 35, 'rows_scanned': 1, 'rows_built': 10, 'rows_probed': 22, 'rows_out': -3, 'd2h_bytes': 524288}, {'base_removed': 1, 'base_added': 0, 'overdeleted': 3, 'rederived': 0, 'inferred_removed': 3, 'inferred_added': 0, 'derivations': 3, 'overdelete_rounds': 1, 'insert_rounds': 0}),
    ],
    "maintain_evict_only_state0": [
        ({'scan_launches': 1, 'build_launches': 7, 'probe_launches': 5, 'other_launches': 3, 'kernel_launches': 28, 'rows_scanned': 3, 'rows_built': 6, 'rows_probed': 9, 'rows_out': 6, 'd2h_bytes': 327680}, {'rounds': 3, 'inferred': 6, 'derivations': 6, 'round_new': [3, 2, 1]}),
        ({'scan_launches': 2, 'build_launches': 12, 'probe_launches': 4, 'filter_launches': 4, 'other_launches': 5, 'kernel_launches': 39, 'rows_scanned': 9, 'rows_built': 5, 'rows_probed': 16, 'rows_out': -3, 'h2d_bytes': 24, 'd2h_bytes': 622592}, {'base_removed': 0, 'base_added': 2, 'overdeleted': 0, 'rederived': 0, 'inferred_removed': 0, 'inferred_added': 3, 'derivations': 3, 'overdelete_rounds': 0, 'insert_rounds': 2}),
        ({'scan_launches': 3, 'build_launches': 13, 'probe_launches': 5, 'filter_launches': 4, 'other_launches': 3, 'kernel_launches': 40, 'rows_scanned': 15, 'rows_built': 10, 'rows_probed': 22, 'rows_out': -3, 'd2h_bytes': 622592}, {'base_removed': 1, 'base_added': 0, 'overdeleted': 3, 'rederived': 0, 'inferred_removed': 3, 'inferred_added': 0, 'derivations': 3, 'overdelete_rounds': 1, 'insert_rounds': 0}),
    ],
    "maintain_add_only_state1": [
        ({'scan_launches': 1, 'build_launches': 3, 'probe_launches': 1, 'other_launches': 1, 'kernel_launches': 10, 'rows_scanned': 1, 'rows_built': 1, 'rows_probed': 1, 'rows_out': 1, 'd2h_bytes': 131072}, {'rounds': 1, 'inferred': 1, 'derivations': 1, 'round_new': [1]}),
        ({'scan_launches': 2, 'build_launches': 12, 'probe_launches': 4, 'filter_launches': 4, 'other_launches': 5, 'kernel_launches': 39, 'rows_scanned': 2, 'rows_built': 4, 'rows_probed': 8, 'rows_out': 2, 'h2d_bytes': 24, 'd2h_bytes': 622592}, {'base_removed': 0, 'base_added': 2, 'overdeleted': 0, 'rederived': 0, 'inferred_removed': 0, 'inferred_added': 3, 'derivations': 3, 'overdelete_rounds': 0, 'insert_rounds': 2}),
        ({'build_launches': 11, 'probe_launches': 6, 'filter_launches': 4, 'other_launches': 6, 'kernel_launches': 43, 'rows_built': 7, 'rows_probed': 19, 'rows_out': 2, 'h2d_bytes': 24, 'd2h_bytes': 622592}, {'base_removed': 0, 'base_added': 2, 'overdeleted': 0, 'rederived': 0, 'inferred_removed': 0, 'inferred_added': 5, 'derivations': 5, 'overdelete_rounds': 0, 'insert_rounds': 3}),
    ],
    "maintain_add_only_state0": [
        ({'scan_launches': 1, 'build_launches': 3, 'probe_launches': 1, 'other_launches': 1, 'kernel_launches': 10, 'rows_scanned': 1, 'rows_built': 1, 'rows_probed': 1, 'rows_out': 1, 'd2h_bytes': 131072}, {'rounds': 1, 'inferred': 1, 'derivations': 1, 'round_new': [1]}),
        ({'scan_launches': 2, 'build_launches': 12, 'probe_launches': 4, 'filter_launches': 4, 'other_launches': 5, 'kernel_launches': 39, 'rows_scanned': 2, 'rows_built': 4, 'rows_probed': 8, 'rows_out': 2, 'h2d_bytes': 24, 'd2h_bytes': 622592}, {'base_removed': 0, 'base_added': 2, 'overdeleted': 0, 'rederived': 0, 'inferred_removed': 0, 'inferred_added': 3, 'derivations': 3, 'overdelete_rounds': 0, 'insert_rounds': 2}),
        ({'scan_launches': 2, 'build_launches': 14, 'probe_launches': 6, 'filter_launches': 4, 'other_launches': 6, 'kernel_launches': 48, 'rows_scanned': 7, 'rows_built': 7, 'rows_probed': 19, 'rows_out': 2, 'h2d_bytes': 24, 'd2h_bytes': 720896}, {'base_removed': 0, 'base_added': 2, 'overdeleted': 0, 'rederived': 0, 'inferred_removed': 0, 'inferred_added': 5, 'derivations': 5, 'overdelete_rounds': 0, 'insert_rounds': 3}),
    ],
    "maintain_add_inferred_state1": [
        ({'scan_launches': 1, 'build_launches': 5, 'probe_launches': 3, 'other_launches': 2, 'kernel_launches': 19, 'rows_scanned': 2, 'rows_built': 3, 'rows_probed': 4, 'rows_out': 3, 'd2h_bytes': 229376}, {'rounds': 2, 'inferred': 3, 'derivations': 3, 'round_new': [2, 1]}),
        ({'scan_launches': 2, 'build_launches': 12, 'probe_launches': 4, 'filter_launches': 4, 'other_launches': 5, 'kernel_launches': 39, 'rows_scanned': 5, 'rows_built': 5, 'rows_probed': 11, 'h2d_bytes': 24, 'd2h_bytes': 622592}, {'base_removed': 0, 'base_added': 2, 'overdeleted': 0, 'rederived': 0, 'inferred_removed': 0, 'inferred_added': 3, 'derivations': 3, 'overdelete_rounds': 0, 'insert_rounds': 2}),
        ({'build_launches': 3, 'filter_launches': 4, 'other_launches': 3, 'kernel_launches': 10, 'rows_out': -3, 'h2d_bytes': 12, 'd2h_bytes': 262144}, {'base_removed': 0, 'base_added': 1, 'overdeleted': 0, 'rederived': 0, 'inferred_removed': 1, 'inferred_added': 0, 'derivations': 0, 'overdelete_rounds': 0, 'insert_rounds': 0}),
    ],
    "maintain_add_inferred_state0": [
        ({'scan_launches': 1, 'build_launches': 5, 'probe_launches': 3, 'other_launches': 2, 'kernel_launches': 19, 'rows_scanned': 2, 'rows_built': 3, 'rows_probed': 4, 'rows_out': 3, 'd2h_bytes': 229376}, {'rounds': 2, 'inferred': 3, 'derivations': 3, 'round_new': [2, 1]}),
        ({'scan_launches': 2, 'build_launches': 12, 'probe_launches': 4, 'filter_launches': 4, 'other_launches': 5, 'kernel_launches': 39, 'rows_scanned': 5, 'rows_built': 5, 'rows_probed': 11, 'h2d_bytes': 24, 'd2h_bytes': 622592}, {'base_removed': 0, 'base_added': 2, 'overdeleted': 0, 'rederived': 0, 'inferred_removed': 0, 'inferred_added': 3, 'derivations': 3, 'overdelete_rounds': 0, 'insert_rounds': 2}),
        ({'scan_launches': 2, 'build_launches': 6, 'filter_launches': 4, 'other_launches': 3, 'kernel_launches': 15, 'rows_scanned': 10, 'rows_out': -3, 'h2d_bytes': 12, 'd2h_bytes': 360448}, {'base_removed': 0, 'base_added': 1, 'overdeleted': 0, 'rederived': 0, 'inferred_removed': 1, 'inferred_added': 0, 'derivations': 0, 'overdelete_rounds': 0, 'insert_rounds': 0}),
    ],
    "maintain_diamond_state1": [
        ({'scan_launches': 1, 'build_launches': 5, 'probe_launches': 3, 'other_launches': 2, 'kernel_launches': 19, 'rows_scanned': 4, 'rows_built': 5, 'rows_probed': 8, 'rows_out': 5, 'd2h_bytes': 229376}, {'rounds': 2, 'inferred': 5, 'derivations': 6, 'round_new': [4, 1]}),
        ({'scan_launches': 2, 'build_launches': 12, 'probe_launches': 4, 'filter_launches': 4, 'other_launches': 5, 'kernel_launches': 39, 'rows_scanned': 9, 'rows_built': 5, 'rows_probed': 17, 'rows_out': -2, 'h2d_bytes': 24, 'd2h_bytes': 622592}, {'base_removed': 0, 'base_added': 2, 'overdeleted': 0, 'rederived': 0, 'inferred_removed': 0, 'inferred_added': 3, 'derivations': 3, 'overdelete_rounds': 0, 'insert_rounds': 2}),
        ({'scan_launches': 1, 'build_launches': 14, 'probe_launches': 8, 'filter_launches': 4, 'other_launches': 5, 'kernel_launches': 48, 'rows_scanned': 1, 'rows_built': 10, 'rows_probed': 35, 'rows_out': -3, 'd2h_bytes': 688128}, {'base_removed': 1, 'base_added': 0, 'overdeleted': 2, 'rederived': 1, 'inferred_removed': 1, 'inferred_added': 0, 'derivations': 3, 'overdelete_rounds': 1, 'insert_rounds': 0}),
    ],
    "maintain_diamond_state0": [
        ({'scan_launches': 1, 'build_launches': 5, 'probe_launches': 3, 'other_launches': 2, 'kernel_launches': 19, 'rows_scanned': 4, 'rows_built': 5, 'rows_probed': 8, 'rows_out': 5, 'd2h_bytes': 229376}, {'rounds': 2, 'inferred': 5, 'derivations': 6, 'round_new': [4, 1]}),
        ({'scan_launches': 2, 'build_launches': 12, 'probe_launches': 4, 'filter_launches': 4, 'other_launches': 5, 'kernel_launches': 39, 'rows_scanned': 9, 'rows_built': 5, 'rows_probed': 17, 'rows_out': -2, 'h2d_bytes': 24, 'd2h_bytes': 622592}, {'base_removed': 0, 'base_added': 2, 'overdeleted': 0, 'rederived': 0, 'inferred_removed': 0, 'inferred_added': 3, 'derivations': 3, 'overdelete_rounds': 0, 'insert_rounds': 2}),
        ({'scan_launches': 3, 'build_launches': 17, 'probe_launches': 8, 'filter_launches': 4, 'other_launches': 5, 'kernel_launches': 53, 'rows_scanned': 15, 'rows_built': 10, 'rows_probed': 35, 'rows_out': -3, 'd2h_bytes': 786432}, {'base_removed': 1, 'base_added': 0, 'overdeleted': 2, 'rederived': 1, 'inferred_removed': 1, 'inferred_added': 0, 'derivations': 3, 'overdelete_rounds': 1, 'insert_rounds': 0}),
    ],
    "repairs": [
        ({'scan_launches': 3, 'build_launches': 6, 'probe_launches': 2, 'other_launches': 2, 'kernel_launches': 13, 'rows_scanned': 18, 'rows_built': 3, 'rows_probed': 6, 'rows_out': 1, 'd2h_bytes': 262144, 'fused_scan_builds': 1}, {'constraints': 2, 'subsets_probed': 0, 'matches': 2, 'conflicts': 2, 'minimal_conflicts': 2, 'conflicted_facts': 4, 'answers': 1}),
    ],
    "refusals": [({}, {}), ({}, {}), ({}, {}), ({}, {}), ({}, {}), ({}, {}), ({}, {}), ({}, {})],
}


@pytest.fixture
def make_ctx(monkeypatch):
    """a fresh context, created after the route switches are set (they are read when a context is created)"""
    made = []

    def make(**env):
        for k, v in {**DEFAULT_ENV, **env}.items():
            monkeypatch.setenv(k, v)
        cx = c.Context(0)
        made.append(cx)
        return cx

    yield make
    for cx in made:
        cx.close()


def returned(st):
    """every field of a returned stats struct except device time (round_new: the rounds' entries)"""
    out = {}
    for name, _ in st._fields_:
        if name.endswith("_ms"):
            continue
        v = getattr(st, name)
        out[name] = [int(x) for x in v[: min(st.rounds, 64)]] if name == "round_new" else int(v)
    return out


def fingerprint(cx, call):
    """(what call() returns, its fingerprint); call() returns (result, stats struct or None)"""
    a = cx.get_stats()
    out, st = call()
    b = cx.get_stats()
    return out, ({f: b[f] - a[f] for f in FIELDS if b[f] != a[f]}, returned(st) if st is not None else {})


def twice(name, make_ctx, run):
    """run(cx, fp) on two fresh contexts; fp(call) fingerprints one call. Both runs' fingerprints must equal ROUTES[name]."""
    for rep in range(2):
        fps = []

        def fp(call):
            out, f = fingerprint(cx, call)
            fps.append(f)
            return out
        cx = make_ctx()
        run(cx, fp)
        cx.close()
        assert fps == ROUTES.get(name), f"{name} run {rep + 1}: {fps!r}"


def rel_rows(rel):
    return rel.to_numpy([0, 1, 2]) if rel.n_rows else np.empty((0, 3), np.uint32)


def assert_blocks(p, what):
    """the p column is runs of one predicate each, in ascending predicate order"""
    assert np.all(np.diff(p.astype(np.int64)) >= 0), f"{what}: predicate blocks out of order"


# ---- kb_datalog_fixpoint
def fixpoint_call(cx, fp, rules, strategy, want_oracle, what):
    rel, st = fp(lambda: (lambda r: (r, r[1]))(cx.datalog_fixpoint(rules, strategy)))
    got = rel_rows(rel)
    H.assert_same_bag(got, want_oracle["facts"], what)
    assert_blocks(got[:, 1], what)
    assert st.rounds == len(want_oracle["round_new"]) and st.inferred == len(got)
    assert [int(x) for x in st.round_new[: st.rounds]] == [int(x) for x in want_oracle["round_new"]]
    if strategy != c.SEMI_NAIVE_OLD_DELTA:
        assert st.derivations == want_oracle["derivations"], what
    return st


def oracle_strategy(strategy):
    return c.SEMI_NAIVE if strategy == c.SEMI_NAIVE_OLD_DELTA else strategy


@pytest.mark.parametrize("strategy", list(STRATEGIES))
@pytest.mark.parametrize("case", FC, ids=[x["name"] for x in FC])
def test_fixpoint_fc(make_ctx, case, strategy):
    d, facts, rules = H.build_fc_case(case)
    kr = [compile_rule(x) for x in rules]
    s = STRATEGIES[strategy]
    want = O.Db(facts[:, 0], facts[:, 1], facts[:, 2], *d.numeric_table()).fixpoint(kr, oracle_strategy(s))
    assert want["status"] == 0

    def run(cx, fp):
        cx.dict_numeric_load(*d.numeric_table())
        cx.store_load(facts[:, 0], facts[:, 1], facts[:, 2])
        fixpoint_call(cx, fp, kr, s, want, case["name"])
    twice(f"{case['name']}_{strategy}", make_ctx, run)


@pytest.mark.parametrize("strategy", list(STRATEGIES))
def test_fixpoint_taxonomy(make_ctx, strategy):
    t = datagen.taxonomy_dataset(fanout=4, depth=4, n_instances=5000)
    rules = datagen.taxonomy_rules(t)
    s = STRATEGIES[strategy]
    want = O.Db(t.s, t.p, t.o).fixpoint(rules, oracle_strategy(s))

    def run(cx, fp):
        cx.store_load(t.s, t.p, t.o)
        fixpoint_call(cx, fp, rules, s, want, "taxonomy")
    twice(f"taxonomy_{strategy}", make_ctx, run)


def test_fixpoint_known_fact_set_grows_mid_launch(make_ctx):
    """a head predicate with no fact and 4 M new facts from one launch: the launch stops at its budget, the set is rebuilt larger and the
    launch repeated"""
    n = 4_000_000
    s = np.arange(10, 10 + n, dtype=np.uint32)
    o = (s * np.uint32(7) + np.uint32(3)) % np.uint32(1 << 22) + np.uint32(10)
    p = np.full(n, 5, np.uint32)
    rule = {"premise": [c.pattern(c.V(0), c.K(5), c.V(1))], "conclusion": [c.pattern(c.V(1), c.K(6), c.V(0))], "filters": []}
    want = {"facts": np.stack([o, np.full(n, 6, np.uint32), s], axis=1), "round_new": [n], "derivations": n}

    def run(cx, fp):
        cx.store_load(s, p, o)
        fixpoint_call(cx, fp, [rule], c.SEMI_NAIVE, want, "grows mid-launch")
    twice("grows_mid_launch", make_ctx, run)


@pytest.mark.parametrize("strategy", ["semi_naive", "naive"])
def test_fixpoint_partitioned_dedup(make_ctx, strategy):
    t = datagen.taxonomy_dataset(fanout=3, depth=5, n_instances=5000)
    rules = datagen.taxonomy_rules(t)
    s = STRATEGIES[strategy]
    want = O.Db(t.s, t.p, t.o).fixpoint(rules, s)
    env = {"KOLIBRIE_DERIVE_PART": "1", "KOLIBRIE_DERIVE_SLICE": "2048", "KOLIBRIE_DERIVE_MIN_ROWS": "16"}

    def run(cx, fp):
        cx.store_load(t.s, t.p, t.o)
        fixpoint_call(cx, fp, rules, s, want, "partitioned")
    twice(f"partitioned_{strategy}", lambda: make_ctx(**env), run)


# ---- kb_datalog_fixpoint_seed
@pytest.mark.parametrize("state", ["1", "0"])
def test_fixpoint_seed_twice(make_ctx, state):
    """a closed taxonomy store, then two seeded calls: each returns its accepted seed facts (the new ones; seed facts the closure holds
    and facts of predicates no rule mentions are dropped) followed by the facts inferred from them"""
    tax = datagen.taxonomy_dataset(fanout=3, depth=4, n_instances=3000)
    rules = datagen.taxonomy_rules(tax)
    typ, sub = tax.ids["rdf:type"], tax.ids["rdfs:subClassOf"]
    base = np.stack([tax.s, tax.p, tax.o], axis=1).astype(np.uint32)
    classes = np.unique(base[base[:, 1] == sub][:, 2])
    rng = np.random.default_rng(21)
    seeds = []
    for k in range(2):
        fresh = np.stack([np.arange(10**6 + 1000 * k, 10**6 + 1000 * k + 300), np.full(300, typ), rng.choice(classes, 300)], axis=1)
        again = base[rng.choice(len(base), 50)]  # facts the store holds already
        other = np.stack([np.arange(40), np.full(40, 999_999), np.arange(40)], axis=1)  # a predicate no rule mentions
        seeds.append(np.concatenate([fresh, again, other]).astype(np.uint32))
    kept = [x[np.isin(x[:, 1], [typ, sub])] for x in seeds]
    closures = [rows_set(base)]
    for k in range(3):
        rows = np.concatenate([base] + kept[:k])
        st, inf = SC.closure_of(rows, rules)
        assert st == 0
        closures.append(rows_set(rows) | rows_set(inf))

    def run(cx, fp):
        cx.store_load(tax.s, tax.p, tax.o)
        fp(lambda: (lambda r: (r, r[1]))(cx.datalog_fixpoint(rules)))
        for k in range(2):
            seed = seeds[k]
            sr = cx.rel_from_host([0, 1, 2], [seed[:, 0], seed[:, 1], seed[:, 2]])
            rel, n_new, st = fp(lambda: (lambda r: (r, r[2]))(cx.datalog_fixpoint_seed(rules, sr)))
            got = rel_rows(rel)
            want = closures[k + 2] - closures[k + 1]
            H.assert_same_bag(got, as_rows(want), f"seed {k}")
            accepted = rows_set(seed) & want
            assert n_new == len(accepted) and rows_set(got[:n_new]) == accepted
            assert_blocks(got[:n_new, 1], f"seed {k}: seed facts")
            assert_blocks(got[n_new:, 1], f"seed {k}: inferred facts")
            assert st.inferred == len(got) - n_new
    twice(f"seed_state{state}", lambda: make_ctx(KOLIBRIE_FIX_STATE=state), run)


# ---- kb_datalog_query
def anc_rules():
    parent, anc = Constant(200), Constant(201)
    X, Y, Z = Variable("X"), Variable("Y"), Variable("Z")
    return [([(X, parent, Y)], [(X, anc, Y)]), ([(X, parent, Y), (Y, anc, Z)], [(X, anc, Z)])]


QUERIES = {
    "variable_predicate": ((Variable("S"), Variable("P"), Variable("O")), 10),
    "open_subject": ((Variable("S"), Constant(201), Constant(7)), 10),
    "ground_stops_early": ((Constant(0), Constant(201), Constant(3)), 10),
    "depth_bound": ((Constant(0), Constant(201), Variable("A")), 3),
}


@pytest.mark.parametrize("case", list(QUERIES))
def test_query(make_ctx, case):
    facts = [(i, 200, i + 1) for i in range(12)] + [(40, 300, 41), (41, 200, 42)]
    rules = anc_rules()
    query, depth = QUERIES[case]
    kr, kq = bc_to_kb(rules, query)
    want = B.device_answers(facts, rules, query, depth)
    a = np.array(facts, np.uint32)

    def run(cx, fp):
        cx.store_load(a[:, 0], a[:, 1], a[:, 2])
        cx.store_append(a[:, 0], a[:, 1], a[:, 2], 1)  # the same triples again: stored duplicates across segments
        rel, st = fp(lambda: (lambda r: (r, r[1]))(cx.datalog_query(kr, kq, depth)))
        n, slots = rel.info()
        rows = rel.to_numpy() if slots else np.zeros((n, 0), np.uint32)
        got = [tuple(int(x) for x in r) for r in rows]
        assert len(got) == len(set(got)) and set(got) == want, case
        assert st.answers == n
        if case == "ground_stops_early":
            assert st.stopped_early and st.rounds == 3
        if case == "depth_bound":
            assert st.rounds == 3 and not st.reached_fixpoint
    twice(f"query_{case}", make_ctx, run)


# ---- kb_datalog_maintain
PAR, ANC = 1, 2
ANCESTOR = [{"premise": [c.pattern(c.V(0), c.K(PAR), c.V(1))], "conclusion": [c.pattern(c.V(0), c.K(ANC), c.V(1))], "filters": []},
            {"premise": [c.pattern(c.V(0), c.K(PAR), c.V(1)), c.pattern(c.V(1), c.K(ANC), c.V(2))],
             "conclusion": [c.pattern(c.V(0), c.K(ANC), c.V(2))], "filters": []}]
A_, B_, C_, D_ = 10, 11, 12, 13
# name -> (segments {tag: rows}, evicted tags, added rows or None); every case first adds the unrelated segment 50 (its kept state)
MAINTAIN = {
    "no_op": ({1: [[A_, PAR, B_], [B_, PAR, C_]]}, [], None),
    "evict_only": ({1: [[A_, PAR, B_]], 2: [[B_, PAR, C_], [C_, PAR, D_]]}, [1], None),
    "add_only": ({1: [[A_, PAR, B_]]}, [], [[B_, PAR, C_], [C_, PAR, D_]]),
    "add_inferred": ({1: [[A_, PAR, B_], [B_, PAR, C_]]}, [], [[A_, ANC, C_]]),
    "diamond": ({1: [[A_, PAR, B_]], 2: [[A_, PAR, C_], [B_, PAR, D_], [C_, PAR, D_]]}, [1], None),
}
PRIME = [[30, PAR, 31], [31, PAR, 32]]


def closure_rows(segs):
    base = set().union(*[rows_set(np.array(r, np.uint32).reshape(-1, 3)) for r in segs.values()])
    st, inf = SC.closure_of(as_rows(base), ANCESTOR)
    assert st == 0
    return base, rows_set(inf) - base


@pytest.mark.parametrize("state", ["1", "0"])
@pytest.mark.parametrize("case", list(MAINTAIN))
def test_maintain(make_ctx, case, state):
    segs0, evict, add = MAINTAIN[case]

    def maintain(cx, fp, segs, evict, add, tag):
        _, before = closure_rows(segs)
        after_segs = {t: r for t, r in segs.items() if t not in evict}
        if add is not None:
            after_segs[tag] = add
        a = None if add is None else np.array(add, np.uint32).reshape(-1, 3)
        gone, new, st = fp(lambda: (lambda r: (r, r[2]))(cx.datalog_maintain(ANCESTOR, evict, a, tag)))
        _, after = closure_rows(after_segs)
        g, n = rel_rows(gone), rel_rows(new)
        assert len(rows_set(g)) == len(g) and rows_set(g) == before - after, case
        assert len(rows_set(n)) == len(n) and rows_set(n) == after - before, case
        assert st.inferred_removed == len(g) and st.inferred_added == len(n)
        s, p, o = cx.store_download()
        live = np.concatenate([np.array(r, np.uint32).reshape(-1, 3) for r in after_segs.values()] + [as_rows(after)])
        H.assert_same_bag(np.stack([s, p, o], axis=1), live, f"{case}: store")
        return after_segs

    def run(cx, fp):
        for t, r in segs0.items():
            r = np.array(r, np.uint32)
            cx.store_append(r[:, 0], r[:, 1], r[:, 2], t)
        rel, _ = fp(lambda: (lambda r: (r, r[1]))(cx.datalog_fixpoint(ANCESTOR)))
        assert rows_set(rel_rows(rel)) == closure_rows(segs0)[1]
        segs = maintain(cx, fp, segs0, [], PRIME, 50)
        maintain(cx, fp, segs, evict, add, 7)
    twice(f"maintain_{case}_state{state}", lambda: make_ctx(KOLIBRIE_FIX_STATE=state), run)


# ---- kb_datalog_query_repairs
def test_query_repairs(make_ctx):
    facts = [(1, 10, 2), (1, 11, 2), (3, 10, 4), (4, 12, 5), (5, 10, 6), (5, 11, 7)]
    constraints = [[("?A", 10, "?B"), ("?A", 11, "?B")], [("?A", 12, "?B"), ("?B", 10, "?C")]]
    query = ("?S", 10, "?O")
    kc, kq = repairs_to_kb(constraints, query)
    want = R.iar(facts, constraints, query)
    a = np.array(facts, np.uint32)

    def run(cx, fp):
        cx.store_load(a[:, 0], a[:, 1], a[:, 2])
        rel, st = fp(lambda: (lambda r: (r, r[1]))(cx.datalog_query_repairs(kc, kq)))
        got = [tuple(int(x) for x in r) for r in rel.to_numpy()]
        assert len(got) == len(set(got)) and set(got) == want
        s = R.stats(facts, constraints)
        assert {k: getattr(st, k) for k in s} == s
    twice("repairs", make_ctx, run)


# ---- refusals: the status code, and what the refused call cost
def refused(call, status):
    def f():
        with pytest.raises(c.KolibrieError) as e:
            call()
        assert e.value.status == status, e.value
        return status, None
    return f


def test_refusals(make_ctx):
    def run(cx, fp):
        r = np.array([[1, PAR, 2], [2, PAR, 3]], np.uint32)
        cx.store_append(r[:, 0], r[:, 1], r[:, 2], 1)
        fp(refused(lambda: cx.datalog_fixpoint(ANCESTOR, 9), c.KB_E_INVALID))
        two = cx.rel_from_host([0, 1], [r[:, 0], r[:, 1]])
        fp(refused(lambda: cx.datalog_fixpoint_seed(ANCESTOR, two), c.KB_E_INVALID))
        fp(refused(lambda: cx.datalog_query(ANCESTOR, c.pattern(c.K(1), c.K(ANC), c.V(5)), 65), c.KB_E_LIMIT))
        fp(refused(lambda: cx.datalog_maintain(ANCESTOR, [1]), c.KB_E_INVALID))  # not closed yet
        cx.datalog_fixpoint(ANCESTOR)
        fp(refused(lambda: cx.datalog_maintain(ANCESTOR, [77]), c.KB_E_NOT_FOUND))
        fp(refused(lambda: cx.datalog_maintain(ANCESTOR, [1], strategy=9), c.KB_E_INVALID))
        fp(refused(lambda: cx.datalog_maintain(ANCESTOR, [1], strategy=c.SEMI_NAIVE_PARALLEL), c.KB_E_UNSUPPORTED))
        fp(refused(lambda: cx.datalog_maintain(ANCESTOR[:1], [1]), c.KB_E_INVALID))  # other rules
        s, p, o = cx.store_download()
        H.assert_same_bag(np.stack([s, p, o], axis=1), np.array([[1, PAR, 2], [2, PAR, 3], [1, ANC, 2], [2, ANC, 3], [1, ANC, 3]], np.uint32),
                          "store after the refusals")
    twice("refusals", make_ctx, run)
