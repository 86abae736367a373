"""The edge selection (glio_select_random_edges, glio_batch_select_random_edges) restated on top of tests/select_reference.py: the
plane rules, unchanged, on edge counts, with the draws taken in Philox domain 3 (window), 4 (batch start/end) or 5 (batch
incremental).  `domain` may be given to check that these are the plane selections but for the domain."""
from tests import select_reference as sr

DOMAIN_WINDOW_EDGES, DOMAIN_BATCH_STARTEND_EDGES, DOMAIN_BATCH_ADD_EDGES = 3, 4, 5


def window_select(n, stream, seed, nonce, F=100, R=300, random_select=True, domain=DOMAIN_WINDOW_EDGES):
    """featureSelection's rule (select_reference.window_select) on a list of n records, the draws taken in `domain`."""
    keep, undefined = sr.window_select(n, stream, seed, nonce, F=F, R=R, random_select=random_select)
    if keep:
        keep = sr.sample_from_draws(int(n), sr.draws(seed, domain, stream, nonce, n, F))
    return keep, undefined


def batch_select(pairs, n, mode, seed, nonce, B=25, BR=400, domain=None):
    """the batch rules (select_reference.batch_select) on record counts n[i], the draws taken in `domain` (default: 4 for mode 0,
    5 for mode 1)."""
    if domain is None:
        domain = DOMAIN_BATCH_STARTEND_EDGES if mode == 0 else DOMAIN_BATCH_ADD_EDGES
    out = []
    for (cur, oth), cnt, (keep, undefined) in zip(pairs, n, sr.batch_select(pairs, n, mode, seed, nonce, B=B, BR=BR)):
        if keep is not None:
            keep = sr.sample_from_draws(int(cnt), sr.draws(seed, domain, sr.stream_of_pair(cur, oth), nonce, cnt, B))
        out.append((keep, undefined))
    return out
