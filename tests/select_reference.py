"""Feature selection of the Estimator (GLIO/src/Estimator.cpp:3894-4116) restated in plain Python, with the seeded sampler the
device uses in place of the reference's std::random_device / std::shuffle draws.

Philox4x64-10 is written out in Python integers (checked against numpy.random.Philox by tests/test_select.py).  The three
functions below follow the reference as written: the window pool is a list that loses the chosen element after every draw
(PCL's ExtractIndices with setNegative keeps the order), the thresholds and R' / BR' clamps are the reference's, a failed
start/end pair `return`s (every later pair of that keyframe keeps all its matches) while the incremental one `continue`s.
Where the reference reads `rand_ids[R'-1]` / `rand_ids[i]` these take the sampler's draw j:

    r_j = mulhi64(u_j, n - 1 - j)          u_j = word j of the (seed, domain, stream, nonce) Philox segment
    index = the r_j-th (0-based) value of 0 .. n-2 not chosen yet, ascending

`undefined` is set for the two sizes where the reference reads out of bounds (window n = F + 1 with R' = 0, start/end
BR' < B); the sampler's result is given there as well.
"""

M64 = (1 << 64) - 1
PHILOX_M0, PHILOX_M1 = 0xD2E7470EE14C6C93, 0xCA5A826395121157
PHILOX_W0, PHILOX_W1 = 0x9E3779B97F4A7C15, 0xBB67AE8584CAA73B

DOMAIN_WINDOW, DOMAIN_BATCH_STARTEND, DOMAIN_BATCH_ADD = 0, 1, 2


def philox4x64_10(ctr, key):
    """Random123's philox4x64_R(10, ctr, key): four 64-bit words."""
    c0, c1, c2, c3 = ctr
    k0, k1 = key
    for r in range(10):
        if r:
            k0 = (k0 + PHILOX_W0) & M64
            k1 = (k1 + PHILOX_W1) & M64
        p0 = PHILOX_M0 * c0
        p1 = PHILOX_M1 * c2
        c0, c1, c2, c3 = ((p1 >> 64) ^ c1 ^ k0) & M64, p1 & M64, ((p0 >> 64) ^ c3 ^ k1) & M64, p0 & M64
    return c0, c1, c2, c3


def words(seed, domain, stream, nonce, count):
    """u_0 .. u_{count-1}: word j is word j % 4 of the block at counter (j // 4 + 1, stream, nonce, 0), key (seed, domain) --
    numpy.random.Philox(key=[seed, domain], counter=[0, stream, nonce, 0]).random_raw(count)."""
    out = []
    for b in range((count + 3) // 4):
        out.extend(philox4x64_10((b + 1, int(stream) & M64, int(nonce) & M64, 0), (int(seed) & M64, int(domain) & M64)))
    return out[:count]


def draws(seed, domain, stream, nonce, n, k):
    """r_0 .. r_{k-1}, r_j = floor(u_j * (n - 1 - j) / 2^64): uniform in [0, n-1-j) up to a bias below 2^-33 for n < 2^31."""
    n = int(n)
    u = words(seed, domain, stream, nonce, k)
    return [(u[j] * (n - 1 - j)) >> 64 for j in range(k)]


def sample_from_draws(n, r):
    """The ordered sample of 0 .. n-2 the draws r define (rank among the values not chosen yet)."""
    pool = list(range(n - 1))
    return [pool.pop(rj) for rj in r]


def stream_of_pair(cur, oth):
    return ((cur & 0xFFFFFFFF) << 32) | (oth & 0xFFFFFFFF)


def window_select(n, stream, seed, nonce, F=100, R=300, random_select=True):
    """featureSelection (Estimator.cpp:3894-3992) for a slot of n matches.  Returns (keep, undefined): keep None = all n matches
    stay active, else the kept match indices in draw order (empty when random_select is off)."""
    n = int(n)
    if n < 1 or n - 1 < F:
        return None, False
    Rp = min(R, n - 1)
    if n - F < Rp:
        Rp = n - F - 1
    undefined = random_select and Rp < 1          # selected_id stays -1: points[-1]
    r = draws(seed, DOMAIN_WINDOW, stream, nonce, n, F) if random_select else []
    pool = list(range(n))                          # vec_surf_cur_pts[idVec], as original match indices
    kept = []
    j = 0
    while len(kept) < F and random_select:
        selected = r[j]                            # rand_ids[R' - 1] of a shuffle of 0 .. len(pool) - 2
        kept.append(pool[selected])
        del pool[selected]                         # ExtractIndices::setNegative(true): order kept
        j += 1
    return kept, undefined


def batch_select(pairs, n_match, mode, seed, nonce, B=25, BR=400):
    """globalFeatureSelection_Batch (mode 0, :3994-4055) / globalFeatureSelectionAdd_Batch (mode 1, :4057-4116) over a pair
    list grouped by cur.  pairs[i] = (cur, oth), n_match[i] its match count; the reference visits the pairs of one idx in
    ascending search_idx, here in list order.  Returns [(keep or None, undefined)] per pair."""
    out = [None] * len(pairs)
    stopped = None                                 # the cur whose start/end loop has `return`ed
    for i, ((cur, oth), n) in enumerate(zip(pairs, n_match)):
        cur, oth, n = int(cur), int(oth), int(n)
        if mode == 0:
            if stopped == cur:
                out[i] = (None, False)
                continue
            if n - 1 < B or n < 50:
                stopped = cur                      # return: this pair and the rest of this idx keep all their matches
                out[i] = (None, False)
                continue
            BRp = min(BR, n - 1)
            if n - B < BRp:
                BRp = n - B - 1
            undefined = BRp < B                    # rand_ids[i] read past its BR' entries
            dom = DOMAIN_BATCH_STARTEND
        else:
            if n <= B:
                out[i] = (None, False)             # continue
                continue
            undefined = False
            dom = DOMAIN_BATCH_ADD
        r = draws(seed, dom, stream_of_pair(cur, oth), nonce, n, B)
        out[i] = (sample_from_draws(n, r), undefined)   # rand_ids[0 .. B) of a shuffle of 0 .. n-2
    return out
