"""The contract of popsift_b200_tracks.h restated with numpy / scipy: connected components of the edges over all features
(scipy.sparse.csgraph), the fork rule (two features of one set drop the component), the length rule, and the output order
(tracks by smallest member, members ascending).  Returns the arrays the C ABI writes."""
import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components


def offsets(n_feat):
    return np.concatenate([[0], np.cumsum(np.asarray(n_feat, np.int64))]).astype(np.int64)


def tracks(n_feat, edges, min_length=2):
    """edges: (E, 2) global ids.  Returns (track_of (N,), track_start (T + 1,), members (M,), counts dict)."""
    off = offsets(n_feat)
    N = int(off[-1])
    e = np.asarray(edges, np.int64).reshape(-1, 2)
    e = e[e[:, 0] != e[:, 1]]
    g = coo_matrix((np.ones(len(e), np.int8), (e[:, 0], e[:, 1])), shape=(N, N))
    _, lab = connected_components(g, directed=True, connection="weak")
    size = np.bincount(lab, minlength=lab.max() + 1 if N else 0)
    active = np.nonzero(size[lab] >= 2)[0] if N else np.zeros(0, np.int64)
    st = np.searchsorted(off, active, side="right") - 1
    # (label, gid) order; a label's first gid is its smallest member
    order = np.lexsort((active, lab[active]))
    a, la, sa = active[order], lab[active][order], st[order]
    heads = np.nonzero(np.r_[True, la[1:] != la[:-1]])[0] if len(a) else np.zeros(0, np.int64)
    lens = np.r_[heads[1:], len(a)] - heads
    fork = np.zeros(len(a), np.int64)
    if len(a) > 1:
        fork[1:] = (la[1:] == la[:-1]) & (sa[1:] == sa[:-1])
    conf = np.add.reduceat(fork, heads) > 0 if len(a) else np.zeros(0, bool)
    short = ~conf & (lens < min_length)
    keep = ~conf & ~short
    # kept segments by their smallest member (their first entry)
    kh, kl = heads[keep], lens[keep]
    o = np.argsort(a[kh], kind="stable")
    kh, kl = kh[o], kl[o]
    start = np.concatenate([[0], np.cumsum(kl)]).astype(np.int32)
    idx = np.repeat(kh - start[:-1], kl) + np.arange(int(start[-1]))
    members = a[idx].astype(np.int32)
    track_of = np.full(N, -1, np.int32)
    track_of[members] = np.repeat(np.arange(len(kh), dtype=np.int32), kl)
    counts = dict(n_tracks=len(kh), n_members=int(start[-1]), n_components=len(heads), n_conflicting=int(conf.sum()),
                  n_short=int(short.sum()))
    return track_of, start, members, counts


def chain_edges(pairs, n_desc, n_feat, match, src, n_corr, mask, rev):
    """The edges ps_tracks_from_matches derives from the chain's arrays (host copies): per pair p = (l, r) and row
    k < start_p + n_corr[p] with mask[k] != 0 (mask None: every row), (off[l] + rev[l][i], off[r] + rev[r][b]) with
    i = src[k], b = match[start_p + i, 0]."""
    off = offsets(n_feat)
    out, start = [], 0
    for p, (l, r) in enumerate(pairs):
        ks = np.arange(start, start + int(n_corr[p]))
        if mask is not None:
            ks = ks[np.asarray(mask[ks]) != 0]
        i = np.asarray(src)[ks]
        b = np.asarray(match).reshape(-1, 3)[start + i, 0]
        out.append(np.stack([off[l] + np.asarray(rev[l])[i], off[r] + np.asarray(rev[r])[b]], axis=1))
        start += int(n_desc[l])
    return np.concatenate(out).astype(np.int64) if out else np.zeros((0, 2), np.int64)
