"""The inverted-file rule of tests/_search_ivf.py checked against itself on exact data, and shown to reject an unstable layout,
ties broken by stored position, ties between lists broken by the higher list index, and unnormalised centroids."""
import numpy as np

import _search_ivf as rule


def _exact(rng, n, dim):
    """integers in [-4, 4] times 2^-3: exact in f16 and bf16, every dot product exact in fp64"""
    return rng.integers(-4, 5, (n, dim)) * 2.0 ** -3


def _index(seed=1, n=600, dim=8, n_lists=12):
    rng = np.random.default_rng(seed)
    db = _exact(rng, n, dim)
    cent = rule.train(db, n_lists, 3, False)
    return rng, db, cent, rule.exact_assign(db, cent)


def test_layout_is_list_major_and_stable():
    _, db, cent, lists = _index()
    off, ids = rule.layout(lists, len(cent))
    assert off[0] == 0 and off[-1] == len(db) and (np.diff(off) >= 0).all()
    for l in range(len(cent)):
        mem = ids[off[l]:off[l + 1]]
        assert (lists[mem] == l).all() and (np.diff(mem) > 0).all()
    # an unstable layout (each list's rows reversed) holds the same lists but is not the rule's
    bad = np.concatenate([ids[off[l]:off[l + 1]][::-1] for l in range(len(cent))])
    assert not np.array_equal(bad, ids)


def test_full_probe_is_the_flat_search():
    rng, db, cent, lists = _index()
    q = _exact(rng, 40, 8)
    for k in (1, 10, 600, 1000):
        s, i = rule.search(q, db, lists, rule.probes(q, cent, len(cent)), k)
        flat = q @ db.T
        order = np.argsort(-flat, axis=1, kind="stable")[:, :min(k, len(db))]
        assert np.array_equal(i, order) and np.array_equal(s, np.take_along_axis(flat, order, 1))


def test_partial_probe_pads_and_ranks_by_original_index():
    rng, db, cent, lists = _index()
    q = _exact(rng, 20, 8)
    probe = rule.probes(q, cent, 2)
    s, i = rule.search(q, db, lists, probe, 1024)
    for r in range(len(q)):
        n_in = np.isin(lists, probe[r]).sum()
        assert (i[r, n_in:] == -1).all() and np.isneginf(s[r, n_in:]).all()
        assert np.isin(lists[i[r, :n_in]], probe[r]).all()
        tie = s[r, 1:n_in] == s[r, :n_in - 1]
        assert (i[r, 1:n_in][tie] > i[r, :n_in - 1][tie]).all()


def test_ties_are_broken_by_original_index_not_stored_position():
    # rows 0 and 1 score alike; row 0 is in list 1 and row 1 in list 0, so stored position puts row 1 first
    db = np.array([[1.0, 0.5], [1.0, -0.5], [-1.0, 0.0]]) * 0.5
    cent = np.array([[0.0, -1.0], [0.0, 1.0]])
    lists = rule.exact_assign(db, cent)
    assert list(lists[:2]) == [1, 0]
    q = np.array([[1.0, 0.0]])
    s, i = rule.search(q, db, lists, rule.probes(q, cent, 2), 2)
    assert list(i[0]) == [0, 1] and s[0, 0] == s[0, 1]
    off, ids = rule.layout(lists, 2)
    by_position = ids[np.argsort(-(db[ids] @ q[0]), kind="stable")][:2]
    assert list(by_position) == [1, 0], "the stored-position order would differ"


def test_ties_between_lists_go_to_the_lower_list():
    cent = np.array([[1.0, 0.0], [1.0, 0.0], [0.0, 1.0]])     # lists 0 and 1 tie for every row near x
    db = np.array([[1.0, 0.25], [0.5, -0.25]])
    assert list(rule.exact_assign(db, cent)) == [0, 0]
    higher = np.argmax((db @ cent.T)[:, ::-1], axis=1)
    assert list(len(cent) - 1 - higher) == [1, 1], "a higher-index tie rule assigns differently"
    assert list(rule.probes(np.array([[1.0, 0.0]]), cent, 1)[0]) == [0]


def test_update_normalises_and_keeps_empty_lists():
    rng = np.random.default_rng(3)
    x = _exact(rng, 300, 8)
    cent0 = rule.init(x, 6)
    cent0[5] = [0.5, 0, 0, 0, 0, 0, 0, 0]                # a centroid no row can prefer once others exist
    lists = rule.exact_assign(x, cent0)
    lists[lists == 5] = 0
    for bf in (False, True):
        cent = rule.update(x, lists, cent0, bf)
        assert np.array_equal(cent[5], cent0[5]), "an empty list keeps its centroid"
        for l in range(5):
            m = x[lists == l].mean(0)
            want = rule.round16(m / np.sqrt((m * m).sum()), bf)
            assert np.array_equal(cent[l], want)
            assert abs(np.linalg.norm(cent[l]) - 1) < 2.0 ** -6
            assert not np.array_equal(cent[l], rule.round16(m, bf)), "unnormalised centroids are not the rule's"


def test_train_is_deterministic_and_round16_is_single_rounding():
    rng = np.random.default_rng(5)
    x = _exact(rng, 200, 16)
    a, b = rule.train(x, 7, 4, True), rule.train(x, 7, 4, True)
    assert np.array_equal(a, b)
    # 1 + 2^-8 + 2^-40 lies just above the bf16 midpoint: one rounding goes up, a detour through f32 would tie to even
    v = 1 + 2.0 ** -8 + 2.0 ** -40
    assert rule.rne_bf16(v) == 1 + 2.0 ** -7
    assert rule.rne_bf16(1 + 2.0 ** -8) == 1.0
    assert rule.round16(1 + 2.0 ** -11 + 2.0 ** -40, False) == 1 + 2.0 ** -10
