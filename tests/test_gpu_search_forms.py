"""The search forms (clip_b200_zero_shot_batch, clip_b200_topk_search, clip_b200_topk_search_16, clip_b200_topk_search_i8) and the
row forms that make their databases (clip_b200_rows_to_16bit, clip_b200_rows_to_int8) run through one table, so that they check
their arguments alike.

  * Every fault is refused by every form it applies to, with a message that starts with the form's name.
  * A call with two faults reports the one the documented order (include/clip_b200.h) puts first, on every form.
  * An empty call returns true and writes nothing, unless a fault that comes before it in that order is present.
  * The fp32 forms keep their clamp: top_k <= 0 and top_k > n_db mean all rows, and top_k > 1024 is ranked on the host.
  * Each search form makes the number of kernel launches it made before the four searches shared one pass driver (LAUNCHES)."""
import ctypes as C

import numpy as np
import pytest

from _util import model_file

pytestmark = pytest.mark.gpu

F16, BF16 = 1, 2
TOO_MANY = 1 << 31
REGION = 8 << 20                              # bytes of device memory behind each pointer argument
GUARD = 64                                    # host output entries past n_q * top_k that a call must leave alone
FP, IP = C.POINTER(C.c_float), C.POINTER(C.c_int)


class Form:
    def __init__(self, name, n_ptr, search=True, knn=False, type_word=None, bad_dims=()):
        self.name, self.n_ptr, self.search, self.knn, self.type_word, self.bad_dims = name, n_ptr, search, knn, type_word, bad_dims
        self.fp32 = search and not knn                            # no alignment rule, no dim, the top_k clamp

    def __repr__(self):
        return self.name


FORMS = [
    Form("clip_b200_zero_shot_batch", 2),
    Form("clip_b200_topk_search", 2),
    Form("clip_b200_topk_search_16", 2, knn=True, type_word="in_type", bad_dims=(60, 0, 2056)),
    Form("clip_b200_topk_search_i8", 4, knn=True, bad_dims=(24, 0, 2064)),
    Form("clip_b200_rows_to_16bit", 2, search=False, type_word="out_type", bad_dims=(62, 0, 2052)),
    Form("clip_b200_rows_to_int8", 3, search=False, bad_dims=(24, 0, 2064)),
]
IDS = [f.name for f in FORMS]
BY_NAME = {f.name: f for f in FORMS}


def faults(f):
    """f's faults in the documented order: [(step, [(call arguments, a word of the message)])].  An empty call comes between
    "count" and "pointer"."""
    out = [("context", [(dict(ctx=False), "null context")])]
    if f.type_word:
        out.append(("type", [(dict(type_=t), f.type_word) for t in (0, 3)]))
    if f.bad_dims:
        out.append(("dim", [(dict(dim=d), "dim") for d in f.bad_dims]))
    if f.knn:
        out.append(("top_k", [(dict(top_k=k), "top_k") for k in (0, 1025)]))
    out.append(("count", [(dict(nq=TOO_MANY), "2^31")] + ([(dict(ndb=TOO_MANY), "2^31")] if f.search else [])))
    ptrs = [dict(null=(i,)) for i in range(f.n_ptr)]
    if not f.fp32:
        ptrs += [dict(shift={i: s}) for i in range(f.n_ptr) for s in (4, 8)]
    out.append(("pointer", [(kw, "null device pointer" if f.fp32 else "aligned") for kw in ptrs]))
    if f.search:
        out.append(("output", [(dict(out=o), "null output") for o in ((False, True), (True, False), (False, False))]))
    return out


class Env:
    """the tiny f16 model (projection dim 128: the fp32 forms' dim), n_ptr zeroed device regions and guarded host outputs"""

    def __init__(self, prod):
        self.prod, self.L = prod, prod.lib
        self.ctx = prod.load(model_file("tiny", "f16", prod), 0)
        self.d = self.L.clip_b200_device_malloc(self.ctx, 4 * REGION)
        zeros = np.zeros(4 * REGION, np.uint8)
        assert self.d and self.L.clip_b200_memcpy_h2d(self.ctx, self.d, zeros.ctypes.data, zeros.nbytes), prod.last_error()
        self.sc = np.zeros(200_000 + GUARD, np.float32)
        self.ix = np.zeros(200_000 + GUARD, np.int32)

    def close(self):
        self.L.clip_b200_device_free(self.ctx, self.d)
        self.prod.free(self.ctx)

    def call(self, f, ctx=True, nq=4, ndb=4, dim=64, type_=F16, top_k=1, null=(), shift=None, out=(True, True)):
        """one call of form f; null: indices of the pointer arguments passed as NULL, shift: {index: bytes added to the pointer}"""
        L, c = self.L, (self.ctx if ctx else None)
        p = [None if i in null else self.d + i * REGION + (shift or {}).get(i, 0) for i in range(f.n_ptr)]
        sp = self.sc.ctypes.data_as(FP) if out[0] else None
        ip = self.ix.ctypes.data_as(IP) if out[1] else None
        if f.name == "clip_b200_zero_shot_batch":
            return L.clip_b200_zero_shot_batch(c, p[0], nq, p[1], ndb, sp, ip, top_k)
        if f.name == "clip_b200_topk_search":
            return L.clip_b200_topk_search(c, p[0], nq, p[1], ndb, top_k, sp, ip)
        if f.name == "clip_b200_topk_search_16":
            return L.clip_b200_topk_search_16(c, p[0], nq, p[1], ndb, dim, type_, top_k, sp, ip)
        if f.name == "clip_b200_topk_search_i8":
            return L.clip_b200_topk_search_i8(c, p[0], p[1], nq, p[2], p[3], ndb, dim, top_k, sp, ip)
        if f.name == "clip_b200_rows_to_16bit":
            return L.clip_b200_rows_to_16bit(c, p[0], nq, dim, type_, p[1])
        return L.clip_b200_rows_to_int8(c, p[0], nq, dim, p[1], p[2])

    def refused(self, f, word, **kw):
        """the call is refused with a message that starts with the form's name and contains word"""
        assert not self.call(f, **kw), (f, word, kw)
        err = self.prod.last_error()
        assert err.startswith(f.name + ": ") and word in err, (f, word, kw, err)

    def guard(self):
        self.sc[:] = 7.0
        self.ix[:] = -7

    def untouched(self, n=0):
        """nothing written from host output entry n on"""
        return (self.sc[n:] == 7.0).all() and (self.ix[n:] == -7).all()

    def launches(self, f, **kw):
        """the kernel launches of one valid call"""
        l0 = self.L.clip_b200_kernel_launches(self.ctx)
        assert self.call(f, **kw), (f, kw, self.prod.last_error())
        return self.L.clip_b200_kernel_launches(self.ctx) - l0


@pytest.fixture(scope="module")
def env(prod):
    e = Env(prod)
    yield e
    e.close()


# ---- 1-3. refusals, their order and empty calls, alike on every form ------------------------------------------------------------

def refusals(env, f):
    """every fault is refused"""
    for _, cases in faults(f):
        for kw, word in cases:
            env.refused(f, word, **kw)


def two_faults(env, f):
    """of two faults, the first in the documented order is reported"""
    steps = faults(f)
    for i, (_, first) in enumerate(steps):
        for _, later in steps[i + 1:]:
            for kw, word in first:
                for kw2, _ in later:
                    if not set(kw) & set(kw2):
                        env.refused(f, word, **{**kw2, **kw})


def empty_calls(env, f):
    """n_q == 0 (or n_db == 0) returns true and writes nothing; the faults before it in the order are still refused, the ones
    after it are not looked at"""
    empties = [dict(nq=0)] + ([dict(ndb=0)] if f.search else [])
    env.guard()
    for e in empties:
        assert env.call(f, **e), (f, e, env.prod.last_error())
        assert env.call(f, null=range(f.n_ptr), out=(False, False), **e), (f, e, env.prod.last_error())
        past = False
        for step, cases in faults(f):
            past |= step == "pointer"
            for kw, word in cases:
                if set(kw) & set(e):
                    continue
                if past:
                    assert env.call(f, **kw, **e), (f, e, kw, env.prod.last_error())
                else:
                    env.refused(f, word, **kw, **e)
    assert env.untouched()


def check_form(prod, name):
    """the three checks above for one form, on a context of its own"""
    env = Env(prod)
    try:
        for check in (refusals, two_faults, empty_calls):
            check(env, BY_NAME[name])
    finally:
        env.close()


@pytest.mark.parametrize("f", FORMS, ids=IDS)
def test_refusals(env, f):
    refusals(env, f)


@pytest.mark.parametrize("f", FORMS, ids=IDS)
def test_two_faults_report_the_first(env, f):
    two_faults(env, f)


@pytest.mark.parametrize("f", FORMS, ids=IDS)
def test_empty_calls(env, f):
    empty_calls(env, f)


@pytest.mark.parametrize("f", [f for f in FORMS if f.fp32], ids=[f.name for f in FORMS if f.fp32])
def test_fp32_top_k_means_all_rows_when_out_of_range(env, f):
    """all scores tie on the zeroed data, so the ranking is the indices in order, at the clamped stride"""
    for top_k, ndb in ((0, 5), (-3, 5), (6, 5), (5, 5), (1500, 5000)):
        w = ndb if top_k <= 0 or top_k > ndb else top_k
        env.guard()
        assert env.call(f, nq=3, ndb=ndb, top_k=top_k), (f, top_k, env.prod.last_error())
        assert env.untouched(3 * w), (f, top_k)
        assert (env.ix[:3 * w].reshape(3, w) == np.arange(w)).all(), (f, top_k)


# ---- 4. kernel launches ---------------------------------------------------------------------------------------------------------
# (form, case, call arguments): fp32 with one sort slice, several slices and a merge stage, and top_k > 1024 over more than one
# slice (ranked on the host); K10 with one database partition, many partitions, and more than 32768 queries (two launches).
LAUNCH_CASES = [(name, case, kw) for name in ("clip_b200_zero_shot_batch", "clip_b200_topk_search") for case, kw in (
    ("one slice", dict(nq=3, ndb=1000, top_k=5)),
    ("slices and a merge", dict(nq=3, ndb=10_000, top_k=100)),
    ("host ranking", dict(nq=3, ndb=5000, top_k=2000)))] + [
    (name, case, kw) for name in ("clip_b200_topk_search_16", "clip_b200_topk_search_i8") for case, kw in (
    ("one partition", dict(nq=4, ndb=100, top_k=5)),
    ("many partitions", dict(nq=4, ndb=20_000, top_k=10)),
    ("over 32768 queries", dict(nq=40_000, ndb=700, top_k=5)))] + [
    (name, "rows", dict(nq=5)) for name in ("clip_b200_rows_to_16bit", "clip_b200_rows_to_int8")]

# clip_b200_kernel_launches deltas of the calls above, recorded with the library built at 8b28512 (before the four searches shared one
# pass driver) on an H100 80GB HBM3 (132 SMs).  The K10 partition counts follow the number of SMs.
LAUNCHES = {
    ("clip_b200_zero_shot_batch", "one slice"): 3,
    ("clip_b200_zero_shot_batch", "slices and a merge"): 4,
    ("clip_b200_zero_shot_batch", "host ranking"): 2,
    ("clip_b200_topk_search", "one slice"): 2,
    ("clip_b200_topk_search", "slices and a merge"): 3,
    ("clip_b200_topk_search", "host ranking"): 1,
    ("clip_b200_topk_search_16", "one partition"): 1,
    ("clip_b200_topk_search_16", "many partitions"): 2,
    ("clip_b200_topk_search_16", "over 32768 queries"): 3,
    ("clip_b200_topk_search_i8", "one partition"): 1,
    ("clip_b200_topk_search_i8", "many partitions"): 2,
    ("clip_b200_topk_search_i8", "over 32768 queries"): 3,
    ("clip_b200_rows_to_16bit", "rows"): 1,
    ("clip_b200_rows_to_int8", "rows"): 1,
}


@pytest.mark.parametrize("name,case,kw", LAUNCH_CASES, ids=["%s-%s" % (n, c) for n, c, _ in LAUNCH_CASES])
def test_kernel_launches_are_unchanged(env, name, case, kw):
    assert env.launches(BY_NAME[name], **kw) == LAUNCHES[name, case]
