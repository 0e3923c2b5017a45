"""The picture engine under the load the encoder puts on it: many pipeline threads in the library at once, slots that
served another kind of call before, an ME residency cache that must evict and re-upload, and the error paths that must
hand a slot back.  Every expectation is computed by the CPU oracle on the main thread before any engine call; every
engine output must equal it bit for bit.  Failures name the phase, the thread, the case and the call kind."""
import ctypes as C
import random
import threading
from collections import Counter

import numpy as np
import pytest

import common as cm
import svtb200 as sb
from test_dlf_gpu import flat_mi
from test_engine_gpu import CdefChain, _host_pic, assert_me_result, lr_boundary_lines, lr_frame_params
from test_oracle_dlf import dlf_case, dlf_params, pick_case, pick_params
from test_oracle_lr_frame import lr_case, run_oracle_lr

pytestmark = pytest.mark.gpu

SVT_B200_ERR_ARG, SVT_B200_ERR_UNSUPPORTED = -2, -3
N_THREADS = 12  # more than the engine's 8 ME slots and 8 filter slots
KINDS = ("dlf", "pick", "cdef", "lr")
# neither dimension a multiple of 64: the device pitch exceeds the width and the 64x64 filter blocks at the edges are partial
FILTER_GEOMETRIES = [(712, 392, 8), (584, 328, 10)]


class Engine:
    def __init__(self, lib):
        self.lib, self.e = lib, C.c_void_p()
        sb.check(lib.svt_b200_engine_create(0, C.byref(self.e)), lib)

    def stats(self):
        st = sb.EngineStats()
        sb.check(self.lib.svt_b200_engine_get_stats(self.e, C.byref(st)), self.lib)
        return st

    def close(self):
        self.lib.svt_b200_engine_destroy(self.e)


def _failed(lib, rc):
    return f"rc={rc}: {lib.svt_b200_last_error().decode()}"


def _frame_diff(got, want):
    for i in range(3):
        bad = np.argwhere(got.plane(i) != want.plane(i))
        if len(bad):
            y, x = bad[0]
            return f"plane {i}: {len(bad)} samples differ, first at (y={y}, x={x}): {got.plane(i)[y, x]} != {want.plane(i)[y, x]}"
    return None


# ---- filter cases: build() runs the oracle, run() makes one engine call on fresh copies and returns None or what went wrong
class DlfCase:
    kind = "dlf"

    def __init__(self, w, h, bd, seed, levels, sharp):
        self.name = f"dlf seed={seed} levels={levels} sharp={sharp}"
        mi_rows, mi_cols, part, self.frame = dlf_case(w, h, bd, seed, levels, sharp)
        self.flat = flat_mi(mi_rows, mi_cols, part, levels)
        self.p = dlf_params(mi_rows, mi_cols, levels, sharp)
        self.want = self.frame.copy()
        ws = self.want.struct()
        cm.oracle().orc_dlf_frame(C.byref(self.p), C.byref(ws), self.flat)

    def run(self, lib, e):
        got = self.frame.copy()
        gs = got.struct()
        rc = lib.svt_b200_engine_dlf_frame(e, C.byref(self.p), C.byref(gs), self.flat)
        return _failed(lib, rc) if rc else _frame_diff(got, self.want)


class PickCase:
    kind = "pick"

    def __init__(self, w, h, bd, seed, mode, last, q_ac):
        self.name = f"dlf_pick seed={seed} method=0 loop_filter_mode={mode} q_ac={q_ac}"
        orc = cm.oracle()
        mi_rows, mi_cols, part, self.src, self.rec = pick_case(w, h, bd, seed)
        self.flat = flat_mi(mi_rows, mi_cols, part, last)
        self.p = pick_params(mi_rows, mi_cols, 0, mode, last, q_ac=q_ac)
        r, t = self.rec.copy(), self.rec.copy()
        rs, ss, ts = r.struct(), self.src.struct(), t.struct()
        lv = (C.c_int32 * 4)()
        orc.orc_pick_filter_level(C.byref(self.p), C.byref(rs), C.byref(ss), C.byref(ts), self.flat, lv)
        self.want_lv = list(lv)
        dp = dlf_params(mi_rows, mi_cols, tuple(self.want_lv), 0)
        self.want = self.rec.copy()
        ws = self.want.struct()
        orc.orc_dlf_frame(C.byref(dp), C.byref(ws), flat_mi(mi_rows, mi_cols, part, tuple(self.want_lv)))

    def run(self, lib, e):
        got = self.rec.copy()
        gs, ss = got.struct(), self.src.struct()
        lv = (C.c_int32 * 4)()
        rc = lib.svt_b200_engine_dlf_pick_frame(e, C.byref(self.p), C.byref(gs), C.byref(ss), self.flat, lv)
        if rc:
            return _failed(lib, rc)
        if list(lv) != self.want_lv:
            return f"levels {list(lv)} != {self.want_lv}"
        return _frame_diff(got, self.want)


class CdefCase:
    kind = "cdef"

    def __init__(self, w, h, bd, seed, with_dlf, apply, pick):
        self.name = f"dlf_cdef_dev seed={seed} dlf={with_dlf} apply={apply} pick={pick}"
        self.with_dlf, self.apply = with_dlf, apply
        self.chain = CdefChain(w, h, bd, with_dlf, pick, seed=seed, part_seed=seed + 50, levels=(16 + seed % 20, 22, 12, 9))

    def run(self, lib, e):
        c = self.chain
        rc, got, dec, idx = c.run(lib, e, self.apply)
        if rc:
            return _failed(lib, rc)
        if not c.decision_matches(dec):
            return "strength decision differs"
        if not np.array_equal(idx, c.want_idx):
            return f"filter-block strength indices differ at {np.flatnonzero(idx != c.want_idx)[:8]}"
        return _frame_diff(got, c.want if self.apply else c.rec)  # apply = 0 leaves the host picture as it was


class LrCase:
    kind = "lr"

    def __init__(self, w, h, bd, seed, unit_sizes, modes, ftypes):
        self.name = f"lr seed={seed} units={unit_sizes} modes={modes} types={ftypes}"
        self.cdef, dblk, self.units = lr_case(w, h, bd, seed, unit_sizes, modes)
        self.ftypes = ftypes
        self.want = run_oracle_lr(self.cdef, dblk, self.units, unit_sizes, ftypes, 0)
        for i in range(3):
            if not ftypes[i]:
                self.want.plane(i)[...] = self.cdef.plane(i)
        self.lines, self.keep = lr_boundary_lines(dblk)
        self.p, self.n_units = lr_frame_params(self.units, unit_sizes, ftypes)

    def run(self, lib, e):
        got = self.cdef.copy()
        gs = got.struct()
        rc = lib.svt_b200_engine_lr_frame(e, C.byref(self.p), self.n_units, C.byref(gs), self.lines)
        return _failed(lib, rc) if rc else _frame_diff(got, self.want)


def filter_cases(w, h, bd):
    """24 seeded cases, six of each call kind."""
    cases = []
    for k in range(6):
        s = 10 * bd + k
        cases.append(DlfCase(w, h, bd, s, ((12, 20, 28, 36, 48, 63)[k], (30, 8, 40, 16, 0, 24)[k], 20 + 3 * k, 14 - 2 * k), k % 8))
        cases.append(PickCase(w, h, bd, s, 3 if k % 2 else 2, (20 + k, 24, 12, 9), 40 + 30 * k))
        cases.append(CdefCase(w, h, bd, s, with_dlf=k % 3 != 1, apply=int(k < 4), pick=(3, 2)[k % 2]))
        us = ((64, 32, 32), (128, 64, 64), (256, 128, 128))[k % 3]
        modes = (("mix", "mix", "mix"), ("wiener", "sgr", "mix"), ("sgr", "mix", "none"))[k % 3]
        ftypes = ((3, 3, 3), (1, 2, 3), (2, 3, 0))[k % 3]
        cases.append(LrCase(w, h, bd, s, us, modes, ftypes))
    return cases


def interleave(cases, seed):
    """An order in which no call follows a call of its own kind, spreading the (previous kind, next kind) pairs."""
    rng = random.Random(seed)
    left = {k: [c for c in cases if c.kind == k] for k in KINDS}
    for v in left.values():
        rng.shuffle(v)
    order, pairs, prev = [], Counter(), None
    while any(left.values()):
        ks = [k for k in KINDS if left[k] and k != prev]
        k = min(ks, key=lambda k: (-len(left[k]), pairs[prev, k], rng.random()))
        pairs[prev, k] += 1
        order.append(left[k].pop())
        prev = k
    assert all(a.kind != b.kind for a, b in zip(order, order[1:]))
    return order


def expected_filter_stats(cases):
    n = Counter(c.kind for c in cases)
    with_dlf = sum(1 for c in cases if c.kind == "cdef" and c.with_dlf)
    return n["dlf"] + n["pick"] + with_dlf, n["cdef"], n["lr"]


def filter_stats(st):
    return st.dlf_frames, st.cdef_frames, st.lr_frames


# ---- the ME program: 120 pictures, keys recycled after 100, long-term references that the cache has evicted
ME_W, ME_H, ME_PICTURES, ME_KEYS = 200, 136, 120, 100


class MeProgram:
    def __init__(self):
        self.geos = sb.me_geometry(ME_W, ME_H)
        self.pics = [cm.me_planes(cm.synth_luma(ME_W, ME_H, i, 77), self.geos) for i in range(ME_PICTURES)]
        self.pool = [C.c_int64() for _ in range(ME_KEYS)]  # the encoder's pooled EbPaReferenceObject*: reused by later pictures
        self.n_sb = ((ME_W + 63) // 64) * ((ME_H + 63) // 64)
        self.calls = []
        for i in range(1, ME_PICTURES):  # picture 0 is only ever a reference
            l0 = [j for j in (i - 1, i - 3) if j >= 0] + ([i - 97] if i >= 100 else [])  # i - 97: long evicted
            l1 = [i - 1] if i % 8 == 4 else [i - 2] if i >= 2 else []  # i % 8 == 4: list1 holds list0's first (key, tag)
            dist = (tuple(i - j for j in l0) + (1,) * (4 - len(l0)), tuple(i - j for j in l1) + (1,) * (4 - len(l1)))
            params = sb.preset8_me_params(ME_W, ME_H, len(l0), len(l1), dist, 1, 1)
            pad = self.pics[0]
            want = cm.run_oracle_me(params, self.pics[i], [self.pics[j] for j in l0] + [pad] * (4 - len(l0)) +
                                    [self.pics[j] for j in l1] + [pad] * (4 - len(l1)))
            self.calls.append((i, l0, l1, params, want))
        self.acquisitions = sum(1 + len(l0) + len(l1) for _, l0, l1, _, _ in self.calls)

    def host(self, i):
        return _host_pic(C.addressof(self.pool[i % ME_KEYS]), i, self.pics[i])

    def run(self, lib, e, call):
        i, l0, l1, params, want = call
        hs = self.host(i)
        hr = (sb.HostMePicture * 8)()
        for j, r in enumerate(l0):
            hr[j] = self.host(r)
        for j, r in enumerate(l1):
            hr[4 + j] = self.host(r)
        got = cm.MeBuffers(self.n_sb)
        rc = lib.svt_b200_engine_me_picture(e, C.byref(params), C.byref(hs), hr, 1, cm.ptr(got.me_mv), cm.ptr(got.me_cand),
                                            cm.ptr(got.total_cand), cm.ptr(got.rc))
        if rc:
            return _failed(lib, rc)
        try:
            assert_me_result(got, want, self.n_sb)
        except AssertionError as ex:
            return " ".join(str(ex).strip().splitlines()[:3])  # "Arrays are not equal", the field, the mismatch count
        return None


class MeCall:
    kind = "me"

    def __init__(self, prog, call):
        self.prog, self.call = prog, call
        i, l0, l1 = call[:3]
        self.name = f"me picture {i} key={i % ME_KEYS} list0={l0} list1={l1}"

    def run(self, lib, e):
        return self.prog.run(lib, e, self.call)


def run_threads(lib, e, programs):
    """programs[t]: the calls of thread t, in order.  The threads start together; each records its own failures (the
    library's error text is thread-local) and the main thread reports them all."""
    barrier = threading.Barrier(len(programs))
    failures = [[] for _ in programs]

    def worker(t):
        barrier.wait()
        for c in programs[t]:
            try:
                msg = c.run(lib, e)
            except Exception as ex:  # reported on the main thread
                msg = f"{type(ex).__name__}: {ex}"
            if msg:
                failures[t].append(f"thread {t} {c.kind} [{c.name}]: {msg}")

    th = [threading.Thread(target=worker, args=(t,)) for t in range(len(programs))]
    for x in th:
        x.start()
    for x in th:
        x.join()
    return [f for per in failures for f in per]


@pytest.fixture(scope="module")
def lib():
    return sb.load()


@pytest.fixture(scope="module", params=FILTER_GEOMETRIES, ids=lambda g: f"{g[0]}x{g[1]}-{g[2]}bit")
def filter_program(request):
    return filter_cases(*request.param)


@pytest.fixture(scope="module")
def filter_program_8bit():
    return filter_cases(*FILTER_GEOMETRIES[0])


@pytest.fixture(scope="module")
def me_program():
    return MeProgram()


def test_filter_calls_serial_then_concurrent(lib, filter_program):
    """Serial: every call runs on slot 0 right after a call of another kind, so whatever the previous call left in the
    slot's device pictures is there to be read by mistake.  Concurrent: 12 threads on a fresh engine, each running all
    the cases in its own order."""
    cases = filter_program
    eng = Engine(lib)
    try:
        fails = [f"serial {c.kind} [{c.name}]: {m}" for c in interleave(cases, 0) for m in [c.run(lib, eng.e)] if m]
        assert not fails, "\n".join(fails)
        assert filter_stats(eng.stats()) == expected_filter_stats(cases)
    finally:
        eng.close()
    eng = Engine(lib)
    try:
        fails = run_threads(lib, eng.e, [interleave(cases, 1 + t) for t in range(N_THREADS)])
        assert not fails, "concurrent:\n" + "\n".join(fails)
        assert filter_stats(eng.stats()) == tuple(N_THREADS * n for n in expected_filter_stats(cases))
    finally:
        eng.close()


def _check_me_stats(st, prog, n_runs=1):
    assert st.me_pictures == n_runs * len(prog.calls)
    assert st.me_plane_uploads + st.me_plane_hits == n_runs * prog.acquisitions
    assert st.me_plane_uploads > ME_PICTURES  # more than one upload per picture: evicted pictures came back


def test_me_eviction_and_key_recycling_serial_then_concurrent(lib, me_program):
    """120 pictures through a 96-entry residency cache: keys recycled after 100 pictures with new tags, long-term references
    that were evicted and must be uploaded again, list0 and list1 naming the same picture.  Serial, then 12 threads on a
    fresh engine (more than the 8 ME slots) taking every 12th picture, so threads wait on each other's uploads."""
    prog = me_program
    calls = [MeCall(prog, c) for c in prog.calls]
    eng = Engine(lib)
    try:
        fails = [f"serial me [{c.name}]: {m}" for c in calls for m in [c.run(lib, eng.e)] if m]
        assert not fails, "\n".join(fails)
        _check_me_stats(eng.stats(), prog)
    finally:
        eng.close()
    eng = Engine(lib)
    try:
        fails = run_threads(lib, eng.e, [calls[t::N_THREADS] for t in range(N_THREADS)])
        assert not fails, "concurrent:\n" + "\n".join(fails)
        _check_me_stats(eng.stats(), prog)
    finally:
        eng.close()


def test_me_and_filter_calls_on_one_engine(lib, me_program, filter_program_8bit):
    """ME pictures and filter calls at once on one engine: both sides wait on the same mutex and condition variable."""
    prog, cases = me_program, filter_program_8bit
    calls = [MeCall(prog, c) for c in prog.calls]
    half = N_THREADS // 2
    programs = [calls[t::half] for t in range(half)] + [interleave(cases, 100 + t) for t in range(half)]
    eng = Engine(lib)
    try:
        fails = run_threads(lib, eng.e, programs)
        assert not fails, "concurrent:\n" + "\n".join(fails)
        st = eng.stats()
        _check_me_stats(st, prog)
        assert filter_stats(st) == tuple(half * n for n in expected_filter_stats(cases))
    finally:
        eng.close()


def test_second_geometry_is_refused_and_the_first_still_served(lib, me_program, filter_program_8bit):
    prog, cases = me_program, filter_program_8bit
    me, dlf = MeCall(prog, prog.calls[5]), next(c for c in cases if c.kind == "dlf")
    eng = Engine(lib)
    try:
        assert me.run(lib, eng.e) is None and dlf.run(lib, eng.e) is None
        # ME at another size
        w, h = ME_W + 64, ME_H
        geos = sb.me_geometry(w, h)
        a, b = (cm.me_planes(cm.synth_luma(w, h, n, 5), geos) for n in (0, 1))
        params = sb.preset8_me_params(w, h, 1, 0)
        hs, hr = _host_pic(1, 1, a), (sb.HostMePicture * 8)()
        hr[0] = _host_pic(2, 0, b)
        n_sb = ((w + 63) // 64) * ((h + 63) // 64)
        got = cm.MeBuffers(n_sb)
        rc = lib.svt_b200_engine_me_picture(eng.e, C.byref(params), C.byref(hs), hr, 1, cm.ptr(got.me_mv), cm.ptr(got.me_cand),
                                            cm.ptr(got.total_cand), cm.ptr(got.rc))
        assert rc == SVT_B200_ERR_UNSUPPORTED and b"geometry" in lib.svt_b200_last_error()
        # deblocking at another size
        other = DlfCase(192, 136, 8, 3, (20, 24, 12, 9), 0)
        got = other.frame.copy()
        gs = got.struct()
        rc = lib.svt_b200_engine_dlf_frame(eng.e, C.byref(other.p), C.byref(gs), other.flat)
        assert rc == SVT_B200_ERR_UNSUPPORTED and b"geometry" in lib.svt_b200_last_error()
        assert _frame_diff(got, other.frame) is None  # the refused call left the picture alone
        for c in [me, MeCall(prog, prog.calls[6])] + [c for c in cases if c.kind != "dlf"][:3] + [dlf]:
            assert c.run(lib, eng.e) is None, c.name
    finally:
        eng.close()


def test_lr_frame_first_then_deblocking_and_cdef(lib, filter_program_8bit):
    """The geometry fixed by a first loop-restoration call serves the deblocking and CDEF calls of the same pictures."""
    cases = filter_program_8bit
    lr = next(c for c in cases if c.kind == "lr")
    rest = [c for c in cases if c.kind == "dlf"][:1] + [c for c in cases if c.kind == "cdef" and c.with_dlf][:2]
    eng = Engine(lib)
    try:
        for c in [lr] + rest:
            msg = c.run(lib, eng.e)
            assert msg is None, f"{c.name}: {msg}"
    finally:
        eng.close()


def _filter_small_bytes(w, h):
    """The per-slot host staging for skip map, CDEF mse, filter-block indices and the decision (ensure_filt's g.small)."""
    al = lambda v: (v + 255) & ~255  # noqa: E731
    mi_rows, mi_cols = 2 * ((h + 7) // 8), 2 * ((w + 7) // 8)
    nfb = ((mi_rows + 15) // 16) * ((mi_cols + 15) // 16)
    skip = al(((mi_rows + 1) // 2) * ((((mi_cols + 1) // 2) + 15) & ~15))
    dec = al(C.sizeof(sb.CdefDecision)) + al(nfb * (16 + 16 * 64) + 64)
    return skip + al(nfb * 2 * 64 * 8) + al(nfb) + dec, al(mi_rows * mi_cols * C.sizeof(sb.DlfMi))


def test_lr_frame_error_after_taking_a_slot_releases_it(lib, filter_program_8bit):
    """Nine loop-restoration calls with more unit bytes than a slot's staging are refused before they take a slot; a
    valid call still completes afterwards, so no refused call kept a slot.  In a thread: a lost slot hangs the call."""
    lr = next(c for c in filter_program_8bit if c.kind == "lr")
    small, mi = _filter_small_bytes(lr.cdef.w, lr.cdef.h)
    n = (small + mi // 2) // C.sizeof(sb.LrUnit)  # more than the staging holds, less than the device side accepts
    units = (sb.LrUnit * n)()
    p = sb.LrFrameParams()
    for i in range(3):
        p.plane[i].frame_restoration_type, p.plane[i].restoration_unit_size, p.plane[i].units = 3, 64, C.addressof(units)
    n_units = (C.c_int32 * 3)(n, 0, 0)
    eng = Engine(lib)
    out = {}

    def body():
        try:
            rcs, errs = [], []
            for _ in range(9):
                got = lr.cdef.copy()
                gs = got.struct()
                rcs.append(lib.svt_b200_engine_lr_frame(eng.e, C.byref(p), n_units, C.byref(gs), lr.lines))
                errs.append(lib.svt_b200_last_error().decode())
            out["rcs"], out["errs"], out["valid"] = rcs, errs, lr.run(lib, eng.e)
        except Exception as ex:
            out["exc"] = ex

    try:
        t = threading.Thread(target=body, daemon=True)
        t.start()
        t.join(timeout=120)
        assert not t.is_alive(), "a call never got a slot: a failed call kept its slot"
        assert "exc" not in out, out.get("exc")
        assert out["rcs"] == [SVT_B200_ERR_ARG] * 9
        assert all("too many restoration units" in m for m in out["errs"]), out["errs"]
        assert out["valid"] is None, out["valid"]
        assert eng.stats().lr_frames == 1
    finally:
        if not t.is_alive():
            eng.close()


def test_me_call_with_a_missing_reference_is_refused_before_any_upload(lib, me_program):
    """Nine ME calls whose second list0 reference has no planes, and one that names more list0 references than
    SvtB200MeParams holds, are refused before they take a slot or upload a picture; a valid call still completes
    afterwards.  In a thread: a lost slot hangs the call."""
    prog = me_program
    call = next(c for c in prog.calls if len(c[1]) == 2 and len(c[2]) == 1)
    i, l0, l1, params = call[:4]
    hs, hr = prog.host(i), (sb.HostMePicture * 8)()
    hr[0], hr[4] = prog.host(l0[0]), prog.host(l1[0])  # hr[1]: list0 reference 1 without planes
    too_many = type(params).from_buffer_copy(params)
    too_many.num_refs[0] = 5
    got = cm.MeBuffers(prog.n_sb)
    eng = Engine(lib)
    out = {}

    def me(p):
        rc = lib.svt_b200_engine_me_picture(eng.e, C.byref(p), C.byref(hs), hr, 1, cm.ptr(got.me_mv), cm.ptr(got.me_cand),
                                            cm.ptr(got.total_cand), cm.ptr(got.rc))
        return rc, lib.svt_b200_last_error().decode()

    def body():
        try:
            out["refused"] = [me(params) for _ in range(9)]
            out["too_many"] = me(too_many)
            out["uploads"] = eng.stats().me_plane_uploads
            out["valid"] = MeCall(prog, call).run(lib, eng.e)
        except Exception as ex:
            out["exc"] = ex

    try:
        t = threading.Thread(target=body, daemon=True)
        t.start()
        t.join(timeout=120)
        assert not t.is_alive(), "a call never got a slot: a refused call kept its slot"
        assert "exc" not in out, out.get("exc")
        assert all(rc == SVT_B200_ERR_ARG and "has no planes" in m for rc, m in out["refused"]), out["refused"]
        assert out["too_many"][0] == SVT_B200_ERR_ARG and "more reference lists or references" in out["too_many"][1], out["too_many"]
        assert out["uploads"] == 0
        assert out["valid"] is None, out["valid"]
        assert eng.stats().me_pictures == 1
    finally:
        if not t.is_alive():
            eng.close()


def _al256(v):
    return (v + 255) & ~255


def _packed_bytes(frame):
    return sum(frame.plane(i).nbytes for i in range(3))


def _filter_call_bytes(c):
    """(H2D, D2H) bytes of one filter call: what the call must move between host staging and the device."""
    mi = C.sizeof(sb.DlfMi)
    if c.kind == "dlf":
        pk = _packed_bytes(c.frame)
        return pk + c.p.mi_rows * c.p.mi_cols * mi, pk
    if c.kind == "pick":  # recon and source up, the mode info, the 768-byte level table of the picked levels
        pk = _packed_bytes(c.rec)
        return 2 * pk + c.p.dlf.mi_rows * c.p.dlf.mi_cols * mi + 3 * 2 * 128, pk
    if c.kind == "cdef":  # recon and source up, the mode info when it deblocks, the skip map; down the index buffer + decision
        ch = c.chain
        pk = _packed_bytes(ch.rec)
        up = 2 * pk + (ch.dp.mi_rows * ch.dp.mi_cols * mi if c.with_dlf else 0) + ((ch.sp.mi_rows + 1) // 2) * ch.skip.shape[1]
        return up, (pk if c.apply else 0) + _al256(ch.nfb) + C.sizeof(sb.CdefDecision)
    # lr: the units of every plane (each array 256-byte aligned, one copy), the picture, and in every restored plane the
    # rows -2 .. +1 around each stripe boundary that lie inside the plane
    pk = _packed_bytes(c.cdef)
    up = sum(_al256(len(u) * C.sizeof(sb.LrUnit)) for u in c.units) + pk
    for i in range(3):
        if c.ftypes[i]:
            plane = c.cdef.plane(i)
            ph, row = plane.shape[0], plane.shape[1] * plane.itemsize
            sh, off = 64 >> (i > 0), 8 >> (i > 0)
            n_boundaries = (ph + off + sh - 1) // sh - 1
            up += row * sum((b + 1) * sh - off - 2 + k < ph for b in range(n_boundaries) for k in range(4))
    return up, pk


def test_byte_counters_count_every_copy_once(lib, filter_program, me_program):
    """h2d_bytes / d2h_bytes grow by exactly the bytes each call moves: every filter case of the geometry, then one ME
    call whose four pictures are all uploaded with their decimations."""
    eng = Engine(lib)
    try:
        fails = []
        for c in filter_program:
            before = eng.stats()
            msg = c.run(lib, eng.e)
            assert msg is None, f"{c.kind} [{c.name}]: {msg}"
            after = eng.stats()
            got = (after.h2d_bytes - before.h2d_bytes, after.d2h_bytes - before.d2h_bytes)
            if got != _filter_call_bytes(c):
                fails.append(f"{c.kind} [{c.name}]: (h2d, d2h) {got} != {_filter_call_bytes(c)}")
        assert not fails, "\n".join(fails)
        prog = me_program
        call = next(c for c in prog.calls if len(set([c[0]] + c[1] + c[2])) == 4)
        geos = prog.geos
        nb = [g.stride * (g.height + 2 * g.origin_y) for g in geos]
        before = eng.stats()
        msg = MeCall(prog, call).run(lib, eng.e)
        assert msg is None, msg
        after = eng.stats()
        assert after.me_plane_uploads - before.me_plane_uploads == 4
        n_sb = prog.n_sb
        want = (4 * (_al256(nb[0]) + _al256(nb[1]) + nb[2]),
                _al256(n_sb * 85 * 7 * 4) + _al256(n_sb * 85 * 23) + _al256(n_sb * 85) + _al256(n_sb * 4))
        assert (after.h2d_bytes - before.h2d_bytes, after.d2h_bytes - before.d2h_bytes) == want
    finally:
        eng.close()
