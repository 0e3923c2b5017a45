"""The picture engine (svt_b200_engine_*: HOST pictures in, host results out - what the reference's process loops call
through integration/svt_cuda_backend.c) against the CPU oracle, without the encoder: the same seeded cases the device-pointer
entries are tested on, passed as plain numpy buffers."""
import ctypes as C

import numpy as np
import pytest

import common as cm
import svtb200 as sb

pytestmark = pytest.mark.gpu


def _host_pic(key, tag, planes, with_decimations=True):
    h = sb.HostMePicture()
    h.key, h.tag, h.full = key, tag, planes[0].ctypes.data
    h.quarter = planes[1].ctypes.data if with_decimations else None
    h.sixteenth = planes[2].ctypes.data if with_decimations else None
    return h


def assert_me_result(got, want, n_sb, what=""):
    """The engine's four ME outputs against the oracle's; candidates beyond total_cand are unspecified."""
    np.testing.assert_array_equal(got.me_mv, want.me_mv, err_msg=f"me_mv {what}")
    np.testing.assert_array_equal(got.total_cand, want.total_cand, err_msg=f"total_cand {what}")
    np.testing.assert_array_equal(got.rc, want.rc, err_msg=f"rc {what}")
    used = np.arange(23) < want.total_cand[:, :, None].astype(np.int64)
    np.testing.assert_array_equal(got.me_cand.reshape(n_sb, 85, 23)[used], want.me_cand.reshape(n_sb, 85, 23)[used],
                                  err_msg=f"me_cand {what}")


def run_me_steps(w, h, steps, uploads, hits):
    """'Pictures' in coding order, each searched against the earlier ones on one engine: every call equals the oracle, and
    the residency counters equal `uploads` / `hits`."""
    lib = sb.load()
    e = C.c_void_p()
    sb.check(lib.svt_b200_engine_create(0, C.byref(e)), lib)
    try:
        dist = ((1, 2, 3, 4), (1, 2, 3, 4))
        geos, src, refs = cm.make_me_case(w, h, 2, 2, seed=21)
        pics = [refs[1], refs[0], src, refs[4]]  # distinct contents; keys = their index
        n_sb = ((w + 63) // 64) * ((h + 63) // 64)
        for step, (cur, l0, l1) in enumerate(steps):
            params = sb.preset8_me_params(w, h, len(l0), len(l1), dist, 1, 1)
            want = cm.run_oracle_me(params, pics[cur], [pics[i] for i in l0] + [pics[0]] * (4 - len(l0)) + [pics[i] for i in l1] + [pics[0]] * (4 - len(l1)))
            hs = _host_pic(1000 + cur, cur, pics[cur])
            hr = (sb.HostMePicture * 8)()
            for j, i in enumerate(l0):
                hr[j] = _host_pic(1000 + i, i, pics[i])
            for j, i in enumerate(l1):
                hr[4 + j] = _host_pic(1000 + i, i, pics[i])
            got = cm.MeBuffers(n_sb)
            sb.check(lib.svt_b200_engine_me_picture(e, C.byref(params), C.byref(hs), hr, 1, cm.ptr(got.me_mv), cm.ptr(got.me_cand),
                                                    cm.ptr(got.total_cand), cm.ptr(got.rc)), lib)
            assert_me_result(got, want, n_sb, f"step {step}")
        st = sb.EngineStats()
        sb.check(lib.svt_b200_engine_get_stats(e, C.byref(st)), lib)
        assert st.me_pictures == len(steps)
        assert st.me_plane_uploads == uploads and st.me_plane_hits == hits
    finally:
        lib.svt_b200_engine_destroy(e)


def test_engine_me_picture_residency_and_results():
    """A picture uploaded once (as source) is found resident when it is a reference later: 4 distinct pictures, 5 reuses."""
    run_me_steps(256, 192, [(1, [0], []), (2, [1, 0], []), (3, [2, 1], [0])], 4, 5)


def test_engine_me_picture_above_copy_split():
    """3840x2160: the full plane (8.7 MB) is staged by the host copy split over threads; 2 list0 + 1 list1 references."""
    run_me_steps(3840, 2160, [(3, [2, 1], [0])], 4, 0)


def test_engine_me_device_side_downsample_matches_uploaded_planes():
    """quarter / sixteenth == NULL: the engine derives them with svt_b200_me_downsample (filtered) - same ME result as with the
    host's planes when those are the filtered downsamples of the full plane."""
    from test_oracle_me import downsample_case, run_downsample
    lib = sb.load()
    e = C.c_void_p()
    sb.check(lib.svt_b200_engine_create(0, C.byref(e)), lib)
    try:
        w, h = 192, 128
        dist = ((1, 2, 3, 4), (1, 2, 3, 4))
        pics = []
        for s in (3, 4):
            geos, full, q0, s0 = downsample_case(w, h, s)
            q, s16 = run_downsample(cm.oracle().orc_me_downsample, geos, full, q0.copy(), s0.copy(), 1)
            pics.append((full, q, s16))
        params = sb.preset8_me_params(w, h, 1, 0, dist, 1, 1)
        want = cm.run_oracle_me(params, pics[1], [pics[0]] * 8)
        n_sb = ((w + 63) // 64) * ((h + 63) // 64)
        hs = _host_pic(1, 1, pics[1], with_decimations=False)
        hr = (sb.HostMePicture * 8)()
        hr[0] = _host_pic(2, 0, pics[0], with_decimations=False)
        got = cm.MeBuffers(n_sb)
        sb.check(lib.svt_b200_engine_me_picture(e, C.byref(params), C.byref(hs), hr, 1, cm.ptr(got.me_mv), cm.ptr(got.me_cand),
                                                cm.ptr(got.total_cand), cm.ptr(got.rc)), lib)
        np.testing.assert_array_equal(got.me_mv, want.me_mv)
        np.testing.assert_array_equal(got.rc, want.rc)
    finally:
        lib.svt_b200_engine_destroy(e)


# 1920x1080 10-bit: the packed picture (6.2 MB) is staged by the split host copy
@pytest.mark.parametrize("case", [(320, 192, 8, 6, (12, 30, 0, 22), 2), (192, 136, 10, 2, (33, 17, 40, 25), 3),
                                  (1920, 1080, 10, 7, (36, 28, 20, 14), 1)])
def test_engine_dlf_frame(case):
    from test_dlf_gpu import flat_mi
    from test_oracle_dlf import dlf_case, dlf_params
    lib = sb.load()
    e = C.c_void_p()
    sb.check(lib.svt_b200_engine_create(0, C.byref(e)), lib)  # one geometry per engine
    try:
        w, h, bd, seed, levels, sharp = case
        mi_rows, mi_cols, part, frame = dlf_case(w, h, bd, seed, levels, sharp)
        flat = flat_mi(mi_rows, mi_cols, part, levels)
        p = dlf_params(mi_rows, mi_cols, levels, sharp)
        want = frame.copy()
        st = want.struct()
        cm.oracle().orc_dlf_frame(C.byref(p), C.byref(st), flat)
        got = frame.copy()
        gs = got.struct()
        sb.check(lib.svt_b200_engine_dlf_frame(e, C.byref(p), C.byref(gs), flat), lib)
        for i in range(3):
            np.testing.assert_array_equal(got.plane(i), want.plane(i), err_msg=f"plane {i}")
    finally:
        lib.svt_b200_engine_destroy(e)


class CdefChain:
    """Inputs of one svt_b200_engine_dlf_cdef_frame_dev call and the oracle's chain on them: deblocking (with_dlf) ->
    strength search -> finish_cdef_search -> apply (damping 5, lambda 3500)."""

    def __init__(self, w, h, bd, with_dlf, pick, seed=9, part_seed=5, levels=(20, 24, 12, 9)):
        from test_dlf_gpu import flat_mi
        from test_oracle_cdef import cdef_picture_case
        from test_oracle_dlf import dlf_params
        lib, orc = sb.load(), cm.oracle()
        self.src, self.rec, mi_rows, mi_cols, skip = cdef_picture_case(w, h, bd, seed)
        # the engine stages skip maps up to the encoder's row stride: (mi_cols + 1) / 2 rounded up to 16
        self.skip = np.ascontiguousarray(skip[:, :((mi_cols + 1) // 2 + 15) & ~15])
        self.skip[0:8, 0:8] = 1  # one filter block entirely skipped
        pre = self.rec.copy()
        self.dp, self.flat = None, None
        if with_dlf:
            part = cm.random_partition(mi_rows, mi_cols, part_seed)
            self.flat = flat_mi(mi_rows, mi_cols, part, levels)
            self.dp = dlf_params(mi_rows, mi_cols, levels, 1)
            ps = pre.struct()
            orc.orc_dlf_frame(C.byref(self.dp), C.byref(ps), self.flat)
        self.sp = sp = sb.CdefSearchParams()
        sp.mi_rows, sp.mi_cols, sp.pri_damping = mi_rows, mi_cols, 5
        orc.orc_cdef_strength_table(pick, C.byref(sp))
        self.dcp = dcp = sb.CdefDecideParams()
        assert lib.svt_b200_cdef_decide_table(pick, C.byref(dcp)) == sp.n_strengths
        ref_tab = sb.CdefDecideParams()
        orc.orc_cdef_decide_table(pick, C.byref(ref_tab))
        assert list(dcp.filter_strength) == list(ref_tab.filter_strength)
        dcp.mi_rows, dcp.mi_cols, dcp.lambda_ = mi_rows, mi_cols, 3500
        self.nfb = nfb = ((mi_rows + 15) // 16) * ((mi_cols + 15) // 16)
        want_mse = np.zeros((2, nfb, 64), np.uint64)
        pres, ss = pre.struct(), self.src.struct()
        orc.orc_cdef_search(C.byref(sp), C.byref(pres), C.byref(ss), cm.ptr(self.skip), self.skip.shape[1], cm.ptr(want_mse))
        self.want_dec, self.want_idx = sb.CdefDecision(), np.zeros(nfb, np.int8)
        orc.orc_cdef_decide(C.byref(dcp), cm.ptr(want_mse), cm.ptr(self.skip), self.skip.shape[1], C.byref(self.want_dec), cm.ptr(self.want_idx))
        pa = sb.CdefApplyParams()
        pa.mi_rows, pa.mi_cols, pa.damping = mi_rows, mi_cols, 5
        for i in range(8):
            pa.y_strength[i], pa.uv_strength[i] = self.want_dec.y_strength[i], self.want_dec.uv_strength[i]
        self.want = pre.copy()
        ws = self.want.struct()
        orc.orc_cdef_apply(C.byref(pa), C.byref(pres), C.byref(ws), cm.ptr(self.skip), self.skip.shape[1], cm.ptr(self.want_idx))

    def run(self, lib, e, apply):
        """One engine call on a copy of the reconstruction: (rc, picture, decision, filter-block indices)."""
        got, dec, idx = self.rec.copy(), sb.CdefDecision(), np.full(self.nfb, 99, np.int8)
        gs, ss = got.struct(), self.src.struct()
        rc = lib.svt_b200_engine_dlf_cdef_frame_dev(e, C.byref(self.dp) if self.dp else None, self.flat, C.byref(self.sp), C.byref(self.dcp),
                                                    5, apply, C.byref(gs), C.byref(ss), cm.ptr(self.skip), self.skip.shape[1],
                                                    C.byref(dec), cm.ptr(idx))
        return rc, got, dec, idx

    def decision_matches(self, dec):
        n = self.want_dec.nb_cdef_strengths
        return ((dec.cdef_bits, dec.nb_cdef_strengths, dec.sb_count) == (self.want_dec.cdef_bits, n, self.want_dec.sb_count) and
                list(dec.y_strength)[:n] == list(self.want_dec.y_strength)[:n] and
                list(dec.uv_strength)[:n] == list(self.want_dec.uv_strength)[:n])


# 1920x1080 10-bit: the packed pictures (6.2 MB) are staged by the split host copy.  The ids of the first four cases
# predate the size parameter.
@pytest.mark.parametrize("w,h,bd,with_dlf,pick", [
    pytest.param(320, 200, 8, False, 3, id="8-False-3"), pytest.param(320, 200, 10, False, 3, id="10-False-3"),
    pytest.param(320, 200, 10, True, 2, id="10-True-2"), pytest.param(320, 200, 8, True, 3, id="8-True-3"),
    pytest.param(1920, 1080, 10, True, 3, id="1920x1080-10-True-3")])
def test_engine_cdef_frame_with_device_decision(w, h, bd, with_dlf, pick):
    """deblocking -> search -> svt_b200_cdef_decide (finish_cdef_search on the device) -> apply in ONE engine call: the
    decision, the per-filter-block choice and the filtered picture against the oracle chain."""
    lib = sb.load()
    c = CdefChain(w, h, bd, with_dlf, pick)
    e = C.c_void_p()
    sb.check(lib.svt_b200_engine_create(0, C.byref(e)), lib)
    try:
        rc, got, dec, idx = c.run(lib, e, 1)
        sb.check(rc, lib)
        assert c.decision_matches(dec)
        np.testing.assert_array_equal(idx, c.want_idx)
        assert c.want_idx[0] == -1 and (c.want_idx >= 0).any()
        for i in range(3):
            np.testing.assert_array_equal(got.plane(i), c.want.plane(i), err_msg=f"plane {i}")
        # apply = 0: decision only, the host picture untouched
        rc, again, dec, idx = c.run(lib, e, 0)
        sb.check(rc, lib)
        assert c.decision_matches(dec)
        np.testing.assert_array_equal(idx, c.want_idx)
        for i in range(3):
            np.testing.assert_array_equal(again.plane(i), c.rec.plane(i))
    finally:
        lib.svt_b200_engine_destroy(e)


@pytest.mark.parametrize("case", [(192, 136, 8, 1, 0, 3, (20, 24, 12, 9)), (128, 128, 10, 3, 0, 3, (40, 40, 33, 20)),
                                  (1920, 1080, 10, 4, 0, 3, (30, 26, 18, 12))])
def test_engine_dlf_pick_frame(case):
    """Level search + deblocking as one call: the levels equal the oracle's svt_av1_pick_filter_level, the picture equals the
    oracle's deblocking with those levels (sharpness 0)."""
    from test_dlf_gpu import flat_mi
    from test_oracle_dlf import dlf_params, pick_case, pick_params
    lib = sb.load()
    e = C.c_void_p()
    sb.check(lib.svt_b200_engine_create(0, C.byref(e)), lib)
    try:
        w, h, bd, seed, method, mode, last = case
        mi_rows, mi_cols, part, src, rec = pick_case(w, h, bd, seed)
        flat = flat_mi(mi_rows, mi_cols, part, last)
        p = pick_params(mi_rows, mi_cols, method, mode, last)
        r, t = rec.copy(), rec.copy()
        rs, ss, ts = r.struct(), src.struct(), t.struct()
        want_lv = (C.c_int32 * 4)()
        cm.oracle().orc_pick_filter_level(C.byref(p), C.byref(rs), C.byref(ss), C.byref(ts), flat, want_lv)
        got = rec.copy()
        gs = got.struct()
        lv = (C.c_int32 * 4)()
        sb.check(lib.svt_b200_engine_dlf_pick_frame(e, C.byref(p), C.byref(gs), C.byref(ss), flat, lv), lib)
        assert list(lv) == list(want_lv)
        flat2 = flat_mi(mi_rows, mi_cols, part, tuple(want_lv))
        dp = dlf_params(mi_rows, mi_cols, tuple(want_lv), 0)
        want = rec.copy()
        ws = want.struct()
        cm.oracle().orc_dlf_frame(C.byref(dp), C.byref(ws), flat2)
        for i in range(3):
            np.testing.assert_array_equal(got.plane(i), want.plane(i), err_msg=f"plane {i}")
    finally:
        lib.svt_b200_engine_destroy(e)


def lr_boundary_lines(dblk):
    """The deblocked lines above / below every stripe boundary as svt_av1_loop_restoration_save_boundary_lines keeps them
    (RestorationStripeBoundaries layout).  Returns the HostLrLines array and the numpy buffers it points into."""
    lines = (sb.HostLrLines * 3)()
    keep = []
    for pl in range(3):
        ss = 1 if pl else 0
        d = dblk.plane(pl)
        ph, pw = d.shape
        SH, off = 64 >> ss, 8 >> ss
        n_stripes = (ph + off + SH - 1) // SH
        stride = pw + 16
        above = np.zeros((2 * n_stripes, stride), d.dtype)
        below = np.zeros((2 * n_stripes, stride), d.dtype)
        for s in range(n_stripes):
            y0, y1 = max(0, s * SH - off), min((s + 1) * SH - off, ph)
            if s > 0:
                above[2 * s, :pw], above[2 * s + 1, :pw] = d[y0 - 2], d[y0 - 1]
            if y1 < ph:
                below[2 * s, :pw], below[2 * s + 1, :pw] = d[y1], d[min(y1 + 1, ph - 1)]
        keep += [above, below]
        lines[pl].above, lines[pl].below, lines[pl].stride = above.ctypes.data, below.ctypes.data, stride
    return lines, keep


def lr_frame_params(units, unit_sizes, ftypes):
    p = sb.LrFrameParams()
    for i in range(3):
        p.plane[i].frame_restoration_type, p.plane[i].restoration_unit_size = ftypes[i], unit_sizes[i]
        p.plane[i].units = C.addressof(units[i])
    p.optimized_lr = 0
    return p, (C.c_int32 * 3)(*[len(u) for u in units])


@pytest.mark.parametrize("case", [(192, 136, 8, 1, (64, 32, 32), ("mix", "mix", "mix"), (3, 3, 3)),
                                  (264, 200, 10, 3, (128, 64, 64), ("mix", "mix", "none"), (3, 3, 0)),
                                  (1920, 1080, 10, 5, (128, 64, 64), ("mix", "mix", "mix"), (3, 3, 3))])
def test_engine_lr_frame_from_boundary_lines(case):
    """The restoration frame filter fed the way rest_kernel feeds it: the CDEF picture plus the two deblocked lines above /
    below every 64-row stripe (RestorationStripeBoundaries layout), not the whole deblocked picture."""
    from test_oracle_lr_frame import lr_case, run_oracle_lr
    lib = sb.load()
    e = C.c_void_p()
    sb.check(lib.svt_b200_engine_create(0, C.byref(e)), lib)
    try:
        w, h, bd, seed, unit_sizes, modes, ftypes = case
        cdef, dblk, units = lr_case(w, h, bd, seed, unit_sizes, modes)
        want = run_oracle_lr(cdef, dblk, units, unit_sizes, ftypes, 0)
        lines, keep = lr_boundary_lines(dblk)
        p, n_units = lr_frame_params(units, unit_sizes, ftypes)
        got = cdef.copy()
        gs = got.struct()
        sb.check(lib.svt_b200_engine_lr_frame(e, C.byref(p), n_units, C.byref(gs), lines), lib)
        for i in range(3):
            exp = want.plane(i) if ftypes[i] else cdef.plane(i)
            np.testing.assert_array_equal(got.plane(i), exp, err_msg=f"plane {i}")
    finally:
        lib.svt_b200_engine_destroy(e)
