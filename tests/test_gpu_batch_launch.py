"""Batched launches the way the benchmark's batch legs call them: the split upload / resident solve / download calls, batches
longer than the device has SMs (so a CTA team solves a second graph after its first), graphs of different shapes, kinds and
settings in one call, and the host-side refusals of malformed batches and of stale uploads.

A launch has one team size and one barrier kind, and whether the block-resident PCG loop runs depends only on the graph and
that team size; so two handles holding the same graph do the same arithmetic wherever they sit in a batch, and their
results must agree bit for bit.  Only their wave, their team and the graph their team solved before them differ."""
import ctypes as C

import numpy as np
import pytest

import oracle_api as O
from oracle_api import OracleAPI
from pop_up_slam_b200 import capi, graphgen as gg
from pop_up_slam_b200.capi import GpuGraphAPI

TOL = 1e-4   # BASELINE.json north_star: final chi2 and estimates within 1e-4 relative
TRACE_KEYS = ("chi2_new", "lam", "accepted", "pcg")


def compare(gpu, orc, ig, io, tol=TOL):
    c_g, c_o = gpu.chi2(), orc.chi2()
    assert abs(c_g - c_o) <= tol * max(abs(c_o), 1e-9), (c_g, c_o)
    P_g, P_o = gpu.get_poses(ig["pose_ids"]), orc.get_poses(io["pose_ids"])
    scale = max(1.0, np.abs(P_o[:, :3]).max())
    assert np.abs(P_g[:, :3] - P_o[:, :3]).max() <= tol * scale
    sq = np.sign(np.sum(P_g[:, 3:] * P_o[:, 3:], axis=1))[:, None]
    assert np.abs(P_g[:, 3:] * sq - P_o[:, 3:]).max() <= tol
    if len(ig["plane_ids"]):
        L_g, L_o = gpu.get_planes(ig["plane_ids"]), orc.get_planes(io["plane_ids"])
        sl = np.sign(np.sum(L_g * L_o, axis=1))[:, None]
        assert np.abs(L_g * sl - L_o).max() <= tol


def num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def set_flags(a, flags):
    o = a.get_solver_options()
    o.reserved[2] = flags
    a._chk(a.lib.pus_set_solver_options(a.h, C.byref(o)))


# A graph and its per-handle settings.  props: Properties overrides; robust: (kind, b); numeric: the reference's
# numerical-difference Jacobians; kind / order: linear solver and direct ordering; flags: solver option reserved[2].
def spec(g, props=None, robust=None, numeric=False, kind=0, order=0, flags=0):
    return dict(g=g, props=props or {}, robust=robust, numeric=numeric, kind=kind, order=order, flags=flags)


def make(sp):
    a = GpuGraphAPI()
    ids = gg.build_bulk(a, sp["g"])
    gg.configure(a, sp["g"], **sp["props"])
    if sp["robust"] is not None:
        a.set_robust(*sp["robust"])
    if sp["numeric"]:
        a.set_jacobian_mode(0)
    if sp["kind"]:
        a.set_linear_solver(sp["kind"])
    if sp["order"]:
        a.set_direct_ordering(sp["order"])
    if sp["flags"]:
        set_flags(a, sp["flags"])
    return a, ids


def oracle(sp):
    o = OracleAPI()
    o.set_jacobian_mode(0 if sp["numeric"] else 1)
    io = gg.build_bulk(o, sp["g"])
    gg.configure(o, sp["g"], **sp["props"])
    if sp["robust"] is not None:
        o.set_robust(*sp["robust"])
    o.batch_optimize()
    return o, io


def reset_values(a, ids, g):
    """back to the generator's initial estimate (a download leaves the solution in the host values)"""
    a.init_poses(ids["pose_ids"], g.poses_init)
    a.init_planes(ids["plane_ids"], g.planes_init)


def result(a, ids):
    t, st = a.trace(), a.stats()
    r = dict(P=a.get_poses(ids["pose_ids"]), L=a.get_planes(ids["plane_ids"]), it=st["lm_iterations"],
             chi2=st["chi2_final"])
    r.update({k: t[k] for k in TRACE_KEYS})
    return r


def assert_bits(r, s, what=""):
    for k in r:
        assert np.array_equal(r[k], s[k]), (what, k, r[k], s[k])


def assert_close(r, s, what=""):
    """the bars of a batched solve against a solo solve of the same graph: the team shapes differ, so the reductions of the
    chi2 and |delta| run in another order (include/popup_gpu.h): same iterations and accept sequence, chi2 within 1e-9
    relative, estimates within 1e-8"""
    assert r["it"] == s["it"], what
    assert np.array_equal(r["accepted"], s["accepted"]), what
    assert abs(r["chi2"] - s["chi2"]) <= 1e-9 * abs(s["chi2"]), (what, r["chi2"], s["chi2"])
    assert np.abs(r["P"] - s["P"]).max() < 1e-8, what
    if len(s["L"]):
        assert np.abs(r["L"] - s["L"]).max() < 1e-8, what


def solo(sp):
    a, ids = make(sp)
    a.batch_optimize()
    return result(a, ids)


_ORACLES = {}


def check_oracle(key, sp, a, ids):
    if key not in _ORACLES:
        _ORACLES[key] = oracle(sp)
    o, io = _ORACLES[key]
    compare(a, o, ids, io)


# ------------------------------------------------------------------------------------------------------------------------
# (a) copies of one graph in a batch longer than the SM count
# ------------------------------------------------------------------------------------------------------------------------
def graph_a():   # 300-pose corridor: 19 pose blocks, the three-level preconditioner forced on PCG handles
    return gg.make_config(2, seed=2)


def graph_b():   # 64-pose corridor: 4 pose blocks, two levels (the block-resident loop can run it)
    return gg.make_config(2, seed=5, n_poses=64, n_planes=16)


MODES = {
    "default": (dict(flags=8), dict()),
    "global_barrier": (dict(flags=8 | 1 << 16), dict(flags=1 << 16)),   # reserved[2] bit 16: no cluster teams
    "general_loop": (dict(flags=8 | 32), dict(flags=32)),               # bit 5: never the block-resident loop
    "direct": (dict(kind=2, order=1), dict(kind=1)),                    # band solve in ND order / dense direct solve
}


@pytest.mark.gpu
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("layout", ["ABA", "BAB"])
def test_copies_of_one_graph_agree_across_waves(layout, mode):
    """[A] + [B]*(n-2) + [A] and [B] + [A]*(n-2) + [B] with n = SMs + 2: teams never outnumber SMs, so some team solves a second
    graph after its first (the team that solved A then solves a B, and the other way round).  Every copy of a graph gives the
    same bits -- estimates, iterations and the whole LM trace -- and one copy of each is checked against the oracle."""
    sms = num_sms()
    n = sms + 2
    ka, kb = MODES[mode]
    specs = {"A": spec(graph_a(), **ka), "B": spec(graph_b(), **kb)}
    outer, inner = layout[0], layout[1]
    names = [outer] + [inner] * (n - 2) + [outer]
    handles = [make(specs[k]) for k in names]
    its = capi.batch_optimize_many([a for a, _ in handles])
    st0 = handles[0][0].stats()
    assert st0["grid_ctas"] <= sms < n, (st0["grid_ctas"], sms, n)   # a second wave is certain
    first = {}
    for i, (k, (a, ids)) in enumerate(zip(names, handles)):
        r = result(a, ids)
        assert its[i] == r["it"]
        assert a.stats()["n_poses"] == specs[k]["g"].n_poses
        if k in first:
            assert_bits(r, first[k][0], (layout, mode, k, i))
        else:
            first[k] = (r, a, ids)
    assert first["A"][0]["it"] > 0 and first["B"][0]["it"] > 0
    assert first["A"][0]["P"].shape != first["B"][0]["P"].shape
    for k in ("A", "B"):
        _, a, ids = first[k]
        check_oracle(k, specs[k], a, ids)


# ------------------------------------------------------------------------------------------------------------------------
# (b) one batch mixing kinds, shapes and settings
# ------------------------------------------------------------------------------------------------------------------------
def mixed_specs():
    return [
        spec(gg.make_config(2, seed=2, n_poses=160, n_planes=32)),                                   # PCG, LM, 10 blocks
        spec(gg.make_config(1, seed=3), props=dict(method=0), numeric=True),                         # PCG, GN, one block
        spec(gg.make_config(2, seed=4, n_poses=48, n_planes=12), robust=(1, 1.0),
             props=dict(max_iterations=5)),                                                          # PCG, Huber, capped
        spec(gg.make_config(2, seed=6, n_poses=96, n_planes=20), kind=1, numeric=True),              # dense direct
        spec(gg.make_config(2, seed=7, n_poses=64, n_planes=16), kind=2, robust=(1, 1.0),
             props=dict(max_iterations=7)),                                                          # band direct
    ]


@pytest.mark.gpu
def test_mixed_batch_gives_each_handle_its_own_answer():
    """SMs + 2 handles of five graphs in turn: PCG, dense-direct and band handles (two launches), a one-block graph
    smaller than the team (CTAs that own no block), GN and LM, Huber and none, numeric and closed-form Jacobians and
    different iteration caps.  Copies agree bit for bit; every handle's statistics, iteration count and result are its own
    graph's (a solo solve of it)."""
    sms = num_sms()
    n = sms + 2
    specs = mixed_specs()
    which = np.arange(n) % len(specs)   # (neighbours in each launch hold different graphs)
    handles = [make(specs[k]) for k in which]
    its = capi.batch_optimize_many([a for a, _ in handles])
    ref = [solo(sp) for sp in specs]
    assert len({r["it"] for r in ref}) > 1 and len({r["chi2"] for r in ref}) == len(specs)
    first = {}
    for i, (k, (a, ids)) in enumerate(zip(which, handles)):
        st = a.stats()
        g = specs[k]["g"]
        assert (st["n_poses"], st["n_planes"]) == (g.n_poses, g.n_planes), (i, k)
        r = result(a, ids)
        assert its[i] == st["lm_iterations"] == ref[k]["it"], (i, k)
        assert abs(st["chi2_final"] - ref[k]["chi2"]) <= 1e-9 * abs(ref[k]["chi2"]), (i, k)
        assert_close(r, ref[k], (i, k))
        if k in first:
            assert_bits(r, first[k], (i, k))
        else:
            first[k] = r
    assert len(first) == len(specs)


# ------------------------------------------------------------------------------------------------------------------------
# (c) the split calls against the one-shot call
# ------------------------------------------------------------------------------------------------------------------------
def split_specs():
    return [
        spec(graph_b()),
        spec(gg.make_config(2, seed=2, n_poses=160, n_planes=32)),
        spec(gg.make_config(2, seed=6, n_poses=96, n_planes=20), kind=1),
        spec(gg.make_config(2, seed=7, n_poses=64, n_planes=16), kind=2, order=1),
    ]


def add_loop_closure(a, ids, g, i=0, j=20):
    """a structural edit: an odometry factor between poses i and j, measured from the true poses"""
    meas = O.pose_vector(O.pose_ominus(g.poses_truth[j], g.poses_truth[i]))
    return a.add_odometry(int(ids["pose_ids"][i]), int(ids["pose_ids"][j]), meas, g.odo_sqrtinf[0])


@pytest.mark.gpu
def test_split_calls_match_the_one_shot_call():
    """upload_many, three solve_resident_many, download_many on one set of handles; batch_optimize_many on a second set built
    the same way: the same bits.  Then a factor is added to one graph, the values reset and the set uploaded and solved
    again: the edited graph gives what a fresh set with the same edit gives, the others what they gave before."""
    specs = split_specs()
    one = [make(sp) for sp in specs]
    two = [make(sp) for sp in specs]
    apis = [a for a, _ in one]
    capi.upload_many(apis)
    runs = []
    for _ in range(3):
        its = capi.solve_resident_many(apis)
        runs.append((its.copy(), [a.stats()["chi2_final"] for a in apis]))
    for its, chi in runs[1:]:
        assert np.array_equal(its, runs[0][0]) and chi == runs[0][1]
    capi.download_many(apis)
    its2 = capi.batch_optimize_many([a for a, _ in two])
    assert np.array_equal(runs[0][0], its2)
    before = []
    for (a, ids), (b, idb) in zip(one, two):
        r = result(a, ids)
        assert_bits(r, result(b, idb))
        before.append(r)
    # structural edit of one graph, then the split route again from the initial values
    k = 1
    add_loop_closure(*one[k], specs[k]["g"])
    for sp, (a, ids) in zip(specs, one):
        reset_values(a, ids, sp["g"])
    capi.upload_many(apis)
    its = capi.solve_resident_many(apis)
    capi.download_many(apis)
    fresh = [make(sp) for sp in specs]
    add_loop_closure(*fresh[k], specs[k]["g"])
    its3 = capi.batch_optimize_many([a for a, _ in fresh])
    assert np.array_equal(its, its3)
    for i, ((a, ids), (b, idb)) in enumerate(zip(one, fresh)):
        r = result(a, ids)
        assert_bits(r, result(b, idb), i)
        if i != k:
            assert_bits(r, before[i], i)
    assert np.abs(result(*one[k])["P"] - before[k]["P"]).max() > 0   # (the loop closure moved the solution)


# ------------------------------------------------------------------------------------------------------------------------
# (d) the benchmark's batch64 leg
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_batch64_leg_matches_solo_solves_and_oracle():
    """64 config-2 graphs (seeds 0-63) on one shared stream, as bench.py's batch64 leg runs them: upload_many,
    solve_resident_many, download_many.  Each graph against its own solo solve (the bars of assert_close), 8 against the
    oracle at BASELINE's 1e-4."""
    import torch
    stream = torch.cuda.Stream()
    specs = [spec(gg.make_config(2, seed=s)) for s in range(64)]
    handles = []
    for sp in specs:
        a, ids = make(sp)
        a.set_stream(stream.cuda_stream)
        handles.append((a, ids))
    apis = [a for a, _ in handles]
    capi.upload_many(apis)
    its = capi.solve_resident_many(apis)
    capi.download_many(apis)
    for s, (sp, (a, ids)) in enumerate(zip(specs, handles)):
        r = result(a, ids)
        assert its[s] == r["it"]
        assert_close(r, solo(sp), s)
    for s in range(0, 64, 8):
        o, io = oracle(specs[s])
        compare(handles[s][0], o, handles[s][1], io)


# ------------------------------------------------------------------------------------------------------------------------
# (e) stream borrowing and the batch scratch
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_handles_get_their_streams_back_after_a_batch():
    """a batch runs on the first handle's stream; afterwards the others have their own again: with the first handle destroyed,
    a solo solve of one of them and a batch of the rest still run and give what the first batch gave"""
    specs = split_specs()[:2] * 2 + [spec(graph_a())]
    handles = [make(sp) for sp in specs]
    capi.batch_optimize_many([a for a, _ in handles])
    before = [result(a, ids) for a, ids in handles]
    handles[0][0].close()
    for sp, (a, ids) in zip(specs[1:], handles[1:]):
        reset_values(a, ids, sp["g"])
    a, ids = handles[1]
    a.batch_optimize()
    assert_close(result(a, ids), before[1], 1)
    capi.batch_optimize_many([a for a, _ in handles[2:]])
    for i in range(2, len(handles)):
        assert_close(result(*handles[i]), before[i], i)


@pytest.mark.gpu
def test_batch_scratch_grows_under_one_first_handle():
    """three batches led by the same handle, of 3, SMs + 2 and 2 graphs: the first handle's batch parameter and result arrays
    grow at the second; every batch's answers are those of solo solves"""
    sms = num_sms()
    sb, sc = spec(graph_b()), spec(gg.make_config(2, seed=9, n_poses=48, n_planes=12))
    ref = {"b": solo(sb), "c": solo(sc)}
    lead = make(sb)
    for n in (3, sms + 2, 2):
        reset_values(*lead, sb["g"])
        names = ["b"] + ["c" if i % 2 else "b" for i in range(1, n)]
        rest = [make(sb if k == "b" else sc) for k in names[1:]]
        handles = [lead] + rest
        its = capi.batch_optimize_many([a for a, _ in handles])
        for i, (k, (a, ids)) in enumerate(zip(names, handles)):
            r = result(a, ids)
            assert its[i] == r["it"]
            assert_close(r, ref[k], (n, i))
        del rest, handles


# ------------------------------------------------------------------------------------------------------------------------
# refusals of stale uploads (GPU: an upload needs the device)
# ------------------------------------------------------------------------------------------------------------------------
STALE = "graph changed since its upload: call pus_upload"


@pytest.mark.gpu
@pytest.mark.parametrize("edit", ["add_factor", "remove_factor", "linear_solver", "direct_ordering"])
def test_resident_solve_and_download_refuse_a_stale_upload(edit):
    """after a structural edit, a switch of linear-solver kind or of direct ordering, the resident solve and the download of
    the uploaded handle (alone or in a batch) are refused and launch nothing: every handle's statistics and host values stay
    as they were; a new upload makes the handle usable again"""
    g = graph_b()
    sp = spec(g, kind=2 if edit == "direct_ordering" else 0)
    a, ids = make(sp)
    b, idb = make(sp)
    a.upload()
    a.solve_resident()
    a.download()
    capi.upload_many([b])
    capi.solve_resident_many([b])
    capi.download_many([b])
    st_a, st_b = a.stats(), b.stats()
    P_a = a.get_poses(ids["pose_ids"])
    if edit == "add_factor":
        add_loop_closure(a, ids, g, 0, 30)
    elif edit == "remove_factor":
        a.remove_factor(int(ids["pp_fids"][5]))
    elif edit == "linear_solver":
        a.set_linear_solver(1)
    else:
        a.set_direct_ordering(1)
    calls = [a.solve_resident, a.download, lambda: capi.solve_resident_many([b, a]),
             lambda: capi.solve_resident_many([a, b]), lambda: capi.download_many([b, a])]
    for call in calls:
        with pytest.raises(capi.ApiError, match=STALE):
            call()
    assert a.stats() == st_a and b.stats() == st_b
    assert np.array_equal(a.get_poses(ids["pose_ids"]), P_a)
    reset_values(a, ids, g)
    a.upload()
    assert a.solve_resident() > 0
    a.download()


@pytest.mark.gpu
def test_resident_solve_starts_from_the_uploaded_snapshot():
    """value and measurement changes after an upload do not make it stale: the resident solve starts again from the uploaded
    estimate with the uploaded measurements (same bits as before) and the download overwrites the new host values; the next
    upload takes them in, giving what a fresh handle built with them gives"""
    g = graph_b()
    sp = spec(g)
    a, ids = make(sp)
    a.upload()
    a.solve_resident()
    a.download()
    r0 = result(a, ids)
    rng = np.random.default_rng(3)
    P1 = g.poses_init.copy()
    P1[:, :3] += rng.normal(0, 0.01, size=(g.n_poses, 3))
    fid = int(ids["pp_fids"][7])
    m1 = O.plane_exmap(a.get_measurement(fid), [0.01, -0.02, 0.005])
    a.init_poses(ids["pose_ids"], P1)
    a.set_measurement(fid, m1)
    assert a.solve_resident() == r0["it"]
    a.download()
    assert_bits(result(a, ids), r0)
    a.init_poses(ids["pose_ids"], P1)
    a.init_planes(ids["plane_ids"], g.planes_init)
    a.upload()
    a.solve_resident()
    a.download()
    r1 = result(a, ids)
    assert np.abs(r1["P"] - r0["P"]).max() > 0
    b, idb = make(sp)
    b.init_poses(idb["pose_ids"], P1)
    b.set_measurement(fid, m1)
    b.upload()
    b.solve_resident()
    b.download()
    assert_bits(r1, result(b, idb))


# ------------------------------------------------------------------------------------------------------------------------
# refusals of malformed batches (host only: no device is needed, and none is touched)
# ------------------------------------------------------------------------------------------------------------------------
def _many_calls(lib):
    its = np.zeros(8, dtype=np.int32)
    ip = its.ctypes.data_as(capi.c_int_p)
    return {
        "pus_upload_many": lambda hs, n: lib.pus_upload_many(hs, n),
        "pus_solve_resident_many": lambda hs, n: lib.pus_solve_resident_many(hs, n, ip),
        "pus_download_many": lambda hs, n: lib.pus_download_many(hs, n),
        "pus_batch_optimize_many": lambda hs, n: lib.pus_batch_optimize_many(hs, n, ip),
        "pus_span_emulate_optimize": lambda hs, n: lib.pus_span_emulate_optimize(hs, n, ip),
    }


def _error(lib):
    lib.pus_last_error.restype = C.c_char_p
    return lib.pus_last_error().decode()


def _small_handles(k):
    g = gg.make_config(1, seed=0)
    out = []
    for _ in range(k):
        a = GpuGraphAPI()
        gg.build_bulk(a, g)
        gg.configure(a, g)
        out.append(a)
    return out


def test_batched_calls_refuse_a_null_array():
    lib = capi.load_library()
    for name, call in _many_calls(lib).items():
        assert call(None, 2) == -1, name
        assert _error(lib) == name + ": null handle array"


@pytest.mark.parametrize("pos", [0, 1, 2])
def test_batched_calls_refuse_a_null_entry(pos):
    apis = _small_handles(3)
    lib = apis[0].lib
    hs = [a.h for a in apis]
    hs[pos] = None
    arr = (C.c_void_p * 3)(*hs)
    for name, call in _many_calls(lib).items():
        assert call(arr, 3) == -1, name
        assert _error(lib) == f"{name}: handle {pos} is null"


@pytest.mark.parametrize("pair", [(0, 1), (0, 2), (1, 2)])
def test_batched_calls_refuse_a_repeated_handle(pair):
    apis = _small_handles(3)
    lib = apis[0].lib
    hs = [a.h for a in apis]
    hs[pair[1]] = hs[pair[0]]
    arr = (C.c_void_p * 3)(*hs)
    for name, call in _many_calls(lib).items():
        assert call(arr, 3) == -1, name
        assert _error(lib) == f"{name}: handles {pair[0]} and {pair[1]} are the same handle"
    for name in ("upload_many", "solve_resident_many", "download_many", "batch_optimize_many"):   # through the binding
        with pytest.raises(capi.ApiError, match="are the same handle"):
            getattr(capi, name)([apis[0], apis[1], apis[0]])


def test_batched_calls_accept_an_empty_batch():
    lib = capi.load_library()
    calls = _many_calls(lib)
    for name in ("pus_upload_many", "pus_solve_resident_many", "pus_download_many", "pus_batch_optimize_many"):
        for n in (0, -1):
            assert calls[name](None, n) == 0, (name, n)


def test_split_calls_refuse_a_graph_never_uploaded():
    """refused as such before any device work (so also where there is no GPU)"""
    a, b = _small_handles(2)
    for call in (a.solve_resident, a.download, lambda: capi.solve_resident_many([a, b]), lambda: capi.download_many([a, b])):
        with pytest.raises(capi.ApiError, match="graph not uploaded"):
            call()
