"""A submission a plain context refuses is refused by the multi-GPU contexts too (a one-GPU group, fq_create_multi, and a
world-1 rank context, fq_comm_init): with the same code and fq_last_error text, and before any output is written, so that
after fq_wait every output still holds its sentinel.  Each refusal sits in the last corridor where it can, runs on every
host entry it applies to (fq_replan_pairs, _assign, _window, sync and async), and afterwards every context still gives
the plain context's bytes for valid submissions."""
import ctypes as C

import numpy as np
import pytest

from faster_b200 import capi

import pair_shape_cases as psc

pytestmark = pytest.mark.gpu
E_ARG = -1
NW, NS, N_PROB = 6, 6, 5
CAP = 1 << 14                      # per-candidate outputs: more than any submission here has candidates
ENTRIES = ["pairs", "pairs_async", "assign", "assign_async", "window", "window_async"]
PAIR_OUT = ("results", "feasible_whole", "cost_whole", "feasible_safe", "cost_safe", "coeffs_whole", "coeffs_safe")
ASSIGN_OUT = ("cand_ofs_whole", "cand_ofs_safe", "sigma_whole", "sigma_safe")
SENTINEL = dict(results=0xAB, feasible_whole=0xCD, feasible_safe=0xCD, cost_whole=-5.0, cost_safe=-5.0, coeffs_whole=-3.0,
                coeffs_safe=-3.0, cand_ofs_whole=-7, cand_ofs_safe=-7, sigma_whole=0xCD, sigma_safe=0xCD, factor_whole=-2.0,
                factor_safe=-2.0, trials_whole=-9, trials_safe=-9, next_init_whole=-4.0, next_final_whole=-4.0,
                next_init_safe=-4.0, next_final_safe=-4.0)


def _family(entry):
    return entry.split("_")[0]


def _inputs(entry):
    w = psc.shared_workload(NW, NS, n=N_PROB) if _family(entry) == "pairs" else psc.mixed_workload(NW, NS, n=N_PROB)
    w = {k: (np.array(v) if isinstance(v, np.ndarray) else v) for k, v in w.items()}          # copies the rows may change
    win = {k: np.ascontiguousarray(v, np.float64) for k, v in psc.mixed_windows(N_PROB, 3).items()}
    return w, win


def _outputs(entry, n=N_PROB):
    out = dict(results=np.full(n * capi.PAIR_RESULT_DTYPE.itemsize, SENTINEL["results"], np.uint8),
               coeffs_whole=np.full(n * NW * 12, SENTINEL["coeffs_whole"]), coeffs_safe=np.full(n * NS * 12, SENTINEL["coeffs_safe"]))
    for k in ("feasible_whole", "feasible_safe"):
        out[k] = np.full(CAP, SENTINEL[k], np.uint8)
    for k in ("cost_whole", "cost_safe"):
        out[k] = np.full(CAP, SENTINEL[k])
    if _family(entry) != "pairs":
        out.update(cand_ofs_whole=np.full(n + 1, -7, np.int32), cand_ofs_safe=np.full(n + 1, -7, np.int32),
                   sigma_whole=np.full(n * NW, 0xCD, np.uint8), sigma_safe=np.full(n * NS, 0xCD, np.uint8))
    if _family(entry) == "window":
        for k in capi.WINDOW_OUT_KEYS:
            out[k] = np.full(n, SENTINEL[k], np.int32 if k.startswith("trials") else np.float64)
    return out


def _submit(h, entry, w, win, out):
    """One host entry on context h, then fq_wait.  -> (return code, fq_last_error text)."""
    L = capi.lib()
    fam = _family(entry)
    skip = {"pairs": (), "assign": ("sigmas_",), "window": ("sigmas_", "factors_")}[fam]
    a = capi.pair_args(w, lambda k: None if k.startswith(skip) else w[k].ctypes.data,
                       {k: v.ctypes.data for k, v in out.items() if k in PAIR_OUT})
    args = [h, C.byref(a)]
    if fam != "pairs":
        a.n_sig_whole = a.n_sig_safe = 0
        s = capi.assign_args(0, {k: out[k].ctypes.data for k in ASSIGN_OUT})
        args.append(C.byref(s))
    if fam == "window":
        a.n_fac_whole = a.n_fac_safe = 0
        wa = capi.window_args(lambda k: win[k].ctypes.data, {k: out[k].ctypes.data for k in capi.WINDOW_OUT_KEYS}, psc.INC, 20.0)
        args.append(C.byref(wa))
    fn = getattr(L, "fq_replan_pairs" + ("" if fam == "pairs" else "_" + fam) + ("_async" if entry.endswith("_async") else ""))
    rc = fn(*args)
    text = L.fq_last_error(h).decode()
    assert L.fq_wait(h) == 0
    return rc, text


# ---- the refusals: (name, families it applies to, expected message, change to (w, win, out))
def _nan_ab_row(w, win, out):
    w["Ab_whole"][w["face_ofs_whole"][w["poly_ofs_whole"][-2]], 1] = np.nan      # first face of the last corridor


def _nan_xf(w, win, out):
    w["xf_safe"][-1, 0] = np.nan


def _zero_limit(w, win, out):
    w["lim"][-1, 1] = 0.0


def _descending_factors(w, win, out):
    w["factors_safe"] = np.ascontiguousarray(w["factors_safe"][::-1])


def _feasible_without_cost(w, win, out):
    del out["cost_whole"]


def _poly_ofs_from_one(w, win, out):
    # the same corridors behind an empty polytope 0: a rebased copy of it is valid, the description is not
    w["poly_ofs_whole"] = w["poly_ofs_whole"] + 1
    w["face_ofs_whole"] = np.concatenate([[0], w["face_ofs_whole"]]).astype(np.int32)


def _face_ofs_from_four(w, win, out):
    w["face_ofs_safe"] = w["face_ofs_safe"] + 4
    w["Ab_safe"] = np.concatenate([np.zeros((4, 4)), w["Ab_safe"].reshape(-1, 4)])


def _zero_window_init(w, win, out):
    win["init_whole"][-1] = 0.0


def _shared_entry_past_p(w, win, out):
    w["sigmas_whole"][-1, -1] = w["poly_ofs_whole"][N_PROB] - w["poly_ofs_whole"][N_PROB - 1]


ROWS = [
    ("nan_in_Ab_whole", ("pairs", "assign", "window"), "non-finite value in Ab", _nan_ab_row),
    ("nan_in_xf_safe", ("pairs", "assign", "window"), "non-finite value in x0/xf", _nan_xf),
    ("limit_zero", ("pairs", "assign", "window"), "limits and factors must be finite and > 0", _zero_limit),
    ("descending_factors_safe", ("pairs", "assign"), "factors_* must be ascending", _descending_factors),
    ("feasible_whole_without_cost", ("pairs", "assign", "window"), "feasible_* and cost_* must be given", _feasible_without_cost),
    ("poly_ofs_whole_from_1", ("pairs", "assign", "window"), "offset arrays must start at 0", _poly_ofs_from_one),
    ("face_ofs_safe_from_4", ("pairs", "assign", "window"), "offset arrays must start at 0", _face_ofs_from_four),
    ("window_init_zero", ("window",), "time-allocation window refused", _zero_window_init),
    ("shared_entry_past_P", ("pairs",), "sigmas_* entry >= number of polytopes", _shared_entry_past_p),
]


@pytest.fixture(scope="module")
def contexts(solver):
    """plain: the session's context; group: fq_create_multi over device 0; rank: a world-1 communicator (None when NCCL
    does not load)."""
    import torch                     # brings torch's NCCL into the process for fq_comm_init's dlopen
    assert torch.cuda.is_available()
    group = capi.Solver(n_gpus=1, devices=[0])
    rank = capi.Solver(0)
    try:
        rank.comm_init(capi.comm_unique_id(), 0, 1)
    except capi.FqError:
        rank.close()
        rank = None
    yield dict(plain=solver, group=group, rank=rank)
    group.close()
    if rank is not None:
        rank.close()


def _context(contexts, kind):
    if contexts[kind] is None:
        pytest.skip("NCCL does not load: no rank context")
    return contexts[kind]


@pytest.mark.parametrize("kind", ["plain", "group", "rank"])
@pytest.mark.parametrize("row", ROWS, ids=[r[0] for r in ROWS])
def test_every_context_refuses_what_a_plain_context_refuses(contexts, kind, row):
    name, families, why, change = row
    ctx = _context(contexts, kind)
    for entry in ENTRIES:
        if _family(entry) not in families:
            continue
        w, win = _inputs(entry)
        out = _outputs(entry)
        change(w, win, out)
        rc0, text0 = _submit(contexts["plain"]._h, entry, w, win, out)
        assert rc0 == E_ARG and why in text0, (entry, text0)
        rc, text = _submit(ctx._h, entry, w, win, out)
        assert rc == E_ARG, (kind, entry)
        assert text == text0, (kind, entry)
        for k, v in out.items():
            assert (v == SENTINEL[k]).all(), (kind, entry, k)


@pytest.mark.parametrize("kind", ["group", "rank"])
def test_every_context_still_gives_the_plain_bytes(contexts, kind):
    ctx = _context(contexts, kind)
    for entry in ENTRIES:
        w, win = _inputs(entry)
        ref, got = _outputs(entry), _outputs(entry)
        assert _submit(contexts["plain"]._h, entry, w, win, ref)[0] == 0, entry
        assert _submit(ctx._h, entry, w, win, got)[0] == 0, (kind, entry)
        assert (np.frombuffer(ref["results"].tobytes(), capi.PAIR_RESULT_DTYPE)["whole_dt_index"] >= 0).any(), entry
        for k in ref:
            assert got[k].tobytes() == ref[k].tobytes(), (kind, entry, k)


def _missing_polytope_workload():
    """Two corridors with P = {0, 1} and a shared whole list whose entry 1 names a polytope the first corridor lacks.  A
    plain context skips the entry bound when some corridor has no polytope; a shard holding only the second corridor
    applies it."""
    seeds = (62000, 62001)
    whole = [psc._corridor(s, p, NW, True) for s, p in zip(seeds, (0, 1))]
    safe = [psc._corridor(s, p, NS, False) for s, p in zip(seeds, (0, 1))]
    sw = np.array([[0] * NW, [0] * (NW - 2) + [1, 1]], np.uint8)
    return capi.make_pair_workload(whole, safe, psc.FACTORS, sw, psc.FACTORS, np.zeros((1, NS), np.uint8), DC=0.01)


def test_a_shard_check_refuses_a_shared_entry_the_whole_batch_lets_through(contexts):
    w = _missing_polytope_workload()
    # one shard of both corridors: accepted as on a plain context, with its bytes
    for kind in ("group", "rank"):
        if contexts[kind] is None:
            continue
        for entry in ("pairs", "pairs_async"):
            ref, got = _outputs(entry, 2), _outputs(entry, 2)
            assert _submit(contexts["plain"]._h, entry, w, None, ref)[0] == 0, entry
            assert _submit(contexts[kind]._h, entry, w, None, got)[0] == 0, (kind, entry)
            for k in ref:
                assert got[k].tobytes() == ref[k].tobytes(), (kind, entry, k)
    # two shards, [0, 1) and [1, 2): the second refuses the entry, before anything is written
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs: only a split batch checks the shard [1, 2) on its own")
    g = capi.Solver(n_gpus=2, devices=[0, 1])
    try:
        for entry in ("pairs", "pairs_async"):
            out = _outputs(entry, 2)
            rc, text = _submit(g._h, entry, w, None, out)
            assert rc == E_ARG and "sigmas_* entry >= number of polytopes" in text, (entry, text)
            for k, v in out.items():
                assert (v == SENTINEL[k]).all(), (entry, k)
    finally:
        g.close()
