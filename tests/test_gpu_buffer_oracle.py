"""GPU: buffered packing (PctBatch(..., buffer=B); DESIGN.md section 18) in lock-step with the buffered env on the oracle
(tests/buffer_oracle.py), which predicts the whole trajectory on the CPU: the items by the refill rule, every slot's leaf block with
Oracle*.set_next, the choices by pct_buffer_policy_random restated.

After the reset and after every step, for every env in lock-step: every byte of the observation (internal rows, all B leaf blocks, the item
rows), buffer_items(), reward, done, counter, the record's flags exactly, the summed n_leaf / n_cand, and at the end a sample of support
graphs.  Unlike the composition twin of tests/test_gpu_buffer.py, the slots the step did not choose are held against an independent
reference too, and so are the flags of their expansions.  An env whose record carries a capacity flag leaves the lock-step (the kernels
have capacities the oracle has none of): its flags must stay set until buffer_reset_envs clears them, and from that reset on it is in
lock-step again."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
from buffer_oracle import MS_CHECK, MS_N, MS_PSEED, MS_STEPS, BufferedOracle, capacity_steps, config, many_support_config, \
    many_support_model, many_support_starts  # noqa: E402
from harness import FLAG_CAND, FLAG_EMS, case_stream, compare_graphs, cont_case_stream, load_capacity_cases  # noqa: E402

pytestmark = pytest.mark.gpu
PSEED = 61
HOLD = 2  # steps a flagged env keeps running before buffer_reset_envs


def _np(t):
    return t.cpu().numpy().copy()


def _batch(c, streams, B, obs_dtype):
    import pct_b200
    cont = c["domain"] == "continuous"
    return pct_b200.PctBatch(len(streams), c["setting"], container_size=c["container"], continuous=cont,
                             item_set=None if cont else c.get("items"), internal_node_holder=c["nb"], leaf_node_holder=c["nl"], obs_dtype=obs_dtype,
                             item_stream=np.stack(streams), size_minimum=c["size_minimum"], LNES=c.get("lnes", "EMS"), buffer=B)


def _check_obs(got, m, npd, where):
    want = m.obs.astype(npd)
    if np.array_equal(got.view(np.uint8), want.view(np.uint8)):
        return
    nb, nl, B = m.nb, m.nl, m.B
    g, w = got.reshape(-1, 9), want.reshape(-1, 9)
    bad = int(np.nonzero((g.view(np.uint8) != w.view(np.uint8)).reshape(len(g), -1).any(1))[0][0])
    part = "internal row %d" % bad if bad < nb else ("slot %d leaf %d" % divmod(bad - nb, nl) if bad < nb + B * nl else "item row %d" % (bad - nb - B * nl))
    raise AssertionError("%s: observation differs first at %s: %s, oracle %s" % (where, part, g[bad].tolist(), w[bad].tolist()))


def lockstep(c, streams, B, steps, obs_dtype=torch.float64, graphs=4, pseed=PSEED, models=None, restore=None):
    """streams[e] drives env e of a buffered batch and its model; pct_buffer_policy_random (seed pseed) chooses.  -> per env, the (step, flag
    bits) of every flag its records carried (step -1: the start).  models: per env a BufferedOracle already in the state the batch starts
    from, or None (an env that is only required to raise no flag); restore(P): puts the reset batch into that state and returns its
    observation (default: every env starts from its model's reset)"""
    n = len(streams)
    npd = np.float64 if obs_dtype == torch.float64 else np.float32
    P = _batch(c, streams, B, obs_dtype)
    rinfo = torch.zeros((n, 8), dtype=torch.int32, device=P.device)
    o = _np(P.reset(info=rinfo))
    fl = P.decode_info(rinfo)["flags"]
    if restore is None:
        models = [BufferedOracle(c, s, B) for s in streams]
        for m in models:
            m.reset()
    else:
        o = _np(restore(P))
        fl = np.array([P.state(e)["flags"] if models[e] is not None else 0 for e in range(n)])
    held = np.full(n, -1)  # step at which the env left the lock-step; -1: in lock-step
    held_bits = np.zeros(n, dtype=np.int64)
    fired = [[] for _ in range(n)]

    def enter(e, t, flags, where):
        """an env's model was just reset (t: the step after which) and its device env too: compare, or hold it on a flag"""
        m = models[e]
        assert flags == m.sticky, "%s: flags %d, the oracle's counts call for %d (slots %s)" % (where, flags, m.sticky, m.slot_fl.tolist())
        if m.sticky:
            fired[e].append((t, m.sticky))
            held[e], held_bits[e] = t, m.sticky
        else:
            _check_obs(o[e], m, npd, where)

    items = _np(P.buffer_items())
    for e in range(n):
        if models[e] is None:
            continue
        enter(e, -1, int(fl[e]), "env %d: %s" % (e, "reset" if restore is None else "restored"))
        if held[e] < 0:
            assert np.array_equal(items[e], models[e].buf), "env %d: buffered items after the reset" % e
    t_dev = torch.zeros((), dtype=torch.int64, device=P.device)
    dev_done = np.zeros(n, dtype=bool)  # a held env's device episode ended (its auto-reset clears the flags)
    for t in range(steps):
        flat = P.random_policy_dev(pseed, t_dev).clone()
        f = _np(flat)
        ob, r, d, info = P.step(leaf_idx=flat)
        t_dev += 1
        o, r, d = _np(ob), _np(r), _np(d).astype(bool)
        inf = P.decode_info(info)
        items = _np(P.buffer_items())
        reset = []
        for e in range(n):
            where = "env %d step %d" % (e, t)
            m = models[e]
            if m is None:
                assert inf["flags"][e] == 0, "%s: flags %d" % (where, inf["flags"][e])
                continue
            if held[e] >= 0:
                dev_done[e] |= d[e]
                if not dev_done[e]:
                    assert inf["flags"][e] & held_bits[e] == held_bits[e], "%s: flags %d lost bits of %d before the reset" % (where, inf["flags"][e], held_bits[e])
                if t - held[e] >= HOLD:
                    reset.append(e)
                continue
            assert f[e] == m.policy(pseed, e, t), where + ": the random policy's flat index"
            _, rr, dd, rec = m.step(int(f[e]))
            # an EMS overflow of the placement leaves the device a truncated EMS list, from which the slots' candidate lists are built: their
            # candidate bit of that step is the device's own
            free = FLAG_CAND if rec["placement_flags"] & FLAG_EMS else 0
            assert inf["flags"][e] & ~free == rec["flags"] & ~free, "%s: flags %d, the oracle's counts call for %d (placement %d, slots %s)" % (
                where, inf["flags"][e], rec["flags"], rec["placement_flags"], rec["slot_flags"].tolist())
            assert d[e] == dd, where + ": done"
            if rec["flags"]:
                fired[e].append((t, rec["flags"]))
            if m.sticky:  # a capacity flag the env still carries: its rows are not the oracle's any more
                held[e], held_bits[e], dev_done[e] = t, m.sticky & ~free, False
                continue
            _check_obs(o[e], m, npd, where)
            assert np.array_equal(items[e], m.buf), where + ": buffered items"
            assert r[e] == np.float32(rr) and inf["counter"][e] == rec["counter"], where + ": reward / counter"
            assert (inf["n_leaf"][e], inf["n_cand"][e], inf["n_ems"][e]) == (rec["n_leaf"], rec["n_cand"], rec["n_ems"]), \
                (where, inf["n_leaf"][e], inf["n_cand"][e], inf["n_ems"][e], rec)
            if dd:
                assert inf["ratio"][e] == np.float32(rec["ratio"]), where + ": ratio"
        if reset:
            pos = {e: P.state(e)["draw_pos"] for e in reset}
            rinfo.zero_()
            o = _np(P.buffer_reset_envs(env_idx=reset, info=rinfo))
            fl = P.decode_info(rinfo)["flags"]
            items = _np(P.buffer_items())
            for e in reset:
                held[e] = -1
                models[e].reset(pos=pos[e])
                enter(e, t, int(fl[e]), "env %d step %d: after buffer_reset_envs" % (e, t))
                if held[e] < 0:
                    assert np.array_equal(items[e], models[e].buf), "env %d step %d: buffered items after buffer_reset_envs" % (e, t)
    live = [e for e in range(n) if held[e] < 0 and models[e] is not None]
    for e in live[:graphs]:
        compare_graphs(P.support_graph(e), models[e].orc.support_graph(), "env %d at the end:" % e)
    P.close()
    return fired


# ---- (a) lock-step at the limits: B = 16 (BUF_MAX) with NL = 64 (NL_MAX), B = 2, large discrete bins, non-unit continuous bins ----------
LIMITS = [(nm, 16, 64, "f64") for nm in ("d1", "d2", "d3", "c1", "c2", "c3")]
LIMITS += [("d2", 2, 50, "f64"), ("c1", 2, 50, "f64"), ("big_s1", 4, 50, "f64"), ("side255", 4, 50, "f64"), ("pallet_s2", 4, 50, "f64"),
           ("mm_s3", 4, 50, "f64"), ("d3", 16, 64, "f32")]


@pytest.mark.parametrize("name,B,nl,dt", LIMITS, ids=["%s-B%d-nl%d-%s" % c for c in LIMITS])
def test_lockstep_at_the_limits(name, B, nl, dt):
    c, mk = config(name, nl)
    n, steps = (8, 90) if B == 16 else (16, 120)
    streams = [mk(19, e, 600) for e in range(n)]
    fired = lockstep(c, streams, B, steps, obs_dtype=torch.float64 if dt == "f64" else torch.float32)
    print(name, B, nl, dt, "flags fired:", fired)  # the 255-cell bin's envs reach the box holder and the EMS capacity


# ---- (b) the capacity cases, flags exact ---------------------------------------------------------------------------------------------------
CAP = load_capacity_cases()


def _mild(c, n):
    """streams of larger items of the case's configuration: neighbours that end their episodes long before any capacity"""
    if c["domain"] == "continuous":
        return [cont_case_stream(dict(c, lo=0.1, hi=0.5), 500 + e, 0, len(c["stream"])) for e in range(n)]
    mild = [(a, b, h) for a in (5, 7) for b in (5, 8) for h in (4, 6)]
    return [case_stream(dict(c, items=mild), 500 + e, 0, len(c["stream"])) for e in range(n)]


@pytest.mark.parametrize("B", [3, 16])
@pytest.mark.parametrize("name", sorted(CAP))
def test_capacity_cases_flags_exact(name, B):
    """the case's stream in env 0 (and again in env 1, where the policy chooses otherwise) next to two mild neighbours: every record's flags
    are the model's, a flagged env keeps its bits until buffer_reset_envs and is exact again after it, the neighbours stay exact"""
    c = dict(CAP[name], items=[tuple(i) for i in CAP[name]["items"]] if "items" in CAP[name] else None)
    streams = [c["stream"]] * 2 + _mild(c, 2)
    fired = lockstep(c, streams, B, capacity_steps(c), graphs=2, pseed=c["pseed"])
    print(name, B, "flags fired:", fired)


# ---- (c) the slots of one env contending for its many-support scratch ----------------------------------------------------------------------
def _buffered_record(hdr, plain, items, n_leaf, stored, cont):
    """a buffered record spliced by the layout of DESIGN.md section 20: the buffered handle's record header, the plain record's body, items
    double[B][4], leaf counts int32[B] padded to 16 bytes, B leaf blocks of NL_MAX x 6 (int16 / double)"""
    B, nl = len(items), stored.shape[1]
    cnt = np.zeros(-(-B // 4) * 4, dtype=np.int32)
    cnt[:B] = n_leaf
    blk = np.zeros((B, 64, 6), dtype=np.float64 if cont else np.int16)  # NL_MAX = 64
    blk[:, :nl] = stored
    return np.concatenate([hdr[:16], plain[16:], np.ascontiguousarray(items, dtype=np.float64).view(np.uint8).reshape(-1), cnt.view(np.uint8),
                           blk.view(np.uint8).reshape(-1)])


@pytest.mark.parametrize("n", [1, MS_N])
@pytest.mark.parametrize("cont,setting", [(False, 1), (False, 3), (True, 1), (True, 3)], ids=["d1", "d3", "c1", "c3"])
def test_many_support_slots(cont, setting, n):
    """the floors of tests/many_supports.py laid by rows on a plain batch, each env's snapshot spliced into a buffered record with 16 items of
    large flat boxes and the model's leaf blocks, restored into a B = 16, NL = 64 batch: its observation is the model's, and then the
    random policy runs in lock-step, where the expansions of most slots visit nodes on more than 8 supports (tests/test_buffer_oracle_cpu.py
    counts them) and so share the env's one many-support scratch under its lock.  With 1024 envs, 16 blocks of every env contend across
    SMs; the envs of MS_CHECK are held against the model, every env must raise no flag."""
    import many_supports as M
    import pct_b200
    c = many_support_config(cont, setting)
    streams = list(M.streams(cont, setting, n))
    # the floors, by rows, on a plain batch
    plain = pct_b200.PctBatch(n, setting, container_size=c["container"], continuous=cont, internal_node_holder=c["nb"], leaf_node_holder=c["nl"],
                              obs_dtype=torch.float64, item_stream=np.stack(streams), size_minimum=c["size_minimum"])
    plain.reset()
    builds = [M.plan(cont, setting, e)[1] for e in range(n)]
    for t in range(max(len(b) for b in builds)):
        act = [e for e in range(n) if t < len(builds[e])]
        rows = np.zeros((n, 9))
        rows[act] = [builds[e][t] for e in act]
        _, _, d, info = plain.step(actions=torch.as_tensor(rows, device=plain.device), env_idx=act)
        assert not _np(d)[act].any() and not plain.decode_info(info)["flags"][act].any(), "build-up step %d" % t
    snaps = _np(plain.snapshot())
    pos = [plain.state(e)["draw_pos"] for e in range(n)]
    plain.close()
    check = [e for e in MS_CHECK if e < n]
    models = [None] * n
    for e in check:
        models[e], _ = many_support_model(cont, setting, e)
        assert pos[e] == models[e].pos, "env %d: draw position after the build-up %d, the model's %d" % (e, pos[e], models[e].pos)
    starts = many_support_starts(cont, setting, n)

    def restore(P):
        hdr = _np(P.buffer_snapshot(env_idx=[0]))[0]
        recs = np.stack([_buffered_record(hdr, snaps[e], *starts[e], cont) for e in range(n)])
        assert recs.shape[1] == P.buffer_snapshot_bytes, (recs.shape, P.buffer_snapshot_bytes)
        return P.buffer_restore(torch.as_tensor(recs, device=P.device))

    fired = lockstep(c, streams, 16, MS_STEPS, graphs=len(check), pseed=MS_PSEED, models=models, restore=restore)
    assert not any(fired), fired
