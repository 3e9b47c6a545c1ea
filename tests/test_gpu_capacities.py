"""The step kernels at their fixed capacities (DESIGN.md section 7), on the cases of tests/golden/capacity_cases.npz, in lock-step with the
oracle, which has no such capacities.  Every step before the first one whose oracle counts cross a capacity (t*) is bit-exact with flags 0
(observation, reward, done, counter, the n_ems / n_cand of the step record, and the discrete EMS list row for row); at t* exactly the
expected flag bit is set; it stays set until the env is reset; after a reset of that env on both sides it is bit-exact again.  Envs of
the same batch that never cross a capacity are not disturbed by the ones that do."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
from harness import FLAG_BOX, capacity_oracle, case_stream, cont_case_stream, expected_flags, load_capacity_cases, oracle_counts, \
    policy_pick  # noqa: E402

pytestmark = pytest.mark.gpu

CASES = load_capacity_cases()

PAST = sorted(n for n, c in CASES.items() if c["flag"])
HOLD = 2       # steps a flagged env keeps running before it is reset
RECOVER = 15   # steps after that reset
MILD = [(a, b, c) for a in (5, 7) for b in (5, 8) for c in (4, 6)]


def _batch(c, streams, obs_dtype=torch.float64):
    import pct_b200
    return pct_b200.PctBatch(len(streams), c["setting"], container_size=c["container"], continuous=c["domain"] == "continuous",
                             item_set=None if c["domain"] == "continuous" else c["items"], internal_node_holder=c["nb"],
                             leaf_node_holder=c["nl"], obs_dtype=obs_dtype, item_stream=np.stack(streams), size_minimum=c["size_minimum"],
                             LNES=c["lnes"], auto_reset=False)


def _other_streams(c, n, seed0, mild=False):
    """streams of the case's configuration from other seeds (each env is judged on its own oracle counts, flagged or not); mild: larger
    items (x, y ~ U(0.1, 0.5) in the continuous domain), which end their episodes long before any capacity"""
    if c["domain"] == "continuous":
        return [cont_case_stream(dict(c, lo=0.1, hi=0.5) if mild else c, seed0 + e, 0, len(c["stream"])) for e in range(n)]
    items = MILD if mild else [tuple(i) for i in c["items"]]
    return [case_stream(dict(c, items=items), seed0 + e, 0, len(c["stream"])) for e in range(n)]


def _lockstep(c, streams, steps, obs_dtype=torch.float64, n_filler=0, check_ems=True, pseeds=None):
    """streams[e] runs in env e against its own oracle; n_filler more envs of other streams share the batch unchecked.
    -> per checked env, the (step, flag bits) of every flag it raised"""
    n = len(streams)
    pseeds = pseeds or [c["pseed"]] * n
    fill = _other_streams(c, n_filler, 9000)
    orcs = [capacity_oracle(dict(c, stream=s)) for s in streams]
    gpu = _batch(c, list(streams) + fill, obs_dtype)
    npd = np.float64 if obs_dtype == torch.float64 else np.float32
    o_ref = [orc.reset() for orc in orcs]
    o = gpu.reset().cpu().numpy()
    for e in range(n):
        assert np.array_equal(o[e], o_ref[e].astype(npd)), "%s env %d: reset" % (c["name"], e)
    flagged = np.full(n, -1)  # step of the env's current flag; -1: in lock-step with its oracle
    fired = [[] for _ in range(n)]
    for t in range(steps):
        idx = np.zeros(n + n_filler, dtype=np.int32)
        rows = [None] * n
        for e in range(n + n_filler):
            src = o_ref[e] if e < n and flagged[e] < 0 else o[e].astype(np.float64)
            idx[e], row = policy_pick(src, c["nb"], c["nl"], pseeds[e] if e < n else 1, 0 if e < n else e, t)
            if e < n:
                rows[e] = row
        ob, r, d, info = gpu.step(leaf_idx=torch.from_numpy(idx).cuda())
        o, r, d = ob.cpu().numpy(), r.cpu().numpy(), d.cpu().numpy().astype(bool)
        inf = gpu.decode_info(info)
        reset = [e for e in range(n, n + n_filler) if d[e]]
        for e in range(n):
            where = "%s env %d step %d" % (c["name"], e, t)
            if flagged[e] >= 0:  # the bit stays set until the env is reset
                assert inf["flags"][e] & fired[e][-1][1], where
                if d[e] or t - flagged[e] >= HOLD:
                    reset.append(e)
                continue
            o_ref[e], r_ref, d_ref, i_ref = orcs[e].step(rows[e])
            cnt = oracle_counts(orcs[e], c["lnes"])
            f = expected_flags(c, cnt, i_ref)
            assert inf["flags"][e] == f, "%s: flags %d, the oracle's counts %s call for %d" % (where, inf["flags"][e], cnt, f)
            if f:
                fired[e].append((t, f))
                flagged[e] = t
                if d[e]:
                    reset.append(e)
                if f == FLAG_BOX:  # IndexError in the reference: the episode ends on the terminal observation of the full holder
                    assert d[e] and d_ref and i_ref.get("error") == 1, where
                    assert np.array_equal(o[e], o_ref[e].astype(npd)), where + ": terminal observation"
                    assert inf["ratio"][e] == np.float32(i_ref["ratio"]) and inf["counter"][e] == i_ref["counter"], where
                continue
            assert d[e] == d_ref, where
            assert np.array_equal(o[e], o_ref[e].astype(npd)), "%s: %d mismatches" % (where, int((o[e] != o_ref[e].astype(npd)).sum()))
            assert r[e] == np.float32(r_ref) and inf["counter"][e] == i_ref["counter"], where
            assert (inf["n_ems"][e], inf["n_cand"][e]) == (cnt["ems"], cnt["cand"]), (where, inf["n_ems"][e], inf["n_cand"][e], cnt)
            if d_ref:
                assert inf["ratio"][e] == np.float32(i_ref["ratio"]), where
                reset.append(e)
            elif check_ems and c["domain"] == "discrete":
                assert np.array_equal(gpu.state(e)["ems"], orcs[e].ems()), where + ": EMS list"
        for e in reset:
            if e < n and flagged[e] >= 0:
                # the oracle stopped at t* while the flagged env kept drawing items: its replacement starts at the env's draw position
                k = gpu.state(e)["draw_pos"]
                orcs[e] = capacity_oracle(dict(c, stream=np.roll(streams[e], -k, axis=0)))
        if reset:
            rinfo = torch.zeros((n + n_filler, 8), dtype=torch.int32, device=gpu.device)
            o = gpu.reset(env_idx=sorted(reset), info=rinfo).cpu().numpy()
            rflags = gpu.decode_info(rinfo)["flags"]
            for e in reset:
                if e < n:  # the overflow left nothing behind: the env is exact again and its flags are those of its new counts
                    o_ref[e] = orcs[e].reset()
                    f = expected_flags(c, oracle_counts(orcs[e], c["lnes"]), {})
                    where = "%s env %d step %d: after the reset" % (c["name"], e, t)
                    assert rflags[e] == f, where
                    flagged[e] = -1
                    if f:  # the first expansion of the new episode already crosses a capacity
                        fired[e].append((t, f))
                        flagged[e] = t
                    else:
                        assert np.array_equal(o[e], o_ref[e].astype(npd)), where
    return fired


def _horizon(c):
    return c["n_steps"] + (HOLD + RECOVER if c["flag"] else 0)


@pytest.mark.parametrize("name", sorted(CASES))
def test_capacity_lockstep(name):
    """one env: exact up to the capacity, the flag at t* (not before), sticky until the reset, then exact again, flagged only where its
    new counts cross a capacity (the FC cases of a 20 x 20 floor may cross it again within a few steps)"""
    c = CASES[name]
    fired = _lockstep(c, [c["stream"]], _horizon(c))[0]
    assert fired[:1] == ([(c["t_star"], c["flag"])] if c["flag"] else []), fired
    if c["lnes"] != "FC":
        assert len(fired) <= 1, fired


@pytest.mark.parametrize("name", ["d_box80_s1", "c_box80_s1", "d_cand_at_fc15_s2"])
def test_capacity_lockstep_float32(name):
    """float32 observations (delta rows): a full box holder writes every internal row"""
    c = CASES[name]
    fired = _lockstep(c, [c["stream"]], _horizon(c), obs_dtype=torch.float32, check_ems=False)[0]
    assert fired[:1] == ([(c["t_star"], c["flag"])] if c["flag"] else [])


@pytest.mark.parametrize("name", PAST)
def test_capacity_in_a_batch_of_64(name):
    """the same stream as env 0 of a 64-env batch flags at the same step and agrees bit for bit up to it (the walk pools are sized by the
    batch: a single env must not run out of them where a larger batch does not)"""
    c = CASES[name]
    fired = _lockstep(c, [c["stream"]], c["n_steps"] + HOLD, n_filler=63, check_ems=False)[0]
    assert fired[:1] == [(c["t_star"], c["flag"])], fired


@pytest.mark.parametrize("names", [("d_ems_s1", "d_box80_s1"), ("c_box80_s1", "c_ems_s1")])
def test_capacity_isolation(names):
    """every third env crosses a capacity; the others (larger items, never flagged) stay bit-exact for the whole horizon"""
    cs = [CASES[nm] for nm in names]
    others = _other_streams(cs[0], 8, 7000, mild=True)
    kinds = [cs[(e // 3) % 2] if e % 3 == 0 else None for e in range(12)]
    streams = [k["stream"] if k else others.pop() for k in kinds]
    pseeds = [k["pseed"] if k else 7 for k in kinds]
    fired = _lockstep(cs[0], streams, max(_horizon(k) for k in cs), check_ems=False, pseeds=pseeds)
    for e, k in enumerate(kinds):
        assert fired[e][:1] == ([(k["t_star"], k["flag"])] if k else []), (e, fired[e])


def test_vec_env_raises_on_the_flagged_step():
    """PctVecEnv: PctError on the step at t*, naming the env and the flag; with raise_on_flags=False the env's info carries the bit"""
    import pct_b200
    from pct_b200.batch import PctError
    c = CASES["d_ems_s1"]
    for raise_on in (True, False):
        env = pct_b200.PctVecEnv(1, c["setting"], container_size=c["container"], item_set=c["items"], item_stream=c["stream"][None],
                                 raise_on_flags=raise_on)
        obs = env.reset().cpu().numpy().astype(np.float64)
        for t in range(c["t_star"] + 1):
            k, _ = policy_pick(obs[0], c["nb"], c["nl"], c["pseed"], 0, t)
            a = torch.tensor([k], dtype=torch.int64)
            if t == c["t_star"] and raise_on:
                with pytest.raises(PctError, match=r"env 0, flags 4 = ems_overflow"):
                    env.step(a)
                break
            obs, _, done, infos = env.step(a)
            obs = obs.cpu().numpy().astype(np.float64)
            assert infos[0].get("flags", 0) == (4 if t == c["t_star"] else 0), t
        env.close()


@pytest.mark.parametrize("name", ["d_ems_s1", "c_cand_s2"])
def test_single_env_facade_reports_flags(name):
    """PackingDiscrete / PackingContinuous put the step record's flags into info"""
    import pct_b200
    c = CASES[name]
    if c["domain"] == "discrete":
        env = pct_b200.PackingDiscrete(setting=c["setting"], container_size=list(c["container"]), item_set=c["items"], item_stream=c["stream"][None])
    else:
        env = pct_b200.PackingContinuous(setting=c["setting"], container_size=list(c["container"]), item_set=None, sample_from_distribution=False,
                                         item_stream=c["stream"][None], size_minimum=c["size_minimum"])
    obs = env.reset()
    for t in range(c["t_star"] + 1):
        _, row = policy_pick(obs, c["nb"], c["nl"], c["pseed"], 0, t)
        obs, _, _, info = env.step(row)
        assert info.get("flags", 0) == (c["flag"] if t == c["t_star"] else 0), t
    env.close()
