"""CPU: the oracle's set_next (`env.next_box = item`) and the buffered env built on it (tests/buffer_oracle.py), which
tests/test_gpu_buffer_oracle.py holds the buffered kernels against.

set_next is pinned against a replay copy: a fresh oracle whose item stream puts the item next, stepped with the episode's rows, must show
the same observation, candidate list, raw-key count and EMS list.  The model with B = 1 must be the plain oracle under policy_pick.  And the
capacity scenarios the GPU test runs must reach what they are there for: a candidate overflow raised by a slot the step did not place from,
an EMS overflow and a box overflow raised by the placement."""
import numpy as np
import pytest

from buffer_oracle import MS_CHECK, MS_PSEED, MS_STEPS, BufferedOracle, capacity_steps, config as _config, make_oracle, many_support_model, \
    slot_census
from harness import FLAG_BOX, FLAG_CAND, FLAG_EMS, load_capacity_cases, policy_pick
from pct_oracle import OracleDiscrete

B_CAP = (3, 16)  # the buffer sizes of the GPU capacity test


PIN = ["d1", "d2", "d3", "c1", "c2", "c3", "big_s2", "holders_s2", "flat_s1", "cp_big_s1", "ep_big_s2", "pallet_s1", "mm_s3"]


def _view(orc):
    cand, feas = orc.candidates()
    out = dict(cand=cand, feas=feas, ems=orc.ems())
    if isinstance(orc, OracleDiscrete):
        out["raw"] = orc.n_raw_candidates()
    return out


def test_set_next_is_a_replay():
    """every state of a few episodes per configuration: set_next(x) equals a fresh oracle whose stream draws x there, stepped with the
    episode's rows; set_next(the episode's own item) then gives the episode's observation back, and the episode goes on"""
    states = {}
    for name in PIN:
        cfg, mk = _config(name)
        n_states, ep = 0, 0
        while n_states < 160:
            L = 400
            st, other = mk(41, ep, L), mk(43, ep, L)
            orc = make_oracle(cfg, st)
            obs = orc.reset()
            rows = []
            for t in range(L - 2):
                x = st[t] if t % 7 == 3 else other[t]  # now and then the item the stream holds anyway
                got = orc.set_next(x)
                v = _view(orc)
                rep_stream = st.copy()
                rep_stream[t] = x
                rep = make_oracle(cfg, rep_stream)
                want = rep.reset()
                for r in rows:
                    want, _, d, _ = rep.step(r)
                    assert not d
                w = _view(rep)
                where = "%s episode %d state %d" % (name, ep, t)
                assert np.array_equal(got.view(np.uint64), want.view(np.uint64)), where + ": observation"
                for k in v:
                    assert np.array_equal(np.asarray(v[k]).view(np.uint8) if np.ndim(v[k]) else v[k],
                                          np.asarray(w[k]).view(np.uint8) if np.ndim(w[k]) else w[k]), "%s: %s" % (where, k)
                back = orc.set_next(st[t])
                assert np.array_equal(back.view(np.uint64), obs.view(np.uint64)), where + ": set_next of the current item"
                n_states += 1
                _, row = policy_pick(obs, cfg["nb"], cfg["nl"], 5, ep, t)
                obs, _, d, _ = orc.step(row)
                if d:
                    break
                rows.append(row)
            ep += 1
        states[name] = n_states
    print("set_next states per configuration:", states)
    assert sum(states.values()) >= 2000


@pytest.mark.parametrize("name", ["d1", "d2", "d3", "c1", "c2", "c3", "cp_big_s1", "pallet_s2"])
def test_b1_model_is_the_plain_oracle(name):
    """B = 1: the buffered model's observation, reward and done are the plain oracle's under policy_pick, step for step"""
    cfg, mk = _config(name)
    for e in range(3):
        st = mk(7, e, 600)
        m, o = BufferedOracle(cfg, st, 1), make_oracle(cfg, st)
        a, b = m.reset(), o.reset()
        dones = 0
        for t in range(250):
            assert np.array_equal(a.view(np.uint64), b.view(np.uint64)), (name, e, t)
            f = m.policy(5, e, t)
            k, row = policy_pick(b, cfg["nb"], cfg["nl"], 5, e, t)
            assert f == k, (name, e, t)
            a, r, d, rec = m.step(f)
            b, r2, d2, _ = o.step(row)
            if d2:
                b = o.reset()
            assert r == r2 and d == d2 and rec["flags"] == 0, (name, e, t)
            dones += d
        assert dones >= 2


def capacity_first_flags(c, B, pseed, steps):
    """the buffered model of a capacity case, driven by pct_buffer_policy_random of env 0, up to its first flag -> None, or dict(t (-1: the
    reset), flags, placement (the placement's bits), slots (slots whose expansion flags), placed (the slot the step placed from), done)"""
    m = BufferedOracle(c, c["stream"], B)
    m.reset()
    if m.sticky:
        return dict(t=-1, flags=m.sticky, placement=0, slots=[int(k) for k in np.nonzero(m.slot_fl)[0]], placed=-1, done=False)
    for t in range(steps):
        f = m.policy(pseed, 0, t)
        _, _, d, rec = m.step(f)
        if rec["flags"]:
            return dict(t=t, flags=rec["flags"], placement=rec["placement_flags"], slots=[int(k) for k in np.nonzero(rec["slot_flags"])[0]],
                        placed=f // m.nl, done=bool(d))
    return None


def test_capacity_scenarios_reach_their_floors():
    """the capacity cases at B = 3 and B = 16 under the buffered random policy raise a candidate overflow in a slot the step did not place
    from (the flag a check of the chosen item's expansion alone misses), and an EMS and a box overflow in the placement"""
    cases = load_capacity_cases()
    reach = dict(cand_unplaced=[], cand_reset_discrete=[], ems=[], box=[])
    for B in B_CAP:
        for name in sorted(cases):
            c = cases[name]
            r = capacity_first_flags(c, B, c["pseed"], capacity_steps(c))
            if r is None:
                continue
            tag = "%s-B%d" % (name, B)
            # a step whose placement overflows the EMS list builds its slots' lists from the device's truncated list: not counted
            if r["flags"] & FLAG_CAND and r["t"] >= 0 and not r["done"] and r["placed"] not in r["slots"] and not r["placement"] & FLAG_EMS:
                reach["cand_unplaced"].append(tag)
            if r["t"] < 0 and c["domain"] == "discrete" and any(k != 0 for k in r["slots"]):  # a slot other than the reset's own draw
                reach["cand_reset_discrete"].append(tag)
            if r["placement"] & FLAG_EMS:
                reach["ems"].append(tag)
            if r["placement"] & FLAG_BOX:
                reach["box"].append(tag)
    print("capacity floors reached:", {k: len(v) for k, v in reach.items()}, reach)
    print("never flagged at either B:", sorted(nm for nm, c in cases.items() if all(capacity_first_flags(c, B, c["pseed"], capacity_steps(c)) is None for B in B_CAP)))
    assert len(reach["cand_unplaced"]) >= 2 and len(reach["cand_reset_discrete"]) >= 2 and len(reach["ems"]) >= 2 and len(reach["box"]) >= 4, reach


MS_CASES = [(cont, setting) for cont in (False, True) for setting in (1, 3)]


@pytest.mark.parametrize("cont,setting", MS_CASES, ids=["d1", "d3", "c1", "c3"])
def test_many_support_slots_reach_their_floors(cont, setting):
    """the checked envs of the GPU test's many-support scenario, every state of it: the (env, step) pairs in which >= 2 and >= 8 of the 16
    slots' expansions make stability visits on more than KSUP_SMALL = 8 supports (a placement on > 8 supports, or one above a box on > 8),
    and the support counts their walks reach; the scenario stays inside every capacity"""
    import many_supports as M
    pairs2 = pairs8 = 0
    ks = set()
    for env in MS_CHECK:
        m, _ = many_support_model(cont, setting, env)
        for t in range(MS_STEPS):
            cs = slot_census(m)
            big = sum(1 for c in cs if any(k > M.KSUP_SMALL for k in c["k"]) or any(c["below_big"]))
            pairs2 += big >= 2
            pairs8 += big >= 8
            for c in cs:
                ks |= set(c["k"])
                assert max(c["k"] + [0]) <= M.KSUP_MAX and c["sup_pool"] <= M.STAB_SUP_POOL and c["depth"] <= M.STAB_DEPTH, (env, t)
            _, _, _, rec = m.step(m.policy(MS_PSEED, env, t))
            assert rec["flags"] == 0, (env, t, rec)
    n = len(MS_CHECK) * MS_STEPS
    print("%s setting %d: of %d (env, step) pairs, %d with >= 2 and %d with >= 8 slots on > 8 supports; support counts %s" % (
        "continuous" if cont else "discrete", setting, n, pairs2, pairs8, sorted(ks)))
    assert pairs2 >= n // 2 and pairs8 >= n // 3, (pairs2, pairs8)
    assert {9, 16, 25, 32} <= ks, sorted(ks)
