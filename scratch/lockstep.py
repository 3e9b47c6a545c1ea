import sys, time
sys.path.insert(0, __import__('os').path.join(__import__('os').path.dirname(__import__('os').path.dirname(__import__('os').path.abspath(__file__))), 'oracle'))
import numpy as np
import ref_shim, pct_oracle
from pct_oracle import OracleDiscrete, policy_pick, rnd_u64
D, C = ref_shim.load_reference()
item_set = [(i,j,k) for i in range(1,6) for j in range(1,6) for k in range(1,6)]

def make_stream(seed, env, n, setting):
    s = np.zeros((n,4))
    for d in range(n):
        it = item_set[rnd_u64(seed, env, d) % 125]
        s[d,:3] = it
        s[d,3] = ((rnd_u64(seed ^ 0xABCDEF, env, d) >> 11) + 1) / float(1<<53) if setting == 3 else 1.0
    return s

LNES='EMS'
def run(setting, seed, envid, steps):
    stream = make_stream(seed, envid, steps+200, setting)
    ref = D.PackingDiscrete(setting=setting, container_size=[10,10,10], item_set=item_set, internal_node_holder=80, leaf_node_holder=50, shuffle=False, LNES=LNES)
    ref.box_creator = ref_shim.make_stream_creator(D, [tuple(r) if setting==3 else tuple(int(v) for v in r[:3]) for r in stream])
    ref.test = True
    orc = OracleDiscrete(setting, stream=stream, lnes=LNES)
    o1 = ref.reset(); o2 = orc.reset()
    nm = 0
    for t in range(steps):
        if not np.array_equal(o1, o2):
            d = np.where(o1 != o2)[0]
            print('OBS MISMATCH setting', setting, 'seed', seed, 'step', t, d[:10], o1[d[:10]], o2[d[:10]]); return False, orc.n_lstsq
        k, a = policy_pick(o1, 80, 50, seed, envid, t)
        o1, r1, d1, i1 = ref.step(a); o2, r2, d2, i2 = orc.step(a)
        if not np.array_equal(o1, o2): print('TERMINAL/STEP OBS MISMATCH', setting, seed, t, d1); return False, orc.n_lstsq
        if r1 != r2 or d1 != d2 or i1 != {k_:v for k_,v in i2.items()}:
            print('RET MISMATCH', setting, seed, t, r1, r2, d1, d2, i1, i2); return False, orc.n_lstsq
        if d1:
            o1 = ref.reset(); o2 = orc.reset()
    return True, orc.n_lstsq

if __name__ == '__main__':
    LNES = sys.argv[5] if len(sys.argv) > 5 else 'EMS'
    setting = int(sys.argv[1]); nseeds = int(sys.argv[2]); steps = int(sys.argv[3]); base = int(sys.argv[4]) if len(sys.argv) > 4 else 0
    t0 = time.time(); ok = 0; nl = 0
    for s in range(base, base+nseeds):
        r, n = run(setting, 1000+s, s, steps); ok += r; nl += n
    print(LNES, 'setting', setting, 'ok', ok, '/', nseeds, 'lstsq calls', nl, 'time', time.time()-t0)
