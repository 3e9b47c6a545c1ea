"""python scratch/sass_summary.py [lib.so] — per kernel of libpct_b200.so: SASS instruction count and the opcodes that
show the Hopper-native paths: UBLKCP (1-D TMA bulk copy, cp.async.bulk), SYNCS (mbarrier), PREEXIT (griddepcontrol.launch_dependents,
programmatic dependent launch), plus the FP64 / vote / shuffle / atomic / local-memory mix.  No GPU needed (cuobjdump -sass)."""
import collections, re, subprocess, sys
lib = sys.argv[1] if len(sys.argv) > 1 else "online-3d-bpp-pct_b200/libpct_b200.so"
sass = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
fn, cnt = None, collections.OrderedDict()
for line in sass.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        fn = m.group(1); cnt[fn] = collections.Counter(); continue
    m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(@!?U?P\d+\s+)?([A-Z0-9_]+)", line)
    if m and fn:
        cnt[fn][m.group(2)] += 1
names = subprocess.run(["c++filt"], input="\n".join(cnt), capture_output=True, text=True).stdout.splitlines()
rev = subprocess.run(["git", "rev-parse", "--short", "HEAD"], capture_output=True, text=True).stdout.strip()
print("# cuobjdump -sass %s (source tree at %s + working changes); counts of static SASS instructions per kernel" % (lib, rev))
cols = ["UBLKCP", "SYNCS", "PREEXIT", "ACQBULK", "DFMA", "DADD", "DMUL", "MUFU", "VOTE", "SHFL", "MATCH", "ATOMS", "ATOMG", "RED", "LDL", "STL", "LDS", "LDG", "BSSY", "WARPSYNC"]
print("%-84s %6s " % ("kernel", "insts") + " ".join("%7s" % c for c in cols))
for (f, c), n in sorted(zip(cnt.items(), names), key=lambda x: x[1]):
    if "kernel" not in n:
        continue
    print("%-84s %6d " % (n.replace("pct::", "")[:84], sum(c.values())) + " ".join("%7d" % c[k] for k in cols))
