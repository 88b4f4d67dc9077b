"""Per-kernel SASS instruction counts, registers and the opcodes that prove the TMA / mbarrier
code paths (cuobjdump here, no GPU needed).  usage: python tools/sass_summary.py > sass_summary.txt"""
import collections, re, subprocess
SO = "zeekstd_b200/libzeekstd_b200.so"
sass = subprocess.run(["cuobjdump", "-sass", SO], capture_output=True, text=True).stdout
res = subprocess.run(["cuobjdump", "-res-usage", SO], capture_output=True, text=True).stdout
regs, cur = {}, None
for l in res.split("\n"):
    m = re.search(r"Function (\S+):", l)
    if m: cur = m.group(1)
    m = re.search(r"REG:(\d+).*SHARED:(\d+)", l)
    if m and cur: regs[cur] = (int(m.group(1)), int(m.group(2)))
kern, cnt = None, collections.OrderedDict()
for l in sass.split("\n"):
    m = re.search(r"Function : (\S+)", l)
    if m: kern = m.group(1); cnt[kern] = collections.Counter(); continue
    m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", l)
    if m and kern:
        cnt[kern][m.group(1).split(".")[0]] += 1; cnt[kern]["_total"] += 1
dem = lambda n: subprocess.run(["c++filt", n], capture_output=True, text=True).stdout.strip().split("(")[0]
print("# SASS summary of zeekstd_b200/libzeekstd_b200.so (cuobjdump -sass, sm_90a) -- tools/sass_summary.py")
print("# UBLKCP = cp.async.bulk (TMA bulk copy global -> shared; K-D1s stages sequence bitstreams with it), SYNCS = mbarrier operations")
print("# (arrive / expect_tx / try_wait: the tile barriers of K-D1s and the event waits of zk_exec2_kernel), REDUX = redux.sync, MATCH = match.any")
print("kernel | SASS instructions | registers | static smem | UBLKCP | SYNCS | REDUX | MATCH | LDS | STS | LDG | STG | ATOM/RED | BAR")
for k, c in cnt.items():
    if "zk_" not in k: continue
    r = regs.get(k, (0, 0))
    print(f"{dem(k)} | {c['_total']} | {r[0]} | {r[1]} | {c['UBLKCP']} | {c['SYNCS']} | {c['REDUX']} | {c['MATCH']} | {c['LDS']} | {c['STS']} | {c['LDG']} | {c['STG']} | {c['ATOMS'] + c['ATOMG'] + c['RED']} | {c['BAR']}")
print()
print("# whole library: UBLKCP %d, SYNCS %d; no HMMA / UTC*MMA / LDTM (integer and byte work: no tensor cores, by design)" % (len(re.findall(r"\bUBLKCP", sass)), len(re.findall(r"\bSYNCS", sass))))
