"""SASS mnemonic counts per kernel of the built library (static evidence that the wgmma / TMA paths are what ships).
usage: python tools/sass_mnemonics.py   (needs cuobjdump + c++filt; no GPU)"""
import os, re, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
so = os.path.join(ROOT, "end-to-end-asr-pytorch_b200", "libb200asr.so")
MN = ["HGMMA", "UTMALDG", "UBLKCP", "SYNCS", "HMMA", "LDGSTS", "UTMACCTL"]


def mnemonic_counts(path=so):
    """{demangled kernel name (without the parameter list): {mnemonic: count}} for every kernel of the library."""
    sass = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True).stdout
    counts, cur = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            counts[cur] = dict.fromkeys(MN, 0)
            continue
        if cur:
            m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)", line)
            if m:
                op = m.group(1)
                for k in MN:
                    if op == k or op.startswith(k + "."):
                        counts[cur][k] += 1
    names = subprocess.run(["c++filt"], input="\n".join(counts), capture_output=True, text=True).stdout.splitlines()
    out = {}
    for raw, nice in zip(counts, names):
        out[re.sub(r"\(.*", "", nice.replace("(anonymous namespace)::", ""))] = counts[raw]
    return out


if __name__ == "__main__":
    print("SASS mnemonic counts per kernel of libb200asr.so (cuobjdump -sass, sm_90a): wgmma = HGMMA,")
    print("cp.async.bulk.tensor = UTMALDG, cp.async.bulk = UBLKCP, cp.async = LDGSTS, mbarrier = SYNCS, mma.sync = HMMA")
    print("%-78s" % "kernel" + "".join("%9s" % k for k in MN))
    for nice, c in sorted(mnemonic_counts().items()):
        if any(c.values()):
            print("%-78s" % nice[-78:] + "".join("%9d" % c[k] for k in MN))
