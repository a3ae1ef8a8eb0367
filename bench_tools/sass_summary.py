"""Per-kernel SASS evidence of the in-tree library (no GPU needed): `python -m bench_tools.sass_summary` rewrites
profiles/sass/mnemonic_summary.txt (mnemonic histogram per kernel) and profiles/sass/listings/<kernel>.sass (the full
`cuobjdump -sass` listing of every kernel, one file each) from dist_mnist_b200/libdmnist_sm90a.so."""
import collections
import re
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
KEEP = re.compile(r"^(UTC|LDTM|STTM|UTMA|UBLKCP|SYNCS|RED|ATOM|MEMBAR|CCTL|UCGABAR|ACQBULK|PREEXIT|MUFU\.(RCP|SQRT|RSQ|EX2|LG2)|"
                  r"ERRBAR|FENCE|LDGMC|LDG\.E\.(\d+\.)?STRONG|STG\.E\.(\d+\.)?STRONG|LD\.E\.STRONG|ST\.E\.STRONG|STS\..*CLUSTER|ST\.E.*CLUSTER|MAPA|"
                  r"UMOV.*SR_CgaCtaId|S2UR)")
HEADER = """SASS mnemonic evidence per kernel of libdmnist_sm90a.so (cuobjdump -sass, sm_90a); regenerate with
`python -m bench_tools.sass_summary`.
HGMMA = wgmma.mma_async, UTMALDG = cp.async.bulk.tensor (TMA), UBLKCP = cp.async.bulk,
SYNCS = mbarrier, UCGABAR = barrier.cluster, ACQBULK / PREEXIT = griddepcontrol.wait / launch_dependents (PDL),
RED/REDG = red.global (atomic push, monotone acks), *.STRONG.SYS = system-scope flag ld/st, MUFU.RCP/SQRT = Adam fast path,
LDGMC.E.ADD.F32x4 = multimem.ld_reduce (in-switch sum over an NVLS multicast team); multimem.st is an STG.E.128.STRONG.SYS whose
address is a multicast mapping (nvls_sm90.cu)
"""


def main() -> int:
    lib = ROOT / "dist_mnist_b200" / "libdmnist_sm90a.so"
    txt = subprocess.run(["cuobjdump", "-sass", str(lib)], capture_output=True, text=True, check=True).stdout
    out = [HEADER]
    name, counts, n = None, None, 0
    # ---- full listings, one file per kernel (demangled name in the header, mangled name in the file name) ----
    ldir = ROOT / "profiles" / "sass" / "listings"
    ldir.mkdir(parents=True, exist_ok=True)
    for old in ldir.glob("*.sass"):
        old.unlink()
    cur_name, cur_lines, n_files = None, [], 0

    def flush_listing():
        nonlocal n_files
        if cur_name:
            dem = subprocess.run(["c++filt", cur_name], capture_output=True, text=True).stdout.strip() or cur_name
            short = re.sub(r"[^A-Za-z0-9_]+", "_", dem.split("(")[0])[:120]
            body = "\n".join(cur_lines)
            (ldir / f"{short}.sass").write_text(f"// {dem}\n// {cur_name}  (sm_90a, cuobjdump -sass)\n{body}\n")
            n_files += 1

    for line in txt.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            flush_listing()
            cur_name, cur_lines = m.group(1), []
            continue
        if cur_name and (line.strip().startswith("....") or line.startswith("Fatbin elf code")):
            flush_listing()          # end of this cubin: what follows is the next ELF's header, not this kernel
            cur_name, cur_lines = None, []
            continue
        if cur_name:
            # keep the instruction text, drop the encoding words (halves the size, loses nothing readable)
            mm = re.match(r"(\s+/\*[0-9a-f]{4,8}\*/\s+.*?;)\s+/\* 0x[0-9a-f]+ \*/", line)
            if mm:
                cur_lines.append(mm.group(1))
            elif re.match(r"\s+/\* 0x[0-9a-f]+ \*/\s*$", line):
                continue
            elif line.strip():
                cur_lines.append(line.rstrip())
    flush_listing()
    print(f"wrote {n_files} listings under {ldir}")

    def flush():
        if name:
            out.append(name)
            out.append(f"    instructions: {n}")
            out.append("    " + ", ".join(f"{k} x{v}" for k, v in sorted(counts.items())))
            out.append("")

    for line in txt.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            flush()
            name, counts, n = m.group(1), collections.Counter(), 0
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,8}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
        if m and name:
            n += 1
            op = m.group(1)
            if KEEP.match(op):
                counts[op] += 1
    flush()
    dst = ROOT / "profiles" / "sass" / "mnemonic_summary.txt"
    dst.parent.mkdir(parents=True, exist_ok=True)
    dst.write_text("\n".join(out) + "\n")
    print(f"wrote {dst} ({len(out)} lines)")
    return 0


if __name__ == "__main__":
    sys.exit(main())
