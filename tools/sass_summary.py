"""Static SASS summary of the compression / decompression kernels of the current build (no GPU needed):
   python tools/sass_summary.py
Per kernel: registers / shared memory / spills (ptxas), static instruction count and the opcode groups that matter for
this path (global / shared loads and stores, shared atomics, shuffles, votes, barriers, integer multiply-adds, branches)."""
import collections, os, re, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "zstd_b200", "csrc")
GROUPS = [("LDG", r"^LDG"), ("STG", r"^STG|^ST\."), ("LDS", r"^LDS"), ("STS", r"^STS"), ("ATOMS", r"^ATOMS"), ("ATOMG/RED", r"^ATOMG|^RED\b|^RED\."),
          ("SHFL", r"^SHFL"), ("VOTE", r"^VOTE"), ("BAR", r"^BAR"), ("IMAD", r"^IMAD"), ("SHF/LOP3", r"^SHF|^LOP3"), ("BRA", r"^BRA|^BSSY|^BSYNC"), ("LDL/STL", r"^LDL|^STL")]
WANT = ["zb_walk_kernelILi7ELi8", "zb_walk_kernelILi8ELi4", "zb_parse_kernelILb0", "zb_parse_dfast_kernelILb0", "zb_merge_segments", "zb_merge_small",
        "zb_literals_kernel", "zb_sequences_kernel", "zb_copy_kernel", "zbd_literals_kernel", "zbd_sequences_kernel", "zbd_place_kernel", "zbd_matches_kernel"]


def ptxas_info():
    info = {}
    for f in os.listdir(CSRC):
        if not f.endswith(".ptxas.log"): continue
        name = None; spill = ""
        for line in open(os.path.join(CSRC, f)):
            m = re.search(r"Compiling entry function '(\S+)'", line)
            if m: name = m.group(1); spill = ""
            if "spill" in line and " 0 bytes spill stores, 0 bytes spill loads" not in line: spill = line.strip()
            m = re.search(r"Used (\d+) registers.*?(?:, (\d+) bytes smem)?$", line.strip())
            if m and name: info[name] = (int(m.group(1)), int(m.group(2) or 0), spill)
    return info


def main():
    info = ptxas_info()
    print("# Static SASS summary of the hot kernels (sm_90a, `cuobjdump -sass` of the in-tree objects; `tools/sass_summary.py`)\n")
    print("Dynamic shared memory (the walk's table: 4 bytes per bucket, 48 KiB at level 1) is not in the ptxas figure.\n")
    print("| kernel | regs | static smem | spills | SASS instr | " + " | ".join(g for g, _ in GROUPS) + " |")
    print("|---|---|---|---|---|" + "---|" * len(GROUPS))
    for obj in ("zb_match.o", "zb_literals.o", "zb_sequences.o", "zb_stitch.o", "zb_decode.o"):
        out = subprocess.run(["cuobjdump", "-sass", os.path.join(CSRC, obj)], capture_output=True, text=True).stdout
        cur, ops = None, None
        funcs = collections.OrderedDict()
        for line in out.splitlines():
            m = re.search(r"Function : (\S+)", line)
            if m: cur = m.group(1); funcs[cur] = []; continue
            m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d\s+)?([A-Z0-9_.]+)", line)
            if m and cur: funcs[cur].append(m.group(1))
        for name, lst in funcs.items():
            if not any(w in name for w in WANT): continue
            cnt = [sum(1 for o in lst if re.search(p, o)) for _, p in GROUPS]
            r, sm, sp = info.get(name, (0, 0, ""))
            short = subprocess.run(["c++filt", name], capture_output=True, text=True).stdout.split("(")[0].replace("void ", "").strip()
            print(f"| `{short}` | {r} | {sm} | {'yes: ' + sp if sp else '0'} | {len(lst)} | " + " | ".join(str(c) for c in cnt) + " |")
    print("\nNo tensor-core (`HMMA`/`UTC*MMA`), TMA (`UBLKCP`) or cluster instructions appear: the path is integer / byte work on")
    print("shared-memory tables and L2-resident windows (DESIGN.md §5, §10); the GPU-specific part of the design is the sizing")
    print("(up to 227 KB of shared memory per block decide the table sizes and CTAs per SM on the 132 SMs of an H100).")


if __name__ == "__main__":
    main()
