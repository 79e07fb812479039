"""Every ld.global.nc (LDG.E...CONSTANT) that a kernel of libstablets_b200.so issues BEFORE its griddepcontrol.wait (ACQBULK).

    python tools/check_pdl_sass.py [objects or the .so]

Such a load reads memory before the predecessor kernel is known to have finished: fine for weights / tables (explicit
__ldg), a race for anything the predecessor writes.  Exit code 1 if a kernel has one that is not allow-listed below."""
import os
import re
import subprocess
import sys

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ALLOW = {            # kernel-name substring -> what its early non-coherent loads are (audited: constants only)
    "gemv_mma_kernel": "explicit __ldg of the WEIGHT fragments, issued ahead of the wait on purpose (gemv.cu:74)",
}
# Asynchronous copies (TMA `UTMALDG`, bulk `UBLKCP`) that are issued ahead of the wait ON PURPOSE -- listed with `--all`:
#   decode_linear_kernel            the WEIGHT tiles of the first ring stages (the activations are loaded after the wait)
#   decode_cross_attn_tc_kernel     the window's cross K / V tiles: written once per window batch by stb_cross_kv, many
#                                   kernels earlier on the same stream (every kernel in between waited on its predecessor)


def main():
    show_all = "--all" in sys.argv
    targets = [a for a in sys.argv[1:] if a != "--all"] or [os.path.join(HERE, "stable-ts_b200", "libstablets_b200.so")]
    bad = 0
    for t in targets:
        out = subprocess.run(["cuobjdump", "-sass", t], capture_output=True, text=True).stdout
        fn, early, other, seen_wait = None, [], [], False
        def flush():
            nonlocal bad
            if fn and seen_wait and other:                 # --all: kernels WITH a wait only
                for o in other:
                    print("early (intentional, see above) in " + fn[:60] + ": " + o)
            if fn and seen_wait and early:
                ok = any(k in fn for k in ALLOW)
                print(("allowed " if ok else "EARLY   ") + fn)
                for e in early:
                    print("        " + e)
                bad += 0 if ok else 1
        for line in out.splitlines():
            m = re.search(r"Function : (\S+)", line)
            if m:
                flush()
                fn, early, other, seen_wait = m.group(1), [], [], False
                continue
            if "ACQBULK" in line:
                seen_wait = True
            elif not seen_wait and re.search(r"LDG\.E[.\w]*CONSTANT", line):
                early.append(line.strip()[:100])
            elif not seen_wait and show_all and re.search(r"UTMALDG|UBLKCP|\bLDG\.|\bLD\.E", line):
                other.append(line.strip()[:70])
        flush()
    print(f"{bad} kernel(s) with non-coherent loads ahead of griddepcontrol.wait")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
