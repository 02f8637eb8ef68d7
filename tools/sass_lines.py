"""Static SASS statistics of one kernel: annotated listing + instructions per source line inside an address range.

    python tools/sass_lines.py <obj-or-cubin> <kernel-name-substring> [--range 0x1e40 0x3f20] [--list out.txt]

Used to iterate on instruction counts of the hot loops without a GPU (nvcc cross-compiles; nvdisasm --print-line-info
maps SASS to source through -lineinfo)."""
import collections
import os
import re
import subprocess
import sys
import tempfile


def main():
    obj, kern = sys.argv[1], sys.argv[2]
    rng = None
    lst = None
    a = sys.argv[3:]
    while a:
        if a[0] == "--range":
            rng = (int(a[1], 16), int(a[2], 16)); a = a[3:]
        elif a[0] == "--list":
            lst = a[1]; a = a[2:]
        else:
            raise SystemExit("unknown argument " + a[0])
    tmp = tempfile.mkdtemp()
    cub = obj
    if not obj.endswith(".cubin"):
        subprocess.check_call(["cuobjdump", "-xelf", "all", os.path.abspath(obj)], cwd=tmp, stdout=subprocess.DEVNULL)
        cub = os.path.join(tmp, sorted(f for f in os.listdir(tmp) if f.endswith(".cubin"))[0])
    txt = subprocess.run(["nvdisasm", "--print-line-info", cub], capture_output=True, text=True).stdout.splitlines()
    rows, cur, on = [], ("?", 0), False
    for ln in txt:
        if ln.split()[:1] == [".section"]:   # (not .sectionflags, which follows it)
            on = ".text." in ln and kern in ln
            continue
        if not on:
            continue
        m = re.match(r'\s*//## File "([^"]+)", line (\d+)', ln)
        if m:
            cur = (os.path.basename(m.group(1)), int(m.group(2)))
            continue
        m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?);", ln)
        if m:
            rows.append((int(m.group(1), 16), m.group(2).strip(), cur))
    print(f"{kern}: {len(rows)} instructions")
    labels = {}
    # backward branches = loops
    for ad, ins, _ in rows:
        pass
    if lst:
        with open(lst, "w") as f:
            for ad, ins, (fn, l) in rows:
                f.write(f"{ad:05x}  {ins:<70s} {fn}:{l}\n")
    sel = [r for r in rows if rng is None or rng[0] <= r[0] <= rng[1]]
    per = collections.Counter((fn, l) for _, _, (fn, l) in sel)
    ops = collections.Counter(re.sub(r"^@!?U?P\d+\s+", "", ins).split()[0].split(".")[0] for _, ins, _ in sel)
    print(f"range: {len(sel)} instructions; opcodes:", ", ".join(f"{k} {v}" for k, v in ops.most_common(24)))
    for (fn, l), c in per.most_common(45):
        print(f"  {c:4d}  {fn}:{l}")


if __name__ == "__main__":
    main()
