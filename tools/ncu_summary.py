"""ncu report -> 'metric,value,unit' summary (one kernel launch), and launch-list shares.
   python tools/ncu_summary.py rep  x.ncu-rep  x_summary.csv
   python tools/ncu_summary.py list gpurun_out/launches.csv            # per-kernel share of the captured launches"""
import csv, subprocess, sys, collections, io, re


def rep(path, out):
    txt = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
    rows = list(csv.reader(io.StringIO(txt)))
    hdr, units, vals = rows[0], rows[1], rows[2]
    with open(out, "w") as f:
        for h, u, v in sorted(zip(hdr, units, vals)):
            if h in ("ID", "Process ID", "Process Name", "Host Name", "Context", "Stream", "Device", "CC"):
                continue
            f.write(f"{h},{v},{u}\n")


def launches(path):
    rows = [r for r in csv.reader(open(path, errors="replace")) if len(r) > 10 and r[0].isdigit()]
    tot = collections.OrderedDict()
    for r in rows:
        name = re.sub(r"\(.*", "", r[4]).replace("<unnamed>::", "")
        name = re.sub(r"<.*", "", name)
        t = float(r[-1].replace(",", ""))
        unit = r[-2]
        t *= {"ns": 1e-6, "us": 1e-3, "ms": 1.0, "s": 1e3}.get(unit, 1e-6)
        c = tot.setdefault(name, [0, 0.0])
        c[0] += 1
        c[1] += t
    s = sum(v[1] for v in tot.values())
    for k, (n, t) in sorted(tot.items(), key=lambda kv: -kv[1][1]):
        print(f"{k:40s} {n:5d} launches {t:10.3f} ms {100 * t / s:6.2f} %")
    print(f"{'total':40s} {sum(v[0] for v in tot.values()):5d} launches {s:10.3f} ms")


if __name__ == "__main__":
    if sys.argv[1] == "rep":
        rep(sys.argv[2], sys.argv[3])
    else:
        launches(sys.argv[2])
