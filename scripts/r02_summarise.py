#!/usr/bin/env python
"""Turn the artefacts of scripts/r02_final.sh (gpurun_out/) into the committed evidence under profiles/ (run in the build
container; ncu reads .ncu-rep files without a GPU).

    python scripts/r02_summarise.py [tag]        # default tag: r02final
"""
import collections
import csv
import json
import os
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
tag = sys.argv[1] if len(sys.argv) > 1 else "r02final"
G = os.path.join(ROOT, "gpurun_out")
P = os.path.join(ROOT, "profiles")


def run(*cmd, **kw):
    return subprocess.run(cmd, capture_output=True, text=True, cwd=kw.get("cwd", ROOT))


def copy(src, dst):
    if os.path.exists(os.path.join(G, src)):
        shutil.copy(os.path.join(G, src), os.path.join(P, dst))
        print("copied", dst)
    else:
        print("MISSING", src)


copy("bench_%s.json" % tag, "r02_bench_final.json")
copy("bench_%s_reference.json" % tag, "r02_bench_final_reference.json")
copy("%s_trace_divergence.md" % tag, "r02_trace_divergence.md")
copy("%s_trace_divergence.json" % tag, "r02_trace_divergence.json")
copy("%s_trace_divergence_6dof.md" % tag, "r02_trace_divergence_6dof.md")
copy("%s_trace_divergence_6dof.json" % tag, "r02_trace_divergence_6dof.json")

# ---- launch list: per-kernel totals and shares
src = os.path.join(G, "launches_%s.csv" % tag)
if os.path.exists(src):
    rows = [r for r in csv.reader(open(src)) if len(r) > 10 and r[0].isdigit()]
    with open(os.path.join(P, "r02_launches.csv"), "w") as f:
        f.write('"ID","Kernel Name","Block Size","Grid Size","gpu__time_duration.sum [ns]"\n')
        for r in rows:
            f.write('"%s","%s","%s","%s","%s"\n' % (r[0], r[4][:110].replace('"', "'"), r[7], r[8], r[-1]))
    agg = collections.OrderedDict()
    for r in rows:
        a = agg.setdefault(r[4], [0, 0.0])
        a[0] += 1
        a[1] += float(r[-1].replace(",", ""))
    tot = sum(v[1] for v in agg.values())
    with open(os.path.join(P, "r02_launches.md"), "w") as f:
        f.write("# ncu launch list summary (profiles/r02_launches.csv): `ncu --metrics gpu__time_duration.sum --clock-control none "
                "-c 120 python bench.py --steps 2 --warmup 1 --no-cpu-baseline --no-configs`\n\nFinal round-2 code.  Per-launch times "
                "under ncu are cold-cache and serialised (the bench's overlapped steps run one after the other here); what must agree "
                "with bench.py is the solve kernel's SHARE of a step.\n\n| kernel | launches | total ms | share |\n|---|---|---|---|\n")
        for k, (n, ns) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
            f.write("| %s | %d | %.3f | %.2f%% |\n" % (k[:70], n, ns * 1e-6, 100 * ns / tot))
    print("wrote r02_launches.{csv,md}")

# ---- full captures
rep = os.path.join(G, "prof_%s_solve.ncu-rep" % tag)
if os.path.exists(rep):
    run(sys.executable, "scripts/ncu_summary.py", rep, os.path.join(P, "r02_solve_ncu_full.md"),
        "frustum_solve_kernel<float,4>, 512 clouds x 20480 points x 60 inits, final round-2 code; "
        "ncu --set full --metrics lts__t_bytes.sum --clock-control none")
    print(run(sys.executable, "scripts/ncu_traffic.py", rep, "512", "60", "1").stdout[-600:])
    srccsv = "/tmp/%s_src.csv" % tag
    open(srccsv, "w").write(run("ncu", "-i", rep, "--page", "source", "--csv").stdout)
    src2 = "/tmp/%s_src2.csv" % tag
    open(src2, "w").write(run("ncu", "-i", rep, "--page", "source", "--csv", "--print-source", "sass,cuda").stdout)
    tmp = "/tmp/%s_cubin" % tag
    os.makedirs(tmp, exist_ok=True)
    run("cuobjdump", "-xelf", "all", os.path.join(ROOT, "deepi2p_b200", "lib", "libdeepi2p_b200.so"), cwd=tmp)
    dis = run("nvdisasm", "-c", os.path.join(tmp, "frustum_solver.sm_90a.cubin")).stdout
    open("/tmp/%s.disasm" % tag, "w").write(dis)
    evals = "1547000"
    try:
        b = json.load(open(os.path.join(G, "bench_%s.json" % tag)))
        evals = str(int(b["roofline"]["mean_cloud_passes_per_solve"] * 512 * 60))
    except Exception:  # noqa: BLE001
        pass
    out = run(sys.executable, "scripts/ncu_by_function.py", srccsv, "/tmp/%s.disasm" % tag,
              "_ZN3dib20frustum_solve_kernelIfLi4EEEvNS_9SolveArgsE", evals).stdout
    open(os.path.join(P, "r02_solve_by_function.txt"), "w").write(out)
    out = run(sys.executable, "scripts/ncu_by_line.py", src2, "45").stdout
    open(os.path.join(P, "r02_solve_by_line.txt"), "w").write(out)
    print("wrote r02_solve_* summaries")
for op in ("index_max", "ball_query"):
    rep = os.path.join(G, "prof_%s_%s.ncu-rep" % (tag, op))
    if os.path.exists(rep):
        run(sys.executable, "scripts/ncu_summary.py", rep, os.path.join(P, "r02_%s_ncu_full.md" % op),
            "%s at BASELINE config 3 (B=64, C=M=64, N=16384, K=64), final round-2 code" % op)
        print("wrote r02_%s_ncu_full.md" % op)
