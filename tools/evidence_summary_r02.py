"""Turn gpurun_out/ev2/ (written by tools/evidence_r02.sh, or its refresh tools/evidence_r02b.sh, on the GPU box) into the tracked
profiles/*_r02.* files.  The refresh does not repeat the `ncu --set full` captures: when gpurun_out/ev2 holds none, the committed
profiles/ncu_top_r02.csv / ncu_traffic_r02.json are kept and quoted as they are.
usage: python tools/evidence_summary_r02.py"""
import collections, csv, json, os, shutil

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EV = os.path.join(ROOT, "gpurun_out", "ev2")
PR = os.path.join(ROOT, "profiles")
TAG = "r02"
WORKLOADS = ("resnet3d50", "r2plus1d34", "nonlocal50", "resnet18", "biggan256", "trn")


def last_json_line(path):
    for ln in reversed(open(path).read().strip().splitlines()):
        if ln.startswith("{"):
            return json.loads(ln)
    raise SystemExit("no JSON line in " + path)


def launch_rows(path):
    rows = []
    with open(path) as f:
        lines = [ln for ln in f if ln.startswith('"')]
    rd = csv.reader(lines)
    hdr = next(rd)
    ik, iv, iu, ig, ib = (hdr.index(k) for k in ("Kernel Name", "Metric Value", "Metric Unit", "Grid Size", "Block Size"))
    for r in rd:
        v = float(r[iv].replace(",", ""))
        us = v / 1e3 if r[iu].startswith("ns") else (v if r[iu].startswith("us") else v * 1e3)
        rows.append((r[ik], us, r[ig], r[ib]))
    return rows


def short(name):
    n = name.replace("void ", "").replace("b2::", "")
    n = n.split("(CUtensorMap")[0].split("(const")[0].split("(b2")[0]
    return n.replace("(int)", "")[:48]


_SCALE = {"byte": 1e-6, "Kbyte": 1e-3, "Mbyte": 1.0, "Gbyte": 1e3, "ns": 1e-3, "us": 1.0, "ms": 1e3, "s": 1e6}


def raw_metrics(path):
    rows = list(csv.reader(open(path)))
    out = {}
    for h, u, v in zip(rows[0], rows[1], rows[2]):
        if u in _SCALE:
            try:
                v = "%.6f" % (float(v.replace(",", "")) * _SCALE[u])
            except ValueError:
                pass
        out[h] = v
    return out


def fnum(x):
    try:
        return float(str(x).replace(",", ""))
    except ValueError:
        return float("nan")


def main():
    os.makedirs(PR, exist_ok=True)
    bench = last_json_line(os.path.join(EV, "bench.json"))
    json.dump(bench, open(os.path.join(PR, "bench_%s.json" % TAG), "w"), indent=1)
    ref = last_json_line(os.path.join(EV, "bench_reference.json"))
    json.dump(ref, open(os.path.join(PR, "bench_reference_%s.json" % TAG), "w"), indent=1)
    shutil.copy(os.path.join(EV, "pytest_gpu.txt"), os.path.join(PR, "pytest_gpu_%s.txt" % TAG))
    lines = {}
    for w in WORKLOADS:
        if not os.path.exists(os.path.join(EV, "line_%s.json" % w)):
            continue
        shutil.copy(os.path.join(EV, "layers_%s.txt" % w), os.path.join(PR, "layers_%s_%s.txt" % (w, TAG)))
        lines[w] = last_json_line(os.path.join(EV, "line_%s.json" % w))
    with open(os.path.join(PR, "workloads_%s.jsonl" % TAG), "w") as f:
        for w in WORKLOADS:
            if w in lines:
                f.write(json.dumps(lines[w]) + "\n")

    # ---- launch lists: the second forward of tools/fwd_once.py (per-kernel device time, cold cache, serialised) ----
    launch_txt = []
    for w in ("resnet3d50", "r2plus1d34"):
        rows = launch_rows(os.path.join(EV, "launches_%s.csv" % w))
        starts = [i for i, r in enumerate(rows) if "ncdhw" in r[0]]
        steady = rows[starts[-1]:]
        with open(os.path.join(PR, "launches_%s_%s.csv" % (w, TAG)), "w") as f:
            f.write("index,kernel,grid,block,duration_us\n")
            for i, (k, us, g, b) in enumerate(steady):
                f.write('%d,"%s","%s","%s",%.3f\n' % (i, short(k), g, b, us))
        agg = collections.OrderedDict()
        for k, us, _, _ in steady:
            a = agg.setdefault(short(k), [0, 0.0]); a[0] += 1; a[1] += us
        tot = sum(a[1] for a in agg.values())
        launch_txt.append("%s: %d launches per forward, %.3f ms of kernel time (cold cache, serialised by ncu; graph replay: %.3f ms)"
                          % (w, len(steady), tot / 1e3, lines[w]["ms_per_step"]))
        for k, (n, us) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
            launch_txt.append("  %-48s n=%3d  %8.3f ms  %5.1f%%" % (k, n, us / 1e3, 100 * us / tot))

    # ---- ncu --set full captures ----
    want = [("duration_us", "gpu__time_duration.sum"), ("grid", "launch__grid_size"), ("regs", "launch__registers_per_thread"),
            ("dram_read_MB", "dram__bytes_read.sum"), ("dram_write_MB", "dram__bytes_write.sum"),
            ("dram_pct", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed"),
            ("tensor_pipe_active_pct", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed"),
            ("l2_throughput_pct", "lts__throughput.avg.pct_of_peak_sustained_elapsed"),
            ("l2_hit_pct", "lts__t_sector_hit_rate.pct"), ("l1tex_pct", "l1tex__throughput.avg.pct_of_peak_sustained_elapsed")]
    captures = [
        ("ncu_stem_poolw", "stemconv<64> conv 7x7x7 s122 C3->64 + BN + ReLU + W max-pool, B=32 16x224x224", "conv 7x7x7 s122 C3->64 M=6422528 +poolW", 154.1e6 + 411.0e6),
        ("ncu_slab64", "slabconv<64> conv 3x3x3 C64->64, 32x8x56x56", "conv 3x3x3 s111 C64->64 M=802816", 2 * 802816 * 64 * 2.0),
        ("ncu_slab128", "slabconv<128> conv 3x3x3 C128->128, 32x4x28x28", "conv 3x3x3 s111 C128->128 M=100352", 2 * 100352 * 128 * 2.0 + 27 * 128 * 128 * 2.0),
        ("ncu_pgemm_64_256", "pgemm<128,0> conv 1x1x1 C64->256, 32x8x56x56 (no residual)", "conv 1x1x1 s111 C64->256 M=802816", 802816 * (64 + 256) * 2.0),
        ("ncu_densem_l4", "densem (split-K cluster) conv 1x3x3 C512->1152, 16x2x4x4 (M = 512)", None, 512 * (512 + 1152) * 2.0 + 9 * 512 * 1152 * 2.0),
        ("ncu_slab_r2p1d_144", "slabconv<0> conv 1x3x3 C64->144 (runtime N = 144), 16x16x28x28", None, 200704 * (64 + 144) * 2.0),
        ("ncu_attention", "attention_online<256> B=8 N=6272 d=256 dv=256", None, 8 * 6272 * (256 * 3 + 256) * 2.0),
        ("ncu_gan_conv1_bn1A", "pgemm<64,1> BigGAN conv1 1x1 C256->64 at 128x128 with bn1+ReLU on the A operand and bn2+ReLU in the epilogue, 64 images", None, 64 * 16384 * (256 + 64) * 2.0),
        ("ncu_gan_conv64", "slabconv<64> BigGAN conv 3x3 C64->64 at 256x256, 64 images, per-sample affine", None, 2 * 64 * 65536 * 64 * 2.0),
    ]
    top_lines, traffic = [], {}
    have_caps = any(os.path.exists(os.path.join(EV, fn + ".raw.csv")) for fn, _, _, _ in captures)
    if not have_caps:          # refresh without new captures: quote the committed summary
        with open(os.path.join(PR, "ncu_top_%s.csv" % TAG)) as f:
            rd = csv.DictReader(f)
            for d in rd:
                top_lines.append("%-100s %8.1f us  dram R %7.1f + W %7.1f MB vs %7.1f algorithmic (dram %4.1f%%)  tensor-pipe %4.1f%%  L2 %4.1f%%  regs %3d" % (
                    d["capture"], float(d["duration_us"]), float(d["dram_read_MB"]), float(d["dram_write_MB"]), float(d["algorithmic_MB"]),
                    float(d["dram_pct"]), float(d["tensor_pipe_active_pct"]), float(d["l2_throughput_pct"]), int(float(d["regs"]))))
    with open(os.path.join(PR, "ncu_top_%s.csv" % TAG), "w" if have_caps else "a") as f:
        if not have_caps:
            captures = []
        else:
            f.write("capture," + ",".join(k for k, _ in want) + ",algorithmic_MB\n")
        for fn, label, desc, alg in captures:
            path = os.path.join(EV, fn + ".raw.csv")
            if not os.path.exists(path) or os.path.getsize(path) < 100:
                continue
            m = raw_metrics(path)
            vals = [fnum(m.get(metric, "nan")) for _, metric in want]
            f.write('"%s",' % label + ",".join("%.3f" % v for v in vals) + ",%.1f\n" % (alg / 1e6))
            d = dict(zip([k for k, _ in want], vals))
            top_lines.append("%-100s %8.1f us  dram R %7.1f + W %7.1f MB vs %7.1f algorithmic (dram %4.1f%%)  tensor-pipe %4.1f%%  L2 %4.1f%%  regs %3d" % (
                label, d["duration_us"], d["dram_read_MB"], d["dram_write_MB"], alg / 1e6, d["dram_pct"], d["tensor_pipe_active_pct"],
                d["l2_throughput_pct"], int(d["regs"])))
            traffic[label] = {"dram_bytes": int((d["dram_read_MB"] + d["dram_write_MB"]) * 1e6), "algorithmic_bytes": int(alg),
                              "bench_desc": desc}
    if have_caps:
      json.dump({"_comment": "dram__bytes_read.sum + dram__bytes_write.sum per launch from `ncu --set full --clock-control none` captures "
                           "(tools/evidence_r02.sh); bench.py leaves roofline.traffic null because DRAM counters cannot be read in an "
                           "un-profiled run -- this file is the ncu measurement of the same kernels at the same shapes",
               "captures": traffic}, open(os.path.join(PR, "ncu_traffic_%s.json" % TAG), "w"), indent=1)

    out = ["# profiles/ -- round 2 evidence (H100, sm_90a)\n",
           "Produced by `tools/evidence_r02.sh` (ncu --set full captures) and its refresh `tools/evidence_r02b.sh` (tests, bench lines, layer "
           "tables, launch lists, sanitizer passes with the final kernels) on H100 machines, summarised by "
           "`tools/evidence_summary_r02.py`.  No throughput number was taken under a profiler.\n",
           "## Bench lines (`python bench.py [--workload W]`, N = 1)\n"]
    for w in WORKLOADS:
        if w not in lines:
            continue
        ln = lines[w]
        e2e = ln["e2e"]
        out.append("* **%s** (%s): **%.0f %s** device-resident (%.3f ms per step); e2e from fp32 pinned host input %.0f%s; parity vs the CPU oracle: %s; "
                   "mixed per-launch roofline fraction %.2f; dominant kernel `%s` at %.2f of its %s peak."
                   % (w, ln["config"]["workload"], ln["value"], ln["unit"], ln["ms_per_step"], e2e["value"],
                      (", %.0f from uint8 frames, %.0f from fp16" % (e2e["uint8_frames_value"], e2e["fp16_input_value"])) if e2e.get("uint8_frames_value") else "",
                      json.dumps({k: ln["parity"][k] for k in ln["parity"] if k not in ("checker", "bound", "tolerance")}) if ln.get("parity") else "n/a",
                      ln["roofline"]["mixed"]["frac"], ln["roofline"]["kernel"].split(" (")[0], ln["roofline"]["frac"], ln["roofline"]["bound"]))
    out.append("\nDefault line (`bench_%s.json`): value %.0f clips/s, e2e %.0f, cpu_baseline %s clips/s on %s host threads (kind %s); sub-lines: %s.\n"
               % (TAG, bench["value"], bench["e2e"]["value"], "%.2f" % bench["cpu_baseline"]["value"] if bench.get("cpu_baseline") else "n/a",
                  bench["cpu_baseline"]["cores"] if bench.get("cpu_baseline") else "?", bench["cpu_baseline"]["kind"] if bench.get("cpu_baseline") else "?",
                  ", ".join("%s %.0f %s" % (k, bench[k]["value"], bench[k]["unit"]) for k in ("biggan256", "r2plus1d34", "nonlocal50") if isinstance(bench.get(k), dict) and "value" in bench[k])))
    # ---- sanitizer passes (tools/sanitize.sh all) ----
    san_dir = os.path.join(ROOT, "gpurun_out", "sanitizer")
    san = []
    for tool in ("memcheck", "synccheck", "racecheck"):
        logp, outp = os.path.join(san_dir, tool + ".log"), os.path.join(san_dir, tool + ".out")
        if not os.path.exists(logp):
            continue
        log = open(logp).read().strip().splitlines()
        summary = [l_ for l_ in log if "ERROR SUMMARY" in l_ or "RACECHECK SUMMARY" in l_]
        cases = [l_ for l_ in open(outp).read().splitlines() if l_.strip() and not l_.startswith("=")] if os.path.exists(outp) else []
        san.append("== compute-sanitizer --tool %s  (kernels of namespace b2 only): %s" % (tool, summary[-1].replace("=========", "").strip() if summary else "no summary line"))
        san += ["   " + c_ for c_ in cases]
        extra = [l_ for l_ in log if l_.startswith("=========") and ("Error" in l_ or "Warning" in l_ or "hazard" in l_.lower() or "Uninitialized" in l_)]
        seen = collections.Counter(" ".join(e.replace("=========", "").split()[:12]) for e in extra)
        san += ["   finding x%d: %s" % (n, k) for k, n in seen.most_common(12)]
    if san:
        san.append("racecheck note: every displayed hazard (40 of 344; the rest are cut by --print-limit) is the write-after-write pair (cp.async operand gather into the ring) / (st.shared::cluster "
                   "partial sums into the same ring reused as reduction staging) of densem_kernel; the two are separated by the MMA-complete mbarrier "
                   "and a barrier.cluster arrive.release / wait.acquire, which racecheck does not model.  Kernels that use CTA-scope barriers only "
                   "report nothing.")
        open(os.path.join(PR, "sanitizer_%s.txt" % TAG), "w").write("\n".join(san) + "\n")
        out.append("## compute-sanitizer (`sanitizer_%s.txt`, tools/sanitize.sh)\n" % TAG)
        out.append("```\n" + "\n".join(l_ for l_ in san if l_.startswith("==") or "finding" in l_ or l_.startswith("racecheck note")) + "\n```\n")
    out.append("## Trunk schedule sweep (`dfs_sweep_%s.txt`, tools/dfs_sweep.py)\n" % TAG)
    out.append("Depth-first (L2-resident) walks of the early stages in clip chunks against the breadth-first walk, CUDA-graph-timed: every "
               "chunked schedule is slower on every workload (DESIGN.md section 3c); breadth-first is the default.\n")
    out.append("## Temporal stack kernel (`tstack_sweep_%s.txt`, tools/conv_sweep.py)\n" % TAG)
    out.append("(kt,1,1) Cout = 64 layers of R(2+1)D-34, CUDA-graph-timed: (7,1,1) C110->64 on 16 clips 263.6 -> 167.8 us, (3,1,1) C144->64 "
               "+ residual 39.3 -> 32.2 us; whole network 7307 -> 7889 clips/s.  The r2plus1d34 line and layer table above are from the run "
               "with the kernel; the `r2plus1d34` sub-line inside `bench_%s.json` and `launches_r2plus1d34_%s.csv` were taken just before it "
               "was added (slab kernel on those 13 launches).\n" % (TAG, TAG))
    out.append("## ncu launch lists (`launches_*_%s.csv`)\n" % TAG)
    out.append("```\n" + "\n".join(launch_txt) + "\n```\n")
    out.append("## ncu --set full captures (`ncu_top_%s.csv`, `ncu_traffic_%s.json`)\n" % (TAG, TAG))
    out.append("```\n" + "\n".join(top_lines) + "\n```\n")
    out.append("Other files: `layers_<workload>_%s.txt` (per-launch CUDA-event tables, `bench.py --layers`; the `roof` column is the launch's "
               "max(FLOP/peak, bytes/BW) over its measured time), `workloads_%s.jsonl` (one full bench line per BASELINE config), "
               "`smallm_sweep_%s.txt` / `slab_mt_sweep_%s.txt` (CUDA-graph-timed single-layer sweeps, tools/conv_sweep.py), `pytest_gpu_%s.txt`.\n"
               % ((TAG,) * 5))
    open(os.path.join(PR, "README_%s.md" % TAG), "w").write("\n".join(out))
    print("\n".join(out))


if __name__ == "__main__":
    main()
