"""Turn gpurun_out/ev/ (written by tools/evidence.sh on the GPU box) into the tracked profiles/ files of a round.
usage: python tools/evidence_summary.py [round_tag]     (default r01)"""
import collections, csv, json, os, shutil, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EV = os.path.join(ROOT, "gpurun_out", "ev")
PR = os.path.join(ROOT, "profiles")
TAG = sys.argv[1] if len(sys.argv) > 1 else "r01"


def read(name):
    with open(os.path.join(EV, name)) as f:
        return f.read()


def last_json_line(text):
    for ln in reversed(text.strip().splitlines()):
        if ln.startswith("{"):
            return json.loads(ln)
    raise SystemExit("no JSON line")


def launch_rows():
    rows = []
    with open(os.path.join(EV, "launches_all.csv")) as f:
        lines = [ln for ln in f if not ln.startswith("==")]
    for r in csv.DictReader(lines):
        if r.get("Metric Name") == "gpu__time_duration.sum":
            v = float(r["Metric Value"].replace(",", ""))
            unit = r["Metric Unit"]
            us = v / 1e3 if unit.startswith("ns") else (v if unit.startswith("us") else v * 1e3)
            rows.append((r["Kernel Name"], us, r["Grid Size"], r["Block Size"]))
    return rows


def short(name):
    n = name.replace("void ", "").replace("b2::", "")
    n = n.split("(CUtensorMap")[0].split("(const")[0].split("(b2")[0]
    return n.replace("(int)", "")[:44]


_SCALE = {"byte": 1e-6, "Kbyte": 1e-3, "Mbyte": 1.0, "Gbyte": 1e3, "ns": 1e-3, "us": 1.0, "ms": 1e3, "s": 1e6}


def raw_metrics(path):
    """metric -> value of the first profiled launch, bytes normalised to MB and times to us (ncu picks the unit per column)."""
    rows = list(csv.reader(open(path)))
    hdr, units, vals = rows[0], rows[1], rows[2]
    out = {}
    for h, u, v in zip(hdr, units, vals):
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
    bench = last_json_line(read("bench.json"))
    json.dump(bench, open(os.path.join(PR, "bench_%s.json" % TAG), "w"), indent=1)
    ref = last_json_line(read("bench_reference.json"))
    json.dump(ref, open(os.path.join(PR, "bench_reference_%s.json" % TAG), "w"), indent=1)
    shutil.copy(os.path.join(EV, "layers.txt"), os.path.join(PR, "layers_%s.txt" % TAG))
    shutil.copy(os.path.join(EV, "others.jsonl"), os.path.join(PR, "others_%s.jsonl" % TAG))
    shutil.copy(os.path.join(EV, "others_layers.txt"), os.path.join(PR, "others_layers_%s.txt" % TAG))
    shutil.copy(os.path.join(EV, "pytest_gpu.txt"), os.path.join(PR, "pytest_gpu_%s.txt" % TAG))

    # ---- launch list: the last two forwards of the run (the eager profiling passes at the end of bench.py) ----
    rows = launch_rows()
    starts = [i for i, r in enumerate(rows) if "ncdhw_to_ndhwc" in r[0]]
    lo = starts[-2] if len(starts) >= 2 else 0
    steady = rows[lo:]
    with open(os.path.join(PR, "launches_%s.csv" % TAG), "w") as f:
        f.write("index,kernel,grid,block,duration_us\n")
        for i, (k, us, g, b) in enumerate(steady):
            f.write('%d,"%s","%s","%s",%.3f\n' % (i, short(k), g, b, us))
    agg = collections.OrderedDict()
    for k, us, _, _ in steady:
        a = agg.setdefault(short(k), [0, 0.0]); a[0] += 1; a[1] += us
    tot = sum(a[1] for a in agg.values())
    launch_txt = ["launches profiled: %d (two steady-state forwards), total %.3f ms" % (len(steady), tot / 1e3)]
    for k, (n, us) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        launch_txt.append("  %-44s n=%3d  %8.3f ms  %5.1f%%" % (k, n, us / 1e3, 100 * us / tot))

    # ---- ncu --set full captures ----
    want = [("duration_us", "gpu__time_duration.sum"), ("grid", "launch__grid_size"), ("regs", "launch__registers_per_thread"),
            ("dram_read_MB", "dram__bytes_read.sum"), ("dram_write_MB", "dram__bytes_write.sum"),
            ("dram_pct", "dram__cycles_active.avg.pct_of_peak_sustained_elapsed"),
            ("tensor_pipe_active_pct", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed"),
            ("sm_throughput_pct", "sm__throughput.avg.pct_of_peak_sustained_elapsed"),
            ("l2_hit_pct", "lts__t_sector_hit_rate.pct"), ("l1tex_pct", "l1tex__throughput.avg.pct_of_peak_sustained_elapsed")]
    top_lines = []
    traffic, gan_traffic = {}, {}
    captures = [("ncu_stem", "stemconv<64>  conv 7x7x7 s122 C3->64, B=32 16x224x224", "conv 7x7x7 s122 C3->64 M=6422528"),
                ("ncu_slab64", "slabconv<64>  conv 3x3x3 C64->64, 32x8x56x56", "conv 3x3x3 s111 C64->64 M=802816"),
                ("ncu_slab128", "slabconv<128> conv 3x3x3 C128->128, 32x4x28x28", "conv 3x3x3 s111 C128->128 M=100352"),
                ("ncu_pgemm_64_256", "pgemm<128>    conv 1x1x1 C64->256, 32x8x56x56 (no residual)", "conv 1x1x1 s111 C64->256 M=802816"),
                ("ncu_slab_r2p1d_144", "slabconv<0>   conv 1x3x3 C64->144 (runtime N=144), 16x16x28x28", None),
                ("ncu_attention", "attention_online<256>  B=8 N=6272 d=256 dv=256", None),
                ("ncu_gan_conv64", "slabconv<64>  BigGAN conv 3x3 C64->64 at 256x256, 64 images, per-sample affine", "gan:conv 1x3x3 s111 C64->64 M=16777216"),
                ("ncu_gan_upconv64", "slabconv<64>  BigGAN conv 3x3 of the upsampled image (4 folded 2x2 phases) C64->64, 128->256, 64 images", "gan:conv 1x3x3 s111 C64->64 M=16777216 up2"),
                ("ncu_gan_conv128", "slabconv<128> BigGAN conv 3x3 C128->128 at 128x128, 64 images", "gan:conv 1x3x3 s111 C128->128 M=4194304"),
                ("ncu_gan_pgemm_64_128", "pgemm<128>    BigGAN conv 1x1 C64->128 at 256x256, 64 images", "gan:conv 1x1x1 s111 C64->128 M=16777216")]
    with open(os.path.join(PR, "ncu_top_%s.csv" % TAG), "w") as f:
        f.write("capture," + ",".join(k for k, _ in want) + "\n")
        for fn, label, desc in captures:
            path = os.path.join(EV, fn + ".raw.csv")
            if not os.path.exists(path):
                continue
            m = raw_metrics(path)
            vals = [fnum(m.get(metric, "nan")) for _, metric in want]
            f.write('"%s",' % label + ",".join("%.3f" % v for v in vals) + "\n")
            d = dict(zip([k for k, _ in want], vals))
            top_lines.append("%-62s %8.1f us  dram R %7.1f W %7.1f MB (%4.1f%%)  tensor-pipe %4.1f%%  L2 hit %4.1f%%  regs %3d" % (
                label, d["duration_us"], d["dram_read_MB"], d["dram_write_MB"], d["dram_pct"], d["tensor_pipe_active_pct"],
                d["l2_hit_pct"], int(d["regs"])))
            if desc and desc.startswith("gan:"):      # captured on 64 images; the bench runs 256: per-launch traffic x 4
                gan_traffic[desc[4:]] = int((d["dram_read_MB"] + d["dram_write_MB"]) * 1e6) * 4
            elif desc:
                traffic[desc] = int((d["dram_read_MB"] + d["dram_write_MB"]) * 1e6)
    json.dump({"_comment": "dram__bytes_read.sum + dram__bytes_write.sum per launch from `ncu --set full --clock-control none` "
                           "captures of single layers at the BASELINE shapes (tools/conv_micro.py, tools/gan_micro.py, "
                           "tools/evidence.sh); the BigGAN layers were captured on 64 images and scaled x4 to the B=256 launch",
               "B=32": traffic, "biggan B=256": gan_traffic}, open(os.path.join(PR, "ncu_traffic_%s.json" % TAG), "w"), indent=1)

    # ---- README body (numbers only; prose lives in profiles/README_<tag>.md, regenerated here) ----
    rl, e2e, cb = bench["roofline"], bench["e2e"], bench.get("cpu_baseline") or {}
    out = []
    out.append("# profiles/ — round %s evidence (H100, sm_90a)\n" % TAG[1:])
    out.append("Produced by `tools/evidence.sh` on an H100 machine and summarised by `tools/evidence_summary.py`; no "
               "throughput number was taken under a profiler.  Files: `bench_%s.json` (the bench line), `bench_reference_%s.json` "
               "(`--impl reference`), `layers_%s.txt` (per-launch CUDA-event table, `bench.py --layers`), `launches_%s.csv` (ncu "
               "`gpu__time_duration.sum` launch list of `bench.py`, last two forwards), `ncu_top_%s.csv` + `ncu_traffic_%s.json` "
               "(`--set full` captures of the top kernels), `others_%s.jsonl` / `others_layers_%s.txt` (the other BASELINE "
               "configs), `pytest_gpu_%s.txt`.\n" % ((TAG,) * 9))
    out.append("## Bench line (`python bench.py`, N=1, K=%d, W=%d)\n" % (bench["steps"], bench["warmup"]))
    out.append("* value **%.0f clips/s** (%.3f ms per 32-clip step, CUDA-graph replay, input resident in HBM); clocks %s/%s MHz, "
               "reasons %s, %.0f W max." % (bench["value"], bench["ms_per_step"], bench["clocks"].get("sm_mhz"),
                                            bench["clocks"].get("sm_max_mhz"), bench["clocks"].get("reasons"),
                                            bench["clocks"].get("power_w_max", float("nan"))))
    out.append("* e2e **%.0f clips/s** with fp16 pinned host clips (%.0f MB H2D + %.0f KB D2H per step, copy of batch i+1 overlapped "
               "with forward i); %.0f clips/s with fp32 host clips (%.0f MB per step)." % (
                   e2e["value"], e2e["h2d_bytes_per_step"] / 1e6, e2e["d2h_bytes_per_step"] / 1e3, e2e["fp32_input_value"],
                   e2e["fp32_input_h2d_bytes_per_step"] / 1e6))
    out.append("* roofline (tensor), dominant kernel `%s`: %.0f TFLOP/s algorithmic = **%.1f %%** of the measured sustained %.0f "
               "TFLOP/s, %.3f ms per launch, %.1f %% of the step; DRAM traffic %s B for %.0f B algorithmic.  Family (%s): %.0f "
               "TFLOP/s = %.1f %%; whole step %.0f TFLOP/s = %.1f %%." % (
                   rl["kernel"], rl["achieved"], 100 * rl["frac"], rl["peak"], rl["ms_per_launch"], 100 * rl["share_of_step"],
                   rl["traffic"], rl["algorithmic_bytes"], rl["family"]["kernels"], rl["family"]["achieved"],
                   100 * rl["family"]["frac"], rl["whole_step_tflops"], 100 * rl["whole_step_frac"]))
    if cb:
        out.append("* cpu_baseline: %.2f %s (%s, %s host threads; %s)." % (cb["value"], cb["unit"], cb["kind"], cb["cores"], cb["sample"]))
    out.append("* reference arm (`--impl reference`): %.2f %s (%s)." % (ref["value"], ref["unit"], ref.get("cpu_baseline", {}).get("sample", "")))
    out.append("\n## Per-launch table of one forward (CUDA events on the launching stream, eager pass)\n\n```")
    out.append(read("layers.txt").rstrip())
    out.append("```\n\n## ncu launch list of the same command (cold-cache, serialised: shares, not absolutes)\n\n```")
    out.extend(launch_txt)
    out.append("```\n\n## ncu --set full, one launch per kernel at the BASELINE shapes\n\n```")
    out.extend(top_lines)
    # ---- BigGAN-deep-256 (BASELINE configs[4]) ----
    try:
        bg = last_json_line(read("biggan.json"))
        json.dump(bg, open(os.path.join(PR, "bench_biggan256_%s.json" % TAG), "w"), indent=1)
        shutil.copy(os.path.join(EV, "biggan_layers.txt"), os.path.join(PR, "layers_biggan256_%s.txt" % TAG))
        bref = last_json_line(read("biggan_reference.json"))
        json.dump(bref, open(os.path.join(PR, "bench_biggan256_reference_%s.json" % TAG), "w"), indent=1)
        brl, be = bg["roofline"], bg["e2e"]
        out.append("```\n\n## BigGAN-deep-256 generator (`python bench.py --workload biggan256`; also the `biggan256` key of the default line)\n")
        out.append("* value **%.0f images/s** (%.2f ms per %d-image step, CUDA-graph replay), e2e **%.0f images/s** (%.0f KB H2D + "
                   "%.0f MB D2H per step); %.1f GFLOP/image algorithmic -> %.0f TFLOP/s = %.1f %% of the sustained tensor peak for the "
                   "whole step." % (bg["value"], bg["ms_per_step"], bg["config"]["global_batch"], be["value"], be["h2d_bytes_per_step"] / 1e3,
                                    be["d2h_bytes_per_step"] / 1e6, brl["whole_step_tflops"] * 1e3 / bg["value"], brl["whole_step_tflops"],
                                    100 * brl["whole_step_frac"]))
        if brl["bound"] == "tensor" and brl["algorithmic_bytes"] / (brl["ms_per_launch"] * 1e-3) / 1e9 > 0.25 * brl["hbm_passes"]["peak_gbs"]:
            # line produced before bench.py classified the dominant kernel by its arithmetic intensity: a 1x1 layer is HBM-bound
            gbs = brl["algorithmic_bytes"] / (brl["ms_per_launch"] * 1e-3) / 1e9
            brl = dict(brl, bound="hbm", achieved=gbs, unit="GB/s", frac=gbs / brl["hbm_passes"]["peak_gbs"])
        out.append("* dominant kernel `%s` (%s-bound): %.0f %s = %.1f %% of the measured peak, %.1f %% of the step, DRAM traffic %s B for %.0f B "
                   "algorithmic; HBM-bound helper passes (%s): %.0f GB/s of %.0f, %.1f %% of the step." % (
                       brl["kernel"], brl["bound"], brl["achieved"], brl["unit"], 100 * brl["frac"], 100 * brl["share_of_step"], brl["traffic"], brl["algorithmic_bytes"],
                       brl["hbm_passes"]["kernels"], brl["hbm_passes"]["achieved_gbs"] or 0, brl["hbm_passes"]["peak_gbs"],
                       100 * brl["hbm_passes"]["share_of_step"]))
        cbb = bg.get("cpu_baseline") or {}
        if cbb:
            out.append("* cpu_baseline: %.2f %s on %s host threads (%s); reference arm: %.2f %s." % (
                cbb["value"], cbb["unit"], cbb["cores"], cbb["sample"], bref["value"], bref["unit"]))
        out.append("\n```")
        out.append(read("biggan_layers.txt").rstrip())
    except (OSError, KeyError, SystemExit) as exc:
        out.append("```\n\n(BigGAN evidence missing: %s)\n\n```" % exc)
    out.append("```\n\n## Other BASELINE configs (parity-test cases; device-resident, CUDA-graph replay, 1 GPU)\n\n```")
    out.append(read("others.jsonl").rstrip())
    out.append("```\n\nPer-layer tables of those runs: `others_layers_%s.txt`.\n" % TAG)
    notes = os.path.join(PR, "NOTES_%s.md" % TAG)
    if os.path.exists(notes):
        out.append(open(notes).read())
    open(os.path.join(PR, "README_%s.md" % TAG), "w").write("\n".join(out) + "\n")
    print("\n".join(out[:12]))


if __name__ == "__main__":
    main()
