#!/usr/bin/env python
"""Turns the scratch output of profiles/capture.sh (gpurun_out/<round>/cap/) into the tracked artefacts:

  profiles/<round>_ncu_<name>.txt    summary of every .ncu-rep (ncu_summary.py)
  profiles/<round>_launches.csv      ncu launch list of the default bench command
  profiles/<round>_clocks.csv        nvidia-smi samples during the plain run
  profiles/<round>_bench*.json       the bench lines themselves
  profiles/<round>_batch_sweep.jsonl throughput / latency against the batch size
  profiles/ncu_traffic.json          dram__bytes_read+write per launch of each workload's top kernel, with the
                                     capture it came from (bench.py reports it as roofline.traffic / traffic_source)
  profiles/<round>_results.md        the table of measured numbers

usage: python profiles/collect.py r02        (run here, where ncu can read the reports)
"""
import csv
import glob
import json
import os
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R = sys.argv[1] if len(sys.argv) > 1 else "r02"
SRC = os.path.join(ROOT, "gpurun_out", R, "cap")
DST = os.path.join(ROOT, "profiles")
UNIT = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}


def raw(rep):
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    return rows[0], rows[1], rows[2:]


def dram_bytes(rep, kernel_substr):
    h, units, rows = raw(rep)
    ki, ri, wi = h.index("Kernel Name"), h.index("dram__bytes_read.sum"), h.index("dram__bytes_write.sum")
    for r in rows:
        if kernel_substr in r[ki]:
            return int(float(r[ri].replace(",", "")) * UNIT[units[ri]] + float(r[wi].replace(",", "")) * UNIT[units[wi]])
    return None


def launch_shares(path):
    """Per-kernel launch count, median and total time from the ncu launch list (cold-cache, serialised: shares, not
    absolutes)."""
    rows = [r for r in csv.reader(open(path, errors="replace")) if len(r) > 10]
    if not rows:
        return {}
    h = rows[0]
    ki, vi, ui = h.index("Kernel Name"), h.index("Metric Value"), h.index("Metric Unit")
    tot = {}
    for r in rows[1:]:
        t = float(r[vi].replace(",", "")) * {"ns": 1e-6, "us": 1e-3, "ms": 1.0, "s": 1e3}.get(r[ui], 1e-6)
        name = r[ki].split("(")[0].replace("void ", "")
        tot.setdefault(name, []).append(t)
    return tot


# what one pipeline_up batch launches (DESIGN.md section 3): kernel -> launches per batch
STEP = (("k_pipe_classify<1, 1, 0>", 1), ("k_rs_hist", 2), ("k_rs_scan", 2), ("k_rs_scatter", 2), ("k_heads", 1),
        ("k_resolve<1, 1, 0, 0>", 1))


def main():
    for rep in sorted(glob.glob(os.path.join(SRC, "*.ncu-rep"))):
        name = os.path.basename(rep)[:-len(".ncu-rep")]
        txt = subprocess.run([sys.executable, os.path.join(DST, "ncu_summary.py"), rep], capture_output=True, text=True).stdout
        open(os.path.join(DST, f"{R}_ncu_{name}.txt"), "w").write(txt)
    for f in ("launches.csv", "clocks.csv", "batch_sweep.jsonl"):
        for p in (os.path.join(SRC, f), os.path.join(ROOT, "gpurun_out", R, f)):
            if os.path.exists(p):
                shutil.copy(p, os.path.join(DST, f"{R}_{f}"))
                break
    for f in glob.glob(os.path.join(SRC, "bench*.json")):
        shutil.copy(f, os.path.join(DST, f"{R}_{os.path.basename(f)}"))

    traffic = {}
    for wl, rep, kern, label in (("pipeline_imix", "classify", "k_pipe_classify", "(k_pipe_classify<true, true>)"),
                                 ("dhcp", "dhcp", "k_dhcp_fastpath", "k_dhcp_fastpath"),
                                 ("antispoof_64", "antispoof_64", "k_antispoof", "k_antispoof"),
                                 ("nat_steady_64", "nat_steady_64", "k_pipe_classify", "(k_pipe_classify<false, false>)"),
                                 ("nat_cold_64", "nat_cold_64", "k_resolve", "(k_resolve<true, false, false>)"),
                                 ("nat_ingress_64", "nat_ingress_64", "k_nat_ingress", "k_nat_ingress")):
        p = os.path.join(SRC, f"{rep}.ncu-rep")
        if os.path.exists(p):
            b = dram_bytes(p, kern)
            if b:
                traffic[wl] = {label: {"bytes": b, "source": f"profiles/{R}_ncu_{rep}.txt (ncu --set full, one launch, "
                                                             f"N=1, 2^22 frames, workload-sized tables)"}}
    json.dump(traffic, open(os.path.join(DST, "ncu_traffic.json"), "w"), indent=1)

    L = [f"# Measured on H100 — round {R}", ""]
    p = os.path.join(DST, f"{R}_bench.json")
    if os.path.exists(p):
        j = json.loads(open(p).readline())
        r = j["roofline"]
        L += ["## The default `python bench.py` line (`profiles/%s_bench.json`)" % R, "",
              "| | |", "|---|---|",
              "| headline: %s, %d frames/step | **%.0f Mpps** device-resident, %.4f ms/step |" % (
                  j["config"]["workload"], j["config"]["frames_per_gpu_per_step"], j["value"], j["ms_per_step"]),
              "| end to end (`bng_prog_run(BNG_MEM_HOST)`, `bng_host_alloc` arena) | %.0f Mpps |" % j["e2e"]["value"],
              "| header-split ring (64-byte slots) | %s Mpps |" % (j.get("e2e_header_split") or {}).get("value"),
              "| kernels (CUDA events around every launch, separate pass) | `%s` |" % json.dumps(r["kernels_ms"]),
              "| dominant kernel | %s: %.4f ms, %.0f GB/s algorithmic = %.3f of %.0f GB/s |" % (
                  r["kernel"], r["kernel_ms"], r["achieved"], r["frac"], r["peak"]),
              "| its DRAM traffic (ncu) | %s bytes per launch = %.0f B/frame |" % (
                  r["traffic"], (r["traffic"] or 0) / j["config"]["frames_per_gpu_per_step"]),
              "| clocks | %s |" % json.dumps(j.get("clocks")),
              "| launches in the timed region | %s (%.1f per step) |" % (j["gpu_launches"], j["gpu_launches"] / j["steps"])]
        rc = j.get("reference_capacities")
        if rc:
            L += ["| same, every table at the reference's compile-time capacity | %.0f Mpps, %.4f ms/step, `%s` |" % (
                rc["value"], rc["ms_per_step"], json.dumps((rc.get("roofline") or {}).get("kernels_ms")))]
        cp = j.get("control_plane") or {}
        if cp:
            L += ["| one `Map.Put` (`bng_map_update`, synchronous) | median %s us, p99 %s us |" % (
                      cp.get("put_single_us", {}).get("median"), cp.get("put_single_us", {}).get("p99")),
                  "| staged upserts (`bng_map_update_staged` x %s + one `bng_sync`) | %s puts/s (staging %s us each through ctypes, apply %s ms) |" % (
                      cp.get("put_staged", {}).get("n"), cp.get("put_staged", {}).get("puts_per_s"),
                      cp.get("put_staged", {}).get("stage_us_each"), cp.get("put_staged", {}).get("apply_ms")),
                  "| batch upsert (`bng_map_update_batch`, %s entries) | %s puts/s |" % (
                      cp.get("put_batch", {}).get("n"), cp.get("put_batch", {}).get("puts_per_s")),
                  "| expiry sweep (`bng_sweep`, %s slots, %s live) | %s ms expiring %s sessions; scan only %s ms = %s GB/s |" % (
                      cp.get("sweep", {}).get("slots"), cp.get("sweep", {}).get("live_sessions"), cp.get("sweep", {}).get("ms"),
                      cp.get("sweep", {}).get("expired"), cp.get("sweep", {}).get("scan_only_ms"), cp.get("sweep", {}).get("scan_GBps"))]
        L += ["", "### The other BASELINE configs, from the same line (`workloads`)", "",
              "| workload | Mpps | ms/step | dominant kernel | its ms | frac of HBM peak | DRAM bytes/launch (ncu) |", "|---|---|---|---|---|---|---|"]
        for w, e in (j.get("workloads") or {}).items():
            L.append("| %s | %.0f | %.4f | %s | %.4f | %.3f | %s |" % (
                w, e["value"], e["ms_per_step"], e["kernel"].strip("()"), e["kernel_ms"], e["frac"], e.get("traffic")))
    L += ["", "## One `bench.py --workload W` line each (10 steps)", "",
          "| workload | Mpps (device-resident) | ms/step | whole-step frac | dominant kernel | its ms | its frac | e2e Mpps |",
          "|---|---|---|---|---|---|---|---|"]
    for n in ("pipeline_64", "nat_ingress_64", "qos_64", "qos_egress_64"):
        p = os.path.join(DST, f"{R}_bench_{n}.json")
        if not os.path.exists(p) or not open(p).readline().strip():
            continue
        j = json.loads(open(p).readline())
        r = j["roofline"]
        L.append("| %s | %.0f | %.4f | %.3f | %s | %.4f | %.3f | %.0f |" % (
            j["config"]["workload"], j["value"], j["ms_per_step"], r["step_frac"], r["kernel"].strip("()"), r["kernel_ms"],
            r["frac"], j["e2e"]["value"]))
    p = os.path.join(DST, f"{R}_bench_reference.json")
    if os.path.exists(p) and open(p).readline().strip():
        j = json.loads(open(p).readline())
        L += ["", "Reference arm (`bench.py --impl reference`, `oracle/_ref` = the reference's eBPF C): **%.1f Mpps** on %s "
              "host threads (%s)." % (j["value"], j["cpu_baseline"]["cores"], j["cpu_baseline"].get("sample", ""))]
    rows = []
    for tag, f in (("1", f"{R}_bench.json"), ("2", f"{R}_bench_2gpu.json"), ("4", f"{R}_bench_4gpu.json"), ("8", f"{R}_bench_8gpu.json")):
        pp = os.path.join(DST, f)
        if os.path.exists(pp) and open(pp).readline().strip():
            jj = json.loads(open(pp).readline())
            pg = jj.get("per_gpu_constant") or {}
            rows.append("| %s | %.0f | %.4f | %s | %.0f | %s | %s |" % (
                jj["n_gpus"], jj["value"], jj["ms_per_step"], (jj.get("details") or jj["config"]).get("subscribers_this_gpu"), jj["e2e"]["value"],
                pg.get("value"), (jj.get("stats_allreduce") or {}).get("matches_torch_allreduce")))
    if len(rows) > 1:
        L += ["", "## GPUs (torchrun, one rank per GPU, shard = splitmix64(mac) % N; each line measured on its own box)", "",
              "| N | Mpps (all GPUs) | ms/step (max over ranks) | subscribers on rank 0 | e2e Mpps | 10 k subscribers PER GPU: Mpps | `bng_sync_reduce` == torch all-reduce |",
              "|---|---|---|---|---|---|---|"] + rows
    p = os.path.join(DST, f"{R}_batch_sweep.jsonl")
    if os.path.exists(p):
        L += ["", "## Batch size (default workload, `tools/batch_sweep.sh`)", "",
              "| frames per batch | Mpps | ms per batch | e2e Mpps | launches per batch |", "|---|---|---|---|---|"]
        for line in open(p):
            if line.strip():
                s = json.loads(line)
                L.append("| %d | %.0f | %.4f | %.0f | %.1f |" % (s["frames"], s["Mpps"], s["ms_per_batch"], s["e2e_Mpps"],
                                                               s["launches_per_batch"]))
    p = os.path.join(DST, f"{R}_launches.csv")
    if os.path.exists(p):
        tot = launch_shares(p)
        med = lambda v: sorted(v)[len(v) // 2]
        L += ["", "## ncu launch list of `bench.py --steps 3 --warmup 3 --no-extra --e2e-steps 0` (`profiles/%s_launches.csv`)" % R, "",
              "Per-launch times under ncu are cold-cache and serialised; the SHARES of a batch are what is compared with the",
              "CUDA-event times above (median launch x launches per batch).", "",
              "| kernel | per batch | median ms | ms per batch | share of the batch (ncu) | share (CUDA events, bench line) |", "|---|---|---|---|---|---|"]
        per = {k: med(tot[k]) * c for k, c in STEP if k in tot}
        allt = sum(per.values()) or 1
        ev = {}
        pj = os.path.join(DST, f"{R}_bench.json")
        if os.path.exists(pj):
            km = json.loads(open(pj).readline())["roofline"]["kernels_ms"]
            tt = sum(km.values())
            ev = {"k_pipe_classify<1, 1, 0>": km.get("(k_pipe_classify<true, true>)", 0) / tt,
                  "k_resolve<1, 1, 0, 0>": km.get("(k_resolve<true, true, false>)", 0) / tt, "group": km.get("group_by_key", 0) / tt}
        for k, c in STEP:
            if k in tot:
                L.append("| %s | %d | %.4f | %.4f | %.1f %% | %s |" % (k, c, med(tot[k]), per[k], 100 * per[k] / allt,
                                                                    "%.1f %%" % (100 * ev[k]) if k in ev else ""))
        grp = sum(per.get(k, 0) for k in ("k_rs_hist", "k_rs_scan", "k_rs_scatter", "k_heads"))
        L.append("| (group-by: the four rows above) | 7 | | %.4f | %.1f %% | %s |" % (grp, 100 * grp / allt,
                                                                                 "%.1f %%" % (100 * ev["group"]) if ev else ""))
        L += ["", "Every kernel in the list:", "", "| kernel | launches | median ms | total ms |", "|---|---|---|---|"]
        for k, v in sorted(tot.items(), key=lambda kv: -sum(kv[1])):
            L.append("| %s | %d | %.4f | %.3f |" % (k, len(v), med(v), sum(v)))
    open(os.path.join(DST, f"{R}_results.md"), "w").write("\n".join(L) + "\n")
    print("\n".join(L))


if __name__ == "__main__":
    main()
