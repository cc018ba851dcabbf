"""Render a bench.py JSON line as a markdown summary (python tools/bench_summary.py line.json)."""
import json
import sys


def f(v, unit=""):
    if v is None:
        return "n/a"
    if abs(v) >= 1e6:
        return "%.2f M%s" % (v / 1e6, unit)
    if abs(v) >= 1e3:
        return "%.1f k%s" % (v / 1e3, unit)
    return "%.3g%s" % (v, unit)


def main(path):
    d = json.loads([l for l in open(path).read().splitlines() if l.startswith("{")][-1])
    print("# bench.py summary (`%s`)\n" % path)
    print("n_gpus %d, steps %d x repeats, warmup %d, dtype %s, data %s\n" % (d["n_gpus"], d["steps"], d["warmup"], d["dtype"], d["data"]))
    print("| workload | scaling | value (device-resident) | e2e pipelined | e2e predict_stream | e2e sync per step | region s | SM MHz (reasons) | CPU baseline (cores) | parity max dp |")
    print("|---|---|---|---|---|---|---|---|---|---|")
    for name, w in d["workloads"].items():
        if "error" in w:
            print("| %s | failed: %s |" % (name, w["error"]))
            continue
        e = w.get("e2e", {})
        ck = w.get("clocks") or {}
        cpu = w.get("cpu_baseline") or {}
        print("| %s | %s | %s | %s | %s | %s | %.2f | %s (%s) | %s (%s) | %s |" % (
            name, w.get("scaling"), f(w["value"], " " + w.get("unit", "sites/s")), f(e.get("value"), ""), f((e.get("predict_stream") or {}).get("value"), ""),
            f((e.get("synchronous_per_step") or {}).get("value"), ""), w.get("timed_region_s", 0), ck.get("sm_mhz"), ",".join(ck.get("reasons") or []) or "none",
            f(cpu.get("value"), ""), cpu.get("cores"), ("%.1e" % w["parity_max_abs_dp"]) if w.get("parity_max_abs_dp") is not None else "n/a"))
    for name, w in d["workloads"].items():
        if "kernels" not in w:
            continue
        r = w["roofline"]
        print("\n## %s: kernels (single stream, CUDA events around every launch)\n" % name)
        print("dominant: `%s` %.1f TFLOP/s = %.3f of the %.0f TFLOP/s burst peak; whole step %.0f TFLOP/s = %.3f of sustained, %.3f of burst; "
              "DRAM bytes per step (ncu, all kernels) %s vs compulsory %s\n" % (
                  r["kernel"], r["achieved"], r["frac"], r["peak"], r["whole_step"]["achieved"], r["whole_step"]["frac_of_sustained"],
                  r["whole_step"]["frac_of_burst"], f(r["whole_step"].get("dram_bytes_per_step_all_kernels"), "B"),
                  f(r["whole_step"].get("compulsory_bytes_per_step"), "B")))
        print("| kernel | us per launch | CTAs | SM-time ms | SM-time share | TFLOP/s | frac of burst (whole GPU) | frac of burst (occupied SMs) |")
        print("|---|---|---|---|---|---|---|---|")
        for kn, k in sorted(w["kernels"].items(), key=lambda kv: -kv[1].get("sm_time_ms", kv[1]["ms_per_launch"])):
            print("| %s | %.1f | %.0f | %.2f | %.1f%% | %s | %s | %s |" % (
                kn, k["ms_per_launch"] * 1e3, k.get("ctas", 0), k.get("sm_time_ms", 0), 100 * k.get("sm_time_share", 0),
                ("%.0f" % k["tflops"]) if "tflops" in k else "", ("%.3f" % k["frac_of_bf16_burst"]) if "frac_of_bf16_burst" in k else "",
                ("%.3f" % k["frac_of_occupied_sms"]) if "frac_of_occupied_sms" in k else ""))
        if "forward_windows" in w.get("e2e", {}):
            fw = w["e2e"]["forward_windows"]
            print("\nforward_windows e2e: %s (%s; %s H2D per step)" % (f(fw["value"], " sites/s"), fw["mode"], f(fw["h2d_bytes_per_step"], "B")))
    pcw = d["workloads"].get("pileup_counts")
    if pcw and "error" not in pcw:
        r = pcw["roofline"]
        print("\n## pileup_counts (SURVEY 8f N4): %s\n" % pcw["config"]["workload"])
        print("%s device-resident, %s columns/s, e2e %s (%s); parity: %s; roofline (HBM): %.1f GB/s of %.0f = %.4f (%s); %s"
              % (f(pcw["value"], " bases/s"), f(pcw["columns_per_s"]), f(pcw["e2e"]["value"], " bases/s"), pcw["e2e"]["mode"], pcw["parity"],
                 r["achieved"], r["peak"], r["frac"], r["kernel"], r["note"]))
    wb = d.get("weight_broadcast") or {}
    if wb.get("bytes"):
        print("\nweight broadcast: %s via %s" % (f(wb["bytes"], "B"), wb.get("how")))


if __name__ == "__main__":
    main(sys.argv[1])
