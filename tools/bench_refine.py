"""Warm re-solve after added or erased seeds (GraphDouble.add_seeds / remove_seeds -> mgc_add_seeds / mgc_remove_seeds)
against a cold rebuild of the same graph.

Config 3 at 512^3 (regional + boundary) and config 2 at 256^3 (boundary only), inputs resident in HBM.  For each
configuration: a cold solve, then five strokes, each applied to a freshly solved graph --
  carve         : a background ball of radius 0.05 n inside blob 1 (inside its foreground markers: fg and bg cancel there),
  line          : a foreground line through the background between the two blobs,
  both          : the two together,
  erase_line    : the line added and solved first (not timed), then erased with remove_seeds,
  erase_markers : the foreground markers of blob 2 erased with remove_seeds,
  soft_line     : the line as a soft stroke, add_tweights_warm(line ids, 50, 0),
  regional_box  : a GrabCut-style regional update inside a box around blob 1: add_tweights_warm(None, (p' - p) alpha,
                  ((1 - p') - (1 - p)) alpha) for p = sigmoid((image - 50) / 15), p' = sigmoid((image - 55) / 15),
                  alpha = 0.1, zero outside the box, as float64 CUDA tensors (config 2 has no regional term: there the
                  same deltas are simply dense t-link calls),
  regional_all  : the same update over the whole lattice.
The add_tweights_warm strokes have no seed call: their cold graph is the fused build with the original markers, then the
same calls staged before the first solve.
Per stroke and run it prints, for the warm path: the wall time of the seed call (which returns after its device work)
with the library's split of it into host work before anything is enqueued (ms_seeds_host) and device time (ms_seeds:
id upload, grouping, claim + materialisation, fold, push-list fix-up); the CUDA-event span of maxflow + mask into device
memory, with its solve time and relabel / push / materialisation / read-out device ms from the library's stats; the
wall time from host id arrays to the mask in device memory and on the host.  For the cold path: the CUDA-event span of
the fused build of the graph the user would otherwise build -- the markers with added seeds merged in, or without the
erased ones -- + solve + mask.  Both spans are host driven (the solve synchronises once per round), so they contain
host gaps.  Also whether the two masks hash equal, the energy difference, both energies as hex (for bit-for-bit
comparisons between builds), and the card name and power limit read in the same run.  Runs alternate warm / cold.

    python tools/bench_refine.py [--runs 3] [--config3 512] [--config2 256] [--strokes carve,line,...] [--out rows.json]
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _sha(a):
    return hashlib.sha256(numpy.ascontiguousarray(a).tobytes()).hexdigest()[:16]


def _card():
    """Name and power limit of cuda:0, read in the same run as the numbers."""
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() if q.returncode == 0 and q.stdout.strip() else "not measured"
    except (OSError, subprocess.SubprocessError):
        power = "not measured"
    return dict(card=name, power_limit_and_max_sm_clock=power)


_STROKES = ("carve", "line", "both", "erase_line", "erase_markers", "soft_line", "regional_box", "regional_all")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--config3", type=int, default=512)
    ap.add_argument("--config2", type=int, default=256)
    ap.add_argument("--strokes", default=",".join(_STROKES), help="comma-separated subset of " + ",".join(_STROKES))
    ap.add_argument("--out", default=None, help="also write the rows to this JSON file")
    args = ap.parse_args()
    names = [x for x in args.strokes.split(",") if x]
    if not set(names) <= set(_STROKES):
        ap.error("unknown stroke in --strokes")
    import torch
    from medpy_b200 import synthetic
    from medpy_b200.graphcut.device import graph_from_device_arrays
    stream = torch.cuda.current_stream()
    card = _card()
    print(json.dumps(card), flush=True)
    out = []
    for name, n, regional in (("config3", args.config3, True), ("config2", args.config2, False)):
        shape = (n, n, n)
        vol = synthetic.two_blob_volume(shape, seed=0, with_prob=regional)
        d_img = torch.from_numpy(vol["image"]).cuda()
        d_prob = torch.from_numpy(vol["prob"]).cuda() if regional else None
        carve = synthetic._ball_mask(shape, (0.3,), 0.05)
        line = numpy.zeros(shape, bool)
        line[n // 2, n // 2, int(0.4 * n):int(0.6 * n)] = True
        blob2 = vol["fg"] & synthetic._ball_mask(shape, (0.7,), 0.09, min_radius=0.5)
        none = numpy.zeros(shape, bool)
        # name: (seed call, fg, bg, strokes added and solved before the timed call, markers of the cold graph)
        strokes = {"carve": ("add", None, carve, None, (vol["fg"], vol["bg"] | carve)),
                   "line": ("add", line, None, None, (vol["fg"] | line, vol["bg"])),
                   "both": ("add", line, carve, None, (vol["fg"] | line, vol["bg"] | carve)),
                   "erase_line": ("remove", line, None, line, (vol["fg"], vol["bg"])),
                   "erase_markers": ("remove", blob2, None, None, (vol["fg"] & ~blob2, vol["bg"]))}
        # add_tweights_warm strokes: (ids or None, src, snk); the regional deltas are built lazily on the device
        def regional(box):
            img = d_img.double()
            p = torch.sigmoid((img - 50.0) / 15.0)
            p2 = torch.sigmoid((img - 55.0) / 15.0)
            src, snk = (p2 - p) * 0.1, ((1.0 - p2) - (1.0 - p)) * 0.1
            if box:
                keep = torch.zeros(shape, dtype=torch.bool, device="cuda")
                keep[tuple(slice(int(0.15 * n), int(0.45 * n)) for _ in shape)] = True
                src, snk = torch.where(keep, src, 0.0), torch.where(keep, snk, 0.0)
            return None, src.contiguous(), snk.contiguous()
        warm_calls = {"soft_line": lambda: (numpy.flatnonzero(line), 50.0, 0.0),
                      "regional_box": lambda: regional(True), "regional_all": lambda: regional(False)}
        for k in warm_calls:
            strokes[k] = ("tweights", None, None, None, (vol["fg"], vol["bg"]))
        strokes = {k: strokes[k] for k in names}
        d_mask = torch.empty(shape, dtype=torch.uint8, device="cuda")

        def dev(m):
            return torch.from_numpy(m.view(numpy.uint8)).cuda()

        def build(d_fg, d_bg, graph=None):
            return graph_from_device_arrays(d_fg, d_bg, image=d_img, boundary="difference_exponential", sigma=vol["sigma"],
                                            prob=d_prob, alpha=vol.get("alpha"), graph=graph, stream=stream.cuda_stream)

        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for sname, (call, sfg, sbg, pre, (cfg, cbg)) in strokes.items():
            fg_ids = numpy.flatnonzero(sfg) if sfg is not None else numpy.zeros(0, numpy.int64)
            bg_ids = numpy.flatnonzero(sbg) if sbg is not None else numpy.zeros(0, numpy.int64)
            d_fg0, d_bg0 = dev(vol["fg"]), dev(vol["bg"])
            d_fg2, d_bg2 = dev(cfg), dev(cbg)
            tw = warm_calls[sname]() if call == "tweights" else None
            if tw is not None and tw[0] is not None:
                fg_ids = tw[0]
            for run in range(args.runs):
                # warm: a freshly solved graph (with the strokes to be erased added and solved), then the stroke
                g = build(d_fg0, d_bg0)
                g.maxflow()
                if pre is not None:
                    g.add_seeds(fg=numpy.flatnonzero(pre))
                    g.maxflow()
                torch.cuda.synchronize()
                s0 = dict(g.stats())
                t0 = time.perf_counter()
                if tw is not None:
                    g.add_tweights_warm(*tw)                    # returns after its device work finished
                else:
                    getattr(g, call + "_seeds")(fg_ids, bg_ids)
                t1 = time.perf_counter()
                ev0.record(stream)
                e_warm = g.maxflow()
                g._nat().get_mask_into(d_mask.data_ptr())
                ev1.record(stream)
                torch.cuda.synchronize()
                t2 = time.perf_counter()
                solve_span = ev0.elapsed_time(ev1)
                m_host = g.get_mask()
                wall = (time.perf_counter() - t0) * 1e3
                s1 = g.stats()
                warm_hash = _sha(m_host)
                del g
                # cold: the same graph built from scratch (seeds merged into the markers), solved, mask into device memory
                torch.cuda.synchronize()
                ev0.record(stream)
                gc_ = build(d_fg2, d_bg2)
                if tw is not None:
                    gc_.add_tweights_warm(*tw)                  # staged before the first solve
                e_cold = gc_.maxflow()
                gc_._nat().get_mask_into(d_mask.data_ptr())
                ev1.record(stream)
                torch.cuda.synchronize()
                cold_dev = ev0.elapsed_time(ev1)
                cold_hash = _sha(d_mask.cpu().numpy())
                del gc_
                d = {k: s1[k] - s0.get(k, 0.0) for k in ("ms_seeds", "ms_seeds_host", "ms_solve", "ms_relabel", "ms_push",
                                                          "ms_caps", "ms_readout", "push_sweeps", "global_relabels")}
                row = dict(config=name, n=n, stroke=sname, call=call, run=run,
                           seeds=int(n ** 3 if tw is not None and tw[0] is None else fg_ids.size + bg_ids.size),
                           seed_call_wall_ms=(t1 - t0) * 1e3, solve_span_ms=solve_span,
                           warm_wall_ms_host_ids_to_device_mask=(t2 - t0) * 1e3,
                           warm_wall_ms_host_ids_to_host_mask=wall, cold_span_ms=cold_dev,
                           masks_equal=warm_hash == cold_hash, warm_mask_sha=warm_hash, energy_diff=e_warm - e_cold,
                           energy=e_cold, energy_warm_hex=float(e_warm).hex(), energy_cold_hex=float(e_cold).hex(),
                           **d, **card)
                print(json.dumps(row), flush=True)
                out.append(row)
        del d_img, d_prob, d_mask
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
