"""cf_batch_pack_device on bench.py's batch (32 768 payloads of 16 KiB, bench.make_payloads), on one GPU:

  pack      Batch.pack_device of the batch's units from a CUDA tensor: kernel time by CUDA events around --launches back-to-back
            calls on one stream, and GB/s from the bytes the algorithm moves (source read + stream written + source offsets read by
            both kernels + offsets and coarse index written).  Beside it, Batch.upload of the same packed stream from pinned host
            memory, timed the same way.
  resubmit  bench.py's chain (SCAN|SUB|TOON, its rules and lexicons) over the batch at a regex_filter hit rate of --hit-rate, then
            TOON over the units it flagged CF_V_RESUBMIT, as wall time per step ending in a device synchronise.  device: the run's
            out / out_offsets packed with pack_device and the stage bytes set on the device.  host: out / out_offsets downloaded,
            engine.pack_units, upload.  Both routes' TOON verdicts and texts are compared on the last step.

    python tools/pack_device_bench.py [--units 32768] [--launches 50] [--steps 10] [--hit-rate 1e-2] [--out DIR]

Prints one JSON document with the card's name, power limit and max SM clock (read in the same run).  Needs a CUDA device.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from run_async_bench import card  # noqa: E402  (tools/ is this script's directory)


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--units", type=int, default=32768)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--hit-rate", type=float, default=1e-2)
    ap.add_argument("--out", help="also write the JSON document to DIR/pack_device_bench.json")
    args = ap.parse_args()

    import numpy as np
    import torch

    import bench
    from mcp_context_forge_b200 import engine
    from mcp_context_forge_b200._native import CF_STAGE_SCAN, CF_STAGE_SUB, CF_STAGE_TOON, CF_V_RESUBMIT
    from mcp_context_forge_b200.plugins.harmful_content_detector import DEFAULT_LEXICONS

    if not torch.cuda.is_available():
        raise SystemExit("pack_device_bench.py: no CUDA device")
    ctx = engine.Context.get(0)
    n = args.units
    s = torch.cuda.Stream()
    doc = {"card": card(), "units": n}

    # ---- pack vs upload of bench.py's stream
    payloads = bench.make_payloads(hit_rate=1e-4)
    units = [payloads[i % len(payloads)] for i in range(n)]
    enc = [engine.encode_unit(u) for u in units]
    stream, offs = engine.pack_units(enc)
    nbytes, src_bytes = len(stream), len(stream) - n
    src = torch.frombuffer(bytearray(b"".join(enc)), dtype=torch.uint8).cuda()
    src_off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum([len(e) for e in enc], out=src_off[1:])
    d_off = torch.from_numpy(src_off).cuda()
    h_stream = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
    h_stream.numpy()[:] = np.frombuffer(stream, dtype=np.uint8)
    batch = engine.Batch(ctx, nbytes, n)
    torch.cuda.synchronize()

    def timed(fn, k):
        fn()
        s.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(s)
        for _ in range(k):
            fn()
        e1.record(s)
        e1.synchronize()
        return e0.elapsed_time(e1) / k

    pack_ms = timed(lambda: batch.pack_device(src, d_off, n, stream=s, src_bytes=src_bytes), args.launches)
    upload_ms = timed(lambda: batch.upload(h_stream.numpy(), offs, cuda_stream=s.cuda_stream), args.launches)
    nc = (nbytes >> 12) + 1
    alg = src_bytes + nbytes + 2 * 8 * (n + 1) + 8 * (n + 1) + 4 * nc
    doc["pack"] = {"stream_bytes": nbytes, "algorithmic_bytes": alg, "pack_device_ms": round(pack_ms, 4),
                   "pack_device_GBps": round(alg / pack_ms / 1e6, 1), "upload_pinned_ms": round(upload_ms, 4),
                   "upload_pinned_GBps": round(nbytes / upload_ms / 1e6, 1), "launches": args.launches}

    # ---- re-submit: device route vs host route
    prog = engine.Program()
    for pats in DEFAULT_LEXICONS.values():
        for pat in pats:
            prog.add_search(pat, re.I)
    for pat, f, r in bench.SUBS:
        prog.add_sub(pat, f, r)
    prog.compile(ctx)
    payloads = bench.make_payloads(hit_rate=args.hit_rate)
    units = [payloads[i % len(payloads)] for i in range(n)]
    stream, offs = engine.pack_units(units)
    nbytes = len(stream)
    b1 = engine.Batch(ctx, nbytes, n)
    b1.upload(stream, offs)
    cap = 2 * nbytes
    run1, run2 = engine.Run(ctx, n, nbytes), engine.Run(ctx, n, cap + n)
    v1 = torch.zeros(n * 24, dtype=torch.uint8, device="cuda")
    oo1 = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    out1 = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    bm1 = torch.zeros(n * prog.words, dtype=torch.int64, device="cuda")
    v2 = torch.zeros(n * 24, dtype=torch.uint8, device="cuda")
    oo2 = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    out2 = torch.zeros(cap + n, dtype=torch.uint8, device="cuda")
    b2 = engine.Batch(ctx, cap + n, n)
    torch.cuda.synchronize()

    def chain():
        run1.enqueue(prog, b1, CF_STAGE_SCAN | CF_STAGE_SUB | CF_STAGE_TOON, None, 0, v1, oo1, out1, bm1, stream=s)
        assert run1.finish() == 0
        with torch.cuda.stream(s):
            return ((v1.view(n, 24)[:, 8] & CF_V_RESUBMIT) != 0).to(torch.uint8) * CF_STAGE_TOON

    def toon(d_us):
        run2.enqueue(None, b2, CF_STAGE_TOON, d_us, 0, v2, oo2, out2, None, stream=s)
        assert run2.finish() == 0

    def device_route():
        d_us = chain()
        b2.pack_device(out1, oo1, stream=s, src_bytes=run1.gathered_bytes)
        toon(d_us)
        torch.cuda.synchronize()

    def host_route():
        d_us = chain()
        s.synchronize()
        oo = oo1.cpu().numpy()
        raw = out1[:int(oo[-1])].cpu().numpy().tobytes()
        hs, ho = engine.pack_units([raw[int(oo[i]):int(oo[i + 1])] for i in range(n)])
        b2.upload(hs, ho, cuda_stream=s.cuda_stream)
        toon(d_us)
        torch.cuda.synchronize()

    res = {}
    for name, fn in (("device", device_route), ("host", host_route)):
        fn()
        res[name] = []
    for _ in range(args.steps):                       # the two routes alternate, step by step
        for name, fn in (("device", device_route), ("host", host_route)):
            t0 = time.perf_counter()
            fn()
            res[name].append((time.perf_counter() - t0) * 1e3)
            res[name + "_out"] = (v2.cpu().numpy().tobytes(), oo2.cpu().numpy().tobytes(), out2[:int(oo2[-1].item())].cpu().numpy().tobytes())
    flags = v1.view(n, 24)[:, 8].cpu().numpy()
    doc["resubmit"] = {"hit_rate": args.hit_rate, "units_resubmitted": int(((flags & CF_V_RESUBMIT) != 0).sum()), "steps": args.steps,
                       "device_ms_per_step": round(float(np.median(res["device"])), 2), "host_ms_per_step": round(float(np.median(res["host"])), 2),
                       "device_ms_all": [round(x, 2) for x in res["device"]], "host_ms_all": [round(x, 2) for x in res["host"]],
                       "outputs_identical": res["device_out"] == res["host_out"]}
    text = json.dumps(doc, indent=1)
    print(text)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "pack_device_bench.json"), "w") as f:
            f.write(text + "\n")
    return 0 if doc["resubmit"]["outputs_identical"] else 1


if __name__ == "__main__":
    sys.exit(main())
