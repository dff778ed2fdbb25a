"""JPEG input on the device against cv2's host decode:
    python scripts/jpeg_input.py [--calls 20] [--warmup 5] [--rounds 2]

Frames: 1920x1440 up-samplings of tests/data/frame_*.png with seeded noise, encoded by cv2 at quality 90 (4:2:0); the
bytes per frame are printed.
  decode    cp_jpeg_decode alone, in us per frame at batch 1 and 32 (CUDA events over 50 calls after 5 of warm-up), with
            the synchronisation rounds it took; cv2.imdecode on this host's CPU at 1 thread and at its core count.
  run       run(path) per call, a host arm (cv2.imread, then run() as for an array) against the device arm (run(path)):
            alternated call by call, `--rounds` times, the median over `--calls` calls after `--warmup`; results are
            checked identical at every call.
  batch     run_batch of 32 JPEGs (pixel_format="jpeg") against a thread-pool cv2.imdecode followed by run_batch of
            the BGR frames, outputs checked identical.
The card name, power limit and maximum SM clock are printed first, in the same run.  Prints JSON lines."""
import argparse
import json
import os
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from centerpose_b200 import _lib  # noqa: E402
from centerpose_b200.engine import jpeg_decode, jpeg_parse  # noqa: E402
from scripts.yuv_input import gpu_state, make_detector  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def frames(n, h=1440, w=1920):
    import cv2
    rng = np.random.default_rng(0)
    out = []
    for i in range(n):
        base = cv2.imread(os.path.join(ROOT, "tests", "data", "frame_%d.png" % (i % 2)))
        img = cv2.resize(base, (w, h)).astype(np.int16) + rng.integers(-6, 7, (h, w, 3)).astype(np.int16)
        ok, buf = cv2.imencode(".jpg", np.clip(img, 0, 255).astype(np.uint8), [cv2.IMWRITE_JPEG_QUALITY, 90])
        out.append(buf.tobytes())
    return out


def decode_us(files, reps=50, warm=5):
    hs = [jpeg_parse(np.frombuffer(f, np.uint8)) for f in files]
    offs = np.cumsum([0] + [len(f) for f in files[:-1]])
    src = torch.from_numpy(np.frombuffer(b"".join(files), np.uint8).copy()).cuda()
    sizes = [h.out_h * h.out_w * 3 for h in hs]
    oo = np.cumsum([0] + sizes[:-1])
    out = torch.empty(sum(sizes), dtype=torch.uint8, device="cuda")
    for _ in range(warm):
        jpeg_decode(hs, src, offs, out, oo)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        jpeg_decode(hs, src, offs, out, oo)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / reps / len(files), _lib.load().cp_jpeg_last_rounds()


def cv2_us(files, threads):
    import cv2
    cv2.setNumThreads(1)
    arrs = [np.frombuffer(f, np.uint8) for f in files]
    with ThreadPoolExecutor(threads) as ex:
        list(ex.map(lambda a: cv2.imdecode(a, cv2.IMREAD_COLOR), arrs))
        t = time.perf_counter()
        list(ex.map(lambda a: cv2.imdecode(a, cv2.IMREAD_COLOR), arrs * 2))
    return (time.perf_counter() - t) * 1e6 / (2 * len(arrs))


def same(a, b):
    return np.asarray(a).tobytes() == np.asarray(b).tobytes()


def main():
    import cv2
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    print(json.dumps({"gpu": gpu_state(), "cpu_cores": os.cpu_count()}))
    files = frames(32)
    print(json.dumps({"frame": "1920x1440 q90 4:2:0", "bytes_per_frame": int(np.mean([len(f) for f in files]))}))
    for B in (1, 32):
        us, rounds = decode_us(files[:B])
        print(json.dumps({"what": "cp_jpeg_decode", "batch": B, "us_per_frame": round(us, 1), "rounds": rounds}))
    for t in (1, os.cpu_count()):
        print(json.dumps({"what": "cv2.imdecode", "threads": t, "us_per_frame": round(cv2_us(files, t), 1)}))

    dev = torch.device("cuda")
    tmp = tempfile.mkdtemp()
    paths = []
    for i, f in enumerate(files[:4]):
        paths.append(os.path.join(tmp, "f%d.jpg" % i))
        open(paths[-1], "wb").write(f)
    dets = {"host": make_detector(dev, False), "device": make_detector(dev, False)}
    cam = {"camera_matrix": np.array([[1500., 0, 960.], [0, 1500., 720.], [0, 0, 1]])}
    for r in range(args.rounds):
        times = {k: [] for k in dets}
        for c in range(args.warmup + args.calls):
            p = paths[c % len(paths)]
            res = {}
            for k in (("host", "device") if c % 2 == 0 else ("device", "host")):
                torch.cuda.synchronize()
                t = time.perf_counter()
                res[k] = dets[k].run(cv2.imread(p) if k == "host" else p, meta_inp=cam)
                times[k].append((time.perf_counter() - t) * 1e3)
            assert len(res["host"]["results"]) == len(res["device"]["results"])
            for x, y in zip(res["host"]["results"], res["device"]["results"]):
                assert all(same(x[q], y[q]) for q in x)
            for q, v in res["host"]["output"].items():
                assert v is None or same(v.cpu().numpy(), res["device"]["output"][q].cpu().numpy()), q
        for k in dets:
            print(json.dumps({"what": "run(path)", "arm": k, "round": r,
                              "ms_median": round(float(np.median(times[k][args.warmup:])), 2)}))

    det = dets["device"]
    cams = np.array([[1500., 0, 960.], [0, 1500., 720.], [0, 0, 1]])
    for r in range(args.rounds):
        t_host, t_dev = [], []
        for c in range(args.warmup + args.calls):
            torch.cuda.synchronize()
            t = time.perf_counter()
            with ThreadPoolExecutor(os.cpu_count()) as ex:
                bgr = list(ex.map(lambda f: cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR), files))
            wp, wn = det.run_batch(bgr, cams)
            t_host.append((time.perf_counter() - t) * 1e3)
            torch.cuda.synchronize()
            t = time.perf_counter()
            gp, gn = det.run_batch(files, cams, pixel_format="jpeg")
            t_dev.append((time.perf_counter() - t) * 1e3)
            assert same(gp, wp) and same(gn, wn)
        print(json.dumps({"what": "run_batch 32 JPEGs", "round": r,
                          "host_decode_ms": round(float(np.median(t_host[args.warmup:])), 2),
                          "device_decode_ms": round(float(np.median(t_dev[args.warmup:])), 2)}))


if __name__ == "__main__":
    main()
