"""Detection of K objects in the same F camera frames of 1440 x 1920, 15 reference views per object, K in {1, 2, 4, 8} and F in
{1, 4}.  Two comparisons, each leg timed with CUDA events around work that ends in a synchronise:
  (a) after the matcher, with matches planted as in tools/detect_bench.py (each object's planted key points are its own part of
      the frame's key points):
        objects     one detect.detect_from_matches_objects call: F * K (frame, object) pairs, one detection and one crop launch;
        per_object  the frames copied K-fold, then K detect.detect_from_matches calls, one per object on its copy of the frames;
      the boxes and crops of the two legs are compared.
  (b) from the frames, with a stub matcher that hands out planted matches (so the extractor and everything after it is what is
      timed; no matcher runs):
        objects     detect.ObjectDetectors.detect: one SuperPoint call on the F frames;
        per_object  K LocalFeatureObjectDetector.detect calls: K SuperPoint calls on the same F frames.
      SuperPoint has seeded synthetic weights (max_keypoints 4096) and runs on synthetic frames; both legs make the same number
      of matcher calls (F * K * 15) and the outputs are compared.
The legs alternate inside every repeat; median and spread over the repeats.  Prints one JSON line with the card's name, power
limit and clocks, and a table on stderr.

    python tools/multi_object_detect_bench.py [--repeats 5] [--iters 5] [--out FILE]"""
import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import detect_bench as db  # noqa: E402
from onepose_b200 import SuperPoint, detect, synthetic  # noqa: E402
from tests import crop_reference as cr  # noqa: E402

H, W, S, V = db.H, db.W, db.S, db.V
OBJECTS, FRAMES = (1, 2, 4, 8), (1, 4)


def planted(rng, K, F, dev):
    """Per object detect_bench's workload; the frame's key points are the objects' planted sets side by side."""
    parts = [db.workload(rng, F) for _ in range(K)]
    q_kp = np.concatenate([p[1] for p in parts], axis=1)
    m0 = [np.where(p[2] >= 0, p[2] + k * db.CAP_Q, -1) for k, p in enumerate(parts)]
    refs = [{"keypoints": torch.from_numpy(p[0]).to(dev), "counts": torch.full((V,), db.CAP_REF, dtype=torch.int32, device=dev),
             "sizes": torch.tensor([[480, 640]] * V, dtype=torch.int32, device=dev)} for p in parts]
    query = {"keypoints": torch.from_numpy(q_kp).to(dev), "counts": torch.full((F,), q_kp.shape[1], dtype=torch.int32, device=dev)}
    return refs, query, [torch.from_numpy(m).to(dev) for m in m0]


def after_matcher(rng, K, F, frames, Kmat, args):
    dev = frames.device
    refs, query, m0 = planted(rng, K, F, dev)
    table = {k: torch.cat([r[k] for r in refs]) for k in refs[0]}
    fi = torch.arange(F, dtype=torch.int32, device=dev).repeat(K)                 # pair k * F + f: object k in frame f
    vf = torch.arange(K, dtype=torch.int32, device=dev).repeat_interleave(F) * V
    vc = torch.full((K * F,), V, dtype=torch.int32, device=dev)
    m_pairs = torch.cat(m0)

    def objects():
        return detect.detect_from_matches_objects(frames, fi, Kmat, table, vf, vc, query, m_pairs, S)

    def per_object():
        rep = frames.repeat(K, 1, 1)
        outs = [detect.detect_from_matches(rep[k * F:(k + 1) * F], Kmat, refs[k], query, m0[k], S) for k in range(K)]
        return tuple(torch.cat([o[i] for o in outs]) for i in range(3))

    t = run_legs({"objects": objects, "per_object": per_object}, args.repeats, args.iters)
    a, b = objects(), per_object()
    t["equal"] = all(torch.equal(x, y) for x, y in zip(a, b))
    return t


class PlantedMatcher(torch.nn.Module):
    """matches0 of a (view, frame) pair from a table keyed by their key-point counts, made on first use: a seeded random half of
    the view's points matched to distinct frame points."""

    def __init__(self):
        super().__init__()
        self.table = {}

    def forward(self, data):
        n0, n1 = data["keypoints0"].shape[1], data["keypoints1"].shape[1]
        if (n0, n1) not in self.table:
            r = np.random.default_rng(n0 * 100003 + n1)
            m = np.full(n0, -1, np.int64)
            k = min(n0 // 2, n1)
            m[r.choice(n0, k, replace=False)] = r.choice(n1, k, replace=False)
            self.table[(n0, n1)] = torch.from_numpy(m).to(data["keypoints0"].device)
        return {"matches0": self.table[(n0, n1)][None]}


def from_frames(K, F, frames, Kmat, sp, matcher, views, args):
    multi = detect.ObjectDetectors(sp, matcher, crop_size=S)
    ids = [multi.add_object(views[k]) for k in range(K)]
    singles = [detect.LocalFeatureObjectDetector(sp, matcher, views[k], crop_size=S) for k in range(K)]
    pairs = [(f, ids[k]) for k in range(K) for f in range(F)]

    def objects():
        return multi.detect(frames, Kmat, pairs)

    def per_object():
        outs = [s.detect(frames, Kmat) for s in singles]
        return tuple(torch.cat([o[i] for o in outs]) for i in range(3))

    t = run_legs({"objects": objects, "per_object": per_object}, args.repeats, max(1, args.iters // 5))
    t["equal"] = all(torch.equal(x, y) for x, y in zip(objects(), per_object()))
    return t


def run_legs(legs, repeats, iters):
    for fn in legs.values():                                                     # warm-up of every shape
        fn()
    t = {k: [] for k in legs}
    for _ in range(repeats):
        for k, fn in legs.items():
            t[k].append(db.timed(fn, iters))
    out = {k: db.stats(v) for k, v in t.items()}
    out["speedup"] = out["per_object"]["median_ms"] / out["objects"]["median_ms"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("multi_object_detect_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(0)
    Kmat = torch.tensor([[1500.0, 0, 960], [0, 1500.0, 720], [0, 0, 1]], dtype=torch.float64, device=dev)
    all_frames = torch.from_numpy(np.stack([cr.synthetic_frame(H, W, 10 + f) for f in range(max(FRAMES))])).to(dev)
    sp = SuperPoint({"max_keypoints": 4096}).eval()
    sp.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in synthetic.make_superpoint_state_dict(0, 4.0).items()})
    sp = sp.to(dev)
    views = [[cr.synthetic_frame(480, 640, 100 + k * V + v) for v in range(V)] for k in range(max(OBJECTS))]
    matcher = PlantedMatcher()
    res = {"card": db.card(), "shape": {"frame": [H, W], "views_per_object": V, "crop": S}, "after_matcher": {}, "from_frames": {}}
    for F in FRAMES:
        frames = all_frames[:F]
        for K in OBJECTS:
            key = f"K{K}_F{F}"
            a = res["after_matcher"][key] = after_matcher(rng, K, F, frames, Kmat, args)
            b = res["from_frames"][key] = from_frames(K, F, frames, Kmat, sp, matcher, views, args)
            print(f"{key}: (a) objects {a['objects']['median_ms']:.2f} ms, per object {a['per_object']['median_ms']:.2f} ms, "
                  f"x{a['speedup']:.2f}, equal {a['equal']}; (b) objects {b['objects']['median_ms']:.1f} ms, per object "
                  f"{b['per_object']['median_ms']:.1f} ms, x{b['speedup']:.2f}, equal {b['equal']}", file=sys.stderr)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
