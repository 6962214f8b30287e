"""The pose-guided crop on one GPU, at B in {1, 8, 32} camera frames of 1440 x 1920 and a 512 x 512 crop: CUDA-event time of
  crop         crop.previous_pose_detect alone (boxes from the previous poses, crop, K_crop);
  step         the live step on the device: previous_pose_detect -> SuperPoint.forward_padded -> match_frames -> poses_from_matches;
  step_host    the same step with the crop done as the reference does it: previous poses to the host, numpy projection and two
               cv2.warpAffine per frame there, the [B,1,512,512] float image back to the device (frames already in host memory).
The legs alternate inside every repeat; median and spread over the repeats.  Prints one JSON line with the card's name, power
limit and clocks.  Weights, object and frames are synthetic: the times depend on shapes, not on content.

    python tools/crop_bench.py [--repeats 7] [--iters 10] [--out FILE]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from onepose_b200 import GATsSuperGlue, SuperPoint, crop, pnp, synthetic  # noqa: E402

H, W, S, N, M, NLEAF = 1440, 1920, 512, 1024, 2500, 8


def card():
    q = "name,power.limit,clocks.max.sm,clocks.sm,clocks.mem"
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return dict(zip(q.split(","), [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]))
    except Exception as e:            # noqa: BLE001
        return {"name": torch.cuda.get_device_name(0), "note": f"nvidia-smi: {e}"}


def timed(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def stats(xs):
    return {"median_ms": statistics.median(xs), "min_ms": min(xs), "max_ms": max(xs)}


def host_crop(cv2, frames_host, K, poses, corners):
    """previous_pose_detect per frame with numpy and cv2 (local_feature_2D_detector.py:232-259) -> float32 [B,1,S,S], K_crop [B,3,3]."""
    def transform(cx, cy, src_w, dst_w, dst_h):
        s = np.float32([[cx, cy], [cx, cy - 0.5 * src_w], [0, 0]])
        d = np.float32([[dst_w * 0.5, dst_h * 0.5], [dst_w * 0.5, dst_h * 0.5 - 0.5 * dst_w], [0, 0]])
        for p in (s, d):
            p[2] = p[1] + np.float32([p[1][1] - p[0][1], p[0][0] - p[1][0]])
        return cv2.getAffineTransform(s, d)

    images, Ks = [], []
    for b in range(len(frames_host)):
        p = K @ (poses[b, :, :3] @ corners.T + poses[b, :, 3:])
        p = (p[:2] / p[2:]).T
        x0, y0, x1, y1 = np.concatenate([p.min(0), p.max(0)]).astype(np.int32)
        w, h = x1 - x0, y1 - y0
        T1 = transform((x0 + x1) / 2.0, (y0 + y1) / 2.0, w, w, h)
        T2 = transform(w / 2.0, h / 2.0, w, S, S)
        im = cv2.warpAffine(cv2.warpAffine(frames_host[b], T1, (int(w), int(h)), flags=cv2.INTER_LINEAR), T2, (S, S), flags=cv2.INTER_LINEAR)
        images.append(im.astype(np.float32) / 255)
        Ks.append(np.vstack([T2, [0, 0, 1]]) @ np.vstack([T1, [0, 0, 1]]) @ K)
    return np.stack(images)[:, None], np.stack(Ks)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("crop_bench.py measures on the GPU and there is none")
    try:
        import cv2
    except ImportError:
        cv2 = None
    dev = torch.device("cuda", 0)
    sp = SuperPoint({"nms_radius": 3, "max_keypoints": N}).eval()
    sp.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in synthetic.make_superpoint_state_dict(0, 4.0).items()})
    sp = sp.to(dev)
    mm = GATsSuperGlue(dict(synthetic.DEFAULT_HPARAMS)).eval()
    mm.load_state_dict({k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in synthetic.make_state_dict(0).items()})
    mm = mm.to(dev)
    db, leaves = synthetic.make_object(2, M, NLEAF)
    kp3d = (torch.rand(M, 3, device=dev) - 0.5) * 0.2
    Knp = np.array([[1500.0, 0, W / 2], [0, 1500.0, H / 2], [0, 0, 1]])
    corners_np = np.array([[sx, sy, sz] for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)], np.float64) * 0.1
    base = (synthetic.make_image(300, H, W)[0] * 255).astype(np.uint8)
    rows = []
    for B in (1, 8, 32):
        mm.set_object(torch.from_numpy(db).to(dev), torch.from_numpy(leaves).to(dev), reserve=(B, N))
        frames_host = np.stack([np.roll(base, 37 * b, axis=1) for b in range(B)])
        frames = torch.from_numpy(frames_host).to(dev)
        # no box edge projects within 0.02 px of an integer: there the projection's last bit would decide the truncated box
        poses_np = np.stack([np.concatenate([np.eye(3), [[0.0213 * (b % 5 - 2)], [0.0117 * (b % 3 - 1)], [0.8031 + 0.0107 * (b % 7)]]], axis=1) for b in range(B)])
        K, poses, corners = torch.from_numpy(Knp).to(dev), torch.from_numpy(poses_np).to(dev), torch.from_numpy(corners_np).to(dev)

        def rest(inp, K_crop):
            det = sp.forward_padded(inp)
            out = mm.match_frames(det["descriptors"], return_conf=False, lengths=det["counts"])
            return pnp.poses_from_matches(K_crop, det["keypoints"], kp3d, out["matches0"], out["matching_scores0"], scale=1000)

        def leg_crop():
            return crop.previous_pose_detect(frames, K, poses, corners, crop_size=S)

        def leg_step():
            _, inp, K_crop = crop.previous_pose_detect(frames, K, poses, corners, crop_size=S)
            return rest(inp, K_crop)

        def leg_step_host():
            im, Kc = host_crop(cv2, frames_host, Knp, poses.cpu().numpy(), corners_np)
            return rest(torch.from_numpy(im).to(dev), torch.from_numpy(Kc).to(dev))

        legs = {"crop": leg_crop, "step": leg_step}
        if cv2 is not None:
            legs["step_host"] = leg_step_host
        for fn in legs.values():
            fn()
        torch.cuda.synchronize()
        t = {k: [] for k in legs}
        for _ in range(a.repeats):
            for k, fn in legs.items():
                t[k].append(timed(fn, a.iters))
        row = {"B": B, "frame": [H, W], "crop_size": S, "N": N, "M": M}
        if cv2 is not None:                                    # the two crops are the same image
            _, inp, K_crop = leg_crop()
            im, Kc = host_crop(cv2, frames_host, Knp, poses_np, corners_np)
            row["same_image_as_cv2"] = bool(np.array_equal(inp.cpu().numpy(), im))
            row["max_dK_crop_over_max_K"] = float(np.abs(K_crop.cpu().numpy() - Kc).max() / np.abs(Kc).max())
        else:
            row["step_host"] = "not measured: cv2 is not installed"
        row.update({k: stats(v) for k, v in t.items()})
        rows.append(row)
        print(json.dumps(row), file=sys.stderr)
    result = {"card": card(), "cv2": cv2.__version__ if cv2 is not None else None, "repeats": a.repeats, "iters_per_repeat": a.iters,
              "note": "CUDA events around iters back-to-back calls, per call; step_host includes its host work and copies "
                      "(the events span them); synthetic weights, object and frames",
              "rows": rows}
    line = json.dumps(result)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
