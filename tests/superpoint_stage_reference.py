"""fp64 references of the SuperPoint extractor's stages, in the device's layout.

Each function restates one stage of the CUDA path (superpoint.cu, gemm_tc.cu EPI_CONV) on the tensors the device works on, so
that a test can feed it the device's own input to that stage and compare that stage's output alone.  Layout (superpoint.cu):
an activation of C channels over an h x w grid is rows [B * P, C], one row per pixel of the zero-bordered (h + 2) x (w + 2)
grid, image b at rows [b P, (b + 1) P), P = round_up((h + 2)(w + 2), 256); border rows and rows [(h + 2)(w + 2), P) are 0.

A "device" result is a dict (``chain`` builds one in fp64, the GPU test reads one through the test hooks):
  image   [B, H, W]                    the input
  act     12 x rows [B P_i, C_i]       output of step i of STEPS (opb_sp_debug_set_stop(i) + debug_read(4))
  logits  rows [B P3, 128]             convPb (65 valid columns; debug_read(2))
  ddesc   rows [B P3, 256]             convDb (debug_read(3))
  scores, nms  [B, H, W]               dense scores, after NMS (debug_read(0), (1))
  kpts [B, cap, 2], kscores [B, cap], desc [B, 256, cap], counts [B]    forward_padded
``check`` compares every stage with its reference on the device's input and returns each error as a multiple of its bar
(<= 1 passes).  Tensors may live on any torch device; the references run in fp64 where their input lives.  ``Defect`` names
plant the errors the stage tests must catch (tests/test_superpoint_stage_reference_cpu.py)."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from oracle import superpoint_oracle as O

STEPS = O.ENCODER + ["convPa|convDa"]
CHANNELS = [64, 64, 64, 64, 64, 64, 128, 128, 128, 128, 128, 512]
LEVEL = [0, 0, 1, 1, 1, 2, 2, 2, 3, 3, 3, 3]          # pooling level of step i's output grid
TILE = 128                                           # output rows per tile of the GEMM core

DEFECTS = (
    "tap_offset",          # tap (2, 1) of every 3x3 convolution reads row offset w + 1 instead of w + 2
    "border_last_tile",    # border / padding rows of the last (partial) row tile of each image are not zeroed
    "pool_hi_only",        # 2x2 pooling compares the hi planes only
    "topk_ties_high",      # top-k breaks score ties toward the HIGHER pixel index
    "align_corners_edge",  # samples touching an edge cell use the other align_corners
    "sample_skip_norm",    # the bilinear sample skips the per-cell normalisation of its fourth neighbour
)

# bars (see check)
E_SPLIT = 2.0 ** -21          # operand split of both operands, the dropped lo.lo pass
E_ACC = 2.0 ** -26            # per reduction step: the truncating fp32 accumulator of the tensor cores
E_OUT = 2.0 ** -22            # output split
E_ABS = 2.0 ** -30
E_CONV1A = 2.0 ** -20         # nine fp32 FMAs
E_SCORE = 2.0 ** -20
E_DESC = 2.0 ** -19


def round_up(x, m):
    return (x + m - 1) // m * m


def stage(H, W, s):
    h, w = H >> s, W >> s
    return h, w, round_up((h + 2) * (w + 2), 256)


def params64(sd, device="cpu"):
    return {k: torch.as_tensor(np.ascontiguousarray(v)).to(device=device, dtype=torch.float64) for k, v in sd.items()}


# ----------------------------------------------------------------------------- layout
def to_grid(x, P):
    """[B, C, h, w] -> rows [B * P, C] of the zero-bordered grid."""
    B, C, h, w = x.shape
    g = torch.zeros(B, P, C, dtype=x.dtype, device=x.device)
    g[:, :(h + 2) * (w + 2)] = F.pad(x, (1, 1, 1, 1)).permute(0, 2, 3, 1).reshape(B, (h + 2) * (w + 2), C)
    return g.reshape(B * P, C)


def grid(rows, B, h, w):
    """rows [B * P, C] -> the whole grid [B, C, h + 2, w + 2] (border included)."""
    C = rows.shape[1]
    P = rows.shape[0] // B
    return rows.reshape(B, P, C)[:, :(h + 2) * (w + 2)].reshape(B, h + 2, w + 2, C).permute(0, 3, 1, 2)


def interior(rows, B, h, w):
    return grid(rows, B, h, w)[:, :, 1:-1, 1:-1]


def border_rows(B, h, w, P, device="cpu"):
    """bool [B * P]: rows that are no interior pixel (grid border and padding)."""
    q = torch.arange(B * P, device=device) % P
    y, x = q // (w + 2), q % (w + 2)
    return (y < 1) | (y > h) | (x < 1) | (x > w)


# ----------------------------------------------------------------------------- encoder and heads
def conv1a(p, image):
    """sp_conv1a: image [B, H, W] -> (rows [B P, 64], sum |w||x| + |b| rows), ReLU."""
    x = image.to(torch.float64)[:, None]
    wt, b = p["conv1a.weight"], p["conv1a.bias"]
    y = F.conv2d(x, wt, b, padding=1).clamp_min(0)
    s = F.conv2d(x.abs(), wt.abs(), b.abs(), padding=1)
    P = stage(image.shape[1], image.shape[2], 0)[2]
    return to_grid(y, P), to_grid(s, P)


def _packed(p, names):
    wt = torch.cat([p[n + ".weight"] for n in names])
    b = torch.cat([p[n + ".bias"] for n in names])
    return wt, b


def conv3x3(p, names, rows, B, h, w, defect=None):
    """EPI_CONV on the device's input rows [B P, C_in]: ReLU(conv + bias) on interior rows, zero elsewhere.  Returns (rows,
    sum |w||x| + |b| rows).  names: one layer, or ["convPa", "convDa"] for the fused heads (512 output columns)."""
    wt, b = _packed(p, names)
    if defect == "tap_offset":            # row offset w + 1 from pixel (y, x) is grid pixel (y + 1, x - 1): tap (2, 0)
        wt = wt.clone()
        wt[:, :, 2, 0] += wt[:, :, 2, 1]
        wt[:, :, 2, 1] = 0
    g = grid(rows, B, h, w).to(torch.float64)
    P = rows.shape[0] // B
    if defect == "border_last_tile":
        full = F.conv2d(g, wt, b, padding=1).clamp_min(0)                     # the product on every grid row
        out = to_grid(full[:, :, 1:-1, 1:-1], P).reshape(B, P, -1)
        allrows = torch.relu(b).expand(B, P, -1).clone()                      # padding rows: taps read zeros, + bias
        n = (h + 2) * (w + 2)
        allrows[:, :n] = full.permute(0, 2, 3, 1).reshape(B, n, -1)
        t0 = (n - 1) // TILE * TILE
        out[:, t0:] = allrows[:, t0:]
        y = out.reshape(B * P, -1)
    else:
        y = to_grid(F.conv2d(g, wt, b).clamp_min(0), P)
    s = to_grid(F.conv2d(g.abs(), wt.abs(), b.abs()), P)
    return y, s


def pool(rows, B, hin, win, defect=None):
    """sp_pool2x2: max of each 2 x 2 block (the winning hi / lo pair is copied: exact)."""
    x = interior(rows, B, hin, win)
    Bc, C = x.shape[:2]
    ho, wo = hin // 2, win // 2
    c = x.reshape(Bc, C, ho, 2, wo, 2).permute(0, 1, 2, 4, 3, 5).reshape(Bc, C, ho, wo, 4)     # candidate d = 2 dy + dx
    if defect == "pool_hi_only":
        hi = (c.to(torch.float32) * 64).to(torch.float16).to(torch.float32)
        y = torch.gather(c, 4, hi.argmax(4, keepdim=True))[..., 0]             # first maximum wins, as `val > best`
    else:
        y = c.max(4).values
    return to_grid(y, stage(ho, wo, 0)[2])


def head_1x1(p, name, rows, B, h, w):
    """convPb / convDb (EPI_F32) on the interior rows of their input: (out [B, C_out, h, w], sum |w||x| + |b|)."""
    x = interior(rows, B, h, w).to(torch.float64)
    wt, b = p[name + ".weight"], p[name + ".bias"]
    return F.conv2d(x, wt, b), F.conv2d(x.abs(), wt.abs(), b.abs())


def dense_scores(logits_rows, B, h, w):
    """sp_scores: 65-way softmax per cell in fp64, dustbin dropped, cell channel c -> pixel (c / 8, c % 8)."""
    lg = interior(logits_rows[:, :65], B, h, w).to(torch.float64)
    s = torch.softmax(lg, 1)[:, :64]
    return s.permute(0, 2, 3, 1).reshape(B, h, w, 8, 8).permute(0, 1, 3, 2, 4).reshape(B, 8 * h, 8 * w)


def nms(scores, r):
    return O.simple_nms(scores, r)


def select(nms_b, thr, border, k, cap, defect=None):
    """sp_count / sp_compact / sp_emit for one image: pixels with score > thr inside the border in row-major order; more
    than k of them: the k best by (score descending, pixel index ascending).  Returns (kpts [n, 2] fp32 (x, y), scores, n)
    with n = min(total, k, cap)."""
    s = np.asarray(nms_b).reshape(-1)
    H, W = np.asarray(nms_b).shape
    pix = np.arange(H * W)
    y, x = pix // W, pix % W
    keep = (s > s.dtype.type(thr)) & (y >= border) & (y < H - border) & (x >= border) & (x < W - border)
    ci, cs = pix[keep], s[keep]
    if 0 <= k < len(ci):
        order = np.lexsort((-ci if defect == "topk_ties_high" else ci, -cs))[:k]
        ci, cs = ci[order], cs[order]
    n = min(len(ci), cap)
    ci, cs = ci[:n], cs[:n]
    return np.stack([ci % W, ci // W], 1).astype(np.float32), cs, n


def sample(ddesc_rows, B, h, w, kpts, align_corners, positions=np.float32, defect=None):
    """sp_sample for every image: kpts = list of [n_b, 2] (x, y).  Grid positions follow the reference's fp32 operation order
    (superpoint.py:79-86 and ATen's un-normalisation; positions=np.float64 evaluates them in fp64), the four cells are
    L2-normalised, weighted, summed and normalised again in fp64; cells outside the grid count as zero.  -> list of [256, n_b]."""
    g = interior(ddesc_rows, B, h, w).to(torch.float64)                      # [B, 256, h, w]
    out = []
    for b in range(B):
        k = np.asarray(kpts[b], np.float64).reshape(-1, 2)
        f = positions
        kx, ky = k[:, 0].astype(f), k[:, 1].astype(f)
        gx = (kx - f(4) + f(0.5)) / f(w * 8 - 4 - 0.5)
        gy = (ky - f(4) + f(0.5)) / f(h * 8 - 4 - 0.5)
        gx, gy = gx * f(2) - f(1), gy * f(2) - f(1)

        def unnorm(ac):
            if ac:
                return ((gx + f(1)) / f(2)) * f(w - 1), ((gy + f(1)) / f(2)) * f(h - 1)
            return ((gx + f(1)) * f(w) - f(1)) / f(2), ((gy + f(1)) * f(h) - f(1)) / f(2)
        ix, iy = unnorm(align_corners)
        if defect == "align_corners_edge":
            x0, y0 = np.floor(ix), np.floor(iy)
            edge = (x0 <= 0) | (x0 + 1 >= w - 1) | (y0 <= 0) | (y0 + 1 >= h - 1)
            ox, oy = unnorm(not align_corners)
            ix, iy = np.where(edge, ox, ix), np.where(edge, oy, iy)
        x0, y0 = np.floor(ix).astype(np.int64), np.floor(iy).astype(np.int64)
        wx1, wy1 = ix.astype(np.float64) - x0, iy.astype(np.float64) - y0
        acc = torch.zeros(256, len(k), dtype=torch.float64, device=g.device)
        for d in range(4):
            yy, xx = y0 + (d >> 1), x0 + (d & 1)
            wgt = (wx1 if d & 1 else 1 - wx1) * (wy1 if d >> 1 else 1 - wy1)
            ok = (yy >= 0) & (yy < h) & (xx >= 0) & (xx < w)
            v = g[b][:, torch.as_tensor(np.clip(yy, 0, h - 1), device=g.device), torch.as_tensor(np.clip(xx, 0, w - 1), device=g.device)]
            if not (defect == "sample_skip_norm" and d == 3):
                v = v / v.norm(dim=0).clamp_min(1e-12)
            acc += v * torch.as_tensor(np.where(ok, wgt, 0.0), device=g.device)
        out.append(acc / acc.norm(dim=0).clamp_min(1e-12))
    return out


# ----------------------------------------------------------------------------- the whole path, and the stage checks
def chain(p, image, cfg, cap, align_corners=True, defect=None, positions=np.float64, score_dtype=torch.float64, quantum=None):
    """The stages composed in fp64 into a device-layout result (the form the GPU test reads); ``defect`` plants one error.
    score_dtype=torch.float32 rounds the dense scores as the device stores them (fp64 sums in different orders separate
    the scores of cells that are equal in exact arithmetic; fp32 ties them again).  quantum: round the dense scores to its
    multiples (a test fixture with many exactly tied candidates)."""
    B, H, W = image.shape
    act = []
    x, _ = conv1a(p, image)
    act.append(x)
    for i in range(1, 12):
        h, w, _ = stage(H, W, LEVEL[i - 1])
        if STEPS[i] == "pool":
            x = pool(x, B, h, w, defect)
        else:
            x, _ = conv3x3(p, ["convPa", "convDa"] if i == 11 else [STEPS[i]], x, B, h, w, defect)
        act.append(x)
    h3, w3, P3 = stage(H, W, 3)
    lg, _ = head_1x1(p, "convPb", act[11][:, :256], B, h3, w3)
    dd, _ = head_1x1(p, "convDb", act[11][:, 256:], B, h3, w3)
    logits = torch.zeros(B * P3, 128, dtype=torch.float64, device=image.device)
    logits[:, :65] = to_grid(lg, P3)
    ddesc = to_grid(dd, P3)
    sc = dense_scores(logits, B, h3, w3).to(score_dtype)
    if quantum:
        sc = torch.round(sc / quantum) * quantum
    nm = nms(sc, cfg["nms_radius"])
    kp = torch.zeros(B, cap, 2, dtype=torch.float32)
    ks = torch.zeros(B, cap, dtype=torch.float64)
    counts = torch.zeros(B, dtype=torch.int32)
    for b in range(B):
        k, s, n = select(nm[b].cpu().numpy(), cfg["keypoint_threshold"], cfg["remove_borders"], cfg["max_keypoints"], cap, defect)
        kp[b, :n], ks[b, :n], counts[b] = torch.from_numpy(k), torch.from_numpy(s), n
    de = sample(ddesc, B, h3, w3, [kp[b, :int(counts[b])].numpy() for b in range(B)], align_corners, positions, defect)
    desc = torch.zeros(B, 256, cap, dtype=torch.float64)
    for b in range(B):
        desc[b, :, :int(counts[b])] = de[b].cpu()
    return {"image": image, "act": act, "logits": logits, "ddesc": ddesc, "scores": sc, "nms": nm, "kpts": kp, "kscores": ks,
            "desc": desc, "counts": counts}


def _ratio(err, bar):
    return float((err / bar).max()) if err.numel() else 0.0


def _exact(a, b):
    """0 if a and b are identical, inf otherwise (a bit-exact bar)."""
    return 0.0 if torch.equal(torch.as_tensor(a), torch.as_tensor(b)) else float("inf")


def check(dev, p, cfg, align_corners=True, stages=None, positions=np.float32):
    """Every stage of ``dev`` against its fp64 reference on ``dev``'s own input to that stage.  Returns {stage: error / bar}
    (<= 1 passes; inf for a bit-exact bar that is missed, or nonzero border rows).  ``stages``: names to check (all: None)."""
    image = dev["image"]
    B, H, W = image.shape
    dv = image.device
    want = (lambda n: True) if stages is None else (lambda n: n in stages)
    r = {}
    act = [a.to(dv, torch.float64) for a in dev["act"]]
    if want("conv1a"):
        ref, s = conv1a(p, image)
        r["conv1a"] = _ratio((act[0] - ref).abs(), E_CONV1A * s + E_OUT * ref.abs() + E_ABS)
    for i in range(1, 12):
        name = STEPS[i]
        tag = name if name != "pool" else f"pool{LEVEL[i]}"
        if not want(tag):
            continue
        h, w, P = stage(H, W, LEVEL[i - 1])
        if name == "pool":
            r[tag] = _exact(act[i], pool(act[i - 1], B, h, w))
            continue
        ref, s = conv3x3(p, ["convPa", "convDa"] if i == 11 else [name], act[i - 1], B, h, w)
        K = 9 * CHANNELS[i - 1]
        bad = border_rows(B, h, w, P, dv)
        ratio = _ratio((act[i] - ref).abs()[~bad], ((E_SPLIT + K * E_ACC) * s + E_OUT * ref.abs() + E_ABS)[~bad])
        r[tag] = ratio if not act[i][bad].any() else float("inf")
    h3, w3, P3 = stage(H, W, 3)
    for name, lo, outd, cols in (("convPb", 0, dev["logits"], 65), ("convDb", 256, dev["ddesc"], 256)):
        if want(name):
            ref, s = head_1x1(p, name, act[11][:, lo:lo + 256], B, h3, w3)
            got = interior(outd.to(dv, torch.float64)[:, :cols], B, h3, w3)
            r[name] = _ratio((got - ref).abs(), (E_SPLIT + 256 * E_ACC) * s + E_ABS)
    if want("scores"):
        ref = dense_scores(dev["logits"].to(dv), B, h3, w3)
        r["scores"] = _ratio((dev["scores"].to(dv, torch.float64) - ref).abs(), E_SCORE * ref.abs() + E_ABS)
    if want("nms"):
        r["nms"] = _exact(dev["nms"].cpu(), nms(dev["scores"].cpu(), cfg["nms_radius"]))
    counts = [int(c) for c in dev["counts"]]
    cap = dev["kpts"].shape[1]
    if want("select"):
        ok = True
        for b in range(B):
            k, s, n = select(dev["nms"][b].cpu().numpy(), cfg["keypoint_threshold"], cfg["remove_borders"], cfg["max_keypoints"], cap)
            ok &= n == counts[b] and np.array_equal(dev["kpts"][b, :n].cpu().numpy(), k) and \
                np.array_equal(dev["kscores"][b, :n].cpu().numpy(), s)
        r["select"] = 0.0 if ok else float("inf")
    if want("sample") and dev.get("desc") is not None:
        ref = sample(dev["ddesc"].to(dv), B, h3, w3, [dev["kpts"][b, :counts[b]].cpu().numpy() for b in range(B)], align_corners,
                     positions)
        r["sample"] = max(_ratio((dev["desc"][b, :, :counts[b]].to(dv, torch.float64) - ref[b]).abs(),
                                 torch.full((), E_DESC, dtype=torch.float64, device=dv)) for b in range(B))
    return r


def table(ratios, title=""):
    return (title + ": " if title else "") + "  ".join(f"{k} {v:.3g}" for k, v in ratios.items())
