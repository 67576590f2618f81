"""Synthetic inputs for the rtpose hot path: seeded weights, frames and injected stride-8 maps.

No datasets or checkpoints exist offline, so (SURVEY.md section 8d):
  * weights  "W-caffe" = the prototxt filler (gaussian std 0.01, bias 0; pose_deploy_linevec.prototxt:19-28)
             "W-he"    = N(0, 2/fan_in), bias 0 (O(1) heat-maps, so NMS sees peaks)
             both from numpy PCG64 seed 1234, conv layers in prototxt order, weight then bias.
  * frames   uint8 BGR noise blended with a low-frequency pattern (so INTER_AREA is not trivially flat).
  * maps     stride-8 part/PAF maps following the training-label recipe (data_transformer.cpp:2002-2019
             putGaussianMaps sigma=7, :2063-2114 putVecMaps thre=1), for parse-stage parity with persons.
This module is shared by tests, bench.py and smoke(); it does not touch the oracle.
"""
import numpy as np

MPI_15, COCO_18 = 0, 1

# (name, cout, cin, k) in prototxt order
_LIMBS = {
    COCO_18: [1, 2, 1, 5, 2, 3, 3, 4, 5, 6, 6, 7, 1, 8, 8, 9, 9, 10, 1, 11, 11, 12, 12, 13, 1, 0, 0, 14, 14, 16, 0, 15, 15, 17, 2, 16, 5, 17],
    MPI_15: [0, 1, 1, 2, 2, 3, 3, 4, 1, 5, 5, 6, 6, 7, 1, 14, 14, 11, 11, 12, 12, 13, 14, 8, 8, 9, 9, 10],
}
_MAPIDX = {
    COCO_18: [31, 32, 39, 40, 33, 34, 35, 36, 41, 42, 43, 44, 19, 20, 21, 22, 23, 24, 25, 26, 27, 28, 29, 30, 47, 48, 49, 50, 53, 54, 51, 52, 55, 56, 37, 38, 45, 46],
    MPI_15: [16, 17, 18, 19, 20, 21, 22, 23, 24, 25, 26, 27, 28, 29, 30, 31, 38, 39, 40, 41, 42, 43, 32, 33, 34, 35, 36, 37],
}


def conv_table(model, stages=6):
    """[(name, cout, cin, k)] for the convolutions of pose_deploy_linevec.prototxt (92 for the 6-stage files; `stages` = 1, 2, 4
    gives model/mpi/pose_deploy_linevec_{1,2,4}.prototxt), in file order."""
    nparts = 18 if model == COCO_18 else 15
    c_l1, c_l2 = len(_LIMBS[model]), nparts + 1
    t = []
    cin = 3
    for b, (co, n) in enumerate([(64, 2), (128, 2), (256, 4), (512, 2)]):
        for i in range(1, n + 1):
            t.append(("conv%d_%d" % (b + 1, i), co, cin, 3))
            cin = co
    t.append(("conv4_3_CPM", 256, 512, 3))
    t.append(("conv4_4_CPM", 128, 256, 3))
    for i in range(1, 6):
        for br in (1, 2):
            name = "conv5_%d_CPM_L%d" % (i, br)
            if i == 1:
                t.append((name, 128, 128, 3))
            elif i <= 3:
                t.append((name, 128, 128, 3))
            elif i == 4:
                t.append((name, 512, 128, 1))
            else:
                t.append((name, c_l1 if br == 1 else c_l2, 512, 1))
    cc = c_l1 + c_l2 + 128
    for s in range(2, stages + 1):
        for i in range(1, 8):
            for br in (1, 2):
                name = "Mconv%d_stage%d_L%d" % (i, s, br)
                if i == 1:
                    t.append((name, 128, cc, 7))
                elif i <= 5:
                    t.append((name, 128, 128, 7))
                elif i == 6:
                    t.append((name, 128, 128, 1))
                else:
                    t.append((name, c_l1 if br == 1 else c_l2, 128, 1))
    return t


def make_weights(model, kind="he", seed=1234, stages=6, bias_std=0.0):
    """dict name -> (w float32 [cout,cin,k,k], b float32 [cout]).

    bias_std: 0 keeps the fillers' zero biases; a number gives every layer N(0, bias_std^2) biases, a dict name -> std one std
    per layer.  The biases come from their own generator (seed + 1), so the weights do not depend on bias_std."""
    rng = np.random.default_rng(seed)
    brng = np.random.default_rng(seed + 1)
    out = {}
    for name, co, ci, k in conv_table(model, stages):
        std = 0.01 if kind == "caffe" else float(np.sqrt(2.0 / (ci * k * k)))
        w = (rng.standard_normal((co, ci, k, k), dtype=np.float32) * np.float32(std)).astype(np.float32)
        bstd = float(bias_std.get(name, 0.0)) if isinstance(bias_std, dict) else float(bias_std)
        b = (brng.standard_normal(co, dtype=np.float32) * np.float32(bstd)).astype(np.float32) if bstd else np.zeros(co, np.float32)
        out[name] = (w, b)
    return out


def netspec_to_prototxt(spec):
    """Deploy prototxt text from a layer table as tests/golden/netspec_*.json stores it (tools/gen_netspec_fixture.py parsed
    those tables from the reference's model/*/pose_deploy_linevec*.prototxt): lets the GPU box, which has no /root/reference,
    feed the engine's prototxt reader the same graphs."""
    out = ['input: "%s"' % spec["input"]] + ["input_dim: %d" % d for d in spec["input_dim"]]
    for l in spec["layers"]:
        out.append("layer {")
        out.append('  name: "%s"\n  type: "%s"' % (l["name"], l["type"]))
        out += ['  bottom: "%s"' % b for b in l["bottom"]] + ['  top: "%s"' % t for t in l["top"]]
        if l["type"] == "Convolution":
            out.append("  param { lr_mult: 1.0 decay_mult: 1 }\n  param { lr_mult: 2.0 decay_mult: 0 }")
            out.append("  convolution_param {\n    num_output: %d\n    pad: %d\n    kernel_size: %d" % (l["num_output"], l["pad"], l["kernel_size"]))
            out.append('    weight_filler { type: "gaussian" std: 0.01 }\n    bias_filler { type: "constant" }\n  }')
        elif l["type"] == "Pooling":
            out.append("  pooling_param {\n    pool: %s\n    kernel_size: %d\n    stride: %d\n  }" % (l["pool"], l["kernel_size"], l["stride"]))
        elif l["type"] == "Concat":
            out.append("  concat_param { axis: %d }" % l.get("axis", 1))
        elif l["type"] == "ImResize":
            out.append("  imresize_param {\n    factor: %g\n    scale_gap: %g\n    start_scale: %g\n    #target_spatial_width: 368\n  }" % (
                l["factor"], l["scale_gap"], l["start_scale"]))
        elif l["type"] == "Nms":
            out.append("  nms_param {\n    threshold: %g" % l["threshold"])
            if "max_peaks" in l and not l.get("max_peaks_default"):
                out.append("    max_peaks: %d\n    num_parts: %d" % (l["max_peaks"], l["num_parts"]))
            out.append("  }")
        out.append("}")
    return "\n".join(out) + "\n"


def make_frame(idx, h=720, w=1280):
    """uint8 BGR HWC synthetic frame `idx`."""
    rng = np.random.default_rng(idx)
    noise = rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8).astype(np.float32)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    ph = rng.uniform(0, 6.28, size=3).astype(np.float32)
    low = np.stack([127.5 + 127.5 * np.sin(xx / (37.0 + 11 * c) + ph[c]) * np.cos(yy / (53.0 - 7 * c)) for c in range(3)], -1)
    return np.clip(0.5 * noise + 0.5 * low, 0, 255).astype(np.uint8)


# --------------------------------------------------------------------------------------- skeletons
# template joint offsets (x, y) in units of "torso length", origin at the neck
_T_COCO = {0: (0, -0.45), 1: (0, 0), 2: (-0.4, 0.02), 3: (-0.5, 0.55), 4: (-0.45, 1.05), 5: (0.4, 0.02), 6: (0.5, 0.55),
           7: (0.45, 1.05), 8: (-0.25, 1.1), 9: (-0.27, 1.9), 10: (-0.27, 2.65), 11: (0.25, 1.1), 12: (0.27, 1.9),
           13: (0.27, 2.65), 14: (-0.1, -0.55), 15: (0.1, -0.55), 16: (-0.22, -0.48), 17: (0.22, -0.48)}
_T_MPI = {0: (0, -0.6), 1: (0, 0), 2: (-0.4, 0.02), 3: (-0.5, 0.55), 4: (-0.45, 1.05), 5: (0.4, 0.02), 6: (0.5, 0.55),
          7: (0.45, 1.05), 8: (-0.25, 1.1), 9: (-0.27, 1.9), 10: (-0.27, 2.65), 11: (0.25, 1.1), 12: (0.27, 1.9),
          13: (0.27, 2.65), 14: (0, 0.55)}


def make_people(model, n_people, net_w, net_h, seed=0, drop_prob=0.1):
    """Random skeletons in net-pixel coordinates: list of dict part -> (x, y)."""
    rng = np.random.default_rng(seed)
    tmpl = _T_COCO if model == COCO_18 else _T_MPI
    people = []
    cols = int(np.ceil(np.sqrt(n_people * net_w / float(net_h))))
    rows = int(np.ceil(n_people / float(cols)))
    cw, ch = net_w / float(cols), net_h / float(rows)
    for p in range(n_people):
        cx = (p % cols + 0.5) * cw + rng.uniform(-0.1, 0.1) * cw
        torso = min(cw / 1.6, ch / 4.2) * rng.uniform(0.8, 1.0)
        cy = (p // cols) * ch + 0.9 * torso + rng.uniform(0, max(ch - 3.9 * torso, 1e-3))
        ang = rng.uniform(-0.25, 0.25)
        ca, sa = np.cos(ang), np.sin(ang)
        person = {}
        for part, (ox, oy) in tmpl.items():
            if part != 1 and rng.uniform() < drop_prob:
                continue
            jx, jy = ox + rng.normal(0, 0.03), oy + rng.normal(0, 0.03)
            x = cx + torso * (ca * jx - sa * jy)
            y = cy + torso * (sa * jx + ca * jy)
            if 6 <= x < net_w - 6 and 6 <= y < net_h - 6:
                person[part] = (float(x), float(y))
        people.append(person)
    return people


def scale_geometry(net_w, net_h, start_scale, scale_gap, i):
    """(tw, th, padw, padh) of scale i inside the net input (rtpose.cpp:508-511, 243-244)."""
    scale = np.float32(start_scale - i * scale_gap)
    tw = int(16 * np.ceil(np.float32(net_w) * scale / np.float32(16)))
    th = int(16 * np.ceil(np.float32(net_h) * scale / np.float32(16)))
    return tw, th, (net_w - tw) // 2, (net_h - th) // 2


def make_maps(model, people, net_w, net_h, num_scales=1, start_scale=1.0, scale_gap=0.3, noise=0.01, seed=0,
              sigma=7.0, stride=8):
    """Stride-8 maps [S, C, H/8, W/8] for `people` (given at scale-0 net-pixel coordinates)."""
    rng = np.random.default_rng(seed + 7919)
    nparts = 18 if model == COCO_18 else 15
    limbs, mapidx = _LIMBS[model], _MAPIDX[model]
    C = nparts + 1 + len(limbs)
    h8, w8 = net_h // stride, net_w // stride
    maps = np.zeros((num_scales, C, h8, w8), np.float32)
    gy, gx = np.mgrid[0:h8, 0:w8].astype(np.float32)
    px, py = gx * stride + stride / 2.0 - 0.5, gy * stride + stride / 2.0 - 0.5
    for s in range(num_scales):
        tw, th, padw, padh = scale_geometry(net_w, net_h, start_scale, scale_gap, s)
        fx, fy = tw / float(net_w), th / float(net_h)
        sig = sigma * min(fx, fy)
        for person in people:
            pts = {k: (padw + v[0] * fx, padh + v[1] * fy) for k, v in person.items()}
            for part, (x, y) in pts.items():
                d2 = (px - x) ** 2 + (py - y) ** 2
                g = np.exp(-d2 / (2.0 * sig * sig))
                g[d2 / (2.0 * sig * sig) > 4.6052] = 0
                maps[s, part] = np.minimum(maps[s, part] + g, 1.0)
            for k in range(len(limbs) // 2):
                a, b = limbs[2 * k], limbs[2 * k + 1]
                if a not in pts or b not in pts:
                    continue
                ax, ay = pts[a][0] / stride, pts[a][1] / stride
                bx, by = pts[b][0] / stride, pts[b][1] / stride
                vx, vy = bx - ax, by - ay
                nrm = np.sqrt(vx * vx + vy * vy)
                if nrm < 1e-3:
                    continue
                vx, vy = vx / nrm, vy / nrm
                ex, ey = gx - ax, gy - ay
                along = ex * vx + ey * vy
                dist = np.abs(ex * vy - ey * vx)
                m = (dist <= 1.0) & (along >= -0.5) & (along <= nrm + 0.5)
                maps[s, mapidx[2 * k]][m] = vx
                maps[s, mapidx[2 * k + 1]][m] = vy
        maps[s, nparts] = 1.0 - maps[s, :nparts].max(0)
    if noise > 0:
        maps += rng.normal(0, noise, size=maps.shape).astype(np.float32)
    return maps
