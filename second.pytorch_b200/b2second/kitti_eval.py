"""KITTI detection formatting and evaluation on the GPU (csrc/kitti_eval.cu).

  convert_detection_to_kitti_annos   second/data/kitti_dataset.py:37-106  (lidar detections -> camera-frame annos)
  get_official_eval_result           second/utils/eval.py:730-816
  get_coco_eval_result               second/utils/eval.py:819-916
  eval_class                         second/utils/eval.py:479-611 (eval_class_v3)

Python packs the annotations into flat float64 rows plus int32 frame offsets (include/b2second.h, B2S_KITTI_ROW),
encodes the names once into a small vocabulary, and formats the result strings.  The overlaps, ignore flags, matching,
thresholds and precision run in libb2second.so.  Unlike the reference (whose 50-part split needs at least 50 frames),
any number of frames >= 1 is accepted, with or without ground truth or detections in each.

clean_data compares each box's height, truncation and occlusion with the difficulty limits in the annotation's own
dtype: for float32 boxes the height y2 - y1 is a float32 difference, which can be exactly 40 where the float64 one is
not.  So pack_limits takes those comparisons on the original arrays, with numpy scalar promotion as clean_data's
scalar code gets it, and hands the kernel one limit bit per (box, difficulty) instead of the widened values.  Under
numpy 1.x a float32 truncation was compared with the Python float in float64 (np.float32(0.15) > 0.15 is True there,
False under numpy 2), so float32 truncation results depend on the numpy version, exactly as they do for the
reference.
"""
import io

import numpy as np
import torch

N_SAMPLE_PTS = 41
ROW = 16                     # B2S_KITTI_ROW
DONTCARE = -2                # B2S_KITTI_DONTCARE
NO_ALT = -3
MAX_DT_PER_FRAME = 2048
# clean_data's difficulty tables (eval.py:38-40), Python numbers as there
MIN_HEIGHT = [40, 25, 25]
MAX_OCCLUSION = [0, 1, 2]
MAX_TRUNCATION = [0.15, 0.3, 0.5]

# clean_data's class table (eval.py:34-37) and get_*_eval_result's class_to_name
CLASS_NAMES = ["car", "pedestrian", "cyclist", "van", "person_sitting", "car", "tractor", "trailer"]
CLASS_TO_NAME = {0: "Car", 1: "Pedestrian", 2: "Cyclist", 3: "Van", 4: "Person_sitting", 5: "car", 6: "tractor",
                 7: "trailer"}
NAME_TO_CLASS = {v: n for n, v in CLASS_TO_NAME.items()}
# names that count as "valid 0" (neither a hit nor a miss) for a class: Van for Car, Person_sitting for Pedestrian
_ALT = {"car": "van", "pedestrian": "person_sitting"}
COCO_RANGES = {0: [0.5, 0.95, 10], 1: [0.25, 0.7, 10], 2: [0.25, 0.7, 10], 3: [0.5, 0.95, 10], 4: [0.25, 0.7, 10],
               5: [0.5, 0.95, 10], 6: [0.5, 0.95, 10], 7: [0.5, 0.95, 10]}


def _lib():
    import spconv
    return spconv._lib, spconv._lib.load()


# ------------------------------------------------------------------------------------------------ host: packing
def vocab_id(lower_name):
    """first index of a lower-cased name in CLASS_NAMES ('car' appears twice), -1 when absent."""
    return CLASS_NAMES.index(lower_name) if lower_name in CLASS_NAMES else -1


def encode_names(names):
    """names -> int32 codes: vocabulary id of the lower-cased name, -1 for others, DONTCARE for exactly 'DontCare'
    (clean_data compares lower-cased names, but don't-care boxes case-sensitively)."""
    uniq, inv = np.unique(np.asarray(names, dtype=str), return_inverse=True)
    codes = np.array([DONTCARE if u == "DontCare" else vocab_id(u.lower()) for u in uniq], dtype=np.int32)
    return codes[inv.reshape(-1)] if len(uniq) else np.zeros(0, np.int32)


def _scalar_dtype(a, value):
    """a's values as clean_data's scalar `a[i] <op> value` compares them: in the dtype numpy's scalar promotion gives a
    scalar of a's dtype and the Python number value (float32 under numpy 2, float64 under numpy 1.x for a float)."""
    t = (a.dtype.type(0) + value).dtype
    return a.astype(t, copy=False), t.type(value)


def _exceeds(a, limit):
    a, v = _scalar_dtype(a, limit)
    return a > v


def difficulty_limits(anno, is_gt):
    """uint8 [n]: bit d set when clean_data puts the box outside difficulty d -- for ground truth occluded >
    MAX_OCCLUSION[d] or truncated > MAX_TRUNCATION[d] or height <= MIN_HEIGHT[d], for detections |height| <
    MIN_HEIGHT[d] -- computed from the anno's own arrays, the height in the bbox's dtype."""
    bbox = np.asarray(anno["bbox"]).reshape(-1, 4)
    height = bbox[:, 3] - bbox[:, 1]
    out = np.zeros(height.shape[0], dtype=np.uint8)
    for d in range(3):
        if is_gt:
            h, v = _scalar_dtype(height, MIN_HEIGHT[d])
            out_d = (_exceeds(np.asarray(anno["occluded"]), MAX_OCCLUSION[d]) |
                     _exceeds(np.asarray(anno["truncated"]), MAX_TRUNCATION[d]) | (h <= v))
        else:
            h, v = _scalar_dtype(np.abs(height), MIN_HEIGHT[d])
            out_d = h < v
        out |= out_d.astype(np.uint8) << d
    return out


def pack_limits(annos, is_gt):
    """list of anno dicts -> difficulty_limits of every box, frame after frame: uint8 [N], in pack_annos' row order."""
    parts = [difficulty_limits(a, is_gt) for a in annos if len(a["name"])]
    return np.concatenate(parts) if parts else np.zeros(0, np.uint8)


def pack_annos(annos, with_score):
    """list of anno dicts -> (rows float64 [N, ROW], name codes int32 [N], offsets int32 [F+1])."""
    counts = np.array([len(a["name"]) for a in annos], dtype=np.int64)
    off = np.zeros(len(annos) + 1, dtype=np.int64)
    np.cumsum(counts, out=off[1:])
    if off[-1] >= 2 ** 31:
        raise ValueError("too many boxes for int32 offsets")
    rows = np.zeros((int(off[-1]), ROW), dtype=np.float64)
    names = []
    for a, lo, hi in zip(annos, off[:-1], off[1:]):
        if hi == lo:
            continue
        r = rows[lo:hi]
        r[:, 0:4] = np.asarray(a["bbox"], dtype=np.float64).reshape(-1, 4)
        r[:, 4:7] = np.asarray(a["location"], dtype=np.float64).reshape(-1, 3)
        r[:, 7:10] = np.asarray(a["dimensions"], dtype=np.float64).reshape(-1, 3)
        r[:, 10] = a["rotation_y"]
        r[:, 11] = a["alpha"]
        if with_score:
            r[:, 12] = a["score"]
        r[:, 13] = a["truncated"]
        r[:, 14] = a["occluded"]
        names.append(np.asarray(a["name"]))
    codes = encode_names(np.concatenate(names)) if names else np.zeros(0, np.int32)
    return rows, codes, off.astype(np.int32)


def task_table(current_classes, difficultys, min_overlaps, metric):
    """(task_info int32 [T, 3], min_overlap float64 [T]) in eval_class_v3's (class, difficulty, overlap) order."""
    info, mo = [], []
    for m, c in enumerate(current_classes):
        name = CLASS_NAMES[c].lower()
        alt = vocab_id(_ALT[name]) if name in _ALT else NO_ALT
        for d in difficultys:
            for k in range(min_overlaps.shape[0]):
                info.append((vocab_id(name), alt, int(d)))
                mo.append(float(min_overlaps[k, metric, m]))
    return np.array(info, dtype=np.int32).reshape(-1, 3), np.array(mo, dtype=np.float64)


def _classes_int(current_classes):
    if not isinstance(current_classes, (list, tuple)):
        current_classes = [current_classes]
    return [NAME_TO_CLASS[c] if isinstance(c, str) else int(c) for c in current_classes]


def compute_aos_of(dt_annos):
    """the reference's switch: the first detection frame with boxes decides (alpha[0] != -10)."""
    for a in dt_annos:
        if np.asarray(a["alpha"]).shape[0] != 0:
            return bool(a["alpha"][0] != -10)
    return False


# ------------------------------------------------------------------------------------------------ device
class _Packed:
    """ground truth and detections of one evaluation on the device, plus the overlaps of each metric once computed."""

    def __init__(self, gt_annos, dt_annos, z_axis, z_center, device):
        if len(gt_annos) != len(dt_annos):
            raise ValueError("gt_annos and dt_annos differ in length (%d vs %d)" % (len(gt_annos), len(dt_annos)))
        if len(gt_annos) == 0:
            raise ValueError("nothing to evaluate: no frames")
        if z_axis not in (1, 2):
            raise ValueError("z_axis must be 1 (camera) or 2 (lidar)")
        self.dev = torch.device(device)
        self.z_axis, self.z_center = int(z_axis), float(z_center)
        gt, gn, go = pack_annos(gt_annos, with_score=False)
        dt, dn, do = pack_annos(dt_annos, with_score=True)
        gl, dl = pack_limits(gt_annos, is_gt=True), pack_limits(dt_annos, is_gt=False)
        self.F, self.G, self.D = len(gt_annos), gt.shape[0], dt.shape[0]
        ng, nd = np.diff(go).astype(np.int64), np.diff(do).astype(np.int64)
        self.max_dt = int(nd.max(initial=0))
        if self.max_dt > MAX_DT_PER_FRAME:
            raise ValueError("a frame has %d detections; at most %d per frame" % (self.max_dt, MAX_DT_PER_FRAME))
        ov_off = np.zeros(self.F + 1, dtype=np.int64)
        np.cumsum(ng * nd, out=ov_off[1:])
        to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(self.dev)
        self.gt, self.gn, self.go, self.gl = to(gt), to(gn), to(go), to(gl)
        self.dt, self.dn, self.do, self.dl = to(dt), to(dn), to(do), to(dl)
        self.ov_off, self.n_ov = to(ov_off), int(ov_off[-1])
        self._ov = {}

    def overlaps(self, metric):
        if metric not in self._ov:
            L, lib = _lib()
            out = torch.zeros(max(self.n_ov, 1), dtype=torch.float64, device=self.dev)
            with torch.cuda.device(self.dev):
                L.check(lib.b2s_kitti_overlaps(int(metric), L.ptr(self.gt), L.ptr(self.go), L.ptr(self.dt),
                                               L.ptr(self.do), self.F, L.ptr(self.ov_off), self.z_axis, self.z_center,
                                               L.ptr(out), L.stream()), "b2s_kitti_overlaps")
            self._ov[metric] = out
        return self._ov[metric]

    def eval(self, metric, current_classes, difficultys, min_overlaps, compute_aos, ignored=False):
        L, lib = _lib()
        info, mo = task_table(current_classes, difficultys, min_overlaps, metric)
        T = info.shape[0]
        prec = torch.zeros(T, N_SAMPLE_PTS, dtype=torch.float64, device=self.dev)
        aos, thr = torch.zeros_like(prec), torch.zeros_like(prec)
        if T:
            ov = self.overlaps(metric)
            ti, tm = torch.from_numpy(info).to(self.dev), torch.from_numpy(mo).to(self.dev)
            ws = torch.empty(lib.b2s_kitti_eval_workspace_bytes(self.F, self.G, self.D, T), dtype=torch.uint8,
                             device=self.dev)
            with torch.cuda.device(self.dev):
                L.check(lib.b2s_kitti_eval(int(metric), L.ptr(self.gt), L.ptr(self.gn), L.ptr(self.gl), L.ptr(self.go),
                                           self.G, L.ptr(self.dt), L.ptr(self.dn), L.ptr(self.dl), L.ptr(self.do),
                                           self.D, self.F, self.max_dt,
                                           L.ptr(ov), L.ptr(self.ov_off), L.ptr(ti), L.ptr(tm), T, int(bool(compute_aos)),
                                           L.ptr(prec), L.ptr(aos), L.ptr(thr), L.ptr(ws), ws.numel(), L.stream()),
                        "b2s_kitti_eval")
        shape = (len(current_classes), len(difficultys), min_overlaps.shape[0], N_SAMPLE_PTS)
        out = {"recall": np.zeros(shape), "precision": prec.cpu().numpy().reshape(shape),
               "orientation": aos.cpu().numpy().reshape(shape), "thresholds": thr.cpu().numpy().reshape(shape),
               "min_overlaps": min_overlaps}
        if ignored:
            # clean_data's flags as the kernel left them in the workspace: after three int32 [T] counters, int8
            # ignored_gt [T, G] then ignored_dt [T, D], each block 256-byte aligned (carve in kitti_eval.cu)
            align = lambda n: (n + 255) // 256 * 256
            w = ws.cpu().numpy().view(np.int8) if T else np.zeros(0, np.int8)
            o = align(12 * T)
            flags = lambda lo, n: w[lo:lo + T * n].reshape(shape[:3] + (n,))
            out["ignored_gt"], out["ignored_dt"] = flags(o, self.G), flags(o + align(T * self.G), self.D)
        return out


def _device(device):
    if device is None:
        device = torch.device("cuda", torch.cuda.current_device())
    if torch.device(device).type != "cuda":
        raise RuntimeError("KITTI evaluation runs on a CUDA device; there is no CPU path")
    return device


def eval_class(gt_annos, dt_annos, current_classes, difficultys, metric, min_overlaps, compute_aos=False, z_axis=1,
               z_center=1.0, device=None, ignored=False):
    """eval_class_v3: {"recall" (zeros, as the reference), "precision", "orientation", "thresholds"} each
    [num_class, num_difficulty, num_minoverlap, 41], and "min_overlaps" [num_minoverlap, 3, num_class].  ignored:
    also clean_data's "ignored_gt" [num_class, num_difficulty, num_minoverlap, num_gt] and "ignored_dt" [..., num_dt]
    (int8, -1 / 0 / 1, all frames' boxes in order) as the kernel computed them."""
    p = _Packed(gt_annos, dt_annos, z_axis, z_center, _device(device))
    return p.eval(metric, list(current_classes), list(difficultys), np.asarray(min_overlaps, dtype=np.float64),
                  compute_aos, ignored)


# ------------------------------------------------------------------------------------------------ host: results
def get_mAP(prec):
    sums = 0
    for i in range(0, prec.shape[-1], 4):
        sums = sums + prec[..., i]
    return sums / 11 * 100


def _line(text):
    out = io.StringIO()
    print(text, file=out)
    return out.getvalue()


def official_min_overlaps(current_classes):
    overlap_mod = np.array([[0.7, 0.5, 0.5, 0.7, 0.5, 0.7, 0.7, 0.7],
                            [0.7, 0.5, 0.5, 0.7, 0.5, 0.7, 0.7, 0.7],
                            [0.7, 0.5, 0.5, 0.7, 0.5, 0.7, 0.7, 0.7]])
    overlap_easy = np.array([[0.7, 0.5, 0.5, 0.7, 0.5, 0.5, 0.5, 0.5],
                             [0.5, 0.25, 0.25, 0.5, 0.25, 0.5, 0.5, 0.5],
                             [0.5, 0.25, 0.25, 0.5, 0.25, 0.5, 0.5, 0.5]])
    return np.stack([overlap_mod, overlap_easy], axis=0)[:, :, current_classes]


def coco_min_overlaps(current_classes):
    ranges = np.zeros([3, 3, len(current_classes)])
    for i, c in enumerate(current_classes):
        ranges[:, :, i] = np.array(COCO_RANGES[c])[:, np.newaxis]
    min_overlaps = np.zeros([10, *ranges.shape[1:]])
    for i in range(ranges.shape[1]):
        for j in range(ranges.shape[2]):
            lo, hi, num = ranges[:, i, j]
            min_overlaps[:, i, j] = np.linspace(lo, hi, int(num))
    return min_overlaps


def format_official(current_classes, min_overlaps, prec_bbox, prec_bev, prec_3d, aos_bbox=None):
    """get_official_eval_result's {"result", "detail"} from the three metrics' precision arrays (and the bbox
    orientation when AOS is computed)."""
    result, detail = "", {}
    for j, curcls in enumerate(current_classes):
        class_name = CLASS_TO_NAME[curcls]
        detail[class_name] = {}
        for i in range(min_overlaps.shape[0]):
            mAPbbox = get_mAP(prec_bbox[j, :, i])
            mAPbev = get_mAP(prec_bev[j, :, i])
            mAP3d = get_mAP(prec_3d[j, :, i])
            detail[class_name][f"bbox@{min_overlaps[i, 0, j]:.2f}"] = mAPbbox.tolist()
            detail[class_name][f"bev@{min_overlaps[i, 1, j]:.2f}"] = mAPbev.tolist()
            detail[class_name][f"3d@{min_overlaps[i, 2, j]:.2f}"] = mAP3d.tolist()
            result += _line(f"{class_name} " + "AP(Average Precision)@{:.2f}, {:.2f}, {:.2f}:".format(
                *min_overlaps[i, :, j]))
            result += _line("bbox AP:" + ", ".join(f"{v:.2f}" for v in mAPbbox))
            result += _line("bev  AP:" + ", ".join(f"{v:.2f}" for v in mAPbev))
            result += _line("3d   AP:" + ", ".join(f"{v:.2f}" for v in mAP3d))
            if aos_bbox is not None:
                mAPaos = get_mAP(aos_bbox[j, :, i])
                detail[class_name]["aos"] = mAPaos.tolist()
                result += _line("aos  AP:" + ", ".join(f"{v:.2f}" for v in mAPaos))
    return {"result": result, "detail": detail}


def format_coco(current_classes, prec_bbox, prec_bev, prec_3d, aos_bbox=None):
    """get_coco_eval_result's {"result", "detail"} from the precision arrays over the 10 overlaps of each class."""
    mAPs = [get_mAP(p).mean(-1) for p in (prec_bbox, prec_bev, prec_3d)]
    mAPaos = get_mAP(aos_bbox).mean(-1) if aos_bbox is not None else None
    result, detail = "", {}
    for j, curcls in enumerate(current_classes):
        class_name = CLASS_TO_NAME[curcls]
        detail[class_name] = {}
        o_range = np.array(COCO_RANGES[curcls])[[0, 2, 1]]
        o_range[1] = (o_range[2] - o_range[0]) / (o_range[1] - 1)
        result += _line(f"{class_name} " + "coco AP@{:.2f}:{:.2f}:{:.2f}:".format(*o_range))
        for label, key, m in (("bbox AP:", "bbox", mAPs[0]), ("bev  AP:", "bev", mAPs[1]), ("3d   AP:", "3d", mAPs[2])):
            result += _line(f"{label}{m[j, 0]:.2f}, {m[j, 1]:.2f}, {m[j, 2]:.2f}")
            detail[class_name][key] = m[j].tolist()
        if mAPaos is not None:
            detail[class_name]["aos"] = mAPaos[j].tolist()
            result += _line(f"aos  AP:{mAPaos[j, 0]:.2f}, {mAPaos[j, 1]:.2f}, {mAPaos[j, 2]:.2f}")
    return {"result": result, "detail": detail}


def get_official_eval_result(gt_annos, dt_annos, current_classes, difficultys=(0, 1, 2), z_axis=1, z_center=1.0,
                             device=None):
    """{"result": str, "detail": dict} as second/utils/eval.py:730-816 prints and returns them."""
    classes = _classes_int(current_classes)
    min_overlaps = official_min_overlaps(classes)
    compute_aos = compute_aos_of(dt_annos)
    p = _Packed(gt_annos, dt_annos, z_axis, z_center, _device(device))
    m = [p.eval(metric, classes, list(difficultys), min_overlaps, compute_aos) for metric in range(3)]
    return format_official(classes, min_overlaps, m[0]["precision"], m[1]["precision"], m[2]["precision"],
                           m[0]["orientation"] if compute_aos else None)


def get_coco_eval_result(gt_annos, dt_annos, current_classes, z_axis=1, z_center=1.0, device=None):
    """{"result": str, "detail": dict} as second/utils/eval.py:819-916 (AP over 10 overlaps per class)."""
    classes = _classes_int(current_classes)
    min_overlaps = coco_min_overlaps(classes)
    compute_aos = compute_aos_of(dt_annos)
    p = _Packed(gt_annos, dt_annos, z_axis, z_center, _device(device))
    m = [p.eval(metric, classes, [0, 1, 2], min_overlaps, compute_aos and metric == 0) for metric in range(3)]
    return format_coco(classes, m[0]["precision"], m[1]["precision"], m[2]["precision"],
                       m[0]["orientation"] if compute_aos else None)


# ------------------------------------------------------------------------------------------------ conversion
def _calib_of(info):
    c = info["calib"]
    return np.stack([np.asarray(c[k], dtype=np.float64).reshape(4, 4) for k in ("R0_rect", "Tr_velo_to_cam", "P2")])


def convert_detection_to_kitti_annos(detections, infos, class_names, device=None):
    """KittiDataset.convert_detection_to_kitti_annos: detections[i] (the dicts net(example) returns, device or host
    tensors) with infos[i]'s calibration and image shape -> list of anno dicts, each with the detection's metadata.
    The inputs are not modified."""
    if len(detections) > len(infos):
        raise ValueError("%d detection frames but only %d infos" % (len(detections), len(infos)))
    F = len(detections)
    if F == 0:
        return []
    dev = torch.device(_device(device))
    L, lib = _lib()
    counts = [int(d["box3d_lidar"].shape[0]) for d in detections]
    code = next((int(d["box3d_lidar"].shape[1]) for d, n in zip(detections, counts) if n), 7)
    rows = []
    for d, n in zip(detections, counts):
        if n == 0:
            continue
        if int(d["box3d_lidar"].shape[1]) != code:
            raise ValueError("detections differ in box code size")
        box = d["box3d_lidar"].detach().to(dev, torch.float32)
        rows.append(torch.cat([box, d["scores"].detach().to(dev, torch.float32)[:, None],
                               d["label_preds"].detach().to(dev).float()[:, None]], 1))
    det = torch.cat(rows, 0).contiguous() if rows else torch.zeros(1, code + 2, device=dev)
    det_off = np.zeros(F + 1, dtype=np.int32)
    np.cumsum(counts, out=det_off[1:])
    calib = torch.from_numpy(np.stack([_calib_of(infos[i]) for i in range(F)])).to(dev)
    shape = torch.from_numpy(np.array([np.asarray(infos[i]["image"]["image_shape"])[:2] for i in range(F)],
                                      dtype=np.int32)).to(dev)
    off_d = torch.from_numpy(det_off).to(dev)
    out = torch.empty(max(int(det_off[-1]), 1), ROW, dtype=torch.float64, device=dev)
    cnt = torch.zeros(F, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        L.check(lib.b2s_kitti_convert(L.ptr(det), code + 2, code, L.ptr(off_d), F, L.ptr(calib), L.ptr(shape),
                                      L.ptr(out), L.ptr(cnt), L.stream()), "b2s_kitti_convert")
    out, cnt = out.cpu().numpy(), cnt.cpu().numpy()
    annos = []
    for i in range(F):
        n = int(cnt[i])
        r = out[det_off[i]:det_off[i] + n]
        if n == 0:
            anno = {"name": np.array([]), "truncated": np.array([]), "occluded": np.array([]), "alpha": np.array([]),
                    "bbox": np.zeros([0, 4]), "dimensions": np.zeros([0, 3]), "location": np.zeros([0, 3]),
                    "rotation_y": np.array([]), "score": np.array([])}
        else:
            anno = {"name": np.array([class_names[int(l)] for l in r[:, 15]]),
                    "truncated": np.zeros(n), "occluded": np.zeros(n, dtype=np.int64),
                    "alpha": r[:, 11].copy(), "bbox": r[:, 0:4].copy(), "dimensions": r[:, 7:10].copy(),
                    "location": r[:, 4:7].copy(), "rotation_y": r[:, 10].copy(),
                    "score": r[:, 12].astype(np.float32)}
        anno["metadata"] = detections[i]["metadata"]
        annos.append(anno)
    return annos
