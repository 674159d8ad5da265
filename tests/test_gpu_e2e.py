"""End-to-end GPU parity against the golden fixtures generated from the unmodified reference network
(tests/golden/make_golden.py) and against the CPU oracle run on the box:
  * module-by-module path: mirror VoxelNet on the CUDA spconv drop-in (same API calls the reference makes)
  * fused engine path: b2second.engine.InferenceEngine (one CUDA graph, no host sync)
Bars: voxel coordinates bit-exact (sha1), BEV features <= 1e-4, boxes <= 1e-4, scores <= 1e-5, labels equal."""
import numpy as np
import pytest
import torch

import golden_util as gu
from b2second import config, models

pytestmark = pytest.mark.gpu
CASES = gu.cases()
IDS = [f"{c[0]}-s{c[1]}-n{c[2]}" for c in CASES]


def build(name, backend, device):
    net = models.build_network(config.get_config(name), backend).eval()
    models.synthetic_weights_(net, name, seed=0)
    return net.to(device)


@pytest.fixture(autouse=True)
def _fp32_convs():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield


@pytest.mark.parametrize("name,seed,n,path", CASES, ids=IDS)
def test_module_path_matches_golden(product, name, seed, n, path):
    fix = np.load(path)
    pts = gu.make_cloud(name, seed, n)
    net = build(name, product, "cuda")
    res = net.voxel_generator.generate(pts, gu.max_voxels_of(fix, name))   # CUDA voxelizer behind the numpy API
    assert res["voxel_num"] == int(fix["voxel_num"])
    assert gu.sha(res["coordinates"]) == str(fix["coords_sha1"])
    assert gu.sha(res["num_points_per_voxel"]) == str(fix["num_points_per_voxel_sha1"])
    assert gu.sha(res["voxels"]) == str(fix["voxels_sha1"])
    coords = np.pad(res["coordinates"], ((0, 0), (1, 0)))
    ex = {"anchors": torch.from_numpy(net.anchors()[None]).cuda(), "voxels": torch.from_numpy(res["voxels"]).cuda(),
          "num_points": torch.from_numpy(res["num_points_per_voxel"]).cuda(),
          "coordinates": torch.from_numpy(coords).cuda()}
    with torch.no_grad():
        vf = net.voxel_feature_extractor(ex["voxels"], ex["num_points"], ex["coordinates"])
        sf = net.middle_feature_extractor(vf, ex["coordinates"], 1)
        pd = net.rpn(sf)
        out = net(ex)[0]
    assert list(sf.shape) == fix["bev_shape"].tolist()
    # active sites are exact; a feature within rounding of the ReLU kink may be +-0 on one side, tiny on the other
    assert abs(int((sf != 0).sum()) - int(fix["bev_nonzero"])) <= max(2, int(fix["bev_nonzero"]) // 20000)
    np.testing.assert_allclose(sf.flatten()[torch.from_numpy(fix["bev_sel_idx"]).cuda()].cpu().numpy(),
                               fix["bev_sel_val"], rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(pd["box_preds"].flatten()[torch.from_numpy(fix["box_sel_idx"]).cuda()].cpu().numpy(),
                               fix["box_sel_val"], rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(pd["cls_preds"].flatten()[torch.from_numpy(fix["cls_sel_idx"]).cuda()].cpu().numpy(),
                               fix["cls_sel_val"], rtol=1e-4, atol=1e-4)
    gu.assert_detections_close({k: (v.cpu().numpy() if hasattr(v, "cpu") else v) for k, v in out.items()}, fix)


def _engine_cases():
    """every fixture on the shipped configuration (wgmma RPN + wgmma sparse conv, CUDA graph); the seed-0 fixture
    of every config additionally on the cross-check configurations (cuDNN RPN / FMA sparse conv, eager)."""
    out, ids = [], []
    for c in CASES:
        combos = [("tc", "tc", True)]
        if c[1] == 0:
            combos += [("cudnn", "fma", False), ("tc", "fma", False), ("tc", "tc", False)]
        for rpn_impl, sparse_impl, graph in combos:
            out.append(c + (rpn_impl, sparse_impl, graph))
            ids.append("%s-s%d-n%d-%s-%s-%s" % (c[0], c[1], c[2], rpn_impl, sparse_impl, "graph" if graph else "eager"))
    return out, ids


_ENG_CASES, _ENG_IDS = _engine_cases()


def _head_values(eng, flat_idx, which, per_anchor):
    """values of the reference's ``box_preds`` / ``cls_preds`` ([B, A_loc, H, W, per_anchor] flattened, rpn.py:400-407)
    at ``flat_idx``, read from the engine's head tensors."""
    idx = np.asarray(flat_idx, dtype=np.int64)
    c = idx % per_anchor
    w = (idx // per_anchor) % eng.fW
    h = (idx // (per_anchor * eng.fW)) % eng.fH
    a = (idx // (per_anchor * eng.fW * eng.fH)) % eng.a_loc
    b = idx // (per_anchor * eng.fW * eng.fH * eng.a_loc)
    if eng.rpn_impl == "tc":
        off = eng.tc_prog["heads"]["offsets"][0 if which == "box" else 1]
        t = eng.tc_heads.cpu().numpy()                       # packed NHWC record [B, H, W, S]
        return t[b, h, w, off + a * per_anchor + c]
    t = eng._keep[1 if which == "box" else 2].cpu().numpy()  # NCHW conv outputs [B, A_loc*per_anchor, H, W]
    return t[b, a * per_anchor + c, h, w]


@pytest.mark.parametrize("name,seed,n,path,rpn_impl,sparse_impl,graph", _ENG_CASES, ids=_ENG_IDS)
def test_engine_matches_golden(product, name, seed, n, path, rpn_impl, sparse_impl, graph):
    from b2second.engine import InferenceEngine
    fix = np.load(path)
    pts = gu.make_cloud(name, seed, n)
    net = build(name, product, "cuda")
    eng = InferenceEngine(net, batch_size=1, max_points=max(n, 1000), max_voxels=gu.max_voxels_of(fix, name),
                          use_cuda_graph=graph, rpn_impl=rpn_impl, sparse_impl=sparse_impl)
    eng.infer([torch.from_numpy(pts).cuda()])
    if graph:   # replay twice: the graph must be re-entrant over its static buffers
        eng.infer([torch.from_numpy(pts).cuda()])
    out = eng.detections()[0]
    assert int(eng.num_voxels[0].item()) == int(fix["voxel_num"])
    assert int(eng.cand_count[0].item()) == int(fix["num_pass_threshold"])
    # the raw regression / classification outputs of the RPN heads against the reference's own tensors: the 1e-4 bar
    # of BASELINE.json applies HERE (decoded boxes below are scaled by the anchor sizes)
    cfg = config.get_config(name)
    np.testing.assert_allclose(_head_values(eng, fix["box_sel_idx"], "box", cfg.box_code_size), fix["box_sel_val"],
                               rtol=0, atol=1e-4)
    np.testing.assert_allclose(_head_values(eng, fix["cls_sel_idx"], "cls", cfg.num_class), fix["cls_sel_val"],
                               rtol=0, atol=1e-4)
    gu.assert_detections_close({k: (v.numpy() if hasattr(v, "numpy") else v) for k, v in out.items()}, fix)


def _example_from_voxels(net, pts, max_voxels, device):
    res = net.voxel_generator.generate(pts, max_voxels)
    coords = np.pad(res["coordinates"], ((0, 0), (1, 0)))
    return {"anchors": torch.from_numpy(net.anchors()[None]).to(device),
            "voxels": torch.from_numpy(res["voxels"]).to(device),
            "num_points": torch.from_numpy(res["num_points_per_voxel"]).to(device),
            "coordinates": torch.from_numpy(coords).to(device)}


@pytest.mark.parametrize("name,seed,n,path", CASES, ids=IDS)
@pytest.mark.parametrize("entry", ["voxels", "points"])
def test_forward_example_runs_fused_engine(product, name, seed, n, path, entry):
    """the reference's own call -- ``net(example)`` -- behind b2second.fastpath.accelerate: the example dict the
    reference's data pipeline produces (voxels / num_points / coordinates / anchors), or raw clouds under 'points'."""
    from b2second import fastpath
    fix = np.load(path)
    pts = gu.make_cloud(name, seed, n)
    net = build(name, product, "cuda")
    mv = gu.max_voxels_of(fix, name)
    ex = _example_from_voxels(net, pts, mv, "cuda" if seed % 2 == 0 else "cpu")     # device- and host-resident examples
    fastpath.accelerate(net, max_points=max(n, 1000), max_voxels=mv)
    if entry == "points":
        ex = {"anchors": ex["anchors"], "points": [torch.from_numpy(pts)], "metadata": [{"token": "f0"}]}
    out = net(ex)
    assert len(net.b2s_fastpath.engines) == 1 and isinstance(out, list) and len(out) == 1
    out = out[0]
    assert out["box3d_lidar"].is_cuda and out["label_preds"].dtype == torch.long
    if entry == "points":
        assert out["metadata"] == {"token": "f0"}
    gu.assert_detections_close({k: (v.cpu().numpy() if hasattr(v, "cpu") else v) for k, v in out.items()}, fix)
    out2 = net(ex)[0]                                   # second call: graph replay
    assert torch.equal(out2["box3d_lidar"], out["box3d_lidar"]) and torch.equal(out2["scores"], out["scores"])


def test_forward_falls_back_for_training_mode_and_padded_layout(product):
    from b2second import fastpath
    name = "car.lite"
    net = build(name, product, "cuda")
    fastpath.accelerate(net)
    pts = gu.make_cloud(name, 0, 6000)
    ex = _example_from_voxels(net, pts, 20000, "cuda")
    ex["num_voxels"] = torch.tensor([[ex["voxels"].shape[0]]])
    padded = dict(ex, voxels=ex["voxels"][None], num_points=ex["num_points"][None], coordinates=ex["coordinates"][None])
    assert not net.b2s_fastpath.applicable(padded)      # DataParallel layout -> module-by-module path
    with torch.no_grad():
        a = net(padded)[0]
        b = net(ex)[0]
    torch.testing.assert_close(a["box3d_lidar"], b["box3d_lidar"], rtol=2e-5, atol=1e-4)
    net.train()
    assert not net.b2s_fastpath.applicable(ex)


@pytest.mark.parametrize("name", ["car.fhd", "pointpillars.car.xyres_16"])
def test_anchors_mask_on_the_fused_path(product, name):
    """anchors_mask (voxelnet.py:397-400,432-439): masked anchors never become candidates.  Fused engine vs the
    module-by-module predict() on the same CUDA backend."""
    from b2second import fastpath
    cfg = config.get_config(name)
    pts = gu.make_cloud(name, 5, 16000)
    net = build(name, product, "cuda")
    ex = _example_from_voxels(net, pts, cfg.max_voxels, "cuda")
    g = torch.Generator().manual_seed(3)
    mask = (torch.rand(1, ex["anchors"].shape[1], generator=g) < 0.6).to(torch.uint8).cuda()
    ex["anchors_mask"] = mask
    with torch.no_grad():
        ref = net(ex)[0]
        fastpath.accelerate(net)
        got = net(ex)[0]
        eng = next(iter(net.b2s_fastpath.engines.values()))
        n_masked = int(eng.cand_count[0].item())
        del ex["anchors_mask"]
        net(ex)
        n_all = int(eng.cand_count[0].item())
    assert 0 < n_masked < n_all
    assert ref["box3d_lidar"].shape[0] > 0
    fixd = {k: ref[k].cpu().numpy() for k in ("box3d_lidar", "scores", "label_preds")}
    gu.assert_detections_close({k: got[k].cpu().numpy() for k in fixd}, fixd)


def test_engine_empty_frame_inside_a_batch(product):
    """a frame with no points (and one with a single point) in the middle of a batch: zero detections for it, the
    neighbours unchanged."""
    from b2second.engine import InferenceEngine
    name = "car.fhd"
    net = build(name, product, "cuda")
    a, c = gu.make_cloud(name, 0, 20000), gu.make_cloud(name, 1, 29000)
    one = np.array([[10.0, 1.0, -1.0, 0.5]], np.float32)
    single = InferenceEngine(net, batch_size=1, max_points=30000, use_cuda_graph=False)
    ref = []
    for cl in (a, c):
        single.infer([torch.from_numpy(cl).cuda()])
        ref.append(single.detections()[0])
    eng = InferenceEngine(net, batch_size=4, max_points=30000, use_cuda_graph=True)
    eng.infer([torch.from_numpy(x).cuda() for x in (a, np.zeros((0, 4), np.float32), one, c)])
    got = eng.detections()
    nv = eng.num_voxels.cpu().tolist()
    assert nv[2] == 0 and nv[3] == 1 and nv[0] == sum(nv[1:])
    assert got[1]["box3d_lidar"].shape[0] == 0 and got[1]["scores"].shape[0] == 0
    for g, r in ((got[0], ref[0]), (got[3], ref[1])):
        assert torch.equal(g["box3d_lidar"], r["box3d_lidar"]) and torch.equal(g["scores"], r["scores"])


def test_engine_batched_frames_match_single_frames(product):
    """frames shard without interaction: a batch of 3 different clouds == the 3 clouds run alone.
    Our kernels are frame-independent and deterministic -> voxels / BEV bit-identical; the cuDNN RPN may pick
    another algorithm for another batch size -> head tensors compared at 1e-4."""
    from b2second.engine import InferenceEngine
    name = "car.fhd"
    net = build(name, product, "cuda")
    clouds = [gu.make_cloud(name, s, n) for s, n in ((0, 20000), (3, 15000), (1, 29000))]
    single = InferenceEngine(net, batch_size=1, max_points=30000, use_cuda_graph=False, rpn_impl="cudnn", sparse_impl="fma")
    ref = []
    for c in clouds:
        single.infer([torch.from_numpy(c).cuda()])
        torch.cuda.synchronize()
        ref.append({"det": single.detections()[0], "nvox": int(single.num_voxels[1].item()),
                    "ncand": int(single.cand_count[0].item()), "bev": single.bev[0].clone(),
                    "box": single._keep[1][0].clone(), "cls": single._keep[2][0].clone()})
    eng = InferenceEngine(net, batch_size=3, max_points=30000, use_cuda_graph=False, rpn_impl="cudnn", sparse_impl="fma")
    eng.infer([torch.from_numpy(c).cuda() for c in clouds])
    got = eng.detections()
    nv = eng.num_voxels.cpu().tolist()
    assert nv[1:] == [r["nvox"] for r in ref] and nv[0] == sum(nv[1:])
    for b, r in enumerate(ref):
        assert torch.equal(eng.bev[b], r["bev"]), "BEV of frame %d differs between batched and single run" % b
        torch.testing.assert_close(eng._keep[1][b], r["box"], rtol=1e-4, atol=1e-4)
        torch.testing.assert_close(eng._keep[2][b], r["cls"], rtol=1e-4, atol=1e-4)
    assert eng.cand_count.cpu().tolist() == [r["ncand"] for r in ref]
    for g, r in zip(got, ref):
        r = r["det"]
        assert g["box3d_lidar"].shape == r["box3d_lidar"].shape and r["box3d_lidar"].shape[0] > 0
        torch.testing.assert_close(g["box3d_lidar"], r["box3d_lidar"], rtol=2e-5, atol=1e-4)
        torch.testing.assert_close(g["scores"], r["scores"], rtol=0, atol=1e-5)
        assert torch.equal(g["label_preds"], r["label_preds"])


def test_module_path_against_live_cpu_oracle(product, oracle):
    """same comparison without fixtures: oracle run on this box's CPU vs the CUDA drop-in, new seed."""
    name = "car.lite"
    cfg = config.get_config(name)
    pts = gu.make_cloud(name, 7, 18000)
    out = {}
    for key, backend, dev in (("cpu", oracle, "cpu"), ("gpu", product, "cuda")):
        net = build(name, backend, dev)
        res = net.voxel_generator.generate(pts, cfg.max_voxels)
        coords = np.pad(res["coordinates"], ((0, 0), (1, 0)))
        ex = {"anchors": torch.from_numpy(net.anchors()[None]).to(dev), "voxels": torch.from_numpy(res["voxels"]).to(dev),
              "num_points": torch.from_numpy(res["num_points_per_voxel"]).to(dev),
              "coordinates": torch.from_numpy(coords).to(dev)}
        with torch.no_grad():
            out[key] = net(ex)[0]
    fix = {k: out["cpu"][k].numpy() for k in ("box3d_lidar", "scores", "label_preds")}
    gu.assert_detections_close({k: out["gpu"][k].cpu().numpy() for k in fix}, fix)
    assert fix["box3d_lidar"].shape[0] > 0
