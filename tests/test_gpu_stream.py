"""FastPath.stream on the H100 against net(example): the same detections bit for bit, in order, for every input form
stream() takes, across batch-size and anchor-mask changes, after closing a stream early, with a post_run hook and
with a status error in the middle of a stream.

Seeded mirror networks of car.fhd and pointpillars.car.xyres_16, B = 4, six batches of distinct seeded clouds whose
point counts differ from frame to frame."""
import numpy as np
import pytest
import torch

import golden_util as gu
from b2second import config, fastpath, models

pytestmark = pytest.mark.gpu
NAMES = ["car.fhd", "pointpillars.car.xyres_16"]
B = 4
BATCHES = 6
MAX_POINTS = 24000
FIELDS = ("box3d_lidar", "scores", "label_preds")


@pytest.fixture(autouse=True)
def _fp32_convs():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield


def _net(product, name, **kw):
    net = models.build_network(config.get_config(name), product).eval()
    models.synthetic_weights_(net, name, seed=0)
    return fastpath.accelerate(net.cuda(), max_points=MAX_POINTS, **kw)


@pytest.fixture(scope="module")
def nets(product):
    """accelerated mirror networks, one per (config, FastPath keywords), shared by the tests of this module"""
    cache = {}

    def get(name, **kw):
        key = (name, tuple(sorted(kw.items())))
        if key not in cache:
            cache[key] = _net(product, name, **kw)
        return cache[key]
    yield get
    cache.clear()
    torch.cuda.empty_cache()


def _place(clouds, memory):
    """the clouds of one batch as `memory` frames: views of one pinned slab, separate pageable tensors, or CUDA"""
    if memory == "pinned":
        slab = torch.from_numpy(np.concatenate(clouds)).pin_memory()
        return list(torch.split(slab, [c.shape[0] for c in clouds]))
    if memory == "pageable":
        return [torch.from_numpy(c) for c in clouds]
    return [torch.from_numpy(c).cuda() for c in clouds]


def _examples(net, name, memory="pinned", sizes=(B,) * BATCHES, seed0=0):
    anchors = torch.from_numpy(net.anchors()[None]).cuda()
    out, seed = [], seed0
    for k, b in enumerate(sizes):
        clouds = []
        for i in range(b):
            clouds.append(gu.make_cloud(name, seed, 6000 + 1700 * ((7 * seed) % 11)))    # 6 000 .. 23 000 points
            seed += 1
        out.append({"points": _place(clouds, memory), "anchors": anchors,
                    "metadata": [{"token": "b%d-f%d" % (k, i)} for i in range(b)]})
    return out


def _assert_same(got, ref, nonempty=True):
    assert len(got) == len(ref)
    boxes = 0
    for k, (g, r) in enumerate(zip(got, ref)):
        assert len(g) == len(r), "batch %d" % k
        for gf, rf in zip(g, r):
            assert gf["metadata"] == rf["metadata"], "batch %d" % k
            for key in FIELDS:
                assert gf[key].device == rf[key].device and gf[key].dtype == rf[key].dtype
                assert torch.equal(gf[key], rf[key]), "batch %d, %s of %s" % (k, key, rf["metadata"])
            boxes += rf["scores"].shape[0]
    assert boxes > 0 or not nonempty, "the examples produced no detections: the comparison would prove nothing"


@pytest.mark.parametrize("memory", ["pinned", "pageable", "cuda"])
@pytest.mark.parametrize("output", ["host", "device"])
@pytest.mark.parametrize("name", NAMES)
def test_stream_equals_net_calls(nets, name, output, memory):
    net = nets(name, output=output)
    examples = _examples(net, name, memory)
    ref = [net(e) for e in examples]
    got = list(net.b2s_fastpath.stream(examples))
    _assert_same(got, ref)
    assert all(f["box3d_lidar"].is_cuda == (output == "device") for r in got for f in r)
    # and again from a generator, after the engine's graphs for both slots exist
    _assert_same(list(net.b2s_fastpath.stream(iter(examples))), ref)


@pytest.mark.parametrize("name", NAMES)
def test_stream_across_batch_size_changes(nets, name):
    net = nets(name, output="host")
    examples = _examples(net, name, sizes=(4, 4, 2, 4, 2, 2), seed0=100)
    ref = [net(e) for e in examples]
    _assert_same(list(net.b2s_fastpath.stream(examples)), ref)
    assert sorted(net.b2s_fastpath.engines) == [2, 4]


@pytest.mark.parametrize("name", NAMES)
def test_stream_with_anchors_mask_on_some_batches(nets, name):
    """given masks on batches 1, 2 and 4, none on the others; xyres_16 computes the anchor-area mask (its eval
    config's threshold) where no mask is given, so its stream switches among three graphs per slot"""
    kw = {"anchor_area_threshold": 1} if name.startswith("pointpillars") else {}
    net = nets(name, output="host", **kw)
    examples = _examples(net, name, seed0=200)
    A = examples[0]["anchors"].shape[1]
    g = torch.Generator().manual_seed(5)
    for k in (1, 2, 4):
        examples[k]["anchors_mask"] = (torch.rand(B, A, generator=g) < 0.5).to(torch.uint8).cuda()
    ref = [net(e) for e in examples]
    _assert_same(list(net.b2s_fastpath.stream(examples)), ref)
    unmasked = [net(dict(examples[k], anchors_mask=None)) for k in (1, 2, 4)]
    assert any(not torch.equal(uf["scores"], rf["scores"])
               for u, k in zip(unmasked, (1, 2, 4)) for uf, rf in zip(u, ref[k])), "the masks changed nothing"


class _CallerError(Exception):
    pass


@pytest.mark.parametrize("how", ["close", "break", "raise"])
@pytest.mark.parametrize("name", NAMES)
def test_closing_a_stream_early_leaves_the_engine_ready(nets, name, how):
    net = nets(name, output="device")
    examples = _examples(net, name, seed0=300)
    ref = [net(e) for e in examples]
    got = []
    if how == "close":
        gen = net.b2s_fastpath.stream(iter(examples))
        got = [next(gen), next(gen)]
        gen.close()
    elif how == "break":
        for r in net.b2s_fastpath.stream(iter(examples)):
            got.append(r)
            if len(got) == 2:
                break
    else:
        try:
            for r in net.b2s_fastpath.stream(iter(examples)):
                got.append(r)
                if len(got) == 2:
                    raise _CallerError()
        except _CallerError:
            pass
    torch.cuda.synchronize()
    _assert_same(got, ref[:2])
    _assert_same([net(examples[3]), net(examples[2])], [ref[3], ref[2]])
    _assert_same(list(net.b2s_fastpath.stream(examples)), ref)


@pytest.mark.parametrize("name", NAMES)
def test_post_run_sees_each_batch_once_in_order(nets, name):
    net = nets(name, output="host")
    fast = net.b2s_fastpath
    examples = _examples(net, name, sizes=(4, 4, 2, 4, 4, 2), seed0=400)
    seen = []
    fast.post_run = lambda eng: seen.append((eng.det_record.clone(), eng.code + 2))
    try:
        ref = [net(e) for e in examples]
        ref_records, seen[:] = list(seen), []
        got = list(fast.stream(examples))
    finally:
        fast.post_run = None
    _assert_same(got, ref)
    assert len(seen) == len(examples)
    for k, ((rec, S), (want, _), res) in enumerate(zip(seen, ref_records, got)):
        # a frame's record: count detections of S floats, then unwritten space, then the count
        counts = rec[:, -1].round().long().tolist()
        assert counts == want[:, -1].round().long().tolist() == [f["scores"].shape[0] for f in res], "batch %d" % k
        for b, n in enumerate(counts):
            assert torch.equal(rec[b, :n * S], want[b, :n * S]), "batch %d: post_run saw another batch's records" % k


def test_status_error_is_raised_at_its_batch(product, nets):
    """a cand_cap that batch 3 overflows (a status word, not a fault): the three earlier results are yielded, then
    RuntimeError; the engine then serves net(example) and a new stream"""
    name = "car.fhd"
    wide = nets(name, output="host")
    examples = _examples(wide, name, seed0=500)
    A = examples[0]["anchors"].shape[1]
    sparse = torch.zeros(B, A, dtype=torch.uint8)
    sparse[:, ::64] = 1                          # earlier batches: one anchor in 64, so few candidates
    for k in (0, 1, 2):
        examples[k]["anchors_mask"] = sparse.cuda()
    eng = wide.b2s_fastpath.engine(B)
    counts = []
    for e in examples:
        wide(e)
        counts.append(int(eng.cand_count.max().item()))
    few, many = max(counts[:3]), counts[3]
    assert many - few >= 2, "candidate counts %s leave no capacity between the batches" % counts
    cap = (few + many) // 2                      # few < cap < many
    net = _net(product, name, output="host", cand_cap=cap)
    ref = [net(e) for e in examples[:3]]
    with pytest.raises(RuntimeError, match="candidate overflow"):
        net(examples[3])
    got = []
    with pytest.raises(RuntimeError, match="candidate overflow"):
        for r in net.b2s_fastpath.stream(examples):
            got.append(r)
    _assert_same(got, ref, nonempty=False)
    torch.cuda.synchronize()
    _assert_same([net(examples[1])], [ref[1]], nonempty=False)
    _assert_same(list(net.b2s_fastpath.stream(examples[:3])), ref, nonempty=False)
