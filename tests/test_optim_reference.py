"""b2second.optim against the reference tree itself (skipped where it is absent): the tabulated schedules against its
schedulers, the parameter groups against its split_bn_bias, and the optimizer block read from its proto message."""
import dataclasses

import pytest

import optim_ref as orf
from b2second import config, models, optim, refcompat
from test_optim import ONE_CYCLE_TEXT, STAIRCASE_TEXT

needs_reference = pytest.mark.skipif(not refcompat.reference_available(), reason="reference tree not present")


@needs_reference
def test_schedule_equals_reference_schedulers(ref_env):
    """the tabulated lr and beta1 are the Python doubles the reference's OneCycle / ExponentialDecay / ManualStepping
    set on their optimizer, bit for bit, and the bias corrections the doubles torch.optim.Adam computes from them"""
    from torchplus.train import learning_schedules_fastai as lsf
    a, b = orf.ONE_CYCLE, orf.STAIRCASE
    manual = dataclasses.replace(b, schedule="manual_stepping", boundaries=(0.8, 0.9), rates=(1e-3, 1e-4, 5e-5))
    cases = [(a, 2320, lambda o, n: lsf.OneCycle(o, n, a.lr_max, list(a.moms), a.div_factor, a.pct_start)),
             (b, 2969, lambda o, n: lsf.ExponentialDecay(o, n, b.initial_learning_rate, b.decay_length, b.decay_factor,
                                                         True)),
             (dataclasses.replace(b, staircase=False), 500,
              lambda o, n: lsf.ExponentialDecay(o, n, b.initial_learning_rate, b.decay_length, b.decay_factor, False)),
             (manual, 500, lambda o, n: lsf.ManualStepping(o, n, list(manual.boundaries), list(manual.rates)))]
    for s, total, make in cases:
        fake = lsf.FakeOptim()
        fake.mom = s.beta1                                           # what Adam is built with
        sched = make(fake, total)
        table = optim.schedule_table(s, total)
        for i in range(total):
            sched.step(i)
            assert (float(fake.lr), float(fake.mom)) == (table[i, 0], table[i, 1]), (s.schedule, i)
            assert table[i, 2] == 1 - fake.mom ** float(i + 1)
            assert table[i, 3] == (1 - s.beta2 ** float(i + 1)) ** 0.5
            assert table[i, 4] == 1 - s.weight_decay * fake.lr


@needs_reference
def test_parameter_groups_equal_split_bn_bias(ref_env):
    """on the mirror network: the same tensors in the same order as the two param groups OptimWrapper.create makes"""
    from second.pytorch.builder.optimizer_builder import get_layer_groups
    from torchplus.train.fastai_optim import split_bn_bias, trainable_params
    net = models.build_network(config.get_config("car.fhd"), ref_env)
    list(net.parameters())[4].requires_grad_(False)
    want = [list(trainable_params(g)) for g in split_bn_bias(get_layer_groups(net))]
    got = optim.parameter_groups(net)
    assert len(want) == 2 and [len(g) for g in got] == [len(g) for g in want]
    for a, b in zip(got, want):
        assert all(x is y for x, y in zip(a, b))


@needs_reference
def test_settings_from_proto_message(ref_env):
    from google.protobuf import text_format
    from second.protos import optimizer_pb2
    for text, want in ((ONE_CYCLE_TEXT, orf.ONE_CYCLE), (STAIRCASE_TEXT, orf.STAIRCASE)):
        body = refcompat._slice_block(refcompat._slice_block(text, "train_config"), "optimizer")
        msg = optimizer_pb2.Optimizer()
        text_format.Merge(body[body.index("{") + 1:body.rindex("}")], msg)
        assert optim.settings(msg) == want
