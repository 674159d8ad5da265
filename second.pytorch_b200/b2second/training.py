"""Training through the CUDA ``spconv`` drop-in.

Upstream ``spconv`` 1.x is mostly used to train: ``second/pytorch/train.py train`` runs ``SubMConv3d`` /
``SparseConv3d`` forward and backward (``torch.ops.spconv.indice_conv_backward``).  The backward here is opt-in, the
same way ``fastpath.accelerate(net)`` is the opt-in for the fused inference engine::

    net = training.enable_sparse_backward(net)
    net = loss.enable_gpu_loss(net)               # b2second.loss: VoxelNet.loss on the GPU
    net = training.enable_rpn_training(net)       # the RPN's 3x3 stride-1 convs on the tensor pipe
    net = training.enable_pfn_training(net)       # PointPillars' pillar feature net and scatter
    net = training.enable_bn_relu_training(net)   # every BatchNorm + ReLU pair of a Sequential
    net.train()
    loss = net(example)["loss"]; loss.backward()

A marked sparse convolution in ``train()`` mode with grad enabled records autograd: its forward runs the inference
kernels with fp32 output rows, its backward computes the input gradient on the same kernels over the transposed
neighbour table (the tensor pipe where the widths allow, with the gradient split under an automatic power-of-two scale)
and the weight gradient with ``b2s_sparse_conv_wgrad``.  The BatchNorm1d and ReLU that follow the conv run as torch
modules, or as one fused train-mode pair after ``enable_bn_relu_training``.  ``eval()`` keeps the fused BN/ReLU
inference path, marked or not; an unmarked conv in training mode still raises
``NotImplementedError``.  Not covered: the fused engine, fp16 parameters / AMP / loss scaling, transposed / inverse
sparse convs.

Half-precision training: ``enable_sparse_backward(net, precision="f16")`` and ``enable_rpn_training(net,
precision="f16")`` run the convolutions that train on the tensor pipe with one f16 ``wgmma`` product per MAC instead of
the 3xF16 split's three: every operand (activations, gradients, weights) is one fp16 plane under its own power-of-two
scale, accumulation stays fp32, and parameters, gradients, BatchNorm, the loss and the optimizer stay fp32.  Which layers
run on the tensor pipe does not change.  The error bound is DESIGN.md §4's f16 bound; ``precision="fp32"`` (the
default) is the fp32-grade path, bit for bit.  The precision is stored per module, and a second call switches it.

The training targets ``VoxelNet.loss`` reads (labels, reg_targets, importance) come from ``b2second.targets`` on the GPU
for a whole batch (``targets.plan(net.target_assigner, feature_map_size).assign_batch(...)``), after
``b2second.inputs.anchor_area_mask``, and the loss they feed runs in csrc/loss.cu through ``b2second.loss`` (the
focal, smooth-L1 and direction terms and their gradient); see INTEGRATION.md, Training.

Several GPUs: ``enable_data_parallel(net)`` trains one process per GPU with the reference's ``--multi_gpu``
(``torch.nn.DataParallel``) semantics; see b2second.dist.
"""


def _products(precision, sparse_impl="tc"):
    """-> the tensor-pipe product count of a training ``precision`` (b2second.engine.check_precision's vocabulary:
    "fp32" -> 3, "f16" -> 1); ValueError for anything else and for "f16" with the fp32 FMA kernels"""
    from .engine import check_precision
    return check_precision(precision, sparse_impl=sparse_impl)


def enable_sparse_backward(module, precision="fp32"):
    """mark every ``spconv.SparseConvolution`` (the CUDA drop-in's) under ``module`` for training; returns ``module``.
    precision: "fp32" (3xF16 on the tensor pipe, fp32-grade) or "f16" (one f16 product per MAC on the tensor pipe;
    ValueError when the drop-in runs the FMA kernels, ``B2S_SPCONV_TC=0``).  Layers the tensor-pipe kernels do not
    cover train in fp32 either way."""
    from . import loader
    sp = loader.product_spconv()
    products = _products(precision, "tc" if sp.USE_TENSOR_CORES else "fma")
    for m in module.modules():
        if isinstance(m, sp.SparseConvolution):
            m._b2s_backward = True
            m._b2s_products = products
    return module


def enable_rpn_training(net, precision="fp32"):
    """train the RPN's 3x3 stride-1 ``nn.Conv2d`` layers under ``net.rpn`` on the tensor pipe (b2second.rpn_train):
    forward, input gradient and weight gradient in 3xF16 on wgmma, fp32-grade (precision "fp32"), or with one f16
    product per MAC (precision "f16").  Layers it does not cover (stride-2 convs, deblocks, heads) stay torch; the
    BatchNorm2d and ReLU that follow the conv are ``enable_bn_relu_training``'s.  Module classes, state-dict keys and
    ``eval()`` are unchanged; idempotent (a second call sets the precision).  Returns ``net``."""
    from . import rpn_train
    return rpn_train.enable(net, _products(precision))


def enable_pfn_training(net):
    """train PointPillars' pillar feature net and scatter on the GPU (b2second.pfn_train): ``PillarFeatureNet`` /
    ``PillarFeatureNetRadius`` with one PFNLayer run the Linear, train-mode BatchNorm1d (batch statistics from the float64
    moments of the decorated inputs, running buffers updated as torch does), ReLU and max without the padded per-point
    map, and their weight gradient in closed form; ``PointPillarsScatter`` runs on b2s_to_bev / b2s_from_bev.  Other
    VFEs stay torch; module classes, state-dict keys and ``eval()`` are unchanged; idempotent.  Returns ``net``."""
    from . import pfn_train
    return pfn_train.enable(net)


def enable_bn_relu_training(net):
    """train every (BatchNorm1d or BatchNorm2d, ReLU) pair of consecutive children of a ``Sequential`` /
    ``SparseSequential`` under ``net`` as one fused pair on the GPU (b2second.bn_train): batch statistics in float64
    with the running buffers updated as torch does, y = relu(BN(x)) in x's layout (rows [M, C] or NCHW), and a backward
    that recomputes the ReLU mask from x, so only x is kept; deterministic, no host sync.  BatchNorms without affine
    parameters, running statistics or a numeric momentum, in-place ReLUs and other norms stay torch; module classes,
    state-dict keys and ``eval()`` are unchanged; idempotent.  Returns ``net``."""
    from . import bn_train
    return bn_train.enable(net)


def enable_data_parallel(net, group=None):
    """train ``net`` data-parallel, one process per GPU over an NCCL process group, with the reference's
    ``torch.nn.DataParallel`` step (b2second.dist.enable_data_parallel); -> the handle ``optim.plan(...,
    data_parallel=)`` takes."""
    from . import dist
    return dist.enable_data_parallel(net, group)
