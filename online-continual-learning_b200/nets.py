"""Model objects of the replay path: Reduced_ResNet18 / SupConResNet with the reference's
constructor signatures (models/resnet.py:112-116,140-168; utils/setup_elements.py:46-68), backed
by the CUDA engine, plus `adopt()` which moves an existing reference nn.Module onto the engine
by aliasing its Parameters and BatchNorm buffers onto the engine's flat arenas (so the
reference's own evaluate(), state_dict() and optimizer objects keep seeing live weights).
"""
import math
import weakref

import torch
import torch.nn as nn

from .engine import Engine, describe
from .memory import input_size_match, n_classes

_ENGINES = weakref.WeakKeyDictionary()


def engine_of(model):
    """The Engine behind a model object (EngineModel or adopted reference module)."""
    if isinstance(model, EngineModel):
        return model.engine
    eng = _ENGINES.get(model)
    if eng is None:
        raise RuntimeError('model is not backed by the b200ocl engine; call b200ocl.nets.adopt(model, in_hw) first')
    return eng


def param_layout(dim_in, num_classes, head=None, feat_dim=128, nf=20):
    """[(state_dict name, shape)] in parameters() order for the networks of
    utils/setup_elements.py:46-68 (dim_in = flattened encoder feature size)."""
    pre = 'encoder.' if head is not None else ''
    out = [(pre + 'conv1.weight', (nf, 3, 3, 3)), (pre + 'bn1.weight', (nf,)), (pre + 'bn1.bias', (nf,))]
    cin = nf
    for li in range(1, 5):
        cout = nf << (li - 1)
        for bi in range(2):
            stride = 2 if (bi == 0 and li > 1) else 1
            b = '%slayer%d.%d.' % (pre, li, bi)
            out += [(b + 'conv1.weight', (cout, cin, 3, 3)), (b + 'bn1.weight', (cout,)), (b + 'bn1.bias', (cout,)),
                    (b + 'conv2.weight', (cout, cout, 3, 3)), (b + 'bn2.weight', (cout,)), (b + 'bn2.bias', (cout,))]
            if stride != 1 or cin != cout:
                out += [(b + 'shortcut.0.weight', (cout, cin, 1, 1)), (b + 'shortcut.1.weight', (cout,)),
                        (b + 'shortcut.1.bias', (cout,))]
            cin = cout
    if head is None:
        out += [('linear.weight', (num_classes, dim_in)), ('linear.bias', (num_classes,))]
    else:
        out += [(pre + 'linear.weight', (100, nf * 8)), (pre + 'linear.bias', (100,))]   # unused encoder classifier
        if head == 'linear':
            out += [('head.weight', (feat_dim, dim_in)), ('head.bias', (feat_dim,))]
        elif head == 'mlp':
            out += [('head.0.weight', (dim_in, dim_in)), ('head.0.bias', (dim_in,)),
                    ('head.2.weight', (feat_dim, dim_in)), ('head.2.bias', (feat_dim,))]
    return out


class EngineModel(nn.Module):
    """nn.Module facade over an Engine: Parameters are views into the parameter arena (their
    .grad views into the gradient arena), features()/forward() run the CUDA kernels.
    forward() follows self.training like the reference modules; it does not build an autograd
    graph -- the learners drive Engine.forward_train / backward / sgd_step directly."""

    def __init__(self, in_hw, num_classes, head=None, feat_dim=128, device='cuda'):
        super().__init__()
        self.engine = Engine(in_hw, num_classes, head=head, feat_dim=feat_dim, device=device)
        self.head_kind = head
        layout = param_layout(self.engine.dim_in, num_classes, head, feat_dim)
        names, shapes = [n for n, _ in layout], [sh for _, sh in layout]
        for (n, sh), (_, numel, _) in zip(layout, self.engine.table):
            assert int(torch.Size(sh).numel()) == numel, 'host/C layout mismatch at ' + n
        self._names = names
        for name, shape, pv, gv in zip(names, shapes, self.engine.param_views(), self.engine.grad_views()):
            p = nn.Parameter(pv.view(shape), requires_grad=True)
            p.grad = gv.view(shape)
            self.register_parameter(name.replace('.', '__'), p)
        self.reset_parameters()

    def reset_parameters(self):
        """Default torch initialisation of the reference layers (kaiming-uniform convs/linears,
        BN weight 1 / bias 0, running mean 0 / var 1)."""
        with torch.no_grad():
            for name, p in zip(self._names, self.parameters()):
                if p.dim() >= 2:
                    fan_in = p[0].numel()
                    bound = 1.0 / math.sqrt(fan_in)          # kaiming_uniform_(a=sqrt(5))
                    p.uniform_(-bound, bound)
                elif name.endswith('.bias') and ('linear' in name or name.startswith('head')):
                    w = self._param(name[:-4] + 'weight')
                    bound = 1.0 / math.sqrt(w.shape[1])
                    p.uniform_(-bound, bound)
                elif name.endswith('.weight'):
                    p.fill_(1.0)
                else:
                    p.zero_()
            for rm, rv in self.engine.bn_views():
                rm.zero_()
                rv.fill_(1.0)
            self.engine.state.bn_tracked.zero_()
        self.engine.pack()

    def _param(self, name):
        return getattr(self, name.replace('.', '__'))

    def named_state(self):
        return dict(zip(self._names, self.parameters()))

    def features(self, x):
        """Encoder features.  Eval mode: running statistics (what ASER and NCM use,
        utils/utils.py:55-58).  Train mode: batch statistics, running stats updated."""
        if self.training:
            raise NotImplementedError('train-mode features() is not on the replay path; use forward()')
        return self.engine.features_eval(x)

    def forward(self, x):
        if self.training:
            out, _ = self.engine.forward_train(x)
            return out
        raise NotImplementedError('eval-mode forward() belongs to evaluate() (SURVEY section 8f); use features()')


def Reduced_ResNet18(nclasses, nf=20, bias=True, in_hw=32):
    """models/resnet.py:112-116 (nf is fixed at 20 there and here)."""
    if nf != 20 or not bias:
        raise NotImplementedError('the engine implements the reference configuration nf=20, bias=True')
    return EngineModel(in_hw, nclasses, head=None)


def SupConResNet(dim_in=160, head='mlp', feat_dim=128, in_hw=None):
    """models/resnet.py:140-157.  in_hw is the input size; without it dim_in selects the dataset like the reference
    does (160: 32x32 inputs, 640: 84x84 inputs; setup_elements.py:49-51).  OpenLORIS's 50x50 inputs also give 160
    features, so setup_architecture always passes in_hw.  The reference builds no SupConResNet for 128x128 inputs: SCR
    on CORe50 is refused by check_supcon."""
    if in_hw is None:
        in_hw = {160: 32, 640: 84}[dim_in]
    return EngineModel(in_hw, 100, head=head, feat_dim=feat_dim)


SUPCON_MAX_DIM = 1024     # b200ocl_supcon's feature limit


def check_supcon(in_hw, head, head_in=None):
    """SCR's network on in_hw x in_hw inputs, refused before anything is allocated where it cannot run:
      * head 'mlp' / 'linear' built for head_in features while the encoder gives reduced_resnet_dim_in(in_hw) (the
        reference's SupConResNet(dim_in=160) on 128x128 inputs): ValueError -- the reference fails at its first forward;
      * head 'None' on features wider than b200ocl_supcon takes (2560 at 128x128): NotImplementedError."""
    dim_in = reduced_resnet_dim_in(in_hw)
    if head in ('mlp', 'linear'):
        if head_in is not None and head_in != dim_in:
            raise ValueError('SupConResNet with a %r head over %d features: the encoder gives %d features for %dx%d '
                             'inputs (the reference fails at its first forward)' % (head, head_in, dim_in, in_hw, in_hw))
    elif dim_in > SUPCON_MAX_DIM:
        raise NotImplementedError('SCR without a head takes the SupCon loss over the %d encoder features of %dx%d inputs; '
                                  'the engine\'s SupCon kernel takes at most %d' % (dim_in, in_hw, in_hw, SUPCON_MAX_DIM))


def setup_architecture(params):
    """utils/setup_elements.py:46-68 for the datasets on the replay path."""
    nclass = n_classes[params.data]
    in_hw = input_size_match[params.data][1]
    if params.agent in ['SCR', 'SCP']:
        dim_in = 640 if params.data == 'mini_imagenet' else 160
        check_supcon(in_hw, params.head, dim_in)
        return SupConResNet(dim_in, head=params.head, in_hw=in_hw)
    if params.data in ('cifar100', 'cifar10', 'mini_imagenet', 'core50', 'openloris'):
        return Reduced_ResNet18(nclass, in_hw=in_hw)
    raise NotImplementedError('dataset %s is outside the replay-path scope (SURVEY section 8)' % params.data)


def reduced_resnet_dim_in(in_hw, nf=20):
    """Flattened encoder feature size of Reduced_ResNet18 for in_hw x in_hw inputs: three stride-2 3x3 convolutions
    (padding 1), then avg_pool2d(4) (models/resnet.py:90-103)."""
    h = int(in_hw)
    for _ in range(3):
        h = (h - 1) // 2 + 1
    return nf * 8 * (h // 4) ** 2


def reference_init(data, num_classes, in_hw):
    """The parameters a fresh setup_architecture(params) draws on the CPU (utils/setup_elements.py:46-68, as
    agents/gdumb.py:61 calls it), in parameters() order, drawn in module construction order from torch's default CPU
    generator by the torch.nn.init calls the layers' reset_parameters() make: kaiming_uniform_(a=sqrt(5)) for every
    convolution and linear weight, uniform_(+-1/sqrt(fan_in)) for the linear bias; BatchNorm weights 1 and biases 0
    take no draws.  For mini_imagenet and core50 the 160-input classifier Reduced_ResNet18 builds is drawn and then
    replaced by a 640- / 2560-input one (setup_elements.py:59-66), so both are drawn and the first is discarded.
    openloris keeps the 160-input classifier (setup_elements.py:67-68): its 50x50 inputs pool to 1x1 like 32x32 ones."""
    dim_in = reduced_resnet_dim_in(in_hw)

    def linear(fan_in):
        w = torch.empty(num_classes, fan_in)
        nn.init.kaiming_uniform_(w, a=math.sqrt(5))
        b = torch.empty(num_classes)
        f, _ = nn.init._calculate_fan_in_and_fan_out(w)
        nn.init.uniform_(b, -1 / math.sqrt(f), 1 / math.sqrt(f))
        return w, b

    out = []
    for name, shape in param_layout(dim_in, num_classes):
        if name.startswith('linear.'):
            continue
        t = torch.empty(shape)
        if len(shape) == 4:
            nn.init.kaiming_uniform_(t, a=math.sqrt(5))
        elif name.endswith('.weight'):
            nn.init.ones_(t)
        else:
            nn.init.zeros_(t)
        out.append(t)
    w, b = linear(20 * 8)
    if data in ('mini_imagenet', 'core50'):
        w, b = linear(dim_in)
    elif dim_in != 20 * 8:
        raise NotImplementedError('reference_init: %dx%d inputs of %s are outside the replay path' % (in_hw, in_hw, data))
    return out + [w, b]


def adopt(module, in_hw):
    """Move a reference nn.Module (models.resnet.ResNet with BasicBlocks, or SupConResNet) onto
    the engine.  Its Parameters / BN buffers are re-pointed at the engine arenas, keeping the
    objects (and therefore an optimizer built on module.parameters(), run.py:40) valid."""
    if isinstance(module, EngineModel):
        return module.engine
    if module in _ENGINES:
        return _ENGINES[module]
    is_supcon = hasattr(module, 'encoder')
    enc = module.encoder if is_supcon else module
    head = None
    if is_supcon:
        h = getattr(module, 'head', None)
        if h is None:
            head = 'None'
        elif isinstance(h, nn.Linear):
            head = 'linear'
        else:
            head = 'mlp'
    num_classes = enc.linear.out_features
    feat_dim = 128
    if head == 'linear':
        feat_dim = module.head.out_features
    elif head == 'mlp':
        feat_dim = module.head[2].out_features
    # the classifier (or SupCon head) must take the features the plan's encoder gives at in_hw
    head_in = enc.linear.in_features if head is None else None
    if head == 'linear':
        head_in = module.head.in_features
    elif head == 'mlp':
        head_in = module.head[0].in_features
    _, info, _ = describe(in_hw, num_classes, head=head, feat_dim=feat_dim)
    if head_in is not None and head_in != info.dim_in:
        raise ValueError('adopt(): the module\'s %s takes %d features, the encoder gives %d for %dx%d inputs'
                         % ('classifier' if head is None else 'head', head_in, info.dim_in, in_hw, in_hw))
    params = list(module.parameters())
    dev = params[0].device
    if dev.type != 'cuda':
        raise RuntimeError('adopt() needs the model on a CUDA device (the reference moves it there, run.py:39)')
    eng = Engine(in_hw, num_classes, head=head, feat_dim=feat_dim, device=dev)
    bns = [m for m in module.modules() if isinstance(m, nn.BatchNorm2d)]
    eng.load(params, [(m.running_mean, m.running_var, int(m.num_batches_tracked)) for m in bns])
    with torch.no_grad():
        for p, pv, gv in zip(params, eng.param_views(), eng.grad_views()):
            p.data = pv.view(p.shape)
            p.grad = gv.view(p.shape)
        for i, (m, (rm, rv)) in enumerate(zip(bns, eng.bn_views())):
            m.running_mean.data = rm
            m.running_var.data = rv
            m.num_batches_tracked.data = eng.state.bn_tracked[i]
    _ENGINES[module] = eng
    return eng
