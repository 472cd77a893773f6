"""CPU: the pieces of the reference's training loop that the native trainer plugs into, without a GPU.

* `FusedSGD` is a `torch.optim.Optimizer`: the reference's PolyLRScheduler (loaded from the reference tree when it is
  present) and torch's PolynomialLR construct on it and write the expected learning rates.
* Its state dict is torch.optim.SGD's: an SGD(nesterov=True) state after two CPU steps loads and comes back unchanged,
  and the mismatches and settings the fused update does not compute are rejected.  None of this launches a kernel.
* `configure_optimizers` returns the scheduler whenever its module imports, and raises when it fails to construct.
* The final validation's DDP key sharding, `val_keys[rank::world]`.
"""
import importlib.util
import os
import sys
import types
from types import SimpleNamespace

import pytest
import torch

from dinounet_b200 import lib as L
from dinounet_b200 import training as TR
from dinounet_b200.train_path import FusedSGD
from oracle.ref_loader import REF_ROOT, reference_available


@pytest.fixture(autouse=True)
def _no_kernels(monkeypatch):
    def refuse():
        raise AssertionError("a CPU optimizer test loaded the native library")
    monkeypatch.setattr(L, "load", refuse)


def _params():
    g = torch.Generator().manual_seed(0)
    return [torch.randn(5, 3, generator=g).requires_grad_(), torch.randn(4, generator=g),   # the second one is frozen
            torch.randn(2, 3, 2, generator=g).requires_grad_(), torch.randn(7, generator=g).requires_grad_()]


def _torch_sgd_state(params, steps=2):
    ref = [p.detach().clone().requires_grad_(p.requires_grad) for p in params]
    opt = torch.optim.SGD(ref, lr=0.01, momentum=0.99, weight_decay=3e-5, nesterov=True)
    g = torch.Generator().manual_seed(1)
    for s in range(steps):
        for i, r in enumerate(ref):
            # parameter 3 first gets a gradient at the second step; the frozen one never does
            r.grad = torch.randn(r.shape, generator=g) if r.requires_grad and (i != 3 or s > 0) else None
        opt.step()
    return opt.state_dict()


def _lrs(sched, opt, n):
    out = []
    for _ in range(n):
        sched.step()
        out.append(opt.param_groups[0]["lr"])
    return out


def test_fused_sgd_is_an_optimizer_with_every_parameter_in_order():
    ps = _params()
    opt = FusedSGD(ps, lr=0.01)
    assert isinstance(opt, torch.optim.Optimizer)
    assert len(opt.param_groups) == 1 and all(a is b for a, b in zip(opt.param_groups[0]["params"], ps))
    assert len(opt.params) == 4 and not opt.state
    assert "max_norm" not in opt.param_groups[0] and opt.max_norm == 12.0
    sd = opt.state_dict()
    assert sd["state"] == {} and sd["param_groups"][0]["params"] == [0, 1, 2, 3]
    assert {k: v for k, v in sd["param_groups"][0].items() if k not in ("params", "lr")} == \
        {k: v for k, v in torch.optim.SGD(ps, lr=0.5, momentum=0.99, weight_decay=3e-5, nesterov=True)
         .state_dict()["param_groups"][0].items() if k not in ("params", "lr")}


def test_torch_polynomial_lr_writes_the_schedule():
    opt = FusedSGD(_params(), lr=0.01)
    sched = torch.optim.lr_scheduler.PolynomialLR(opt, total_iters=10, power=0.9)
    assert opt.param_groups[0]["lr"] == 0.01
    got = _lrs(sched, opt, 4)
    want = [0.01 * (1 - k / 10) ** 0.9 for k in range(1, 5)]
    assert got == pytest.approx(want, rel=1e-12)


def _reference_polylr():
    if not reference_available():
        pytest.skip("reference tree not present")
    spec = importlib.util.spec_from_file_location(
        "_ref_polylr", os.path.join(REF_ROOT, "dinounet", "training", "lr_scheduler", "polylr.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_reference_poly_lr_scheduler_writes_the_schedule():
    PolyLRScheduler = _reference_polylr().PolyLRScheduler
    opt = FusedSGD(_params(), lr=0.01)
    sched = PolyLRScheduler(opt, 0.01, 1000)
    assert opt.param_groups[0]["lr"] == 0.01          # the constructor's own step(): epoch 0
    got = []
    for epoch in range(1, 5):                          # on_train_epoch_start: lr_scheduler.step(current_epoch)
        sched.step(epoch)
        got.append(opt.param_groups[0]["lr"])
    assert got == [0.01 * (1 - e / 1000) ** 0.9 for e in range(1, 5)]


def test_torch_sgd_state_loads_and_round_trips():
    ps = _params()
    sd = _torch_sgd_state(ps)
    assert sorted(sd["state"]) == [0, 2, 3]
    opt = FusedSGD(ps, lr=0.5, weight_decay=1.0)
    opt.load_state_dict(sd)
    assert opt.param_groups[0]["lr"] == 0.01 and opt.param_groups[0]["weight_decay"] == 3e-5
    assert ps[1] not in opt.state                    # no buffer for the frozen parameter
    back = opt.state_dict()
    assert back["param_groups"] == sd["param_groups"]
    assert back["state"].keys() == sd["state"].keys()
    for k, v in sd["state"].items():
        assert back["state"][k].keys() == v.keys()
        assert torch.equal(back["state"][k]["momentum_buffer"], v["momentum_buffer"])
    # and the reverse: the native optimizer's state resumes on torch.optim.SGD
    other = torch.optim.SGD([p.detach().clone() for p in ps], lr=1.0, momentum=0.9, nesterov=True)
    other.load_state_dict(back)
    assert other.param_groups[0]["lr"] == 0.01 and other.param_groups[0]["momentum"] == 0.99
    assert torch.equal(other.state[other.param_groups[0]["params"][2]]["momentum_buffer"],
                       sd["state"][2]["momentum_buffer"])
    # a round trip through FusedSGD alone
    again = FusedSGD(_params(), lr=0.5)
    again.load_state_dict(back)
    assert again.state_dict()["param_groups"] == back["param_groups"]


def test_reference_trainer_optimizer_state_loads_on_the_native_network(monkeypatch):
    """The reference trainer's `torch.optim.SGD(self.network.parameters())` state, over the reference's own network,
    loads on FusedSGD over the native network: same parameter order and shapes."""
    if not reference_available():
        pytest.skip("reference tree not present")
    import dinounet_b200
    from dinounet_b200 import config
    from oracle import ref_loader
    monkeypatch.setenv("DINOUNET_B200_ALLOW_RANDOM_BACKBONE", "1")
    ref = ref_loader.build_reference_model("dinounet_s", 2)
    nat = dinounet_b200.DinoUNet.from_config({"architecture": dict(config.DEFAULT_ARCHITECTURE)}, 3, 2, None, "dinounet_s")
    sgd = torch.optim.SGD(ref.parameters(), lr=0.01, momentum=0.99, weight_decay=3e-5, nesterov=True)
    for p in ref.parameters():
        p.grad = torch.full_like(p, 1e-3) if p.requires_grad else None
    sgd.step()
    sd = sgd.state_dict()
    opt = FusedSGD(nat.parameters(), lr=0.5)
    opt.load_state_dict(sd)
    trainable = [p for p in nat.parameters() if p.requires_grad]
    assert len(opt.state) == len(trainable) == 289 and all(p in opt.state for p in trainable)


def test_mismatched_state_is_rejected():
    ps = _params()
    sd = _torch_sgd_state(ps)
    with pytest.raises(ValueError):
        FusedSGD(ps[:3], lr=0.01).load_state_dict(sd)
    wrong = [ps[0], ps[1], torch.randn(3, 2, 2, requires_grad=True), ps[3]]
    with pytest.raises(ValueError, match="shape"):
        FusedSGD(wrong, lr=0.01).load_state_dict(sd)
    orphan = {"state": {**sd["state"], 7: {"momentum_buffer": torch.zeros(3)}}, "param_groups": sd["param_groups"]}
    with pytest.raises(ValueError, match="no parameter group"):
        FusedSGD(ps, lr=0.01).load_state_dict(orphan)
    for key, value in (("nesterov", False), ("dampening", 0.1)):
        bad = {"state": sd["state"], "param_groups": [dict(sd["param_groups"][0], **{key: value})]}
        opt = FusedSGD(ps, lr=0.5)
        with pytest.raises(NotImplementedError):
            opt.load_state_dict(bad)
        assert opt.param_groups[0]["lr"] == 0.5 and not opt.state    # left as it was


class _Trainer(TR.DinoUNetTrainer_s):
    """The attributes `configure_optimizers` reads from the reference's trainer."""

    def __init__(self):
        self.network = torch.nn.Linear(3, 2)
        self.initial_lr, self.weight_decay, self.num_epochs = 0.01, 3e-5, 1000


def _install_scheduler_module(monkeypatch, cls):
    names = ["dinounet", "dinounet.training", "dinounet.training.lr_scheduler", "dinounet.training.lr_scheduler.polylr"]
    for n in names:
        monkeypatch.setitem(sys.modules, n, types.ModuleType(n))
    sys.modules[names[-1]].PolyLRScheduler = cls


def test_configure_optimizers_returns_the_scheduler():
    if reference_available():
        cls = _reference_polylr().PolyLRScheduler
    else:
        class cls(torch.optim.lr_scheduler.LRScheduler):   # the published PolyLRScheduler's contract
            def __init__(self, optimizer, initial_lr, max_steps):
                self.initial_lr, self.max_steps = initial_lr, max_steps
                super().__init__(optimizer)

            def get_lr(self):
                return [self.initial_lr * (1 - self.last_epoch / self.max_steps) ** 0.9]
    with pytest.MonkeyPatch.context() as mp:
        _install_scheduler_module(mp, cls)
        opt, sched = _Trainer().configure_optimizers()
    assert isinstance(opt, FusedSGD) and isinstance(sched, cls)
    assert opt.param_groups[0]["lr"] == 0.01


def test_configure_optimizers_raises_when_the_scheduler_fails():
    class Broken:
        def __init__(self, *a):
            raise TypeError("FusedSGD is not an Optimizer")
    with pytest.MonkeyPatch.context() as mp:
        _install_scheduler_module(mp, Broken)
        with pytest.raises(TypeError):
            _Trainer().configure_optimizers()


@pytest.mark.parametrize("world,rank", [(1, 0), (3, 0), (3, 1), (3, 2), (4, 3)])
def test_validation_keys_are_sharded_by_rank(monkeypatch, world, rank):
    keys = [f"case_{i:03d}" for i in range(10)]
    tr = TR.DinoUNetTrainer_s.__new__(TR.DinoUNetTrainer_s)
    tr.do_split = lambda: (["train"], list(keys))
    tr.is_ddp, tr.local_rank = True, rank
    monkeypatch.setattr(TR.dist, "get_world_size", lambda group=None: world)
    got, last = tr._validation_keys()
    assert got == keys[rank::world] and last == len(keys) // world - 1
    assert sorted(k for r in range(world) for k in keys[r::world]) == keys
    tr.is_ddp, tr.local_rank = False, 0
    assert tr._validation_keys() == (keys, None)


def test_cascaded_and_next_stage_configurations_are_rejected_first():
    tr = TR.DinoUNetTrainer_s.__new__(TR.DinoUNetTrainer_s)
    tr.is_cascaded = True
    tr.configuration_manager = SimpleNamespace(next_stage_names=None)
    with pytest.raises(NotImplementedError, match="cascade"):
        tr.perform_actual_validation()
    tr.is_cascaded = False
    tr.configuration_manager = SimpleNamespace(next_stage_names=["3d_lowres"])
    with pytest.raises(NotImplementedError, match="next stages"):
        tr.perform_actual_validation()
