"""The owner-side exchange step of PeerShardedVariable (attach_exchange(insert="push"), det_peer_xchg_apply_*) has the
Adagrad and Adam rules only.  Over the emulated library, with one fake shard: AdamW, AMSGrad (FusedAdamW(amsgrad=True)
and FusedAdam(amsgrad=True)) and Lion are refused with a TypeError before anything changes -- no row, no slot and no
step count is written -- instead of being run as plain Adam; plain FusedAdam still takes the step, bit for bit like the
oracle's Adam step."""
import numpy as np
import pytest
import torch

from oracle import oracle as O
from tests.emu import backend

DIM, CAP = 8, 128


@pytest.fixture(autouse=True)
def _emu():
  with backend.installed():
    yield


def _exchange_variable(name):
  from recommenders_addons_b200 import dynamic_embedding as de
  var = de.Variable(dim=DIM, init_size=1024, initializer=0.05, num_slot_planes=3, name=name, devices=["cpu"])
  pv = de.PeerShardedVariable(fake_shards=[var])
  nbytes = int(pv._lib.det_peer_xchg_bytes(1, CAP, DIM * 4))
  raw = torch.zeros(nbytes + 256, dtype=torch.uint8)
  off = (-raw.data_ptr()) % 256
  pv.attach_exchange(CAP, mailbox_ptrs=[raw.data_ptr() + off], keepalive=raw, insert="push")
  return var, pv


def _batch(seed):
  rng = np.random.default_rng(seed)
  keys = torch.from_numpy(rng.choice(1 << 40, size=40, replace=False).astype(np.int64))
  grads = torch.from_numpy(rng.normal(0, 1e-2, (40, DIM)).astype(np.float32))
  return keys, grads


MAKERS = {
    "adamw": lambda de: de.FusedAdamW(0.01),
    "adamw_amsgrad": lambda de: de.FusedAdamW(0.01, amsgrad=True),
    "adam_amsgrad": lambda de: de.FusedAdam(0.01, amsgrad=True),
    "adamw_no_decay": lambda de: de.FusedAdamW(0.01, weight_decay=0.0),
    "lion": lambda de: de.FusedLion(1e-3, weight_decay=0.1),
}


@pytest.mark.parametrize("kind", sorted(MAKERS))
def test_exchange_step_refuses_rules_it_does_not_have(kind):
  from recommenders_addons_b200 import dynamic_embedding as de
  var, pv = _exchange_variable("xchg-refuse-" + kind)
  opt = MAKERS[kind](de)
  assert not isinstance(opt, de.FusedAdam) or opt.amsgrad   # AdamW is not an Adam subclass
  keys, grads = _batch(3)
  with pytest.raises(TypeError, match="de.FusedAdagrad / de.FusedAdam"):
    pv.apply_gradients(opt, keys, grads)
  assert opt.iterations == 0
  assert int(var.size()) == 0
  for plane in range(4):
    k, _ = var.tables[0].export(plane=plane)
    assert k.numel() == 0
  pv.close()


def test_exchange_step_still_runs_plain_adam():
  """FusedAdam without amsgrad keeps the owner-side det_peer_xchg_apply_adam step: param, m and v as the oracle's"""
  from recommenders_addons_b200 import dynamic_embedding as de
  var, pv = _exchange_variable("xchg-plain-adam")
  opt = de.FusedAdam(0.01, 0.9, 0.999, 1e-8)
  tabs = [O.PortTable(DIM) for _ in range(3)]
  ip = np.full(DIM, 0.05, np.float32)
  for step in (1, 2):
    keys, grads = _batch(step)
    pv.apply_gradients(opt, keys, grads)
    O.sparse_adam_step(tabs[0], tabs[1], tabs[2], keys.numpy(), grads.numpy(), O.adam_scalars(0.01, 0.9, 0.999, step),
                       0.9, 0.999, 1e-8, ip)
  assert opt.iterations == 2
  for plane in range(3):
    k, v = var.tables[0].export(plane=plane)
    o = torch.argsort(k)
    ek, ev = tabs[plane].export()
    eo = np.argsort(ek)
    np.testing.assert_array_equal(k[o].numpy(), ek[eo])
    np.testing.assert_array_equal(v[o].numpy().view(np.uint32), ev[eo].view(np.uint32))
  pv.close()
