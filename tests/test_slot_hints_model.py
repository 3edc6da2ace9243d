"""Sequential property test of the slot-hint rule (csrc/table.cu), modelled on top of tests/layout_model.LayoutModel:
interleaved streams of batch finds, inserts, removes and in-place rewrites of the key buffer leave the same table and
return the same results with hints on and with hints off."""
import numpy as np
import pytest

from tests.layout_model import EMPTY, TOMB, LayoutModel


class HintedLayoutModel(LayoutModel):
  """LayoutModel plus the slot-hint rule of table.cu: a batch find records (key, slot) per position and the table
  generation; every mutation advances the generation; the insert of a batch that follows uses the hint of position i
  only if the generation is unchanged and the hint's key is the key now at position i -- otherwise it probes."""

  def __init__(self, nb, hints=True):
    super(HintedLayoutModel, self).__init__(nb)
    self.hints = hints
    self.gen = 0
    self.record = None
    self.hinted = 0

  def find_batch(self, keys):
    slots = [self.find(k) for k in keys]
    self.record = (self.gen, list(zip(keys, slots)))
    return slots

  def insert_batch(self, keys, values):
    rec, self.record = self.record, None   # one find gives at most one hinted insert
    usable = self.hints and rec is not None and rec[0] == self.gen and len(rec[1]) == len(keys)
    for i, (k, v) in enumerate(zip(keys, values)):
      if usable and rec[1][i][0] == k and rec[1][i][1] >= 0:
        self.vals[rec[1][i][1]] = v
        self.hinted += 1
      else:
        self.insert(k, v)
    self.gen += 1

  def remove_batch(self, keys):
    for k in keys:
      self.remove(k)
    self.gen += 1


def run(seed, hints, nb=16, n_ops=300):
  rng = np.random.default_rng(seed)
  m = HintedLayoutModel(nb, hints=hints)
  universe = [int(x) for x in rng.integers(-(1 << 40), 1 << 40, 40)] + [EMPTY, TOMB]
  buf = [universe[int(i)] for i in rng.integers(0, len(universe), 12)]
  results = []
  for step in range(n_ops):
    op = rng.integers(0, 6)
    if m.size > nb * 8 * 0.7:
      op = 3
    if op in (0, 1):
      results.append(("find", m.find_batch(list(buf))))
    elif op == 2:
      m.insert_batch(list(buf), [step * 100 + i for i in range(len(buf))])
    elif op == 3:
      m.remove_batch([universe[int(i)] for i in rng.integers(0, len(universe), 6)])
    elif op == 4:   # rewrite a few positions of the key buffer in place (same buffer, same length)
      for i in rng.integers(0, len(buf), 3):
        buf[int(i)] = universe[int(rng.integers(0, len(universe)))]
    else:           # a find immediately followed by the insert of the same buffer: the hinted pattern
      results.append(("find", m.find_batch(list(buf))))
      m.insert_batch(list(buf), [step * 100 + i for i in range(len(buf))])
    m.check_invariants()
  return m, results


@pytest.mark.parametrize("seed", range(12))
def test_hints_on_and_off_give_the_same_table_and_results(seed):
  on, r_on = run(seed, True)
  off, r_off = run(seed, False)
  assert r_on == r_off
  assert list(on.keys) == list(off.keys)
  assert on.live() == off.live()
  assert (on.size, on.used, on.special) == (off.size, off.used, off.special)
  assert on.hinted > 0 and off.hinted == 0
