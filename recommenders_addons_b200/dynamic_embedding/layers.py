"""Callers of the hot path, mirrored as thin torch modules (reference: python/keras/layers/embedding.py:111-595 --
`Embedding`, `SquashedEmbedding`, `HvdAllToAllEmbedding` are thin wrappers over embedding_lookup_unique on a
ShadowVariable / HvdVariable).  Training flow, like the reference's TrainableWrapper: forward fills a dense scratch
of the UNIQUE rows from the table, autograd produces the gradient of that scratch, `apply_gradients(optimizer)`
writes the update back with the fused find-or-insert + optimizer kernel."""
import torch

from .ops import trainable_embedding_lookup_sparse
from .optimizer import _FUSED_DTYPES, ComposedOptimizer, _FusedBase
from .sharded import PeerShardedVariable, ShardedVariable
from .table import slot_dtype_of
from .variable import Variable, default_partition_fn, embedding_lookup_unique, gather_unique, unique


class Embedding(torch.nn.Module):
  """de.keras.layers.Embedding: dynamic embedding space, arbitrary ids shape -> ids.shape + [embedding_size].

  num_slot_planes: float32 optimizer slot planes beside the rows, for the fused Adagrad / Adam step; kept for float32,
  float16 and bfloat16 rows (the step widens a half row, updates it in float32 and rounds it once), 0 for any other
  value_dtype.  slot_dtype: None (float32 planes) or the layer's own float16 / bfloat16 value_dtype (planes in that
  dtype, rounded once per step like the rows; the reference's slot layout)."""

  def __init__(self, embedding_size, key_dtype=torch.int64, value_dtype=torch.float32, combiner="sum", initializer=None,
               devices=None, name="DynamicEmbeddingLayer", with_unique=True, trainable=True, bp_v2=False,
               init_capacity=0, partitioner=default_partition_fn, kv_creator=None, max_norm=None, num_slot_planes=2,
               restrict_policy=None, short_file_name=False, slot_dtype=None):
    super().__init__()
    if combiner not in ("sum", "mean", "sqrtn"):
      raise ValueError("combiner must be one of 'mean', 'sqrtn' or 'sum'")
    self.embedding_size = int(embedding_size)
    self.combiner = combiner
    self.with_unique = with_unique
    self.max_norm = max_norm
    self.params = Variable(key_dtype=key_dtype, value_dtype=value_dtype, dim=self.embedding_size, devices=devices,
                           partitioner=partitioner, name=name, initializer=initializer, trainable=trainable,
                           init_size=init_capacity, kv_creator=kv_creator, bp_v2=bp_v2, restrict_policy=restrict_policy,
                           num_slot_planes=num_slot_planes if value_dtype in _FUSED_DTYPES else 0,
                           short_file_name=short_file_name, slot_dtype=slot_dtype)
    self._wrappers = []

  def call(self, ids):
    """the Keras entry point of the reference layer (embedding.py:300-335)"""
    return self.forward(ids)

  def get_config(self):
    """embedding.py:327-335"""
    return {"embedding_size": self.embedding_size, "key_dtype": self.params.key_dtype, "value_dtype": self.params.value_dtype,
            "combiner": self.combiner, "initializer": self.params.initializer, "devices": self.params.devices,
            "name": self.params.name, "with_unique": self.with_unique}

  def forward(self, ids):
    out, tw = embedding_lookup_unique(self.params, ids, max_norm=self.max_norm, return_trainable=True)
    if self.training and self.params.trainable:
      self._wrappers.append(tw)
    return out

  def apply_gradients(self, optimizer):
    """optimizer: de.FusedAdagrad / de.FusedAdam (or DynamicEmbeddingOptimizer(torch optimizer))."""
    if not isinstance(optimizer, (_FusedBase, ComposedOptimizer)):
      raise TypeError("use de.DynamicEmbeddingOptimizer(...) / de.FusedAdagrad / de.FusedAdam")
    gv = [(tw.values.grad, tw) for tw in self._wrappers if tw.values.grad is not None]
    self._wrappers = []
    if gv:
      optimizer.apply_gradients(gv)


class SquashedEmbedding(Embedding):
  """embedding.py:337-362: ids [batch, n] -> [batch, embedding_size], reduced over axis 1 with the combiner."""

  def forward(self, ids):
    emb = super().forward(ids)
    if self.combiner == "sum":
      return emb.sum(dim=1)
    if self.combiner == "mean":
      return emb.mean(dim=1)
    return emb.sum(dim=1) / (emb.shape[1] ** 0.5)


BasicEmbedding = Embedding  # embedding.py:340-343


class SparseEmbedding(Embedding):
  """Bags of ids -> [batch, embedding_size], combined with `combiner`, trained through the fused kernels:
  `forward(sp_ids, sp_weights=None)` is `trainable_embedding_lookup_sparse` (the fused embedding_lookup_sparse), and
  `apply_gradients(optimizer)` steps the table from the output gradient -- one det_apply_*_sparse call per forward with
  a fused optimizer.  One shard, float32 / float16 / bfloat16 rows, a constant or keyed initializer, embedding_size a
  multiple of 4 up to 128.  `max_norm` clips every looked-up row, and the step trains through the clip (float32)."""

  def __init__(self, embedding_size, combiner="mean", **kwargs):
    super().__init__(embedding_size, combiner=combiner, **kwargs)

  def forward(self, sp_ids, sp_weights=None):
    out, h = trainable_embedding_lookup_sparse(self.params, sp_ids, sp_weights, combiner=self.combiner,
                                               max_norm=self.max_norm)
    if self.training and self.params.trainable:
      self._wrappers.append(h)
    return out

  def apply_gradients(self, optimizer):
    """optimizer: a fused optimizer or DynamicEmbeddingOptimizer(torch optimizer)."""
    if not isinstance(optimizer, (_FusedBase, ComposedOptimizer)):
      raise TypeError("use de.DynamicEmbeddingOptimizer(...) / de.FusedAdagrad / de.FusedAdam")
    gv = [(h.out.grad, h) for h in self._wrappers if h.out.grad is not None]
    self._wrappers = []
    if gv:
      optimizer.apply_gradients(gv)


class FieldWiseEmbedding(Embedding):
  """embedding.py:365-515: every feature id belongs to one of `nslots` fields (`slot_map_fn`, element-wise); the rows
  of the ids of a sample that fall into the same field are combined: ids [batch, n] -> [batch, nslots, embedding_size]
  (fields without ids give zeros, like the reference's sparse_segment_* with num_segments)."""

  def __init__(self, embedding_size, nslots, slot_map_fn=None, name="SlotDynamicEmbeddingLayer", **kwargs):
    if not callable(slot_map_fn):
      raise ValueError("slot_map_fn is not callable.")
    try:
      nslots = int(nslots)
    except Exception:
      raise TypeError("nslots should be convertible to int, but get {}".format(type(nslots)))
    super().__init__(embedding_size, name=name, **kwargs)
    self.slot_map_fn = slot_map_fn
    self.nslots = nslots

  def forward(self, ids):
    if ids.dim() > 2:
      raise NotImplementedError("Input dimension higher than 2 is not implemented yet.")
    if ids.dim() == 1:
      ids = ids.reshape(1, -1)
    batch = ids.shape[0]
    rows = super().forward(ids.reshape(-1))                                     # [batch * n, dim]
    slots = self.slot_map_fn(ids).to(torch.int64)
    seg = (slots + torch.arange(batch, device=ids.device, dtype=torch.int64).reshape(batch, 1) * self.nslots).reshape(-1)
    out = torch.zeros((batch * self.nslots, self.embedding_size), dtype=rows.dtype, device=rows.device)
    out = out.index_add(0, seg, rows)
    if self.combiner != "sum":
      cnt = torch.zeros(batch * self.nslots, dtype=rows.dtype, device=rows.device).index_add(
          0, seg, torch.ones_like(seg, dtype=rows.dtype)).clamp_(min=1).reshape(-1, 1)
      out = out / (cnt if self.combiner == "mean" else cnt.sqrt())
    return out.reshape(batch, self.nslots, self.embedding_size)


class AllToAllEmbedding(torch.nn.Module):
  """HvdAllToAllEmbedding (embedding.py:545-595) over the one-sided sharded table: ids owned by ANY rank.
  forward: unique -> det_peer_find -> gather; apply_gradients: per-unique gradients routed to their owners
  (det_peer_route), combined and stepped there.

  With a `kv_creator` whose config has an eviction strategy (the reference's HkvHashTableCreator) every rank owns an
  ordinary, evicting HkvHashTable and the layer runs on the COLLECTIVE exchange (ShardedVariable: all-to-all of ids,
  owner-side find / fused step, all-to-all of rows back) -- a shard peers write one-sidedly cannot evict (DESIGN.md 4b)."""

  def __init__(self, embedding_size, capacity_per_shard=None, group=None, initializer=None, name="AllToAllEmbedding",
               num_slot_planes=2, with_unique=True, with_secondary_unique=True, mpi_size=None, batch_size=None,
               key_dtype=torch.int64, value_dtype=torch.float32, init_capacity=0, kv_creator=None, devices=None,
               exchange_impls=None, evict_strategy=None, max_ids_per_rank=None, slot_dtype=None, **kwargs):
    """The reference's arguments (embedding.py:545-563: with_unique, with_secondary_unique, mpi_size, batch_size and the
    base layer's) are accepted; the world size comes from `group`, lookups always dedupe once (unique -> one-sided
    find), and a published shard has a FIXED capacity: capacity_per_shard (default: init_capacity, else 1M slots)."""
    super().__init__()
    from .keyed_init import refuse_keyed
    refuse_keyed(initializer, "AllToAllEmbedding")
    if key_dtype != torch.int64 or value_dtype != torch.float32:
      raise TypeError("AllToAllEmbedding: int64 keys and float32 rows")
    slot_dtype_of(value_dtype, slot_dtype)   # float32 rows: float32 slot planes only
    self.embedding_size = int(embedding_size)
    self.with_unique, self.with_secondary_unique, self.batch_size = with_unique, with_secondary_unique, batch_size
    capacity_per_shard = int(capacity_per_shard or init_capacity or (1 << 20))
    evicting = getattr(getattr(kv_creator, "config", None), "evict_strategy", None) is not None
    self.collective = kv_creator is not None
    if self.collective:
      # `exchange_impls` (tests): partition_impl / gather_impl / scatter_impl / unique_impl of ShardedVariable
      local = Variable(key_dtype=key_dtype, value_dtype=value_dtype, dim=self.embedding_size, devices=devices, name=name,
                       initializer=initializer, init_size=capacity_per_shard, kv_creator=kv_creator,
                       num_slot_planes=num_slot_planes)
      if len(local.tables) != 1:
        raise ValueError("AllToAllEmbedding: one local shard per rank (devices must name one device)")
      self.params = ShardedVariable(local, group, **(exchange_impls or {}))
      self.evicting = evicting
    else:
      # evict_strategy without a kv_creator: fixed-capacity shards that evict, served by their owners over the owner-side
      # exchange (max_ids_per_rank = the mailbox capacity: the most unique ids one rank sends in one call)
      self.evicting = evict_strategy is not None
      self.params = PeerShardedVariable.create(self.embedding_size, capacity_per_shard, group=group,
                                               initializer=initializer, num_slot_planes=num_slot_planes, name=name,
                                               evict_strategy=evict_strategy)
      if self.evicting:
        if not max_ids_per_rank:
          raise ValueError("AllToAllEmbedding(evict_strategy=...): max_ids_per_rank (the exchange mailbox capacity) is required")
        self.params.attach_exchange(int(max_ids_per_rank), insert="push")
    self._pending = []
    self._inbox_items = 0

  def forward(self, ids):
    flat = ids.reshape(-1)
    uniq, idx = unique(flat)
    rows = self.params.lookup(uniq).reshape(-1, self.embedding_size)
    if not self.collective:
      self.params.phase_barrier()
    rows = rows.detach().requires_grad_(self.training)
    if self.training:
      self._pending.append((uniq, rows))
    return gather_unique(rows, idx).reshape(tuple(ids.shape) + (self.embedding_size,))

  def apply_gradients(self, optimizer, max_unique_per_rank=None):
    """COLLECTIVE: every rank calls it once per forward, whatever happened to its own gradients.  The inbox capacity is
    agreed by all ranks (an all-reduce MAX of the largest per-rank unique count, unless `max_unique_per_rank` is given
    identically everywhere): attach_inbox is itself collective and the inbox segment offsets depend on the capacity,
    so a rank-local decision could hang the job or misplace remote writes.  A rank whose rows received no gradient
    routes zeros instead of skipping the exchange."""
    import torch.distributed as dist
    if self.collective:           # the all-to-all sizes itself; a rank without gradients still takes part, with zeros
      for uniq, rows in self._pending:
        self.params.apply_gradients(optimizer, uniq, rows.grad if rows.grad is not None else torch.zeros_like(rows))
      self._pending = []
      return
    if getattr(self.params, "_xchg", False) and self.params._xchg_insert:   # owner-side exchange: no inbox to size
      for uniq, rows in self._pending:
        self.params.apply_gradients(optimizer, uniq, rows.grad if rows.grad is not None else torch.zeros_like(rows))
      self._pending = []
      return
    for uniq, rows in self._pending:
      grad = rows.grad if rows.grad is not None else torch.zeros_like(rows)
      if max_unique_per_rank is not None:
        need = int(max_unique_per_rank)
      else:
        t = torch.tensor([uniq.numel()], dtype=torch.int64, device=uniq.device)
        if dist.is_available() and dist.is_initialized() and self.params.world > 1:
          dist.all_reduce(t, op=dist.ReduceOp.MAX, group=self.params._group)
        need = int(t.item())
      if uniq.numel() > need:
        raise ValueError("AllToAllEmbedding.apply_gradients: %d unique ids exceed max_unique_per_rank=%d" % (uniq.numel(), need))
      if need > self._inbox_items:
        self._inbox_items = max(need, 2 * self._inbox_items)   # same value on every rank: a function of agreed numbers
        self.params.attach_inbox(self._inbox_items)            # collective
      self.params.apply_gradients(optimizer, uniq, grad)
    self._pending = []
