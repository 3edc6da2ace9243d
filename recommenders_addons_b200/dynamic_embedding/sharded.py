"""Key-hash sharding of one logical table across the GPUs of a box: one process per GPU, each owning the
shard `owner(key) == rank` (reference: HvdVariable.__alltoall_embedding_lookup__,
python/ops/shadow_embedding_ops.py:397-447, with Horovod alltoall replaced by NCCL through
torch.distributed).  Exchange per lookup: all-to-all of keys (8 B/key) -> local find -> all-to-all of rows
back (dim*4 B/key); per update: all-to-all of keys + rows/grads to the owners -> local insert / fused
optimizer.  Works with the `gloo` backend on CPU tensors for the exchange logic tests only when a
`local_table` stub is injected; the real table is always on the GPU."""
import torch
import torch.distributed as dist

from .variable import Variable, combine_rows, gather_rows, partition, scatter_rows


def _alltoall_counts(counts, group):
  """send counts [W] -> recv counts [W] (the 8x8 size exchange)."""
  recv = torch.empty_like(counts)
  dist.all_to_all_single(recv, counts, group=group)
  return recv


def exchange_keys(grouped_keys, send_counts, group=None):
  """all-to-all(v) of keys grouped by owner.  Returns (received keys, recv_counts list)."""
  recv_counts = _alltoall_counts(send_counts, group)
  sc, rc = send_counts.tolist(), recv_counts.tolist()
  out = torch.empty(int(sum(rc)), dtype=grouped_keys.dtype, device=grouped_keys.device)
  dist.all_to_all_single(out, grouped_keys, output_split_sizes=rc, input_split_sizes=sc, group=group)
  return out, rc, sc


def exchange_rows(rows, in_splits, out_splits, group=None):
  out = torch.empty((int(sum(out_splits)),) + tuple(rows.shape[1:]), dtype=rows.dtype, device=rows.device)
  dist.all_to_all_single(out, rows.contiguous(), output_split_sizes=out_splits, input_split_sizes=in_splits,
                         group=group)
  return out


def agree_on(value, group=None, device=None, what="value"):
  """COLLECTIVE.  Every rank must pass the same integer (mailbox / inbox capacities fix the segment offsets peers write
  to, so a rank-local choice would misplace remote stores): MAX(v) == -MAX(-v) over the group, else ValueError on
  every rank."""
  value = int(value)
  if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
    return value
  t = torch.tensor([value, -value], dtype=torch.int64, device=device)
  dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
  hi, lo = int(t[0].item()), -int(t[1].item())
  if hi != lo:
    raise ValueError("%s differs between ranks (min %d, max %d, this rank %d): it must be agreed" % (what, lo, hi, value))
  return value


class ShardedVariable(object):
  """One shard of a key-hash-sharded variable per rank; lookups / updates take keys owned by ANY rank."""

  def __init__(self, local_variable, group=None, partition_impl=None, gather_impl=None, scatter_impl=None,
               unique_impl=None):
    from .keyed_init import refuse_keyed
    refuse_keyed(getattr(local_variable, "initializer", None), "ShardedVariable")
    self.local = local_variable
    self._unique = unique_impl
    self.group = group
    self.world = dist.get_world_size(group)
    self.rank = dist.get_rank(group)
    self._partition = partition_impl or (lambda k: partition(k, self.world, True))
    self._gather = gather_impl or gather_rows
    self._scatter = scatter_impl or scatter_rows

  @property
  def dim(self):
    return self.local.dim

  def lookup(self, keys):
    """rows for `keys` [n] in request order, wherever they live."""
    grouped, perm, counts = self._partition(keys.reshape(-1))
    recv_keys, rc, sc = exchange_keys(grouped, counts, self.group)
    rows = self.local.lookup(recv_keys)                      # local shard: find (no insert)
    back = exchange_rows(rows, rc, sc, self.group)          # rows return on the reverse pattern
    return self._scatter(back, perm)

  def upsert(self, keys, values):
    grouped, perm, counts = self._partition(keys.reshape(-1))
    vals = self._gather(values.reshape(-1, self.dim), perm)
    recv_keys, rc, sc = exchange_keys(grouped, counts, self.group)
    recv_vals = exchange_rows(vals, sc, rc, self.group)
    self.local.upsert(recv_keys, recv_vals)

  def apply_gradients(self, optimizer, keys, grads):
    """route row-gradients to the owning rank, which applies the fused optimizer locally (half-sync:
    sparse rows are never all-reduced, dynamic_embedding_optimizer.py:580-595).  Keys that several ranks
    send for the same row are combined (summed) on the owner before the update."""
    grouped, perm, counts = self._partition(keys.reshape(-1))
    g = self._gather(grads.reshape(-1, self.dim), perm)
    recv_keys, rc, sc = exchange_keys(grouped, counts, self.group)
    recv_g = exchange_rows(g, sc, rc, self.group)
    if self._unique is None:
      from .variable import unique
      self._unique = unique
    uniq, idx = self._unique(recv_keys)
    gsum = combine_rows(recv_g, idx, uniq.numel())
    optimizer.iterations += 1
    optimizer.apply_sparse(self.local, uniq, gsum)

  def size(self):
    s = self.local.size().to(torch.int64)
    t = s.clone().to(next(iter(self.local.tables)).device) if hasattr(self.local, "tables") else s.clone()
    dist.all_reduce(t, group=self.group)
    return t


class PeerShardedVariable(object):
  """The peer-memory sharded table: every rank maps its peers' shards over NVLink (CUDA IPC) and ONE kernel per
  call probes the owner's key plane and moves the row over NVLink -- no partition / all-to-all / stitch
  (det_peer_find / det_peer_insert).  `local_variable` must be single-shard, pre-sized (a published table cannot
  grow) and created identically on every rank.  With `fake_shards` (a list of Variables on ONE GPU, the way the
  reference's tests fake devices) no process group is needed.

  lookup()/upsert() are stream-ordered on the current stream; phase_barrier() separates a phase in which ranks
  read from a phase in which ranks write (the ordering the reference gets from its collectives)."""

  @classmethod
  def create(cls, dim, capacity, group=None, value_dtype=torch.float32, initializer=None, num_slot_planes=0,
             name="PeerShardedVariable", gpu_mode=True, evict_strategy=None):
    """Preferred constructor: the local shard (fixed `capacity` slots) is built inside a torch symmetric-memory
    region (CUDA VMM, mapped by every rank with 2 MB pages); peers are addressed through the rendezvous
    handle's buffer pointers.  Collective over `group`.

    evict_strategy (de.HkvEvictStrategy): every shard keeps a score plane and evicts its lowest-scored keys at
    `capacity` instead of failing with DET_TABLE_FULL.  Such shards are served by their owners only: call
    attach_exchange() (insert="push"); lookup() and apply_gradients() then run as det_peer_xchg_find /
    det_peer_xchg_apply_* -- the step's find-or-insert makes room (evict_room) and writes the scores -- and upsert() as
    det_peer_xchg_insert, where the owner compacts what arrived and runs its own scored insert (one host sync per
    call).  The one-sided kernels are refused by the library (DESIGN.md 4b)."""
    from .keyed_init import refuse_keyed
    refuse_keyed(initializer, "PeerShardedVariable")
    import torch.distributed._symmetric_memory as symm_mem
    from .table import CuckooHashTable
    from .variable import Variable
    dev = torch.device("cuda", torch.cuda.current_device())
    nbytes = CuckooHashTable.region_bytes(value_dtype, dim, capacity, num_slot_planes, dev.index)
    region = symm_mem.empty(nbytes, dtype=torch.uint8, device=dev)
    hdl = symm_mem.rendezvous(region, group if group is not None else dist.group.WORLD)

    from .table import KVCreator

    class _RegionCreator(KVCreator):
      """builds the (single) shard table inside the symmetric region"""

      def create(self, key_dtype=None, value_dtype=None, default_value=None, name=None, checkpoint=None,
                 init_size=None, config=None, device=None, shard_saveable_object_fn=None, num_slot_planes=0):
        return CuckooHashTable(key_dtype, value_dtype, default_value, name=name, init_size=capacity, device=device,
                               num_slot_planes=num_slot_planes, region=region, evict_strategy=evict_strategy,
                               max_capacity=capacity if evict_strategy is not None else 0)

    creator = _RegionCreator()
    var = Variable(dim=dim, value_dtype=value_dtype, init_size=capacity, initializer=initializer, name=name,
                   kv_creator=creator, num_slot_planes=num_slot_planes, devices=[dev])
    self = cls.__new__(cls)
    self._init_common(var, group, gpu_mode)
    import ctypes
    ptrs = (ctypes.c_void_p * self.world)(*[int(p) for p in hdl.buffer_ptrs])
    g = ctypes.c_void_p()
    self._libmod.check(self._lib.det_peer_group_create_regions(ctypes.byref(g), var.tables[0].handle, ptrs, self.world,
                                                               self.rank, 1 if gpu_mode else 0))
    self._g = g
    self._symm = (region, hdl)
    self._tables = [None] * self.world
    self._tables[self.rank] = var.tables[0]
    self.backing = "symmetric-memory"
    self._create_args = dict(dim=dim, group=group, value_dtype=value_dtype, initializer=initializer,
                             num_slot_planes=num_slot_planes, name=name, gpu_mode=gpu_mode, evict_strategy=evict_strategy)
    self.evict_strategy = evict_strategy
    self.capacity = int(capacity)
    return self

  # ---- lifecycle of a sharded table: a shard has a FIXED capacity (its planes are mapped by every peer) ------------
  def load(self):
    """COLLECTIVE.  Highest load (live keys / slots) over all shards, agreed by every rank."""
    t = torch.tensor([float(self.local.size()) / float(self.capacity)], dtype=torch.float64, device=self.device)
    if self.world > 1:
      dist.all_reduce(t, op=dist.ReduceOp.MAX, group=self._group)
    return float(t.item())

  def grow(self, new_capacity, window=1 << 22):
    """COLLECTIVE.  The reference's cuckoo shards double under the hood (cuckoohash_map.hh:1774+); a shard that peers have
    mapped cannot: every rank builds a NEW symmetric region of `new_capacity` slots, re-rendezvouses, streams its own shard
    across in bounded windows (rows and optimizer slot planes), and swaps the peer group, mailbox and inbox over.  Keys
    keep their owner, so no row crosses NVLink.  Call it between steps (maybe_grow does, on an agreed load)."""
    if self.backing != "symmetric-memory":
      raise RuntimeError("grow needs the symmetric-memory backing (PeerShardedVariable.create)")
    if getattr(self, "evict_strategy", None) is not None:
      raise RuntimeError("grow: shards with an eviction strategy stay at their capacity and evict")
    new_capacity = int(new_capacity)
    if new_capacity <= self.capacity:
      raise ValueError("grow: new_capacity must exceed the current %d slots" % self.capacity)
    torch.cuda.synchronize(self.device)
    dist.barrier(group=self._group)                       # nobody is still reading or writing the old shards
    fresh = PeerShardedVariable.create(capacity=new_capacity, **self._create_args)
    told, tnew = self.local.tables[0], fresh.local.tables[0]
    planes = int(self._create_args["num_slot_planes"])
    first = 0
    while True:
      k, v = told.export_window(first, window)
      if k.numel() == 0:
        break
      tnew.insert(k, v)
      for pl in range(1, planes + 1):
        k2, sv_ = told.export_window(first, window, plane=pl)
        tnew.import_plane(pl, k2, sv_)
      first += k.numel()
    torch.cuda.synchronize(self.device)
    xitems = getattr(self, "_xchg_items", 0) if getattr(self, "_xchg", False) else 0
    xins = "push" if getattr(self, "_xchg_insert", True) else "pull"
    inbox_items = getattr(self, "_inbox_items", 0)
    self.close()                                          # old group; the old region dies with its last reference
    old_table = told
    for attr in ("local", "_g", "_symm", "_tables", "capacity", "_default"):
      setattr(self, attr, getattr(fresh, attr))
    fresh._g = None                                       # ownership moved
    self._xchg = False
    for attr in ("_xbox", "_inbox", "_xapply_ws"):
      if hasattr(self, attr):
        delattr(self, attr)
    old_table.close()
    if xitems:
      self.attach_exchange(xitems, insert=xins)
    if inbox_items:
      self.attach_inbox(inbox_items)
    dist.barrier(group=self._group)

  def maybe_grow(self, threshold=0.6, factor=2.0):
    """COLLECTIVE.  Grows every shard by `factor` once the fullest shard has passed `threshold` (the decision is an
    all-reduce MAX, so all ranks take it together).  Returns True when it grew."""
    if getattr(self, "evict_strategy", None) is not None:
      return False                                   # shards with an eviction strategy evict instead
    if self.load() > threshold:
      self.grow(int(self.capacity * factor))
      return True
    return False

  def _init_common(self, local_variable, group, gpu_mode):
    from .. import _lib
    from .keyed_init import refuse_keyed
    refuse_keyed(getattr(local_variable, "initializer", None), "PeerShardedVariable")
    self._lib = _lib.lib()
    self._libmod = _lib
    self.local = local_variable
    self.world = dist.get_world_size(group)
    self.rank = dist.get_rank(group)
    self.dim = local_variable.dim
    self.device = local_variable.tables[0].device
    self.value_dtype = local_variable.value_dtype
    self._group = group
    self._default = local_variable.tables[0]._default_value

  def __init__(self, local_variable=None, group=None, fake_shards=None, gpu_mode=True):
    import ctypes
    from .. import _lib
    self._lib = _lib.lib()
    self._libmod = _lib
    self.backing = "cuda-ipc" if fake_shards is None else "same-process"
    if fake_shards is not None:
      self.world, self.rank = len(fake_shards), 0
      tables = [v.tables[0] for v in fake_shards]
      self.local = fake_shards[0]
      blobs = None
    else:
      self.local = local_variable
      self.world = dist.get_world_size(group)
      self.rank = dist.get_rank(group)
      t = local_variable.tables[0]
      nbytes = self._lib.det_peer_handle_bytes()
      mine = (ctypes.c_ubyte * nbytes)()
      _lib.check(self._lib.det_peer_export(t.handle, ctypes.cast(mine, ctypes.c_void_p)))
      send = torch.tensor(list(bytes(mine)), dtype=torch.uint8, device=t.device)
      gathered = [torch.empty_like(send) for _ in range(self.world)]
      dist.all_gather(gathered, send, group=group)
      blobs = b"".join(bytes(g.cpu().numpy().tobytes()) for g in gathered)
      tables = [None] * self.world
      tables[self.rank] = t
    self._tables = tables
    self.dim = self.local.dim
    self.device = self.local.tables[0].device
    self.value_dtype = self.local.value_dtype
    arr = (ctypes.c_void_p * self.world)(*[(tb.handle if tb is not None else None) for tb in tables])
    self._blob_buf = ctypes.create_string_buffer(blobs, len(blobs)) if blobs is not None else None
    g = ctypes.c_void_p()
    _lib.check(self._lib.det_peer_group_create(ctypes.byref(g), arr,
                                               ctypes.cast(self._blob_buf, ctypes.c_void_p) if blobs else None,
                                               self.world, self.rank, 1 if gpu_mode else 0))
    self._g = g
    self._group = group
    self._default = self.local.tables[0]._default_value

  def _sp(self):
    import ctypes
    return ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

  # ---- owner-side exchange (det_peer_xchg_*): ids travel to the owner, the owner probes locally and pushes rows ----
  def attach_exchange(self, max_items, mailbox_ptrs=None, keepalive=None, insert="push"):
    """Collective.  Gives every rank a MAILBOX all peers map (request / insert segments per source rank, a 2-entry
    output ring, flag words); afterwards lookup() / upsert() run through the owners with posted NVLink stores only
    (HvdVariable.__alltoall_embedding_lookup__, shadow_embedding_ops.py:397-447, without a collective library).
    Every rank must then issue the same sequence of lookup / upsert calls (n may differ), as with the reference's
    alltoall ops.  `mailbox_ptrs` (tests): explicit pointers instead of a symmetric-memory allocation."""
    import ctypes
    rb = self.dim * torch.empty(0, dtype=self.value_dtype).element_size()
    nbytes = int(self._lib.det_peer_xchg_bytes(self.world, int(max_items), rb))
    if nbytes == 0:
      raise ValueError("attach_exchange: bad max_items / world")
    if mailbox_ptrs is not None:
      ptrs, self._xbox = [int(p) for p in mailbox_ptrs], keepalive
    elif self.backing == "symmetric-memory":
      import torch.distributed._symmetric_memory as symm_mem
      agree_on(max_items, self._group, self.device, "attach_exchange: max_items")
      box = symm_mem.empty(nbytes, dtype=torch.uint8, device=self.device)
      box.zero_()
      hdl = symm_mem.rendezvous(box, self._group if self._group is not None else dist.group.WORLD)
      ptrs = [int(p) for p in hdl.buffer_ptrs]
      self._xbox = (box, hdl)
      torch.cuda.synchronize(self.device)
      dist.barrier(group=self._group)   # every mailbox is zeroed before any rank may write into it
    else:
      raise RuntimeError("the exchange mailbox needs the symmetric-memory backing (PeerShardedVariable.create)")
    arr = (ctypes.c_void_p * self.world)(*ptrs)
    self._libmod.check(self._lib.det_peer_xchg_attach(self._g, arr, int(max_items), rb))
    self._xchg_items = int(max_items)
    self._xchg = True
    # insert="pull" (the HYBRID exchange): lookups go through the owners (pushes only), upserts keep the one-sided kernel
    # that probes the owner's key plane remotely and posts the row.  Reads and remote writes then need phase_barrier() between them again.
    if insert not in ("push", "pull"):
      raise ValueError("attach_exchange: insert must be 'push' or 'pull'")
    self._xchg_insert = insert == "push"

  def _ring_view(self, ptr, n):
    """torch view of n rows of the output ring (lives inside the mailbox allocation)"""
    box = self._xbox[0]
    es = torch.empty(0, dtype=self.value_dtype).element_size()
    off = int(ptr) - box.data_ptr()
    return box[off:off + n * self.dim * es].view(self.value_dtype).reshape(n, self.dim)

  def lookup(self, keys, return_exists=False, default=None, copy=True):
    import ctypes
    flat = keys.reshape(-1).contiguous()
    n = flat.numel()
    d = self._default if default is None else default.contiguous()
    full = 1 if (n > 0 and d.numel() == n * self.dim) else 0
    if getattr(self, "_xchg", False):
      # copy=False: the rows are a VIEW of the output ring, valid until the next-but-one lookup (no extra HBM pass)
      p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
      zero_copy = (not copy) and isinstance(self._xbox, tuple) and torch.is_tensor(self._xbox[0])
      out = None if zero_copy else torch.empty((n, self.dim), dtype=self.value_dtype, device=self.device)
      ex = torch.empty(n, dtype=torch.bool, device=self.device) if return_exists else None
      view = ctypes.c_void_p()
      self._libmod.check(self._lib.det_peer_xchg_find(self._g, p(flat), n, p(d), full, p(out), p(ex),
                                                      ctypes.byref(view), self._sp()))
      if zero_copy:
        out = self._ring_view(view.value, n)
      out = out.reshape(tuple(keys.shape) + (self.dim,))
      return (out, ex.reshape(keys.shape)) if return_exists else out
    out = torch.empty((n, self.dim), dtype=self.value_dtype, device=self.device)
    ex = torch.empty(n, dtype=torch.bool, device=self.device) if return_exists else None
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
    self._libmod.check(self._lib.det_peer_find(self._g, p(flat), n, p(d), full, p(out), p(ex), self._sp()))
    out = out.reshape(tuple(keys.shape) + (self.dim,))
    return (out, ex.reshape(keys.shape)) if return_exists else out

  def upsert(self, keys, values):
    import ctypes
    flat = keys.reshape(-1).contiguous()
    vals = values.reshape(-1, self.dim).contiguous()
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    if getattr(self, "_xchg", False) and self._xchg_insert:
      self._libmod.check(self._lib.det_peer_xchg_insert(self._g, p(flat), p(vals), flat.numel(), self._sp()))
      return
    self._libmod.check(self._lib.det_peer_insert(self._g, p(flat), p(vals), flat.numel(), self._sp()))

  def phase_barrier(self):
    """Separates a phase in which ranks read from one in which they write (one-sided kernels).  With the owner-side
    exchange attached it is a no-op: every shard is read and written by its OWNER's kernels only, in stream order."""
    if getattr(self, "_xchg", False) and self._xchg_insert:
      return
    self._libmod.check(self._lib.det_peer_barrier(self._g, self._sp()))

  # ---- one-sided all-to-all-v: (key, row) pairs travel to the owner's inbox (backward path) ---------------
  def attach_inbox(self, max_items):
    """Collective.  Gives every rank an inbox of `max_items` (key, row) pairs per source rank that all peers map."""
    import ctypes
    rb = self.dim * torch.empty(0, dtype=self.value_dtype).element_size()
    nbytes = int(self._lib.det_peer_inbox_bytes(self.world, int(max_items), rb))
    if self.backing == "symmetric-memory":
      import torch.distributed._symmetric_memory as symm_mem
      agree_on(max_items, self._group, self.device, "attach_inbox: max_items")
      box = symm_mem.empty(nbytes, dtype=torch.uint8, device=self.device)
      box.zero_()
      hdl = symm_mem.rendezvous(box, self._group if self._group is not None else dist.group.WORLD)
      ptrs = [int(p) for p in hdl.buffer_ptrs]
      self._inbox = (box, hdl)
    elif self.backing == "same-process":
      boxes = [torch.zeros(nbytes, dtype=torch.uint8, device=t.device) for t in self._tables]
      ptrs = [b.data_ptr() for b in boxes]
      self._inbox = boxes
    else:
      raise RuntimeError("the inbox needs the symmetric-memory backing (PeerShardedVariable.create)")
    torch.cuda.synchronize(self.device)
    arr = (ctypes.c_void_p * self.world)(*ptrs)
    self._libmod.check(self._lib.det_peer_inbox_attach(self._g, arr, int(max_items), rb))
    self._inbox_items = int(max_items)
    if self._group is not None or self.backing == "symmetric-memory":
      dist.barrier(group=self._group)

  def route(self, keys, rows):
    """partition by owner + pack + send in one kernel; follow with phase_barrier() before inbox_take()."""
    import ctypes
    flat = keys.reshape(-1).contiguous()
    r = rows.reshape(-1, self.dim).contiguous()
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    self._libmod.check(self._lib.det_peer_route(self._g, p(flat), p(r), flat.numel(), self._sp()))

  def inbox_take(self, shard=None):
    """(keys, rows) every source routed to this rank's shard (concatenated in source-rank order)."""
    import ctypes
    shard = self.rank if shard is None else int(shard)
    counts = (ctypes.c_int64 * self.world)()
    self._libmod.check(self._lib.det_peer_inbox_counts(self._g, shard, counts, self._sp()))
    total = int(sum(counts))
    dev = self.device if self._tables[shard] is None else self._tables[shard].device
    keys = torch.empty(total, dtype=torch.int64, device=dev)
    rows = torch.empty((total, self.dim), dtype=self.value_dtype, device=dev)
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t.numel() else None
    self._libmod.check(self._lib.det_peer_inbox_gather(self._g, shard, counts, p(keys), p(rows), self._sp()))
    return keys, rows, [int(c) for c in counts]

  def apply_gradients(self, optimizer, keys, grads):
    """Backward of the sharded lookup: route the row-gradients to their owners over NVLink, combine the gradients
    that several ranks sent for the same key, then run the fused optimizer on the local shard (half-sync: sparse
    rows are never all-reduced, dynamic_embedding_optimizer.py:580-595)."""
    if getattr(self, "_xchg", False) and self._xchg_insert and self.value_dtype == torch.float32:
      return self._apply_gradients_xchg(optimizer, keys, grads)
    from .variable import unique
    self.route(keys, grads)
    self.phase_barrier()
    rk, rg, _ = self.inbox_take()
    self.phase_barrier()  # every owner has emptied its inbox: the next route may overwrite it
    if rk.numel():
      uniq, idx = unique(rk)
      gsum = combine_rows(rg, idx, uniq.numel())
      optimizer.iterations += 1
      optimizer.apply_sparse(self.local, uniq, gsum)
    else:
      optimizer.iterations += 1

  def _apply_gradients_xchg(self, optimizer, keys, grads):
    """owner-side step in ONE collective C call (det_peer_xchg_apply_*): route -> compact -> unique -> position-order
    gradient sum -> fused optimizer, every count on the device (no host synchronisation, no inbox round trip)"""
    import ctypes
    from .optimizer import FusedAdagrad, FusedAdam
    # the owner-side exchange step has the Adagrad and Adam rules only: AMSGrad, AdamW and the other optimizers are
    # refused, before any state changes, rather than run as another rule
    adagrad = isinstance(optimizer, FusedAdagrad)
    if not adagrad and not (isinstance(optimizer, FusedAdam) and not optimizer.amsgrad):
      raise TypeError("PeerShardedVariable.apply_gradients: de.FusedAdagrad / de.FusedAdam (without amsgrad), got %s" %
                      type(optimizer).__name__)
    flat = keys.reshape(-1).contiguous()
    g = grads.reshape(-1, self.dim).to(torch.float32).contiguous()
    need = int(self._lib.det_peer_xchg_apply_workspace_bytes(self._g))
    ws = getattr(self, "_xapply_ws", None)
    if ws is None or ws.numel() < need:
      raw = torch.empty(need + 256, dtype=torch.uint8, device=self.device)
      off = (-raw.data_ptr()) % 256
      ws = self._xapply_ws = raw[off:off + need]
    init = self._default.to(self.device).contiguous()
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t.numel() else None
    optimizer.iterations += 1
    if adagrad:
      self._libmod.check(self._lib.det_peer_xchg_apply_adagrad(self._g, p(flat), p(g), flat.numel(), optimizer.learning_rate,
                                                               optimizer.epsilon, p(init), optimizer.initial_accumulator_value,
                                                               p(ws), ws.numel(), self._sp()))
    else:
      self._libmod.check(self._lib.det_peer_xchg_apply_adam(self._g, p(flat), p(g), flat.numel(), optimizer.alpha(),
                                                            optimizer.beta_1, optimizer.beta_2, optimizer.epsilon, p(init),
                                                            p(ws), ws.numel(), self._sp()))

  def size(self):
    if self._group is None and self.world > 1 and all(t is not None for t in self._tables):
      return sum(int(t.size()) for t in self._tables)
    s = self.local.size().to(self.device)
    if self.world > 1:
      dist.all_reduce(s, group=self._group)
    return int(s)

  def close(self):
    if getattr(self, "_g", None):
      self._lib.det_peer_group_destroy(self._g)
      self._g = None

  def __del__(self):
    try:
      self.close()
    except Exception:
      pass
