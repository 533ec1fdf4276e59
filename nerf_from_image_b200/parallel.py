"""Multi-GPU: one process per GPU, rays sharded by image (or, with fewer images than GPUs, by
row tiles of each image: ``render_row_sharded``), one all-gather.

The reference scales with nn.DataParallel: scatter on the batch dimension,
replicate the module, gather the outputs on GPU 0 (run.py:636-644).  The render
path has no cross-image arithmetic (SURVEY.md section 8e), so the H100 version
is: every rank renders its own contiguous slice of the batch with the fused
kernels and the output tiles are all-gathered so every rank holds the full
batch (``gather=True``); inversion needs no gradient collective because latents
and poses are per image.

Two forms of the exchange:

* in place (``render_sharded(..., inplace=True)``, equal shards): the full-batch
  rgb / depth / mask buffers are allocated first, the render kernel writes this
  rank's tiles DIRECTLY into its slice of them (``fused_render(out=...)``) and
  NCCL all-gathers each buffer in place -- the collective is the epilogue of the
  render stream, with no pack / pad / concatenate kernels and no second copy of
  the outputs around it;
* packed (ragged shards, or a ``render_fn`` without ``out``): one all-gather of
  the padded [rgb(3), depth, mask] tiles, then trim.
"""

import torch
import torch.distributed as dist


def shard_range(batch, world_size, rank):
    """Contiguous [start, stop) of images for ``rank``; remainders go to the
    lowest ranks (same split nn.DataParallel's scatter produces)."""
    if not (0 <= rank < world_size):
        raise ValueError('rank %d outside world of %d' % (rank, world_size))
    base, rem = divmod(batch, world_size)
    start = rank * base + min(rank, rem)
    return start, start + base + (1 if rank < rem else 0)


def shard_inputs(tensors, world_size, rank):
    """Slices every [B, ...] tensor (None passes through) to this rank's images."""
    batch = next(t.shape[0] for t in tensors.values() if t is not None)
    a, b = shard_range(batch, world_size, rank)
    return {k: (None if t is None else t[a:b]) for k, t in tensors.items()}


def pack_outputs(rgb, depth, mask):
    """[b,H,W,3], [b,H,W], [b,H,W] -> [b,H,W,5] (one buffer, one collective)."""
    return torch.cat((rgb, depth.unsqueeze(-1), mask.unsqueeze(-1)), dim=-1)


def unpack_outputs(packed):
    return packed[..., :3], packed[..., 3], packed[..., 4]


def all_gather_outputs(rgb, depth, mask, batch, group=None):
    """All ranks end up with the full-batch (rgb, depth, mask).

    Shards may be ragged (batch not divisible by the world size): every rank
    pads its packed tile to the largest shard, gathers, and trims.
    """
    world = dist.get_world_size(group)
    packed = pack_outputs(rgb, depth, mask)
    sizes = [shard_range(batch, world, r) for r in range(world)]
    longest = max(b - a for a, b in sizes)
    if packed.shape[0] < longest:
        pad = packed.new_zeros((longest - packed.shape[0],) + tuple(packed.shape[1:]))
        packed = torch.cat((packed, pad), dim=0)
    out = [torch.empty_like(packed) for _ in range(world)]
    dist.all_gather(out, packed.contiguous(), group=group)
    full = torch.cat([o[: b - a] for o, (a, b) in zip(out, sizes)], dim=0)
    return unpack_outputs(full)


def gathered_buffers(batch, height, width, device, dtype=torch.float32):
    """Full-batch (rgb [B,H,W,3], depth [B,H,W], mask [B,H,W]) the ranks fill in place."""
    return (torch.empty(batch, height, width, 3, device=device, dtype=dtype),
            torch.empty(batch, height, width, device=device, dtype=dtype),
            torch.empty(batch, height, width, device=device, dtype=dtype))


def shard_views(full, batch, world, rank):
    """This rank's contiguous slices of the full-batch buffers (no copy)."""
    a, b = shard_range(batch, world, rank)
    return tuple(t[a:b] for t in full)


def all_gather_inplace(full, batch, group=None):
    """Every rank has written ``full[i][a:b]`` for its own [a, b); afterwards every rank
    holds all of ``full``.  Needs equal shards (the in-place form of the collective
    requires rank r's contribution at offset r * count of the receive buffer)."""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    if batch % world:
        raise ValueError('in-place all-gather needs batch %% world == 0 (got %d, %d)'
                         % (batch, world))
    a, b = shard_range(batch, world, rank)
    if dist.get_backend(group) == 'nccl':
        # the three collectives as ONE NCCL group launch (one kernel, one ring/tree set-up):
        # at 1.3 MB per rank they are latency-bound, three back-to-back launches cost ~3x
        with dist._coalescing_manager(group=group, device=full[0].device, async_ops=False):
            for t in full:
                dist.all_gather_into_tensor(t, t[a:b], group=group)
    else:
        for t in full:
            dist.all_gather_into_tensor(t, t[a:b], group=group)
    return full


def all_reduce_grads(params, group=None, average=False):
    """Sums (or averages) the ``.grad`` of ``params`` over the ranks with ONE all-reduce of a
    flat bucket -- what nn.DataParallel's replica reduction does for the generator parameters
    in the reference's GAN step (run.py:636-644,1044).  Parameters without a gradient
    contribute zeros, so that every rank sends the same bucket layout."""
    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        return
    params = list(params)
    flat = torch.cat([(p.grad if p.grad is not None else torch.zeros_like(p)).reshape(-1).float()
                      for p in params])
    dist.all_reduce(flat, group=group)
    if average:
        flat /= dist.get_world_size(group)
    off = 0
    for p in params:
        n = p.numel()
        g = flat[off:off + n].view_as(p).to(p.dtype)
        if p.grad is None:
            p.grad = g.clone()
        else:
            p.grad.copy_(g)
        off += n


def render_sharded(render_fn, batch_inputs, batch, gather=True, group=None, inplace=False,
                   height=None, width=None):
    """Runs ``render_fn(**shard)`` on this rank's images; ``render_fn`` returns
    (rgb, depth, mask, ...).  With ``gather`` the full batch comes back.

    ``inplace`` (with ``height`` / ``width``): ``render_fn`` is called with an extra
    ``out=(rgb, depth, mask)`` -- this rank's slices of the gathered buffers -- and must
    write its outputs there (``fused_render(..., out=out)`` does); ragged batches fall back
    to the packed exchange."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    shard = shard_inputs(batch_inputs, world, rank)
    if inplace and gather and world > 1 and batch % world == 0:
        device = next(t.device for t in shard.values() if t is not None)
        full = gathered_buffers(batch, height, width, device)
        out = shard_views(full, batch, world, rank)
        res = render_fn(**shard, out=out)[:3]
        for got, want in zip(res, out):
            if got.data_ptr() != want.data_ptr():
                raise RuntimeError('render_fn ignored out=: outputs must be written in place')
        return all_gather_inplace(full, batch, group)
    if inplace:
        rgb, depth, mask = render_fn(**shard, out=None)[:3]
    else:
        rgb, depth, mask = render_fn(**shard)[:3]
    if world == 1 or not gather:
        return rgb, depth, mask
    return all_gather_outputs(rgb, depth, mask, batch, group)


def row_range(height, world_size, rank, align=8):
    """Contiguous rows [r0, r1) of an image for ``rank`` when ONE image's rays are split over the
    GPUs (fewer images than GPUs: SURVEY.md section 8e).  Shards are multiples of ``align`` rows
    (the kernels' tile height), the remainder goes to the lowest ranks; a rank may get none."""
    if not (0 <= rank < world_size):
        raise ValueError('rank %d outside world of %d' % (rank, world_size))
    blocks = -(-height // align)
    base, rem = divmod(blocks, world_size)
    b0 = rank * base + min(rank, rem)
    b1 = b0 + base + (1 if rank < rem else 0)
    return min(b0 * align, height), min(b1 * align, height)


def slice_rows(noise_t, noise_u, batch, height, width, r0, r1):
    """The two noise tensors of render() restricted to rows [r0, r1): noise_t [B,H,W,S] ->
    [B,h,W,S], noise_u [B*H*W,S] -> [B*h*W,S]."""
    nt = None if noise_t is None else noise_t[:, r0:r1].contiguous()
    nu = None
    if noise_u is not None:
        S = noise_u.shape[-1]
        nu = noise_u.view(batch, height, width, S)[:, r0:r1].reshape(-1, S).contiguous()
    return nt, nu


def render_row_sharded(render_fn, height, group=None, align=8):
    """Splits every image's ROWS over the ranks: ``render_fn(r0, r1)`` renders rows [r0, r1) of
    the whole batch (``fused_render(..., height=r1 - r0, rows=(r0, height))``) and returns
    (rgb [B,h,W,3], depth [B,h,W], mask [B,h,W]); every rank gets the full images back (one
    all-gather of the padded packed tiles, then trim + concatenate along the rows)."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    r0, r1 = row_range(height, world, rank, align)
    if world == 1:
        return tuple(render_fn(r0, r1)[:3])
    ranges = [row_range(height, world, r, align) for r in range(world)]
    longest = max(b - a for a, b in ranges)
    if r1 > r0:
        packed = pack_outputs(*render_fn(r0, r1)[:3])            # [B,h,W,5]
        shape = (packed.shape[0], longest) + tuple(packed.shape[2:])
    else:  # nothing to render on this rank: it still takes part in the exchange
        shape = None
    # every rank must know the tile shape: ranks without rows learn it from rank 0
    meta = [shape]
    dist.broadcast_object_list(meta, src=0, group=group)
    shape = shape or meta[0]
    dev = packed.device if r1 > r0 else torch.device(
        'cuda', torch.cuda.current_device()) if dist.get_backend(group) == 'nccl' else 'cpu'
    tile = torch.zeros(shape, device=dev, dtype=torch.float32)
    if r1 > r0:
        tile[:, :r1 - r0] = packed
    out = [torch.empty_like(tile) for _ in range(world)]
    dist.all_gather(out, tile, group=group)
    full = torch.cat([o[:, :b - a] for o, (a, b) in zip(out, ranges) if b > a], dim=1)
    return unpack_outputs(full)


class PeerExchange:
    """The all-gather of the output tiles WITHOUT a collective call: every rank's render kernel
    stores its tiles straight into all ranks' full-batch buffers over NVLink (peer mappings of
    symmetric memory; ``fused_render(out=..., peers=...)``) and the kernels themselves shake hands
    before they finish (the last CTA of a rank signals every peer and waits for their signals:
    ``nfi_render_params.peer_signal``).  A completed kernel = every rank's tiles are here.  What
    ``nn.DataParallel``'s gather does in the reference (run.py:636-644), fused into the render.

    Two buffer sets alternate between calls, so that a rank still reading step k's images cannot be
    overwritten by a faster peer's step k+1: that peer's step k+1 kernel cannot complete before
    this rank's step k+1 kernel has signalled, and step k+2 reuses the set only after that.
    Equal shards only (batch % world == 0), world <= 8."""

    FLAG_WORDS = 64

    def __init__(self, batch, height, width, device, group=None, handshake='kernel'):
        import torch.distributed._symmetric_memory as symm_mem
        self.group = group if group is not None else dist.group.WORLD
        self.world, self.rank = dist.get_world_size(self.group), dist.get_rank(self.group)
        if batch % self.world:
            raise ValueError('PeerExchange needs batch %% world == 0 (got %d, %d)' % (batch, self.world))
        if self.world - 1 > 7:
            raise ValueError('PeerExchange: at most 8 ranks')
        self.batch, self.h, self.w = batch, height, width
        self.handshake = handshake          # 'kernel' | 'barrier' (symmetric-memory barrier launch)
        n = batch * height * width
        self.n = n
        self.sets = []
        for _ in range(2):
            buf = symm_mem.empty(5 * n + self.FLAG_WORDS, dtype=torch.float32, device=device)
            buf.zero_()
            hdl = symm_mem.rendezvous(buf, self.group)
            self.sets.append([buf, hdl, 0])     # epoch of the set
        self.done = torch.zeros(1, dtype=torch.int32, device=device)
        torch.cuda.synchronize(device)
        dist.barrier(self.group)               # every rank's flag words are zero before anyone signals
        self.turn = 0

    def _views(self, buf):
        n, B, H, W = self.n, self.batch, self.h, self.w
        return (buf[:3 * n].view(B, H, W, 3), buf[3 * n:4 * n].view(B, H, W), buf[4 * n:5 * n].view(B, H, W))

    def begin(self):
        """-> (full buffers, this rank's slices (``out=``), the ``peers=`` argument)."""
        st = self.sets[self.turn]
        if len(st) == 3:   # first use of this set: views and peer addresses are fixed from here on
            buf, hdl = st[0], st[1]
            full = self._views(buf)
            a, b = shard_range(self.batch, self.world, self.rank)
            out = tuple(t[a:b] for t in full)
            rays0 = a * self.h * self.w
            slices, signal, ranks = [], [], []
            for r in range(self.world):
                if r == self.rank:
                    continue
                base = int(hdl.buffer_ptrs[r])
                slices.append((base + 4 * (3 * rays0), base + 4 * (3 * self.n + rays0),
                               base + 4 * (4 * self.n + rays0)))
                signal.append(base + 4 * (5 * self.n + self.rank))   # our word in peer r's flag area
                ranks.append(r)
            peers = {'slices': slices}
            if self.handshake == 'kernel':
                peers.update(signal=signal, ranks=ranks, done=self.done.data_ptr(),
                             self_signal=int(hdl.buffer_ptrs[self.rank]) + 4 * 5 * self.n)
            st.append((full, out, peers))
        st[2] += 1
        full, out, peers = st[3]
        if self.handshake == 'kernel':
            peers['epoch'] = st[2]
        return full, out, peers

    def finish(self):
        """With the in-kernel handshake nothing is left to do; with ``handshake='barrier'`` a
        stream-ordered symmetric-memory barrier stands in for it."""
        if self.handshake != 'kernel':
            self.sets[self.turn][1].barrier(channel=0)
        self.turn ^= 1
