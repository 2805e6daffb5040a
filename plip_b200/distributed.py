"""Multi-GPU data parallelism for the encode path: one process per GPU, batch sharding, and an
all-gather of embeddings only where a cross-batch similarity matrix / global embedding table is needed.

The reference is single-device (``plip.py:15``; SURVEY.md §2a) — this layer is new.  Every image and
caption is an independent unit and the packed weights (354 MB) are replicated per GPU, so the towers need
no collective at all; the only exchange is ``all_gather`` of ``[n_local,512]`` float32 rows
(NCCL over NVLink on GPUs; gloo in the CPU tests).  Rows are block-partitioned contiguously with the
remainder on the low ranks, so a gather restores the original order.
"""
from __future__ import annotations

from typing import Callable, Iterable, List, Optional, Sequence, Tuple, Union

import torch
import torch.distributed as dist


def world() -> Tuple[int, int]:
    """``(rank, world_size)``; ``(0, 1)`` when torch.distributed is not initialised."""
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def shard_counts(n: int, world_size: int) -> List[int]:
    """Rows per rank: contiguous blocks, remainder spread over the low ranks."""
    base, rem = divmod(int(n), int(world_size))
    return [base + (1 if r < rem else 0) for r in range(world_size)]


def shard_range(n: int, rank: int, world_size: int) -> Tuple[int, int]:
    """Half-open row range ``[lo, hi)`` owned by ``rank``."""
    counts = shard_counts(n, world_size)
    lo = sum(counts[:rank])
    return lo, lo + counts[rank]


def merge_topk_candidates(cand_i: torch.Tensor, cand_v: torch.Tensor, k: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """Merge per-shard top-k lists: ``cand_i`` int64 / ``cand_v`` ``[n_queries, shards * k]`` in shard-major order
    (global indices, -1 for an exhausted list) -> the best ``k`` by score, equal scores by lower global index."""
    cand_v = torch.where(cand_i < 0, torch.full_like(cand_v, float("-inf")), cand_v)
    # shard-major candidate order = ascending global index among equal scores; a stable sort keeps it
    order = torch.sort(cand_v, dim=1, descending=True, stable=True).indices[:, :k]
    return torch.gather(cand_i, 1, order), torch.gather(cand_v, 1, order)


def all_gather_rows(local: torch.Tensor, counts: Optional[Sequence[int]] = None, group=None) -> torch.Tensor:
    """Concatenate per-rank row blocks ``[n_r, d]`` in rank order -> ``[sum n_r, d]`` on every rank.

    Uneven blocks are padded to the largest block for a single ``all_gather_into_tensor`` (one NCCL
    call, NVLS-eligible) and trimmed afterwards.  ``counts`` avoids an extra size exchange."""
    rank, ws = world()
    if ws == 1:
        return local
    local = local.contiguous()
    if counts is None:
        sizes = torch.tensor([local.shape[0]], device=local.device, dtype=torch.int64)
        all_sizes = [torch.zeros_like(sizes) for _ in range(ws)]
        dist.all_gather(all_sizes, sizes, group=group)
        counts = [int(s.item()) for s in all_sizes]
    counts = list(counts)
    if local.shape[0] != counts[rank]:
        raise ValueError(f"rank {rank}: local block has {local.shape[0]} rows, expected {counts[rank]}")
    mx = max(counts)
    d = local.shape[1:]
    if local.shape[0] < mx:
        pad = torch.zeros((mx - local.shape[0], *d), device=local.device, dtype=local.dtype)
        send = torch.cat([local, pad], dim=0)
    else:
        send = local
    recv = torch.empty((ws * mx, *d), device=local.device, dtype=local.dtype)
    dist.all_gather_into_tensor(recv, send, group=group)
    if all(c == mx for c in counts):
        return recv
    return torch.cat([recv[r * mx: r * mx + counts[r]] for r in range(ws)], dim=0)


def all_gather_rows_async(local: torch.Tensor, group=None):
    """Equal-sized row blocks only: start ``all_gather_into_tensor`` on NCCL's stream and return
    ``(gathered, work)``; call ``work.wait()`` before reading ``gathered`` on the current stream.  Lets the
    exchange (and any skew between ranks) overlap with whatever is launched in between — e.g. the vision tower
    while the text embeddings travel."""
    rank, ws = world()
    if ws == 1:
        return local, None
    local = local.contiguous()
    recv = torch.empty((ws * local.shape[0], *local.shape[1:]), device=local.device, dtype=local.dtype)
    work = dist.all_gather_into_tensor(recv, local, group=group, async_op=True)
    return recv, work


def _encode_chunks(encode: Callable, rows: Union[torch.Tensor, Iterable[torch.Tensor]]) -> torch.Tensor:
    """``rows`` is one tensor or an iterable of tensors (a gallery streamed chunk by chunk): embeddings in order."""
    if torch.is_tensor(rows):
        return encode(rows)
    return torch.cat([encode(c) for c in rows], dim=0)


class ShardedCLIP:
    """Batch-sharded encode + similarity flows of BASELINE.json's multi-GPU configs.

    ``encode_images`` / ``encode_text`` are callables ``rows -> [n,512]`` NORMALISED embeddings of the *local* shard
    (on GPUs: ``Engine.encode_images`` / ``Engine.encode_text`` with ``normalize=True`` — see :meth:`from_engine`);
    ``similarity(a, b, scale)`` returns ``scale * a @ b.T`` (``Engine.similarity``); ``topk(query, space, k)`` returns
    ``(idx, val)`` of the k best ``space`` rows per query (``Engine.similarity_topk``).  The class only does the
    partitioning / gathering; image arguments may be one tensor or an iterable of chunks."""

    def __init__(self, encode_images: Callable, encode_text: Callable, similarity: Callable, logit_scale_exp: float,
                 topk: Optional[Callable] = None, encode_pair: Optional[Callable] = None):
        self.encode_images = encode_images
        self.encode_text = encode_text
        self.encode_pair = encode_pair  # (pixels, ids) -> (image, text) embeddings, both towers at once
        self.similarity = similarity
        self.topk = topk
        self.logit_scale_exp = float(logit_scale_exp)
        self.rank, self.world_size = world()

    @classmethod
    def from_engine(cls, engine) -> "ShardedCLIP":
        """The real thing: this rank's CUDA engine behind the sharding logic (NCCL process group already initialised)."""
        return cls(lambda x: engine.encode_images(x, normalize=True),
                   lambda ids: engine.encode_text(ids, normalize=True),
                   lambda a, b, s: engine.similarity(a, b, scale=s, normalize_image=False, normalize_text=False),
                   engine.logit_scale_exp,
                   topk=lambda q, sp, k: engine.similarity_topk(q, sp, k, scale=1.0, normalize_query=False,
                                                                normalize_space=False),
                   encode_pair=lambda x, ids: engine.encode_pair(x, ids, normalize=True))

    def clip_forward(self, local_pixels, local_ids):
        """``CLIPModel.forward`` over a batch sharded across the ranks (TF:867-944): returns this rank's row block
        ``logits_per_image[n_local, n_text_total]``.  The text embeddings travel (async all-gather on NCCL's stream)
        while the vision tower runs, so the exchange and any skew between ranks hide behind ~9 ms of compute.  On one
        rank with both inputs single tensors, the two towers run side by side (``encode_pair``) when available."""
        if self.world_size == 1 and self.encode_pair is not None and torch.is_tensor(local_pixels) \
                and torch.is_tensor(local_ids):
            img, txt = self.encode_pair(local_pixels, local_ids)
            return self.similarity(img, txt, self.logit_scale_exp)
        txt = self.encode_text(local_ids)
        txt_all, work = all_gather_rows_async(txt)
        img = _encode_chunks(self.encode_images, local_pixels)
        if work is not None:
            work.wait()
        return self.similarity(img, txt_all, self.logit_scale_exp)

    def local_slice(self, n_total: int) -> slice:
        lo, hi = shard_range(n_total, self.rank, self.world_size)
        return slice(lo, hi)

    def zero_shot(self, local_images, class_token_ids, n_total_images: int, gather_embeddings: bool = True):
        """cfg4: images sharded, class prompts replicated (64 x 77 ids: cheaper to recompute than to ship).
        Returns ``(pred_local [n_local], logits_local [n_local, n_classes], image_embeds_all or None)``."""
        txt = self.encode_text(class_token_ids)                      # replicated
        img = _encode_chunks(self.encode_images, local_images)       # this rank's block
        logits = self.similarity(img, txt, self.logit_scale_exp)     # [n_local, n_classes]
        pred = logits.argmax(dim=-1)
        all_img = None
        if gather_embeddings:
            all_img = all_gather_rows(img, shard_counts(n_total_images, self.world_size))
        return pred, logits, all_img

    def retrieval(self, local_gallery_images, local_query_ids, n_total_queries: int):
        """cfg5: gallery and queries sharded; query embeddings are all-gathered (small: 10k x 512 fp32 =
        20.5 MB), the gallery stays sharded and each rank returns its row block of the
        ``[n_gallery, n_queries]`` similarity matrix."""
        q_local = self.encode_text(local_query_ids)                  # queries first: their exchange overlaps the gallery
        counts = shard_counts(n_total_queries, self.world_size)
        if self.world_size > 1 and len(set(counts)) == 1:
            q_all, work = all_gather_rows_async(q_local)
            gal = _encode_chunks(self.encode_images, local_gallery_images)
            work.wait()
        else:
            gal = _encode_chunks(self.encode_images, local_gallery_images)
            q_all = all_gather_rows(q_local, counts)
        block = self.similarity(gal, q_all, self.logit_scale_exp)    # [n_gallery_local, n_queries]
        return block, gal, q_all

    def retrieval_topk(self, gal_local: torch.Tensor, q_all: torch.Tensor, k: int, n_total_gallery: int):
        """The reference's retrieval head over the SHARDED gallery (``retrieval.py:13-16``: per text query,
        ``argsort()[-k:][::-1]`` over all images): every rank takes the fused top-k of all queries over its own
        gallery rows (never materialising ``[n_queries, n_gallery]``), the ``[n_queries, k]`` candidates (score +
        global image index) are all-gathered (8 x 10k x 50 x 8 B = 32 MB at cfg5) and merged.  Ties resolve to the
        lower global index.  The result equals the one-GPU result bit for bit when every shard takes the path the
        whole gallery takes (``plip_similarity_topk``: the tensor-core chunks for >= 256 queries and >= 8192 rows);
        a shard below that runs the fp32 kernels, whose scores differ in the last bits, so near-ties may then
        resolve differently than on one GPU (every score stays within its kernel's bound).  Returns ``(idx int64 [n_queries,k], val [n_queries,k])`` on every rank."""
        if self.topk is None:
            raise RuntimeError("ShardedCLIP was built without a top-k kernel")
        idx, val = self.topk(q_all, gal_local, k)                    # local candidates, descending
        lo, _ = shard_range(n_total_gallery, self.rank, self.world_size)
        gidx = idx.to(torch.int64) + lo
        gidx = torch.where(idx < 0, torch.full_like(gidx, -1), gidx)
        if self.world_size == 1:
            return gidx, val
        nq = q_all.shape[0]
        cand_v = all_gather_rows(val.contiguous()).view(self.world_size, nq, k).permute(1, 0, 2).reshape(nq, -1)
        cand_i = all_gather_rows(gidx.contiguous()).view(self.world_size, nq, k).permute(1, 0, 2).reshape(nq, -1)
        return merge_topk_candidates(cand_i, cand_v, k)
