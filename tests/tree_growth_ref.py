"""Plain torch reference of draft-tree growth (the level loop of cnets.py:703-757 as restated by
oracle/eagle_oracle.py:topk_generate), driven by per-level top-k TABLES instead of draft forwards, so that the integer
kernels tree_seed / tree_expand (eb200_k_tree_grow) can be held to it bit for bit.

Two things differ from a literal transcription, both on purpose:
  * torch.topk leaves the order of equal values unspecified; the kernels document (value desc, flat index asc), so the
    frontier is selected with a STABLE descending sort;
  * everything is returned per level (frontier ids / source rows / flat indices / scores / dense ancestor mask), which the
    reference keeps only as loop variables.
cu_scores = topk_p + scores[:, None] is evaluated in the model dtype exactly like the oracle (cnets.py:740).

tests/test_tree_growth_cpu.py holds this file to the oracle; tests/test_tree_growth_gpu.py holds the kernels to this file.
"""
import torch
import torch.nn.functional as F


def stable_topk(flat: torch.Tensor, k: int):
    """Indices of the k largest values in (value desc, index asc) order."""
    return torch.sort(flat.double(), descending=True, stable=True).indices[:k]


def make_tables(k: int, depth: int, dtype, seed: int, draft_vocab: int = 512):
    """Seeded top-k tables [1 + depth*k, k]: log-softmax rows of random logits rounded to the model dtype (so cumulative
    scores tie naturally in bf16/fp16), each row's top-k in (value desc, index asc) order.  Returns (topk_p fp32, topk_i int32)."""
    g = torch.Generator().manual_seed(seed)
    rows = 1 + depth * k
    logp = F.log_softmax((torch.randn(rows, draft_vocab, generator=g) * 2).to(dtype), dim=-1)
    order = torch.sort(logp.double(), dim=-1, descending=True, stable=True).indices[:, :k]
    return torch.gather(logp, 1, order).float().contiguous(), order.int().contiguous()


def pack_mask(dense: torch.Tensor) -> torch.Tensor:
    """[k, cols] bool -> [k, 2] int64: bit c of word c // 64 (two's-complement view of the kernels' uint64 words).  The
    kernels keep 128 columns, all a draft forward ever attends over (depth * top_k <= 128); the frontier left by the LAST level
    has (depth + 1) * top_k columns, is never attended over, and its columns from 128 on (the level's own) are dropped."""
    out = []
    for row in dense.tolist():
        words = [0, 0]
        for c, bit in enumerate(row):
            if bit and c < 128:
                words[c // 64] |= 1 << (c % 64)
        out.append([w - (1 << 64) if w >= (1 << 63) else w for w in words])
    return torch.tensor(out, dtype=torch.int64)


def grow(topk_p: torch.Tensor, topk_i: torch.Tensor, d2t, k: int, depth: int, dtype, last_row: int = 0):
    """topk_p [1 + depth*k, k] (values representable in `dtype`), topk_i same shape (draft-vocab ids), d2t [Vd] int64 or None.
    Returns the pool (scores_flat fp32, tokens_flat int64, parents_flat int64) and `levels`: depth + 1 dicts, entry 0 after
    the seed, entry l + 1 after level l, each with ids / src / cs (int64 [k]), scores (fp32 [k]) and mask (bool [k, (l+2)*k])."""
    def to_target(idx):
        idx = idx.long()
        return idx + d2t[idx] if d2t is not None else idx

    p = topk_p.to(dtype)
    idx = topk_i.long()
    scores = p[0]
    scores_list = [scores[None]]
    parents_list = [torch.zeros(1, dtype=torch.long)]
    ss_token = [to_target(idx[:1])]
    tree_mask = torch.eye(k, dtype=torch.bool)
    tree_mask_init = tree_mask
    topk_cs_index = torch.arange(k)
    levels = [dict(ids=to_target(idx[0]), src=torch.full((k,), last_row, dtype=torch.long), cs=topk_cs_index.clone(),
                   scores=scores.float(), mask=tree_mask.clone())]
    for i in range(depth):
        bias = 1 + k ** 2 * max(0, i - 1) + (k if i > 0 else 0)
        parents_list.append(topk_cs_index + bias)
        lp, li = p[1 + i * k: 1 + (i + 1) * k], idx[1 + i * k: 1 + (i + 1) * k]
        cu_scores = lp + scores[:, None]  # model dtype
        flat = cu_scores.reshape(-1)
        topk_cs_index = stable_topk(flat, k)
        scores = flat[topk_cs_index]
        out_ids = topk_cs_index // k
        level_ids = to_target(li.reshape(-1)[topk_cs_index])
        ss_token.append(to_target(li))
        scores_list.append(cu_scores)
        tree_mask = torch.cat((tree_mask[out_ids], tree_mask_init), dim=1)
        levels.append(dict(ids=level_ids, src=out_ids.clone(), cs=topk_cs_index.clone(), scores=scores.float(), mask=tree_mask.clone()))
    scores_flat = torch.cat([s.reshape(-1) for s in scores_list]).float()
    tokens_flat = torch.cat([t.reshape(-1) for t in ss_token])
    parents_flat = torch.cat(parents_list)
    return scores_flat, tokens_flat, parents_flat, levels
