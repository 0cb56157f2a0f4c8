"""The oracle's generation cycle (OracleEaModel.eagenerate, oracle/eagle_oracle.py) split at its decisions, so a test can drive
it with decisions taken elsewhere.

`Shadow` keeps the oracle's target KV, draft stable KV and committed ids.  Per cycle the caller runs `verify` over a draft tree
(the engine's own, so the verify rows align one to one with the engine's), takes (best, accept_length, bonus) from wherever
it wants (the engine, or the oracle's own posterior as in tests/test_sampled_cycles_cpu.py), then `commit`s them: the KV is
compacted as update_inference_inputs does (utils.py:418-473) and the next draft tree is grown from the accepted features.
tests/test_sampled_cycles_cpu.py holds this restatement to OracleEaModel.eagenerate on the oracle's own decisions.
"""
from __future__ import annotations

import math

import torch

from oracle import eagle_oracle as orc


class Shadow:
    def __init__(self, ref: orc.OracleEaModel, sampling: bool = True):
        self.ref, self.sampling = ref, sampling
        self.kv = None
        self.ids = None
        self.tree = None  # (draft_tokens [1,T], retrieve, tree_mask [1,1,T,T], tree_pos [T]) grown by the oracle
        self.scores = None  # the dynamic tree's candidate pool: (scores_flat, top_k, total); None for a static tree
        self._feats = None

    def _grow(self, feats, ids):
        ref = self.ref
        ref.head.trace = {}
        self.tree = ref._tree(feats, ids, self.sampling)
        tr, ref.head.trace = ref.head.trace, None
        self.scores = (tr["scores_flat"], ref.head.top_k, ref.head.total_tokens) if "scores_flat" in tr else None
        self._feats = None

    def prefill(self, prompt: torch.Tensor, max_length: int) -> torch.Tensor:
        """Target prefill (utils.py:232-245); returns the last row's logits [V] (model dtype).  `first_token` follows."""
        ref = self.ref
        ref.head.reset_kv()
        self.kv = ref._kv(max_length)
        self.ids = prompt.clone()
        hidden, taps = ref.target.forward(prompt, self.kv)
        self._feats = ref._features(hidden, taps)
        return ref.target.lm_head(hidden)[0, -1]

    def first_token(self, token: int):
        """The first draft tree, rooted at the first token (utils.py:248-254)."""
        self._grow(self._feats, torch.cat((self.ids, torch.tensor([[int(token)]], dtype=torch.long)), dim=1))

    def verify(self, draft_tokens, tree_mask, tree_pos) -> torch.Tensor:
        """tree_decoding (utils.py:306-331) over the given tree: the verify logits [T, V] (model dtype), in node order."""
        ref = self.ref
        position_ids = tree_pos + self.ids.shape[1]
        hidden, taps = ref.target.forward(draft_tokens, self.kv, position_ids=position_ids[None], tree_mask=tree_mask)
        self._feats = ref._features(hidden, taps)
        return ref.target.lm_head(hidden)[0]

    def commit(self, draft_tokens, retrieve, best: int, accept_length: int, bonus: int):
        """update_inference_inputs (utils.py:418-473) with the given decisions, then the next draft tree."""
        a = int(accept_length)
        prev_len = self.ids.shape[1]
        cands = torch.cat((draft_tokens, torch.full((1, 1), -1, dtype=torch.long)), dim=1)[0, retrieve]
        select = retrieve[best, : a + 1] + prev_len
        self.ids = torch.cat([self.ids, cands[None, best, : a + 1]], dim=-1)
        self.kv.compact(select, prev_len)
        accept_feats = self._feats[:, retrieve][:, best, : a + 1]
        self._grow(accept_feats, torch.cat((self.ids, torch.tensor([[int(bonus)]], dtype=torch.long)), dim=1))
        return cands[best, : a + 1]


def tree_paths(draft_tokens, tree_mask):
    """Token path (root first) of every node: [T] tuples."""
    T = draft_tokens.shape[-1]
    toks = draft_tokens.reshape(-1).tolist()
    m = tree_mask.reshape(T, T)
    return [tuple(toks[j] for j in range(T) if m[i, j] > 0) for i in range(T)]


def certain_chain(draft_tokens, tree_mask, scores, margin: float):
    """The prefix of top_score_chain whose membership no rounding of the cumulative scores can change.  scores: Shadow.scores
    (None for a static tree, whose structure is fixed: the whole chain).  A chain node is kept while its cumulative score exceeds
    by `margin` both the best score left out of the tree (cnets.py:760: top total of the pool) and, for a node with children,
    the best score of its level that was not expanded (top_k beams per level, cnets.py:737-742)."""
    chain = top_score_chain(draft_tokens, tree_mask)
    if scores is None:
        return chain
    flat, k, total = scores
    order = torch.topk(flat, total + 1).values
    left_out = float(order[-1]) if flat.numel() > total else -math.inf
    top_idx = torch.sort(torch.topk(flat, total).indices).values
    T = draft_tokens.shape[-1]
    paths = tree_paths(draft_tokens, tree_mask)
    node_of = {p: i for i, p in enumerate(paths)}
    out = [chain[0]]
    for depth, path in enumerate(chain[1:], start=1):
        f = int(top_idx[node_of[path] - 1])
        s = float(flat[f])
        if s - left_out <= margin:
            break
        if depth < len(chain) - 1 and depth >= 1:  # this node was expanded: a beam of its level
            lo = 0 if f < k else k + ((f - k) // (k * k)) * k * k
            hi = k if f < k else lo + k * k
            level = flat[lo:hi]
            if level.numel() > k and s - float(torch.topk(level, k + 1).values[-1]) <= margin:
                out.append(path)
                break
        out.append(path)
    assert len(out) <= T
    return out


def top_score_chain(draft_tokens, tree_mask):
    """Token paths of the root and, level by level, of the first child of the previous chain node.  Within one parent the draft
    tree keeps its children in descending score order (cnets.py:760-785 sorts the selected flat indices, and each parent's
    children are one top-k block), so the first child is the parent's top-score child."""
    T = draft_tokens.shape[-1]
    m = tree_mask.reshape(T, T) > 0
    depth = m.sum(-1) - 1
    paths = tree_paths(draft_tokens, tree_mask)
    chain, node = [paths[0]], 0
    while True:
        kids = [i for i in range(node + 1, T) if m[i, node] and int(depth[i]) == int(depth[node]) + 1]
        if not kids:
            return chain
        node = kids[0]
        chain.append(paths[node])
