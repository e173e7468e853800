"""Prefix caching: requests whose prompts share a prefix share its KV pages.

``PrefixCache`` is one radix tree per model over token ids, at page granularity.  A node holds the tokens of one page
and that page's id in every layer's pool; a child is either full (``page_size`` tokens) or partial (fewer, always a
leaf).  Full pages chain from position 0, so a node's K/V is valid only under its exact ancestry.  K/V computed under
one LoRA adapter is wrong under another, so the tree has one root per adapter id (-1: the base model): a lookup under
one adapter never sees pages indexed under another.

* ``lookup(prompt)`` walks full pages by exact match and, where the prompt leaves the tree, picks the child (full or
  partial) with the longest common token prefix ``r``: its first ``r`` slots are copied on write into a private page.
  The reused length is capped at ``n - 1``: the last prompt token is always recomputed, since its logits give the first
  generated token.
* ``adopt(match, caches)`` hands the shared pages to a fresh request (``TinyKvPagedCache.adopt_prefix``) and copies the
  partly shared page of every layer in one ``paged_cache_copy_prefix`` launch.  The request then prefills from the
  reused length.
* ``insert(prompt, caches)``, once the prompt is prefilled, indexes its full pages and its partial tail page with the
  tail's length.  Only prompt tokens are indexed.  Where a node with the same tokens already exists under other pages,
  the existing node stays, the request's page stays private, and nothing deeper is indexed: so every request holding
  an indexed page holds that page's whole ancestry, and an index-only node never has a request-held descendant.

The index holds one reference on each of its pages (``TinyKvPagedPool.extra_refs``).  Pages no request holds are
evicted least recently used, leaves first, when a pool runs out of free pages; until then they use only the slack of
the pool's slab.
"""

from __future__ import annotations

from dataclasses import dataclass, field

from .paged_kv_cache import adopt_with_copies, copy_pages


class _Node:
    __slots__ = ("parent", "tokens", "pages", "children", "last_used")

    def __init__(self, parent, tokens: tuple, pages: list[int] | None, tick: int):
        self.parent = parent
        self.tokens = tokens
        self.pages = pages
        self.children: dict[tuple, _Node] = {}
        self.last_used = tick


@dataclass
class PrefixMatch:
    """What ``lookup`` found: ``shared`` full-page nodes from position 0, then optionally ``cow``, a node whose first
    ``cow_slots`` slots are copied.  ``reused`` = ``page_size * len(shared) + cow_slots``."""

    shared: list = field(default_factory=list)
    cow: _Node | None = None
    cow_slots: int = 0
    reused: int = 0


def _common_prefix(a, b) -> int:
    n = min(len(a), len(b))
    i = 0
    while i < n and a[i] == b[i]:
        i += 1
    return i


class PrefixCache:
    """The prefix index over one model's per-layer page pools (module docstring)."""

    def __init__(self, pools):
        if not pools:
            raise ValueError("a prefix cache needs the model's page pools")
        for pool in pools:
            if pool.prefix_index is not None:
                raise ValueError("a page pool already has a prefix cache")
        self.pools = list(pools)
        self.page_size = pools[0].page_size
        self._root = _Node(None, (), None, 0)
        self._roots = {-1: self._root}  # adapter id -> root of its subtree
        self._nodes: set[_Node] = set()
        self._tick = 0
        self.lookups = self.hits = self.reused_tokens = 0
        self.cow_copies = self.cow_slots = self.evictions = 0
        for pool in pools:
            pool.prefix_index = self

    def _touch(self, node: _Node) -> None:
        self._tick += 1
        node.last_used = self._tick

    def _held(self, node: _Node) -> bool:
        """Whether a request holds the node's pages (layer 0 stands for all: requests hold every layer of a page)."""
        return self.pools[0].extra_refs.get(node.pages[0], 0) > 0

    # ---- lookup and adoption -------------------------------------------------------
    def _root_of(self, adapter: int) -> _Node:
        root = self._roots.get(adapter)
        if root is None:
            root = self._roots[adapter] = _Node(None, (), None, 0)
        return root

    def lookup(self, prompt_ids, adapter: int = -1) -> PrefixMatch:
        ids = [int(t) for t in prompt_ids]
        P, cap = self.page_size, len(ids) - 1
        self.lookups += 1
        match = PrefixMatch()
        node, pos = self._root_of(adapter), 0
        while pos + P <= cap:
            child = node.children.get(tuple(ids[pos : pos + P]))
            if child is None:
                break
            match.shared.append(child)
            node, pos = child, pos + P
        limit = min(P, cap - pos)
        if limit > 0:
            want = ids[pos : pos + limit]
            for child in node.children.values():
                r = _common_prefix(child.tokens, want)
                if r > match.cow_slots:
                    match.cow, match.cow_slots = child, r
        match.reused = pos + match.cow_slots
        for n in match.shared:
            self._touch(n)
        if match.cow is not None:
            self._touch(match.cow)
        return match

    def adopt(self, match: PrefixMatch, caches) -> int:
        """Give the fresh request ``caches`` (one per layer) the matched prefix: shared references on the full pages
        and, per layer, a private copy of the first ``cow_slots`` slots of the partly matched page, all layers in one
        copy launch.  Returns the reused length, the offset the request prefills from."""
        if match.reused == 0:
            return 0
        cow = match.cow
        if cow is not None:  # pinned while the destinations are allocated, so no eviction can take the source
            for layer, pool in enumerate(self.pools):
                pool.share_page(cow.pages[layer])
        try:
            copies = []
            pages = [[n.pages[layer] for n in match.shared] for layer in range(len(caches))]
            tails = [None if cow is None else cow.pages[layer] for layer in range(len(caches))]
            adopt_with_copies(caches, pages, match.reused, tails, copies)
            copy_pages(self.pools, copies)
        finally:
            if cow is not None:  # the copy is enqueued ahead of every later write to the source page
                for layer, pool in enumerate(self.pools):
                    pool.free_page(cow.pages[layer])
        self.hits += 1
        self.reused_tokens += match.reused
        if cow is not None:
            self.cow_copies += 1
            self.cow_slots += match.cow_slots
        return match.reused

    # ---- insertion -----------------------------------------------------------------
    def insert(self, prompt_ids, caches, adapter: int = -1) -> int:
        """Index the prompt's pages from the request's ``caches`` (prefilled through the whole prompt under ``adapter``).
        Returns the number of nodes added."""
        ids = [int(t) for t in prompt_ids]
        P = self.page_size
        if caches[0].offset < len(ids):
            raise ValueError("insert needs the whole prompt prefilled")
        node, pos, added = self._root_of(adapter), 0, 0
        for index in range(-(-len(ids) // P)):
            key = tuple(ids[pos : pos + P])
            pages = [c.page_ids[index] for c in caches]
            child = node.children.get(key)
            if child is not None:
                if child.pages != pages:
                    break  # a duplicate: the existing node stays, the request's page stays private
                self._touch(child)
            else:
                child = _Node(node, key, pages, 0)
                self._touch(child)
                for pool, page_id in zip(self.pools, pages):
                    pool.share_page(page_id)
                    pool.indexed[page_id] = len(key)
                node.children[key] = child
                self._nodes.add(child)
                added += 1
            node, pos = child, pos + P
        return added

    # ---- eviction ------------------------------------------------------------------
    def _drop(self, node: _Node) -> None:
        del node.parent.children[node.tokens]
        self._nodes.discard(node)
        for pool, page_id in zip(self.pools, node.pages):
            del pool.indexed[page_id]
            pool.free_page(page_id)

    def evictable_pages(self) -> int:
        """Pages per layer that eviction can free: the nodes no request holds (their descendants are unheld too)."""
        return sum(1 for n in self._nodes if not self._held(n))

    def evict_one(self) -> bool:
        """Free the least recently used leaf no request holds (its page in every layer).  False if there is none."""
        victim = None
        for n in self._nodes:
            if not n.children and not self._held(n) and (victim is None or n.last_used < victim.last_used):
                victim = n
        if victim is None:
            return False
        self._drop(victim)
        self.evictions += 1
        return True

    def clear(self) -> None:
        """Drop the index's reference on every page: pages no request holds go back to their pools."""
        stack = [n for root in self._roots.values() for n in root.children.values()]
        order = []
        while stack:
            n = stack.pop()
            order.append(n)
            stack.extend(n.children.values())
        for n in reversed(order):  # children before parents
            self._drop(n)

    def stats(self) -> dict:
        return {
            "lookups": self.lookups,
            "hits": self.hits,
            "reused_tokens": self.reused_tokens,
            "cow_copies": self.cow_copies,
            "cow_slots": self.cow_slots,
            "evictions": self.evictions,
            "cached_pages": len(self._nodes),  # per layer
        }
