"""Shared prompt prefixes for continuous batching: a radix tree over token ids whose nodes hold the fp16 post-RoPE K / V
of their span for every layer, so that an insert whose prompt starts with tokens the server has already run computes only
the rest (LlamaForCausalLM_KIVI.insert(seq, ids, prefix_cache)).

K / V at positions 0 .. r - 1 depend on the tokens 0 .. r - 1 only -- not on the slot, the shared length or what follows
-- so a stored prefix stays valid for every later prompt that starts with it.  A node's storage is one tensor
[layers, 2, Hkv, span, 128] (K then V).  A prompt that diverges inside a node splits it into two views of that storage,
which counts in full until both halves are gone; `stored_bytes` is therefore a bound on the memory the tree holds, and
it never exceeds `max_bytes`.  When a new span does not fit, the least recently used leaves are evicted first, never a node on the
path of the insert in progress; a span that does not fit even then is not stored.  A block is charged the most that
PyTorch's caching allocator can hand out for it (`charge`), computed from its size alone.  "Recently" is a use counter
bumped once per operation, and every decision depends on token ids, that counter and the model's shapes only -- never on
a clock or on the allocator's state -- so tensor-parallel ranks that see the same prompts decide the same way.

The tree itself runs no kernel: it slices, copies and allocates tensors on the device it is bound to (CPU tensors in the
CPU tests).  Nodes hold no reference to their parent, so a dropped cache frees its memory at once."""
from __future__ import annotations

import weakref
from typing import NamedTuple

import torch

# The shortest stored prefix an insert reuses; below it the insert runs the whole prompt, as without a cache.  The suffix
# pass runs the prompt-attention kernel where the whole prompt would run SDPA's faster flash kernel, a cost that grows with
# the prompt, while r reused tokens save r / n of the weight GEMMs.  On an H100 (tools/prefix_bench.py, DESIGN.md "Prefix
# reuse in continuous batching") a 8192-token prompt breaks even at r = 1024 and loses 4-12 % at r = 64 .. 512, while
# shorter prompts already gain from r = 256.
MIN_REUSE = 1024


def charge(nbytes: int) -> int:
    """The bytes a stored block of `nbytes` counts: the most torch.cuda.memory_allocated can grow by when PyTorch's caching
    allocator (its default configuration) serves the request.  It rounds a request up to 512 bytes, and serves a
    request over 1 MiB from its large pool without splitting off a remainder of 1 MiB or less, so such a block may hold
    up to 1 MiB more.  Charging that bound makes max_bytes bound the memory the tree holds, whatever the pool's state."""
    rounded = -(-nbytes // 512) * 512
    return rounded + (1 << 20) if rounded > (1 << 20) else rounded


def reuse_length(matched: int, n: int) -> int:
    """The number of leading tokens an insert of an n-token prompt takes from the tree when `matched` of them are stored:
    at most n - 1 (the last position is always computed: its logits start the sequence), and 0 below MIN_REUSE."""
    r = min(matched, n - 1)
    return r if r >= MIN_REUSE else 0


class _Block:
    """One allocation of K / V, shared by the nodes a split made of it; it counts until the last of them is freed."""
    __slots__ = ("nbytes", "refs")

    def __init__(self, nbytes: int):
        self.nbytes, self.refs = nbytes, 1


class _Node:
    __slots__ = ("tokens", "kv", "block", "children", "used", "serial")

    def __init__(self, tokens, kv, block, used, serial):
        self.tokens, self.kv, self.block = tokens, kv, block
        self.children: dict[int, _Node] = {}
        self.used, self.serial = used, serial


class Match(NamedTuple):
    """The longest stored prefix of a prompt: `length` tokens along `path`, a list of (node, tokens taken from it) from
    the root down; only the last node may be taken in part."""
    length: int
    path: list


class PrefixCache:
    """A radix tree of prompt prefixes' K / V within `max_bytes` bytes of device memory (see the module docstring).

    Counters: `hits` (inserts that reused a prefix), `reused_tokens` (their reused tokens, summed), `stored_bytes` (the
    storage held now), `peak_bytes` (its maximum) and `evictions` (nodes evicted).  The cache binds to the first model
    that uses it (bind); the caller owns it, so it may outlive serve() calls."""

    def __init__(self, max_bytes: int):
        if int(max_bytes) < 0:
            raise ValueError(f"max_bytes must be >= 0, got {max_bytes}")
        self.max_bytes = int(max_bytes)
        self.hits = self.reused_tokens = self.stored_bytes = self.peak_bytes = self.evictions = 0
        self._root = _Node((), None, None, 0, 0)
        self._clock = 0
        self._serial = 0
        self._owner = None
        self.layers = self.kv_heads = self.device = None

    # ------------------------------------------------------------------ binding
    def bind(self, owner, layers: int, kv_heads: int, device):
        """Tie the cache to the model `owner` with `layers` layers and `kv_heads` KV heads (of its rank) on `device`; a
        later call with another model or other shapes raises ValueError (its K / V would not be this model's)."""
        device = torch.device(device)
        if self._owner is None:
            self._owner = weakref.ref(owner)
            self.layers, self.kv_heads, self.device = int(layers), int(kv_heads), device
            return
        if self._owner() is not owner or (self.layers, self.kv_heads, self.device) != (layers, kv_heads, device):
            raise ValueError(f"this PrefixCache holds the K / V of another model ({self.layers} layers, {self.kv_heads} "
                             f"KV heads on {self.device}): use one cache per model")

    def span_bytes(self, tokens: int) -> int:
        """The bytes of `tokens` stored tokens: layers * 2 * Hkv * 128 fp16 values each."""
        return self.layers * 2 * self.kv_heads * 128 * 2 * tokens

    # ------------------------------------------------------------------ lookup
    def match(self, tokens) -> Match:
        """The longest stored prefix of `tokens` (a sequence of ints).  Changes nothing."""
        node, pos, path = self._root, 0, []
        while pos < len(tokens):
            child = node.children.get(tokens[pos])
            if child is None:
                break
            take, span = 0, min(len(child.tokens), len(tokens) - pos)
            while take < span and child.tokens[take] == tokens[pos + take]:
                take += 1
            path.append((child, take))
            pos += take
            if take < len(child.tokens):
                break
            node = child
        return Match(pos, path)

    def copy_prefix(self, match: Match, r: int, layer: int, k_out, v_out):
        """Copy layer `layer`'s K and V of the first r matched tokens into k_out / v_out [Hkv, >= r, 128]."""
        pos = 0
        for node, take in match.path:
            take = min(take, r - pos)
            if take <= 0:
                break
            k_out[:, pos:pos + take].copy_(node.kv[layer, 0, :, :take])
            v_out[:, pos:pos + take].copy_(node.kv[layer, 1, :, :take])
            pos += take

    # ------------------------------------------------------------------ insertion
    def reserve(self, match: Match, tokens: int):
        """Room for `tokens` new tokens after `match`: evict least recently used leaves off the match's path until they
        fit, then allocate their storage [layers, 2, Hkv, tokens, 128] fp16.  Returns it, or None when nothing is to be
        stored or it does not fit (nothing is added; leaves evicted on the way stay evicted)."""
        need = charge(self.span_bytes(tokens))
        if tokens <= 0 or need > self.max_bytes:
            return None
        if not self._make_room(need, {id(node) for node, _ in match.path}):
            return None
        return torch.empty((self.layers, 2, self.kv_heads, tokens, 128), dtype=torch.float16, device=self.device)

    def _make_room(self, nbytes: int, keep) -> bool:
        """Evict least recently used leaves outside `keep` until nbytes more fit; False if they cannot."""
        while self.stored_bytes + nbytes > self.max_bytes:
            leaf = self._lru_leaf(keep)
            if leaf is None:
                return False
            self._evict(*leaf)
        return True

    def insert(self, tokens, match: Match, storage=None):
        """Record an insert of `tokens` that matched `match`: every node of its path counts as used now, and with
        `storage` (reserve()'s tensor, filled with the K / V of tokens[match.length:]) those tokens become a new leaf --
        splitting the last node of the path where the prompt diverges inside it."""
        self._clock += 1
        parent = self._root
        for node, take in match.path:
            if take < len(node.tokens):
                if storage is None:
                    node.used = self._clock
                    break
                node = self._split(parent, node, take)
            node.used = self._clock
            parent = node
        if storage is None:
            return
        assert storage.shape[3] == len(tokens) - match.length
        self._serial += 1
        leaf = _Node(tuple(tokens[match.length:]), storage, _Block(charge(storage.numel() * storage.element_size())),
                     self._clock, self._serial)
        parent.children[leaf.tokens[0]] = leaf
        self.stored_bytes += leaf.block.nbytes
        self.peak_bytes = max(self.peak_bytes, self.stored_bytes)

    def _split(self, parent, node, at: int):
        """Cut `node` (a child of `parent`) after `at` tokens: a new head node (the first `at` tokens) takes its place
        under `parent`, and `node` keeps the rest under the head.  Both are views of the one block."""
        self._serial += 1
        head = _Node(node.tokens[:at], node.kv[:, :, :, :at], node.block, node.used, self._serial)
        parent.children[head.tokens[0]] = head
        node.tokens, node.kv = node.tokens[at:], node.kv[:, :, :, at:]
        head.children[node.tokens[0]] = node
        node.block.refs += 1
        return head

    # ------------------------------------------------------------------ eviction
    def _edges(self):
        """(parent, node) for every node below the root."""
        stack = [(self._root, c) for c in self._root.children.values()]
        while stack:
            parent, node = stack.pop()
            yield parent, node
            stack.extend((node, c) for c in node.children.values())

    def _nodes(self):
        return (node for _, node in self._edges())

    def _lru_leaf(self, keep):
        """(parent, leaf) of the least recently used leaf not in `keep` (ids), oldest serial first among equals; None
        if there is none."""
        leaves = [(p, nd) for p, nd in self._edges() if not nd.children and id(nd) not in keep]
        return min(leaves, key=lambda e: (e[1].used, e[1].serial), default=None)

    def _evict(self, parent, node):
        del parent.children[node.tokens[0]]
        node.block.refs -= 1
        if node.block.refs == 0:
            self.stored_bytes -= node.block.nbytes
        node.kv = None
        self.evictions += 1

    def __len__(self):
        """The number of nodes."""
        return sum(1 for _ in self._edges())
