"""greedy_decode (Codebook/AudiocaptionLoss/tools/utils.py) and beam_decode (tools/beam.py) on the caption engine.

beam_decode keeps the reference's best-first search exactly: each clip has its own heap of (score, node) on the host, ordered as the reference's
PriorityQueue orders it (score, then BeamSearchNode.__lt__ on logp), with the score -logp / (leng - 1 + 1e-6) in Python floats from the fp32
log-probs, the qsize > 2000 cut-off, endnodes and top_k.  The clips are independent, so instead of one clip at a time each round pops the next
node of every unfinished clip and expands all of them in one GPU step; the output equals running the reference clip by clip.  Where the
reference re-runs the decoder over a node's whole prefix, the engine keeps every expanded node's K / V in a slot pool and attends over the slots
of its ancestor path."""
from __future__ import annotations

import heapq
import operator
from typing import Callable, List, Sequence, Tuple

import torch
from torch.nn.utils.rnn import pad_sequence

QUEUE_CAP = 2000  # beam.py: `if qsize > 2000: break`


class BeamSearchNode(object):
    """beam.py's node: wordid here is the node's last word (the prefix is the chain of prevNode words)."""

    def __init__(self, previousNode, wordId, logProb, length):
        self.prevNode = previousNode
        self.wordid = wordId
        self.logp = logProb
        self.leng = length
        self.slot = None  # engine bookkeeping: the K / V slot this node's expansion wrote
        self.path = None

    def __lt__(self, other):
        return self.logp < other.logp

    def eval(self, alpha=1.0):
        reward = 0
        return self.logp / float(self.leng - 1 + 1e-6) + alpha * reward

    def words(self) -> List[int]:
        out, n = [], self
        while n is not None:
            out.append(n.wordid)
            n = n.prevNode
        return out[::-1]


class _ClipSearch:
    __slots__ = ("nodes", "endnodes", "qsize", "done")

    def __init__(self, sos_ind):
        node = BeamSearchNode(None, sos_ind, 0, 1)
        self.nodes = [(-node.eval(), node)]
        self.endnodes = []
        self.qsize = 1
        self.done = False


def beam_search(expand: Callable[[Sequence[Tuple[int, BeamSearchNode]]], Tuple[Sequence[Sequence[float]], Sequence[Sequence[int]]]], n_clips: int,
                sos_ind: int, eos_ind: int, beam_width: int = 5, top_k: int = 1) -> List[List[int]]:
    """beam.py's search for n_clips independent clips.  expand(items), items a list of (clip, node) with at most one node per clip, returns the
    top beam_width (log-prob, word) of every item's next position, each row in descending order.  Returns top_k word lists per clip, clip-major."""
    number_required = min((top_k + 1), top_k)
    clips = [_ClipSearch(sos_ind) for _ in range(n_clips)]
    while True:
        items = []
        for c, st in enumerate(clips):
            while not st.done:
                if st.qsize > QUEUE_CAP:
                    st.done = True
                    break
                if not st.nodes:
                    raise RuntimeError("beam search: the queue ran empty before top_k sentences ended (the reference's PriorityQueue.get would block)")
                score, n = heapq.heappop(st.nodes)
                if n.wordid == eos_ind and n.prevNode is not None:
                    st.endnodes.append((score, n))
                    if len(st.endnodes) >= number_required:
                        st.done = True
                    continue
                items.append((c, n))
                break
        if not items:
            break
        logps, words = expand(items)
        for (c, n), lp, wd in zip(items, logps, words):
            st = clips[c]
            nextnodes = []
            for new_k in range(beam_width):
                node = BeamSearchNode(n, int(wd[new_k]), n.logp + float(lp[new_k]), n.leng + 1)
                nextnodes.append((-node.eval(), node))
            for i in range(len(nextnodes)):
                heapq.heappush(st.nodes, nextnodes[i])
            st.qsize += len(nextnodes) - 1
    decoded = []
    for st in clips:
        endnodes = st.endnodes if st.endnodes else [heapq.heappop(st.nodes) for _ in range(top_k)]
        utterances = [n.words() for score, n in sorted(endnodes, key=operator.itemgetter(0))]
        for i in range(top_k):
            decoded.append(utterances[i])
    return decoded


def _engine_of(model):
    from .models import _refuse_training
    _refuse_training(model)
    return model.engine


@torch.no_grad()
def greedy_decode(model, src, sos_ind=0, eos_ind=9, max_len=30):
    """tools/utils.py greedy_decode: (B, max_len + 1) int64 with ys[:, 0] = sos_ind and argmax(softmax(logits)) after it, no early stop."""
    model.eval()
    eng = _engine_of(model)
    return eng.greedy(eng.encode(src), sos_ind, max_len)


@torch.no_grad()
def beam_decode(x, model, sos_ind, eos_ind, beam_width=5, top_k=1):
    """tools/beam.py beam_decode: x (B, T, 80) -> the top_k sentences of every clip (clip-major), padded with eos_ind, int64 on x.device."""
    eng = _engine_of(model)
    seqs = eng.beam(eng.encode(x), sos_ind, eos_ind, beam_width, top_k)
    return pad_sequence([torch.tensor(s, dtype=torch.int64, device=x.device) for s in seqs], batch_first=True, padding_value=eos_ind)
