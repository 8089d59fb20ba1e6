"""A minimal `pqdict` (min-heap priority-queue dict) for running the reference's `pq_astar.solve_single` here.

ASSUMPTION: pqdict 1.2.0 is not available to this project, so its heap moves are restated from heapq, whose
algorithm pqdict's own code follows:
  * additem: append, then _swim: move the parent down while the node's priority is < the parent's;
  * popitem: take the root, move the last node to the root, then _sink it Floyd's way: walk the hole down to a leaf,
    taking the right child unless left < right, put the node there and _swim it up with a strict <;
  * __setitem__ on an existing key (_reheapify): swim when the new priority is < the parent's, else sink when the
    smaller child's priority is < the new one.  The reference only ever lowers a key, so it swims.
These moves decide every tie between equal priorities.  The only check against the real library is indirect: the
reference's own test asserts that its heap A* equals its differentiable A* on the 64x64 fixture
(tests/golden/fixture64_vanilla.npz), which upstream passes with the real pqdict, and this shim reproduces that output.

Only what solve_single uses: additem, popitem, __getitem__, __setitem__, __contains__, __len__ and keys.
"""
from __future__ import annotations


class _Node:
    __slots__ = ("key", "value")

    def __init__(self, key, value):
        self.key = key
        self.value = value


class pqdict:  # noqa: N801  the name the reference imports
    def __init__(self):
        self._heap = []
        self._position = {}

    def __len__(self):
        return len(self._heap)

    def __contains__(self, key):
        return key in self._position

    def __getitem__(self, key):
        return self._heap[self._position[key]].value

    def keys(self):
        return self._position.keys()

    def additem(self, key, value):
        if key in self._position:
            raise KeyError(f"{key!r} is already in the queue")
        self._heap.append(_Node(key, value))
        self._position[key] = len(self._heap) - 1
        self._swim(len(self._heap) - 1)

    def __setitem__(self, key, value):
        if key not in self._position:
            self.additem(key, value)
            return
        pos = self._position[key]
        self._heap[pos].value = value
        self._reheapify(pos)

    def popitem(self):
        heap = self._heap
        if not heap:
            raise KeyError("pqdict is empty")
        end = heap.pop(-1)
        if heap:
            node = heap[0]
            heap[0] = end
            self._position[end.key] = 0
            self._sink(0)
        else:
            node = end
        del self._position[node.key]
        return node.key, node.value

    def _reheapify(self, pos):
        heap = self._heap
        parent = (pos - 1) >> 1
        child = 2 * pos + 1
        if parent > -1 and heap[pos].value < heap[parent].value:
            self._swim(pos)
        elif child < len(heap):
            other = child + 1
            if other < len(heap) and not heap[child].value < heap[other].value:
                child = other
            if heap[child].value < heap[pos].value:
                self._sink(pos)

    def _sink(self, top=0):
        heap, position = self._heap, self._position
        pos = top
        node = heap[pos]
        child = 2 * pos + 1
        while child < len(heap):
            other = child + 1
            if other < len(heap) and not heap[child].value < heap[other].value:
                child = other
            heap[pos] = heap[child]
            position[heap[pos].key] = pos
            pos = child
            child = 2 * pos + 1
        heap[pos] = node
        position[node.key] = pos
        self._swim(pos, top)

    def _swim(self, pos, top=0):
        heap, position = self._heap, self._position
        node = heap[pos]
        while pos > top:
            parent = (pos - 1) >> 1
            if node.value < heap[parent].value:
                heap[pos] = heap[parent]
                position[heap[pos].key] = pos
                pos = parent
                continue
            break
        heap[pos] = node
        position[node.key] = pos
