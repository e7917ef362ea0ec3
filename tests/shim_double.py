"""The C test double of the Go shim (integration/shim_double.c) as a backend of tests/scenario.py: it replays, per
verb, the C calls the shim makes against libegs.so."""
import subprocess

from oracle_harness import egs


def build_double() -> str:
    return egs()._build.build_shim_double()


def _req(shape):
    """GPUUnit -> the (gpu-core, gpu-memory) requests NewGPURequest maps to it (allocate.go:38-53)."""
    out = []
    for core, mem, cnt in shape:
        if cnt > 0:
            out += [100 * cnt, 0]
        elif core == -1:
            out += [0, 0]
        else:
            out += [core, mem]
    return f"{len(shape)} " + " ".join(str(x) for x in out)


class ShimDoubleBackend:
    """A scenario backend (tests/scenario.py) over the double's line protocol.  g_max, when given, is the widest node
    (the double's second argument); the double prints each mask as one integer of up to 16 bits."""

    def __init__(self, policy, g_max=None):
        args = [build_double(), str(policy)] + ([str(g_max)] if g_max else [])
        self.p = subprocess.Popen(args, stdin=subprocess.PIPE, stdout=subprocess.PIPE, text=True)
        self.n = 0
        self.g = {}

    def close(self):
        self.p.stdin.close()
        self.p.wait(timeout=20)

    def _ask(self, line):
        self.p.stdin.write(line + "\n")
        self.p.stdin.flush()
        return self.p.stdout.readline().split()

    def add_node(self, core_alloc, mem_alloc):
        st = int(self._ask(f"NODE n{self.n} {core_alloc} {mem_alloc}")[1])
        if st != 0:
            return -1
        self.g[self.n] = core_alloc // 100
        self.n += 1
        return self.n - 1

    def set_rows(self, node, core, mem):
        assert self._ask(f"ROWS n{node} {len(core)} " + " ".join(map(str, list(core) + list(mem))))[1] == "0"

    def rows(self, node):
        for ent in self._ask("STATUS")[1:]:
            name, *gp = ent.split(":")
            if name == f"n{node}":
                return [tuple(int(x) for x in g.split(",")) for g in gp]
        return []

    def filter(self, ids, shape):
        return [int(c) for c in self._ask(f"ASSUME {_req(shape)} | " + " ".join(f"n{i}" for i in ids))[1]]

    def score(self, ids, shape):
        a = self._ask(f"SCORE {_req(shape)} | " + " ".join(f"n{i}" for i in ids))
        return (9 if a[0] == "SCORE!" else 0), [int(x) for x in a[1:]]

    @staticmethod
    def _lists(masks):
        return [[g for g in range(16) if m >> g & 1] for m in masks]

    def bind(self, node, shape, uid):
        a = self._ask(f"BIND {uid} n{node} {_req(shape)}")
        st = int(a[1])
        return st, (self._lists([int(x) for x in a[2:]]) if st == 0 else None)

    def peek(self, node, shape):
        a = self._ask(f"PEEK n{node} {_req(shape)}")
        if a[1] == "0":
            return None
        return self._lists([int(x) for x in a[3:]]), int(a[2])

    def _alloc(self, shape, alloc):
        parts = [str(len(shape))]
        for (core, mem, cnt), ids in zip(shape, alloc):
            c, m = (100 * cnt, 0) if cnt > 0 else (0, 0) if core == -1 else (core, mem)
            parts += [str(c), str(m), str(len(ids or []))] + [str(i) for i in (ids or [])]
        return " ".join(parts)

    def add_pod(self, node, shape, alloc, uid):
        self._ask(f"ADD {uid} n{node} {self._alloc(shape, alloc)}")

    def forget_pod(self, node, shape, alloc, uid):
        self._ask(f"FORGET {uid} n{node} {self._alloc(shape, alloc)}")

    def known(self, uid):
        return self._ask(f"KNOWN {uid}")[1] == "1"

    def released(self, uid):
        return self._ask(f"RELEASED {uid}")[1] == "1"
