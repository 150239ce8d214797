"""An exact reference for the equi-join and the semi-join, in plain Python over host Pages: a dictionary from key tuples to build
positions.  It shares no code with the library and none with oracle/oracle.cpp (no row hash, no table), so it pins what the hash
tables must compute, whatever their layout:

* a row joins only when no key channel is NULL and no DOUBLE / REAL key channel is NaN; DOUBLE / REAL compare by value (-0.0 == 0.0),
  VARCHAR by its bytes, long DECIMAL and the integer types as integers (EQUAL: M/operator/SimplePagesHashStrategy.java:194-260);
* the build positions of one key form a chain in DESCENDING position order: the head is the last row, links lead to lower positions
  (M/operator/join/ArrayPositionLinks.java:45-50);
* LookupJoinOperator emits, per probe row in order, one row per chain position (the head only with outputSingleMatch), or one row
  with a NULL build side when nothing matched and the join is PROBE_OUTER / FULL_OUTER (M/operator/join/PageJoiner.java:203-242);
* the LookupOuterOperator returns the build positions no probe emitted, ascending (M/operator/join/OuterLookupSource.java:109-139);
* HashSemiJoinOperator.java:155-201 answers TRUE / FALSE / NULL; its ChannelSet compares with IDENTICAL, so over DOUBLE / REAL every
  NaN is one member of the set (M/operator/FlatSet.java:54,374).
"""
import numpy as np

from trino_b200 import abi
from trino_b200.page import Page

_NAN = "NaN"        # the one member every NaN is under IDENTICAL


def channel_values(block, identical=False):
    """One hashable Python value per row of a key channel; None where the row cannot join through this channel (NULL, and NaN unless
    `identical`, where every NaN becomes one value)."""
    b = block.flatten()
    n = b.position_count
    if b.type == abi.UTF8:
        data, offs = b.values.tobytes(), b.offsets.tolist()
        vals = [data[offs[i]:offs[i + 1]] for i in range(n)]
    elif b.type == abi.INT128:
        vals = [(int(h) << 64) | (int(l) & ((1 << 64) - 1)) for h, l in b.values.tolist()]
    elif b.type == abi.FLOAT32:
        with np.errstate(invalid="ignore"):         # (widening a signalling NaN)
            vals = np.asarray(b.values, dtype=np.float32).astype(np.float64).tolist()      # REAL: the float32 value, exactly
    else:
        vals = b.values.tolist()
    if b.type in (abi.FLOAT64, abi.FLOAT32):
        vals = [(_NAN if identical else None) if v != v else v for v in vals]           # -0.0 == 0.0 and hash(-0.0) == hash(0.0)
    if b.nulls is not None:
        vals = [None if z else v for v, z in zip(vals, b.nulls.tolist())]
    return vals


def keys_of(page, channels):
    """key tuple per row, None for a row that cannot join"""
    cols = [channel_values(page.get_block(c)) for c in channels]
    return [None if any(v is None for v in row) else row for row in zip(*cols)]


def key_of(page, channels, row):
    return keys_of(page, channels)[row]


class JoinReference:
    def __init__(self, build_pages, key_channels):
        """build_pages: the pages of the build side in arrival order (positions run on across pages), or one Page"""
        pages = [build_pages] if isinstance(build_pages, Page) else list(build_pages)
        self.key_channels = list(key_channels)
        self.chains = {}                    # key -> build positions, ascending while building
        self.position_count = 0
        for page in pages:
            for key in keys_of(page, self.key_channels):
                if key is not None:
                    self.chains.setdefault(key, []).append(self.position_count)
                self.position_count += 1
        self._links = [-1] * self.position_count
        for chain in self.chains.values():
            chain.reverse()                 # descending: head first
            for a, b in zip(chain, chain[1:]):
                self._links[a] = b

    def positions(self, probe_page, key_channels):
        """head of the probe row's chain, or -1"""
        chains = self.chains
        out = [-1 if key is None or key not in chains else chains[key][0] for key in keys_of(probe_page, key_channels)]
        return np.array(out, dtype=np.int32).reshape(-1)

    def links(self):
        return np.array(self._links, dtype=np.int32).reshape(-1)

    def has_links(self):
        return any(len(c) > 1 for c in self.chains.values())

    def expand(self, positions, join_type, single_match):
        """(probe rows, build positions) of the operator's output rows in order; build position -1 = NULL build side"""
        outer = join_type in (abi.JOIN_PROBE_OUTER, abi.JOIN_FULL_OUTER)
        links = self._links
        out_probe, out_build = [], []
        for i, pos in enumerate(np.asarray(positions).tolist()):
            if pos < 0:
                if outer:
                    out_probe.append(i)
                    out_build.append(-1)
                continue
            while pos >= 0:
                out_probe.append(i)
                out_build.append(pos)
                pos = -1 if single_match else links[pos]
        return np.array(out_probe, dtype=np.int32).reshape(-1), np.array(out_build, dtype=np.int32).reshape(-1)

    def unvisited(self, emitted_build_positions):
        """build positions the LookupOuterOperator returns after probes that emitted these build positions (arrays, one per page)"""
        visited = np.zeros(self.position_count, dtype=bool)
        for b in emitted_build_positions:
            b = np.asarray(b)
            visited[b[b >= 0]] = True
        return np.nonzero(~visited)[0].astype(np.int32)


def semi(set_block, probe_block):
    """The BOOLEAN channel HashSemiJoinOperator appends: True / False / None per probe row"""
    members = channel_values(set_block, identical=True)
    has_null = any(v is None for v in members)
    values = {v for v in members if v is not None}
    empty = not members
    out = []
    for v in channel_values(probe_block, identical=True):
        if v is None:
            out.append(False if empty else None)        # a NULL probe key is unknown, unless there is nothing to compare with
        elif v in values:
            out.append(True)
        else:
            out.append(None if has_null else False)
    return out
