"""set_lcas -a / -A restated in Python — TEST INFRASTRUCTURE ONLY.

What `krakenuniq-build --taxids-for-sequences --taxids-for-genomes` (build_db.sh: set_lcas -a -A) does to the
taxonomy, from the taxDB rows, the seqid2taxid.map lines and the library's FASTA records:

* ``Extension(rows, map_lines, add_sequences, add_assembly)``: the taxa read_seqid_to_taxid_map adds before any
  sequence is read (set_lcas.cpp:205-266, get_new_taxid :183-203), the seq id → taxid map and the stdout lines;
* ``Extension.assign(records, min_len)``: the taxid each record's k-mers get (process_single_file, :268-381) and the
  names the headers give taxa under -a (:344-353);
* ``Extension.taxdb_text()``: the taxDB the reference writes back (writeTaxonomyIndex, taxdb.hpp:533-547);
* ``Extension.parent_map()``: Parent_map with the new taxa, for the oracle's LCA.

Where new ids start depends on the iteration order of an unordered_map when the taxDB already holds ids
>= 1 000 000 000; such a taxDB is refused here."""
from __future__ import annotations

import re

import numpy as np

HUMAN, MOUSE = 9606, 10090
FIRST_NEW = 1_000_000_000
PREFIX = "kraken:taxid|"
_MAP_LINE = re.compile(r"^\s*(\S+)\s+(\d+)(.*)$", re.S)


class Extension:
    def __init__(self, rows, map_lines, add_sequences: bool, add_assembly: bool):
        # readTaxonomyIndex_ (taxdb.hpp:563-605): the first row of a taxid wins; taxid 0 'unclassified' is added;
        # a parent pointer exists when the parent is another taxon of the file (or 0)
        self.entries = {}
        for t, p, name, rank in rows:
            self.entries.setdefault(int(t), [int(p), name, rank])
        self.entries.setdefault(0, [0, "unclassified", "no rank"])
        for t, e in self.entries.items():
            e[0] = e[0] if (e[0] != t and e[0] in self.entries) else None
        self.add_sequences, self.add_assembly = add_sequences, add_assembly
        add = add_sequences or add_assembly
        if add and max(self.entries) >= FIRST_NEW:
            raise ValueError("the taxDB already holds new-style taxids: where new ids start depends on hash order")
        self.next_id = FIRST_NEW
        cache = {}

        def new_taxid(name, parent, rank):
            if name in cache:
                return cache[name]
            self.next_id += 1                                    # used up even when nothing is added
            if parent == self.next_id or parent not in self.entries:
                return 0
            self.entries[self.next_id] = [parent, name, rank]
            cache[name] = self.next_id
            return self.next_id

        self.seq_map, out = {}, []
        for line in map_lines:
            if not line:
                break
            m = _MAP_LINE.match(line)
            assert m, f"map line outside what this restatement parses: {line!r}"
            seq_id, taxid, rest = m.group(1), int(m.group(2)), m.group(3)
            if seq_id in self.seq_map:
                continue
            orig = taxid
            if add_assembly and rest:                           # one separator, then the rest of the line
                name = rest[1:]
                if name:
                    taxid = new_taxid(name, taxid, "assembly")
            if add_sequences and orig not in (HUMAN, MOUSE):
                taxid = new_taxid(seq_id, taxid, "sequence")
            if add:
                out.append(f"{seq_id}\t{taxid}\n")
            self.seq_map[seq_id] = taxid
        self.stdout = "".join(out)

    def _pmap(self, t):
        p = self.entries[t][0]
        return 0 if p is None else p

    def assign(self, records, min_len=0):
        """records: (header line after '>', sequence bytes) in file order → the taxid each record is processed
        with, 0 = skipped.  Renames taxa under -a."""
        out = []
        for header, seq in records:
            words = header.split()
            sid = words[0] if words else ""
            if not seq:
                out.append(0)
                continue
            taxid = self.seq_map.get(sid)
            if taxid is None:
                taxid = 0
                head, dot, tail = sid.rpartition(".")
                if dot and all(c.isdigit() for c in tail):
                    taxid = self.seq_map.get(head, 0)
            if taxid == 0 and sid.startswith(PREFIX):
                m = re.match(r"[+-]?\d+", sid[len(PREFIX):])
                taxid = int(m.group(0)) if m else 0
                header = header.lstrip("\t ") or header
            if taxid == 0 or (min_len > 0 and len(seq) < min_len) or taxid not in self.entries:
                out.append(0)
                continue
            if self.add_sequences:
                par = self._pmap(taxid)
                if taxid not in (HUMAN, MOUSE) and par not in (HUMAN, MOUSE):
                    self.entries[taxid][1] = header
            out.append(taxid)
        return out

    def rows(self):
        """(taxid, parent, name, rank) as written: a taxon without a parent pointer is its own parent"""
        return [(t, t if e[0] is None else e[0], e[1], e[2]) for t, e in sorted(self.entries.items())]

    def taxdb_text(self):
        return "".join(f"{t}\t{p}\t{n}\t{r}\n" for t, p, n, r in self.rows())

    def parent_map(self):
        ids = sorted(t for t in self.entries if t != 0)
        return np.array(ids, np.uint32), np.array([self._pmap(t) for t in ids], np.uint32)
