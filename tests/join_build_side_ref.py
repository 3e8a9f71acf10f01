"""Reference results of the build-side ("right") hash joins for the tests (probe = left, build =
right), restated from the reference rather than derived from inner-join pairs:

  RIGHT        new_hash_join/memory/right_join.rs       every match, then every build row never matched
  RIGHT SEMI   new_hash_join/memory/right_join_semi.rs  every build row matched at least once, once
  RIGHT ANTI   new_hash_join/memory/right_join_anti.rs  every build row never matched
  FULL         hash_join/hash_join_probe_state.rs:455-567 with probe_join/left_join.rs:
               LEFT during the probe, then RIGHT's final scan

The probe walk sets scan_map[build row] for every match (right_join.rs: `scan_map`); final_probe
then scans EVERY build row, inserted or not, so a build row with a NULL key (never inserted,
fixed_keys.rs) counts as unmatched.  Keys compare by their 64-bit image (signed keys sign-extended,
unsigned ones zero-extended), as the device join and the C oracle do.

Also `derive_build_side_join_rows`: the same results derived from the C oracle's INNER pairs and
the mask of build rows they match, which the CPU test holds the restatement against."""
import numpy as np

from databend_b200 import abi


def _key_words(col):
    v = col.values()
    words = v.astype(np.int64) if v.dtype.kind == "i" else v.astype(np.uint64).view(np.int64)
    return words, col.valid_mask()


def hash_join_build_side(kind: int, build_key, probe_key):
    """kind: abi.JOIN_RIGHT / JOIN_RIGHT_SEMI / JOIN_RIGHT_ANTI / JOIN_FULL; build_key and probe_key
    are Columns.  Returns (probe_idx, build_idx) as int64 arrays, -1 on the side the output row does
    not carry.  Row order is unspecified, as for the operator."""
    if kind not in (abi.JOIN_RIGHT, abi.JOIN_RIGHT_SEMI, abi.JOIN_RIGHT_ANTI, abi.JOIN_FULL):
        raise ValueError(kind)
    bw, bvalid = _key_words(build_key)
    pw, pvalid = _key_words(probe_key)
    n_build, n_probe = len(bw), len(pw)
    # the table: every build row with a valid key, ordered by key so one key's entries are adjacent
    inserted = np.nonzero(bvalid)[0]
    table = inserted[np.argsort(bw[inserted], kind="stable")]
    table_keys = bw[table]
    # the probe walk: entries [lo, hi) of each probe row's key; a NULL probe key walks nothing
    lo = np.searchsorted(table_keys, pw, side="left")
    hi = np.searchsorted(table_keys, pw, side="right")
    n_match = np.where(pvalid, hi - lo, 0)
    total = int(n_match.sum())
    first = np.cumsum(n_match) - n_match
    match_probe = np.repeat(np.arange(n_probe, dtype=np.int64), n_match)
    match_build = table[np.repeat(lo, n_match) + (np.arange(total) - np.repeat(first, n_match))].astype(np.int64)
    scan_map = np.zeros(n_build, dtype=bool)
    scan_map[match_build] = True
    # final_probe: scan every build row
    if kind == abi.JOIN_RIGHT_SEMI:
        final = np.nonzero(scan_map)[0]
    else:
        final = np.nonzero(~scan_map)[0]
    final_pairs = (np.full(len(final), -1, dtype=np.int64), final.astype(np.int64))
    if kind in (abi.JOIN_RIGHT_SEMI, abi.JOIN_RIGHT_ANTI):
        return final_pairs
    probe_parts, build_parts = [match_probe], [match_build]
    if kind == abi.JOIN_FULL:  # the unmatched probe rows are kept with a NULL build side
        unmatched_probe = np.nonzero(n_match == 0)[0].astype(np.int64)
        probe_parts.append(unmatched_probe)
        build_parts.append(np.full(len(unmatched_probe), -1, dtype=np.int64))
    probe_parts.append(final_pairs[0])
    build_parts.append(final_pairs[1])
    return np.concatenate(probe_parts), np.concatenate(build_parts)


def derive_build_side_join_rows(kind: str, n_probe: int, n_build: int, pairs):
    """Expected output rows (probe_idx or None, build_idx or None) of a build-side join from the C
    oracle's INNER pairs (probe_idx, build_idx) and the mask of build rows they match.
      right      -> pairs + (None, b) for unmatched build rows;  right_semi -> (None, b) matched, once;
      right_anti -> (None, b) unmatched;  full -> the LEFT rows + (None, b) for unmatched build rows."""
    pi, bi = pairs
    build_matched = np.zeros(n_build, dtype=bool)
    build_matched[bi] = True
    probe_matched = np.zeros(n_probe, dtype=bool)
    probe_matched[pi] = True
    both = [(int(p), int(b)) for p, b in zip(pi, bi)]
    unmatched_build = [(None, int(b)) for b in np.nonzero(~build_matched)[0]]
    if kind == "right":
        return both + unmatched_build
    if kind == "right_semi":
        return [(None, int(b)) for b in np.nonzero(build_matched)[0]]
    if kind == "right_anti":
        return unmatched_build
    if kind == "full":
        return both + [(int(p), None) for p in np.nonzero(~probe_matched)[0]] + unmatched_build
    raise ValueError(kind)
