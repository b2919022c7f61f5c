"""Plain model of vector find, vector comparisons and the key-value store on
Python integers: the results `tfhe-rs_b200/radix_find.py` computes, each
rule with the tfhe-rs function it restates (tfhe/src/integer/server_key/
radix_parallel/).  Results are (value, num_blocks) for radix integers and
0 / 1 for booleans."""


def num_blocks_for(value):
    """mod.rs `num_blocks_to_represent_unsigned_value`: ceil(bits / 2), at
    least one bit"""
    return (max(int(value).bit_length(), 1) + 1) // 2


def _digits(v, n):
    return [(v >> (2 * j)) & 3 for j in range(n)]


def _one_hot_sum(indices, values, width):
    """scalar_dot_prod.rs `unchecked_boolean_scalar_one_hot_dot_prod_parallelized`:
    block-wise sums without carries, so duplicate matches add digit by digit
    mod 4"""
    out = 0
    for j in range(width):
        out |= (sum(_digits(values[i], width)[j] for i in indices) % 4) << (2 * j)
    return out


def match_value(x, matches):
    """vector_find.rs `unchecked_match_value_parallelized`: empty -> (0 on one
    block, false); else enough blocks for the largest output"""
    if not matches:
        return (0, 1), 0
    width = num_blocks_for(max(o for _, o in matches))
    hit = [i for i, (inp, _) in enumerate(matches) if inp == x]
    return (_one_hot_sum(hit, [o for _, o in matches], width), width), int(bool(hit))


def match_value_or(x, matches, or_value):
    """vector_find.rs `unchecked_match_value_or_parallelized`: empty ->
    or_value on its own blocks; else max(blocks of the match, of or_value)"""
    if not matches:
        return or_value, num_blocks_for(or_value)
    (v, w), found = match_value(x, matches)
    return (v if found else or_value), max(w, num_blocks_for(or_value))


def contains(values, x):
    """vector_find.rs `unchecked_contains_parallelized` (and `_clear`): false
    for an empty list"""
    return int(x in values)


def is_in_clears(x, clears):
    """vector_find.rs `unchecked_is_in_clears_parallelized`"""
    return int(x in clears)


def index_in_clears(x, clears, n):
    """vector_find.rs `unchecked_index_in_clears_parallelized`: empty -> (0 on
    ct's n blocks, false); else blocks for len - 1 (`compute_final_index_from_selectors`);
    0 when absent"""
    if not clears:
        return (0, n), 0
    hit = [i for i, c in enumerate(clears) if c == x]
    width = num_blocks_for(len(clears) - 1)
    return (_one_hot_sum(hit, list(range(len(clears))), width), width), int(bool(hit))


def first_index_in_clears(x, clears, n):
    """vector_find.rs `unchecked_first_index_in_clears_parallelized`: later
    duplicates dropped first (`unique_by`), blocks for the largest kept index"""
    if not clears:
        return (0, n), 0
    kept = {}
    for i, c in enumerate(clears):
        kept.setdefault(c, i)
    width = num_blocks_for(max(kept.values()))
    return ((kept.get(x, 0), width), int(x in kept))


def index_of(values, x, n):
    """vector_find.rs `unchecked_index_of_parallelized`: empty -> (0 on the
    value's n blocks, false); `unchecked_index_of_clear_parallelized` passes
    n = 1"""
    return index_in_clears(x, values, n)


def first_index_of(values, x, n):
    """vector_find.rs `unchecked_first_index_of_parallelized` (`only_keep_first_true`,
    then blocks for len - 1); `_clear` passes n = 1 for the empty list"""
    if not values:
        return (0, n), 0
    width = num_blocks_for(len(values) - 1)
    return ((values.index(x) if x in values else 0), width), int(x in values)


def all_eq_slices(lhs, rhs):
    """vector_comparisons.rs `unchecked_all_eq_slices_parallelized`: false on
    different lengths, true for two empty slices (entries are (value,
    num_blocks): a pair of different block counts is unequal)"""
    return int(len(lhs) == len(rhs) and all(a == b for a, b in zip(lhs, rhs)))


def contains_sub_slice(lhs, pattern):
    """vector_comparisons.rs `unchecked_contains_sub_slice_parallelized`: false
    when the pattern is longer (an empty pattern is refused)"""
    assert pattern
    P = len(pattern)
    return int(any(lhs[w:w + P] == pattern for w in range(len(lhs) - P + 1)))


def kv_store_get(store, key, key_blocks):
    """kv_store.rs `kv_store_get_impl`: empty -> (0 on the encrypted key's
    blocks, false); else (store[key] or 0, found) on the values' blocks"""
    if not store:
        return (0, key_blocks), 0
    return store.get(key, 0), int(key in store)


def kv_store_update(store, key, new):
    """kv_store.rs `kv_store_update`: returns found; the store changes in place"""
    if key in store:
        store[key] = new
        return 1
    return 0


def kv_store_map(store, key, f, key_blocks):
    """kv_store.rs `kv_store_map`: (old, f(old), found), old as `kv_store_get`"""
    old, found = kv_store_get(store, key, key_blocks)
    old_v = old[0] if isinstance(old, tuple) else old
    new = f(old_v)
    if found:
        store[key] = new
    return old_v, new, found
