"""An encrypted key-value store on the GPU: clear keys mapped to encrypted
radix values, the values resident on the device (tfhe-rs' `CudaKVStore`).

The host-side operations (`insert`, `remove`, `get`, `len`) take clear keys.
The encrypted-key operations are methods of `integer.CudaRadixServerKey`:
`kv_store_get`, `kv_store_update`, `kv_store_map`, `kv_store_contains_key`,
`kv_store_contains_value` and `kv_store_contains_clear_value`, compiled to
KS -> PBS layers by `radix_find`.  Entries are kept in key order, as
tfhe-rs' BTreeMap keeps them."""
from __future__ import annotations

from typing import Dict, List, Optional

import numpy as np

from . import integer


class CudaKVStore:
    """Clear integer keys -> encrypted values of one kind (unsigned or
    signed) and one block count, set by the first insert."""

    def __init__(self):
        self._data: Dict[int, object] = {}   # key -> blocks [num_blocks, big + 1]
        self.kind = None
        self.num_blocks: Optional[int] = None

    @staticmethod
    def _key(key) -> int:
        if isinstance(key, bool) or not isinstance(key, (int, np.integer)):
            raise ValueError(f"a store key is a clear integer, got {key!r}")
        return int(key)

    def _ct(self, blocks):
        return self.kind(blocks, 1)

    def insert(self, key, value) -> Optional[integer.CudaUnsignedRadixCiphertext]:
        """Store `value` (a radix ciphertext holding one integer) under `key`;
        returns the value it replaces, or None.  A value of no blocks is not
        inserted (None is returned); one of another kind or block count than
        the stored values raises ValueError."""
        key = self._key(key)
        if not isinstance(value, integer.CudaUnsignedRadixCiphertext) or value.num_inputs != 1:
            raise ValueError("a store value is a radix ciphertext holding one integer (num_inputs = 1)")
        n = value.blocks.shape[0]
        if n == 0:
            return None
        if self.kind is None:
            self.kind, self.num_blocks = type(value), n
        elif type(value) is not self.kind or n != self.num_blocks:
            raise ValueError(f"the store holds {self.num_blocks}-block {self.kind.__name__} values, "
                             f"got a {n}-block {type(value).__name__}")
        old = self._data.get(key)
        self._data[key] = value.blocks
        return None if old is None else self._ct(old)

    def remove(self, key) -> Optional[integer.CudaUnsignedRadixCiphertext]:
        old = self._data.pop(self._key(key), None)
        return None if old is None else self._ct(old)

    def get(self, key) -> Optional[integer.CudaUnsignedRadixCiphertext]:
        """the value stored under the clear `key`, or None"""
        old = self._data.get(self._key(key))
        return None if old is None else self._ct(old)

    def __len__(self) -> int:
        return len(self._data)

    def keys(self) -> List[int]:
        return sorted(self._data)

    def values(self) -> List[integer.CudaUnsignedRadixCiphertext]:
        return [self._ct(self._data[k]) for k in self.keys()]

    def stacked(self):
        """the values' blocks in key order, [len * num_blocks, big + 1]"""
        import torch

        return torch.cat([self._data[k] for k in self.keys()])

    def _set_values(self, blocks):
        """replace every value, in key order, from [len, num_blocks, big + 1]"""
        for k, b in zip(self.keys(), blocks.reshape(len(self), self.num_blocks, -1)):
            self._data[k] = b
