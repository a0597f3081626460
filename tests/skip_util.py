"""TEST INFRASTRUCTURE for skip mode (REGK_SKIP_BAD): the oracle's fence, record by record."""
import ctypes as C

import numpy as np

from oracle import oracle


def fence_bits(batch, flags: int = 0) -> np.ndarray:
    """REGK_BAD_* of every record of a host RecordBatch (uint8[n]) for the batch flags `flags` (REGK_NODE_ALIAS
    also comes from batch.alias; REGK_NO_JSON / REGK_NO_PATH drop the checks of the half not composed): one
    call of the oracle's ro_validate_record per record.  What a skip-mode batch must skip."""
    L = oracle.lib()
    alias = int(bool(batch.alias or flags & (1 << 2)))
    no_json, no_path = int(bool(flags & (1 << 3))), int(bool(flags & (1 << 4)))
    db, ab, hb = batch.domain_bytes.tobytes(), batch.addr_bytes.tobytes(), batch.host_bytes.tobytes()
    out = np.zeros(batch.n, np.uint8)
    for i in range(batch.n):
        d = db[int(batch.domain_off[i]):int(batch.domain_off[i + 1])]
        a = ab[int(batch.addr_off[i]):int(batch.addr_off[i + 1])]
        if alias:
            h = b""
        elif batch.host_off is not None:
            h = hb[int(batch.host_off[i]):int(batch.host_off[i + 1])]
        else:
            h = hb[i * batch.host_stride:(i + 1) * batch.host_stride]
        out[i] = L.ro_validate_record(d, C.c_size_t(len(d)), h, C.c_size_t(len(h)), C.c_int(alias), a,
                                      C.c_size_t(len(a)), C.c_uint32(int(batch.type_id[i])),
                                      C.c_uint32(len(batch.types)), C.c_int(no_json), C.c_int(no_path))
    return out
