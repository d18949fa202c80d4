"""CPU statement of the stop-mode cut of the batched walks (sq_accept_*_batch_stop, DESIGN.md §3a) -- TEST
INFRASTRUCTURE, never imported by the product.

The walk commits tokens[P .. n) without an end rule (n = a + 1, or a when the NaN flag ended the walk).  The sequence then
ends at j + 1 for the first j in [P, n) whose token is a stop id, and at its absolute length limit E when 0 < E <= n;
the earlier end wins, the stop id on a tie."""
from typing import Iterable, Sequence, Tuple

FINISH_NONE, FINISH_STOP, FINISH_LENGTH = 0, 1, 2


def cut(tokens: Sequence[int], P: int, n: int, stop_ids: Iterable[int], end_limit: int) -> Tuple[int, int]:
    """-> (finish, end): the state words SQ_ST_FINISH and SQ_ST_END a stop walk writes.  stop_ids may hold -1 padding
    (never a token); end_limit <= 0 is no limit."""
    stop = {int(t) for t in stop_ids if int(t) >= 0}
    finish, end = FINISH_NONE, 0
    for j in range(P, n):
        if int(tokens[j]) in stop:
            finish, end = FINISH_STOP, j + 1
            break
    if 0 < end_limit <= n and (finish == FINISH_NONE or end_limit < end):
        finish, end = FINISH_LENGTH, end_limit
    return finish, end
