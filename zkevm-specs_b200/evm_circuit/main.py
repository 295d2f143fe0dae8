"""verify_steps — the reference's EVM-circuit entry point (evm_circuit/main.py:14-44), with
the per-step loop running on the device.

The reference builds one `Instruction` per (curr, next) pair in Python and stops at the first
AssertionError; other exception types propagate.  Here all steps are packed into a 13-cell
matrix, the tables into cell matrices, ONE zk_check(ZK_CIRCUIT_EVM) evaluates every step, and
the smallest failing (step, constraint) is turned back into the exception class the reference
would have raised first (SURVEY.md Appendix B)."""
from __future__ import annotations

from typing import List, Optional

import numpy as np

from .. import native, packing
from ..util.arithmetic import FQ
from .spec import ExecutionState
from .step import StepState
from .table import LookupAmbiguousFailure, LookupUnsatFailure, Tables, fixed_table_matrix


class ConstraintUnsatFailure(Exception):
    def __init__(self, message: str) -> None:
        self.message = message
        super().__init__(message)


DUMMY_STEP_STATE = StepState(ExecutionState.EndBlock, rw_counter=-1)


def step_row(s: StepState) -> List[int]:
    c = packing.cell_int
    return [int(s.execution_state), c(s.rw_counter), c(s.call_id), int(s.is_root), int(s.is_create),
            c(s.code_hash.lo), c(s.code_hash.hi), c(s.program_counter), c(s.stack_pointer), c(s.gas_left),
            c(s.memory_word_size), c(s.reversible_write_counter), c(s.log_id)]


def pack_steps(steps: List[StepState]) -> np.ndarray:
    return packing.matrix_from_ints([step_row(s) for s in steps], 13)


def step_aux_rows(steps: List[StepState], row_base: int = 0) -> List[List[int]]:
    """StepState.aux_data (reference step.py:45) as the step-aux side table: one row (step row, lo, hi) per step that carries
    a Word (CREATE / CREATE2 read it as the init code's hash, create.py:107) or an int (ErrorOutOfGasSloadSstore: the slot's
    committed value, error_oog_sload_sstore.py:33) there"""
    c = packing.cell_int
    rows = []
    for k, s in enumerate(steps):
        a = getattr(s, "aux_data", None)
        if isinstance(a, int) and not isinstance(a, bool) and 0 <= a < (1 << 256):
            rows.append([row_base + k, a & ((1 << 128) - 1), a >> 128])
        elif a is not None and hasattr(a, "lo") and hasattr(a, "hi"):
            rows.append([row_base + k, c(a.lo), c(a.hi)])
    return rows


def upload_tables(ctx: native.Context, tables: Tables) -> None:
    """Python row sets -> cell matrices -> device (tables are replicated per GPU)."""
    ctx.upload_table(native.TABLE_BYTECODE, packing.pack(tables.bytecode_table, packing.bytecode_table_row, 6))
    rws = list(tables.rw_table)
    ctx.upload_table(native.TABLE_RW, packing.pack(rws, packing.rw_table_row, 14),
                     flags=np.array([packing.rw_table_flags(r) for r in rws], dtype=np.uint8))
    ctx.upload_table(native.TABLE_COPY, packing.pack(tables.copy_table, packing.copy_table_row, 14))
    ctx.upload_table(native.TABLE_KECCAK, packing.pack(tables.keccak_table, packing.keccak_table_row, 5))
    # tx / block tables: the ORIGIN / GASPRICE / BlockCtx gadgets (tables.tx_lookup / block_lookup, table.py:691-705)
    # (+ BeginTx / EndTx / EndBlock; the value type flags carry WordOrValue.is_word for their .value() asserts)
    txs, blks = list(getattr(tables, "tx_table", ()) or ()), list(getattr(tables, "block_table", ()) or ())
    ctx.upload_table(native.TABLE_TX, packing.pack(txs, packing.tx_table_row, 5),
                     flags=np.array([packing.word_flag(r.value) for r in txs], dtype=np.uint8))
    ctx.upload_table(native.TABLE_BLOCK, packing.pack(blks, packing.block_table_row, 4),
                     flags=np.array([packing.word_flag(r.value) for r in blks], dtype=np.uint8))
    wds = list(getattr(tables, "withdrawal_table", ()) or ())
    c = packing.cell_int
    ctx.upload_table(native.TABLE_WITHDRAWAL,
                     packing.matrix_from_ints([[c(w.id), c(w.validator_id), c(w.address), c(w.amount)] for w in wds], 4))
    # exp table of the EXP gadget: one row per exp-circuit row (reference table.py:654-671)
    ctx.upload_table(native.TABLE_EXP, packing.matrix_from_ints(exp_table_rows(getattr(tables, "exp_circuit", None) or ()), 11))
    upload_fixed_table(ctx)


def exp_table_rows(exp_circuit) -> List[List[int]]:
    """ExpTableRow cells of an exp circuit (is_step = 1, identifier, is_last, the base as four 64-bit limbs, exponent lo / hi,
    exponentiation lo / hi), identical rows once like the reference's set"""
    c = packing.cell_int
    rows = set()
    for r in exp_circuit:
        lo, hi = c(r.base.lo), c(r.base.hi)
        m64 = (1 << 64) - 1
        rows.add((1, c(r.identifier), c(r.is_last), lo & m64, lo >> 64, hi & m64, hi >> 64,
                  c(r.exponent.lo), c(r.exponent.hi), c(r.exponentiation.lo), c(r.exponentiation.hi)))
    return [list(r) for r in sorted(rows)]


def upload_fixed_table(ctx: native.Context) -> None:
    if not getattr(ctx, "_fixed_uploaded", False):
        ctx.upload_table(native.TABLE_FIXED, fixed_table_matrix())
        ctx._fixed_uploaded = True


def raise_first_failure(first_fail: np.ndarray, circuit_id: int, what: str) -> None:
    hit = native.first_failure(first_fail, circuit_id)
    if hit is None:
        return
    row, cid, cls, name = hit
    msg = f"{what} {row}: {name}"
    if cls == native.ERR_ASSERT:
        raise AssertionError(msg)
    if cls == native.ERR_LOOKUP_UNSAT:
        raise LookupUnsatFailure(name, msg)
    if cls == native.ERR_LOOKUP_AMBIGUOUS:
        raise LookupAmbiguousFailure(name, msg)
    if cls == native.ERR_RANGE_RAISE:
        raise ConstraintUnsatFailure(msg)
    if cls == native.ERR_VALUE:
        raise ValueError(msg)
    raise NotImplementedError(msg)


def check_steps(ctx: native.Context, steps_matrix: np.ndarray, begin_with_first_step: bool = False,
                end_with_last_step: bool = False):
    """steps already packed (and tables already uploaded): returns (first_fail, fail_count)."""
    ctx.upload_columns(native.CIRCUIT_EVM, steps_matrix)
    flags = (native.FLAG_EVM_FIRST_STEP if begin_with_first_step else 0) | (
        native.FLAG_EVM_LAST_STEP if end_with_last_step else 0)
    n = steps_matrix.shape[1]
    return ctx.check(native.CIRCUIT_EVM, 0, max(n - 1, 0), 0, flags)


def verify_steps(tables: Tables, steps: List[StepState], begin_with_first_step: bool = False,
                 end_with_last_step: bool = False, success: bool = True,
                 ctx: Optional[native.Context] = None) -> None:
    """Reference signature and error convention (main.py:14-44): mutates `steps` when
    end_with_last_step; an AssertionError-class failure is re-raised when success=True and
    required when success=False; every other failure class propagates."""
    ctx = ctx or native.default_context()
    upload_tables(ctx, tables)
    verify_steps_resident(steps, ctx, begin_with_first_step, end_with_last_step, success)


def verify_steps_resident(steps: List[StepState], ctx: native.Context, begin_with_first_step: bool = False,
                          end_with_last_step: bool = False, success: bool = True) -> None:
    """verify_steps against the tables already resident in `ctx` (uploaded, or built on the device: assign.assign_tx_table,
    assign_copy_table, assign_exp_circuit, ...): only the steps and their step-aux table are uploaded (and the fixed
    table, once per context).  Same error convention, and `steps` is mutated the same way"""
    if end_with_last_step:
        steps.append(DUMMY_STEP_STATE)
    upload_fixed_table(ctx)
    ctx.upload_table(native.TABLE_STEP_AUX, packing.matrix_from_ints(step_aux_rows(steps), 3))
    ff, _ = check_steps(ctx, pack_steps(steps), begin_with_first_step, end_with_last_step)
    exception = None
    try:
        raise_first_failure(ff, native.CIRCUIT_EVM, "step")
    except AssertionError as e:
        exception = e
    if success:
        if exception:
            raise exception
    else:
        assert exception is not None
