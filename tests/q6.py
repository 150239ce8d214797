"""TPC-H Q6 through the GPU AggregationOperator (fused scan filter + project + global sum), shared by tests and tools/bench_q6.py.

Input channels are those of the synthetic lineitem (tgpu_synth_lineitem_q1): 0 shipdate (INTEGER days), 1 returnflag, 2 linestatus,
3 quantity, 4 extendedprice, 5 discount, 6 tax."""
import numpy as np

from trino_b200 import abi
from trino_b200 import operators as ops

SHIP_LO, SHIP_HI = 8766, 9131          # DATE '1994-01-01', DATE '1995-01-01' as days since 1970-01-01
DISC_LO, DISC_HI, QTY_HI = 0.05, 0.07, 24.0
INPUT_TYPES = [abi.INT32, abi.INT8, abi.INT8, abi.FLOAT64, abi.FLOAT64, abi.FLOAT64, abi.FLOAT64]


def q6_filter(ship_lo=SHIP_LO, ship_hi=SHIP_HI):
    """shipdate >= lo AND shipdate < hi AND discount BETWEEN 0.05 AND 0.07 AND quantity < 24"""
    B, D = abi.V_BIGINT, abi.V_DOUBLE
    sd, qty, disc = ops.Col(0, B), ops.Col(3, D), ops.Col(5, D)
    return ops.Call(abi.EX_AND,
                    ops.Call(abi.EX_AND, ops.Call(abi.EX_GE, sd, ops.Const(ship_lo, B)), ops.Call(abi.EX_LT, sd, ops.Const(ship_hi, B))),
                    ops.Call(abi.EX_AND, ops.Call(abi.EX_BETWEEN, disc, ops.Const(DISC_LO, D), ops.Const(DISC_HI, D)),
                             ops.Call(abi.EX_LT, qty, ops.Const(QTY_HI, D))))


def q6_program(ship_lo=SHIP_LO, ship_hi=SHIP_HI):
    """the Q6 filter; projection extendedprice * discount"""
    D = abi.V_DOUBLE
    return ops.PageProcessorProgram(q6_filter(ship_lo, ship_hi), [ops.Call(abi.EX_MUL, ops.Col(4, D), ops.Col(5, D))])


def q6_aggregators():
    # sum(extendedprice * discount), count(*)
    return [ops.Aggregator(abi.AGG_SUM, 0), ops.Aggregator(abi.AGG_COUNT_STAR)]


def q6_factory(ctx, ship_lo=SHIP_LO, ship_hi=SHIP_HI):
    return ops.AggregationOperatorFactory(ctx, abi.STEP_SINGLE, q6_aggregators(), pre=q6_program(ship_lo, ship_hi), input_types=INPUT_TYPES)


def q6_selected(cols, ship_lo=SHIP_LO, ship_hi=SHIP_HI):
    sd, disc, qty = cols["shipdate"], cols["discount"], cols["quantity"]
    return (sd >= ship_lo) & (sd < ship_hi) & (disc >= DISC_LO) & (disc <= DISC_HI) & (qty < QTY_HI)


def q6_oracle(cols, ship_lo=SHIP_LO, ship_hi=SHIP_HI):
    """(revenue or None, count) through the oracle's left fold: every selected row in group 0"""
    from helpers import oracle_agg_rows
    from trino_b200.page import Block, Page
    sel = q6_selected(cols, ship_lo, ship_hi)
    rev = cols["extendedprice"][sel] * cols["discount"][sel]
    page = Page(Block.bigint(np.zeros(len(rev), dtype=np.int64)), Block.double(rev))
    rows = oracle_agg_rows([page], [0], [(abi.AGG_SUM, 1, -1), (abi.AGG_COUNT_STAR, -1, -1)]) if len(rev) else [(0, None, 0)]
    return rows[0][1], rows[0][2]
