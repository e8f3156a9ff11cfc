"""Nexmark q0 / q1 / q2 / q3 / q4 / q6 / q7 / q18, and q5 as its SQL states it (q5_hop), on the Stream API; and
`rolling_bids`, a rolling aggregate over the bid stream that no reference query has.

The reference's `NexmarkStream` is one stream of `Event` enum rows
(crates/nexmark/src/queries/mod.rs:12); here it is three column tables
(person / auction / bid) per step, which is the same data column-major.
Column order: see generator.PERSON_COLS / AUCTION_COLS / BID_COLS.
"""
from __future__ import annotations

from dataclasses import dataclass

from ..circuit import Fold, Linear, Max, Min, RootCircuit, Stream, TableStream
from ..zset import Before, Proj, RelRange, Schema, acc, col, const, fanout_index, key, lval, rval

WATERMARK_INTERVAL_SECONDS = 4  # queries/mod.rs:12
TUMBLE_SECONDS = 10             # queries/q7.rs:43
CATEGORY_OF_INTEREST = 10       # queries/q3.rs:31
AUCTION_ID_MODULO = 123         # queries/q2.rs:21
HOP_SLIDE_MS = 2_000            # queries/q5.rs:24-60: HOP(dateTime, INTERVAL '2' SECOND, INTERVAL '10' SECOND)
HOP_SIZE_MS = 10_000
NUM_AUCTIONS_PER_SELLER = 10    # queries/q6.rs:39


@dataclass
class NexmarkTables:
    person: TableStream
    auction: TableStream
    bid: TableStream


def add_nexmark_input(circuit: RootCircuit):
    p, hp = circuit.add_input_table(5)
    a, ha = circuit.add_input_table(5)
    b, hb = circuit.add_input_table(5)
    return NexmarkTables(p, a, b), {"person": hp, "auction": ha, "bid": hb}


def q0(inp: NexmarkTables) -> Stream:
    """q0 pass-through of bids (queries/q0.rs): plumbing only."""
    return inp.bid.flat_map_index(Proj(Schema("uuuuu"), [col(0), col(1), col(2), col(3), col(4)]))


def q1(inp: NexmarkTables) -> Stream:
    """q1 currency conversion (queries/q1.rs:31-39): every bid with price * 89 / 100, in u64 arithmetic."""
    return inp.bid.flat_map_index(Proj(Schema("uuuuu"), [col(0), col(1), (col(2) * 89).divu(100), col(3), col(4)]))


def q2(inp: NexmarkTables) -> Stream:
    """q2 selection (queries/q2.rs:23-31): (auction, price) of the bids whose auction % 123 == 0."""
    return inp.bid.flat_map_index(Proj(Schema("uu"), [col(0), col(2)], where=[col(0).remu(AUCTION_ID_MODULO).eq(0)]))


def q3(inp: NexmarkTables, states_of_interest=(1, 2, 3)) -> Stream:
    """queries/q3.rs:35-63.  States of interest OR, ID, CA = codes 3, 2, 1."""
    # Select auctions of interest and index them by seller id (q3.rs:37-40).
    auction_by_seller = inp.auction.flat_map_index(
        Proj(Schema("u", "u"), [col(1), col(0)], where=[col(2).eq(CATEGORY_OF_INTEREST)]))
    # Select people from states of interest, indexed by person id (q3.rs:43-50).
    person_by_id = inp.person.flat_map_index(
        Proj(Schema("u", "uuu"), [col(0), col(1), col(2), col(3)], where=[col(3).isin(states_of_interest)]))
    # (name, city, state, auction_id) (q3.rs:53-63)
    return auction_by_seller.join(person_by_id, Proj(Schema("uuuu"), [rval(0), rval(1), rval(2), lval(0)]))


def q4(inp: NexmarkTables) -> Stream:
    """queries/q4.rs:43-83."""
    # (a.id, (a.category, a.date_time, a.expires))  (q4.rs:45-48)
    auctions_by_id = inp.auction.flat_map_index(Proj(Schema("u", "uuu"), [col(0), col(2), col(3), col(4)]))
    # (b.auction, (b.price, b.date_time))  (q4.rs:51-54)
    bids_by_auction = inp.bid.flat_map_index(Proj(Schema("u", "uu"), [col(0), col(2), col(3)]))
    # ((auction_id, category), bid_price) for bids inside [date_time, expires]  (q4.rs:58-67)
    bids_for_auctions = auctions_by_id.join_index(
        bids_by_auction,
        Proj(Schema("uu", "u"), [key(0), lval(0), rval(0)], where=[rval(1).ge(lval(1)), rval(1).le(lval(2))]))
    winning_bids = bids_for_auctions.aggregate(Max)                                    # q4.rs:73-74
    by_category = winning_bids.map_index(Proj(Schema("u", "u"), [key(1), lval(0)]))    # q4.rs:75-76
    avg = by_category.average(lval(0))                                                 # q4.rs:80-81
    return avg.map(Proj(Schema("uu"), [key(0), lval(0)]))                              # q4.rs:82


def q7(inp: NexmarkTables) -> Stream:
    """queries/q7.rs:45-94."""
    # (date_time, (auction, bidder, price, extra))  (q7.rs:47-55)
    bids_by_time = inp.bid.flat_map_index(Proj(Schema("u", "uuuu"), [col(3), col(0), col(1), col(2), col(4)]))
    watermark = bids_by_time.watermark_monotonic(lambda dt: dt - WATERMARK_INTERVAL_SECONDS * 1000)   # q7.rs:60-61

    def bounds(wm):   # q7.rs:64-70
        rounded = wm - (wm % (TUMBLE_SECONDS * 1000))
        return (max(rounded - TUMBLE_SECONDS * 1000, 0), rounded)

    windowed = bids_by_time.window(watermark.apply(bounds))                            # q7.rs:73
    # (price, (auction, bidder, price, date_time, extra))  (q7.rs:74-79)
    bids_by_price = windowed.map_index(Proj(Schema("u", "uuuuu"), [lval(2), lval(0), lval(1), lval(2), key(0), lval(3)]))
    # ((), -price) -> Min -> max price  (q7.rs:82-91)
    neg_price = windowed.map_index(Proj(Schema("", "i"), [-lval(2)]))
    if windowed.circuit.workers > 1:
        # The single group () would shard every windowed bid to one worker.  Min is a
        # semigroup (aggregate/min.rs:17-27): aggregate per worker first, then
        # aggregate the <= P partial minima (SURVEY §8e).
        neg_price = neg_price.aggregate(Min, local=True)
    max_price = neg_price.aggregate(Min).map(Proj(Schema("u"), [-lval(0)]))
    # all bids with the max price  (q7.rs:92-93)
    return max_price.join(bids_by_price, Proj(Schema("uuuuu"), [rval(0), rval(1), rval(2), rval(3), rval(4)]))


def q5_hop(inp: NexmarkTables) -> Stream:
    """The SQL of queries/q5.rs:24-60 (hot items): per HOP(dateTime, 2 s, 10 s) window, the auctions with the most
    bids, as (auction, num).  Every window is kept (no watermark).  A row's weight is the number of windows in which
    the auction had `num` bids and no auction had more.  (The reference's DBSP q5 uses one sliding window instead.)"""
    last = col(3) - col(3).remu(HOP_SLIDE_MS)   # the start of the latest window that holds the bid
    j = fanout_index()
    # (auction, starttime) for each of the size / slide windows of a bid; no window starts below 0
    bid_windows = inp.bid.flat_map_index(Proj(Schema("uu"), [col(0), last - j * HOP_SLIDE_MS],
                                              where=[(j * HOP_SLIDE_MS).le(last)], fanout=HOP_SIZE_MS // HOP_SLIDE_MS))
    counts = bid_windows.aggregate_linear(const(1))                                      # ((auction, starttime), num)
    auction_bids = counts.map_index(Proj(Schema("u", "ui"), [key(1), key(0), lval(0)]))  # starttime -> (auction, num)
    max_bids = counts.map_index(Proj(Schema("u", "i"), [key(1), lval(0)])).aggregate(Max)   # starttime -> maxn
    # endtime = starttime + size, so the join on starttime is the SQL's join on both
    return auction_bids.join(max_bids, Proj(Schema("ui"), [lval(0), lval(1)], where=[lval(1).ge(rval(0)).signed()]))


def q6(inp: NexmarkTables) -> Stream:
    """queries/q6.rs:41-107: per seller, the average winning price of its last 10 auctions (by auction id), as
    (seller, avg), u64 division."""
    # (a.id, (a.seller, a.date_time, a.expires)) and (b.auction, (b.price, b.date_time))  (q6.rs:43-52)
    auctions_by_id = inp.auction.flat_map_index(Proj(Schema("u", "uuu"), [col(0), col(1), col(3), col(4)]))
    bids_by_auction = inp.bid.flat_map_index(Proj(Schema("u", "uu"), [col(0), col(2), col(3)]))
    # ((auction_id, seller), bid_price) for bids inside [date_time, expires]  (q6.rs:58-79)
    bids_for_auctions = auctions_by_id.join_index(
        bids_by_auction,
        Proj(Schema("uu", "u"), [key(0), lval(0), rval(0)], where=[rval(1).ge(lval(1)), rval(1).le(lval(2))]))
    # seller -> (auction, winning price)  (q6.rs:86-88)
    winning = bids_for_auctions.aggregate(Max).map_index(Proj(Schema("u", "uu"), [key(1), key(0), lval(0)]))
    # the VecDeque of the last 10 prices as words 0..9, newest in word 9 (words of a deque shorter than 10 that were
    # never pushed stay 0), and its length in word 10  (q6.rs:93-106)
    n = NUM_AUCTIONS_PER_SELLER
    last_prices = Fold([0] * (n + 1), [acc(i + 1) for i in range(n - 1)] + [lval(1), (acc(n) + 1).min(n)],
                       output=Proj(Schema("", "u"), [sum((acc(i) for i in range(1, n)), acc(0)).divu(acc(n))]))
    return winning.aggregate(last_prices)


def q18(inp: NexmarkTables) -> Stream:
    """queries/q18.rs:37-50: the last bid (latest date_time) of every (auction, bidder).  The accumulator starts as
    Bid::default() (zeros) and takes a value iff its date_time is strictly later, so of two bids at one date_time the
    first in value order wins."""
    bids = inp.bid.flat_map_index(Proj(Schema("uu", "uuuuu"), [col(0), col(1), col(0), col(1), col(2), col(3), col(4)]))
    last = Fold([0] * 5, [key(0), key(1), lval(2), lval(3), lval(4)], where=lval(3).gt(acc(3)))
    return bids.aggregate(last).map(Proj(Schema("uuuuu"), [lval(i) for i in range(5)]))


ROLLING_RANGE = RelRange(Before(1000), Before(0))   # the last second of bids, the bid's own millisecond included


def rolling_bids(inp: NexmarkTables, watermark: bool = False) -> tuple[Stream, Stream]:
    """Per auction and bid time, over the auction's bids of the last second (ROLLING_RANGE): (auction, (date_time,
    some, count, sum of price)) from a Linear aggregate and (auction, (date_time, some, max price)) from Max.
    watermark=True: the same outputs from partitioned_rolling_aggregate_with_watermark over the bids indexed by
    date_time, with a watermark WATERMARK_INTERVAL_SECONDS behind the latest bid, so the state stays bounded.
    Not in QUERIES: the reference's Nexmark suite has no rolling aggregate."""
    count_sum = Linear(Proj(Schema("", "ii"), [const(1), lval(0)]))
    if not watermark:
        by_auction = inp.bid.flat_map_index(Proj(Schema("u", "uu"), [col(0), col(3), col(2)]))   # (auction, (ts, price))
        return (by_auction.partitioned_rolling_aggregate(count_sum, ROLLING_RANGE),
                by_auction.partitioned_rolling_aggregate(Max, ROLLING_RANGE))
    by_time = inp.bid.flat_map_index(Proj(Schema("u", "uu"), [col(3), col(0), col(2)]))          # (ts, (auction, price))
    wm = by_time.watermark_monotonic(lambda dt: dt - WATERMARK_INTERVAL_SECONDS * 1000)
    partition = Proj(Schema("u", "u"), [lval(0), lval(1)])                                        # (auction, price)
    return (by_time.partitioned_rolling_aggregate_with_watermark(wm, partition, count_sum, ROLLING_RANGE),
            by_time.partitioned_rolling_aggregate_with_watermark(wm, partition, Max, ROLLING_RANGE))


QUERIES = {"q0": q0, "q1": q1, "q2": q2, "q3": q3, "q4": q4, "q7": q7, "q5_hop": q5_hop, "q6": q6, "q18": q18}
