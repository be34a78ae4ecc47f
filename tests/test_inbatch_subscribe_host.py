"""PCDN_FLAG_INBATCH_SUBSCRIBE on a host-only engine (no device, no batches): the engine accepts the flag,
and its mirror and sync maps go through exactly the states of an engine without it."""
import random

from oracle import oracle as orc


def run(pcdn, flags, seed):
    rng = random.Random(seed)
    e = pcdn.Engine(device=-1, max_conns=512, max_topics=64, max_keys=1024, n_valid_topics=32, flags=flags)
    keys = [b"k%03d" % i for i in range(40)]
    trace = []
    for k in keys:
        e.add_user(k, [rng.randrange(32)])
    e.add_broker("p/p")
    for step in range(300):
        k = rng.choice(keys)
        topics = [rng.randrange(40) for _ in range(rng.randrange(1, 5))]
        op = rng.randrange(6)
        try:
            if op == 0:
                e.subscribe_user_to(k, [t % 32 for t in topics])
            elif op == 1:
                e.unsubscribe_user_from(k, topics)
            elif op == 2:
                trace.append(e.user_receive(k, orc.serialize(orc.KIND_SUBSCRIBE if step % 2 else orc.KIND_UNSUBSCRIBE, bytes(topics))))
            elif op == 3:
                e.subscribe_broker_to("p/p", [t % 32 for t in topics])
            elif op == 4:
                e.unsubscribe_broker_from("p/p", topics)
            else:
                e.add_user(k, topics[:1])   # a kick
        except pcdn.PcdnError as ex:
            trace.append(("error", ex.args[0]))
        if step % 10 == 0:
            trace.append([sorted(e.debug_interested([t], to_users_only=uo)) for t in range(32) for uo in (False, True)])
            trace.append(sorted(e.get_topic_sync(full=False)))
    trace.append(sorted(e.get_topic_sync(full=True)))
    trace.append(sorted(map(repr, e.get_user_sync(full=True))))
    e.close()
    return trace


def test_host_only_engine_accepts_the_flag(pcdn):
    for seed in range(3):
        assert run(pcdn, pcdn.FLAG_INBATCH_SUBSCRIBE, seed) == run(pcdn, 0, seed)
