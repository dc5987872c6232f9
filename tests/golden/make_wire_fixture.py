"""Copies records of the reference's captured Lab3 stream into tests/golden/ as the Avro codec's known-answer fixtures.
These are DATA records captured from Kafka (base64 Confluent-framed Avro, assets/lab3/data/ride_requests.jsonl of the
reference repository, 30 873 records), not source code.

  ride_requests_head.jsonl    200 records: the first 120, and two runs of 40 further in
  ride_requests_sample.jsonl  every 256th record, plus the records with the earliest and the latest request_ts

    python tests/golden/make_wire_fixture.py <reference checkout>/assets/lab3/data/ride_requests.jsonl
"""
import base64
import itertools
import os
import struct
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))


def request_ts(line):
    import json
    sys.path.insert(0, ROOT)
    from qsa_b200.wire import avro, schemas
    raw = base64.b64decode(json.loads(line)["value"])
    assert struct.unpack(">I", raw[1:5])[0] == 100008
    return avro.CompiledSchema(schemas.RIDE_REQUESTS_VALUE).decode(raw, 5)["request_ts"]


if __name__ == "__main__":
    with open(sys.argv[1]) as f:
        lines = f.readlines()
    head = list(itertools.islice(lines, 20000))
    picked = head[:120] + head[5000:5040] + head[19960:20000]
    with open(os.path.join(HERE, "ride_requests_head.jsonl"), "w") as out:
        out.writelines(picked)
    ts = [request_ts(line) for line in lines]
    keep = sorted(set(range(0, len(lines), 256)) | {ts.index(min(ts)), ts.index(max(ts))})
    with open(os.path.join(HERE, "ride_requests_sample.jsonl"), "w") as out:
        out.writelines(lines[i] for i in keep)
    print("wrote", len(picked), "+", len(keep), "records")
