"""H100-native vector search for the Lab2 RAG path of confluentinc/quickstart-streaming-agents.

Import as ``qsa_b200`` (see qsa_b200/__init__.py).  Modules:
  capi      ctypes binding of libsa_b200.so (include/sa_api.h)
  engine    VectorIndex: device-memory holder + calls into the C ABI
  operator  VECTOR_SEARCH_AGG drop-in over topic records
  wire      Avro / Confluent wire codec, schemas
  transport file-log topics with Kafka semantics
"""
