"""WordCount whose result comes out in one global key order: a first-letter key-range partitionfn (see init.py)."""
