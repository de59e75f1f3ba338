"""Key-number sum: the numbers of text lines "key number" summed per key -- bytes per URL, sales per product, edge
weights per node (see init.py)."""
