"""Inverted index: for every word, the files it occurs in -- the classic second MapReduce program (see init.py)."""
