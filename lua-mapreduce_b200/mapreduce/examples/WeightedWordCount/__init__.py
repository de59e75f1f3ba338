"""Weighted word count: every word of a line weighs 1 / (words in the line), summed per word (see init.py)."""
