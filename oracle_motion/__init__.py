"""The motion-vector oracle (test infrastructure): oracle_motion/motion.cpp + pymotion.py."""
