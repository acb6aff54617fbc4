"""gnss_ins_sim_b200: H100-native Monte-Carlo strapdown-INS engine behind the
gnss-ins-sim plugin API (free integration + IMU error generation + ensemble error
statistics + Allan variance).  See DESIGN.md."""
__version__ = '0.1.0'
