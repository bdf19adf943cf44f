/*
 * Catalyst plan fragment -> sd_plan_desc (include/snappy_gpu.h, SD_ABI_VERSION 2), and the per-batch / per-row traffic
 * across the JNI boundary.
 *
 * Lives under org.apache.spark.sql.* because it uses private[sql] members of the reference exactly like the generated
 * code does: ColumnBatchIterator.getColumnBuffer (core/.../columnar/ColumnBatchIterator.scala:102-120), ParamLiteral
 * internals (core/.../catalyst/expressions/ParamLiteral.scala:244-250).
 *
 * NOT COMPILED in this repository's container (no JDK / scalac here).  Written against the signatures in
 * /root/reference (SnappyData 1.3.0, snappy-spark 2.1.1.9) -- every reference member used is cited where it is used; the
 * byte layouts of the C structs are the ones tests/test_abi_exports.py pins (offsets in jvm/abi_offsets.txt).
 */
package org.apache.spark.sql.execution.columnar.gpu

import java.nio.{ByteBuffer, ByteOrder}

import scala.collection.mutable.ArrayBuffer

import com.gemstone.gemfire.internal.shared.unsafe.UnsafeHolder
import io.snappydata.gpu.SnappyGpuNative

import org.apache.spark.sql.catalyst.InternalRow
import org.apache.spark.sql.catalyst.expressions._
import org.apache.spark.sql.catalyst.expressions.aggregate._
import org.apache.spark.sql.catalyst.expressions.codegen.{BufferHolder, UnsafeRowWriter}
import org.apache.spark.sql.catalyst.util.DateTimeUtils
import org.apache.spark.sql.collection.SharedUtils
import org.apache.spark.sql.execution.{ExpandExec, FilterExec, ProjectExec, SparkPlan}
import org.apache.spark.sql.execution.aggregate.SnappyHashAggregateExec
import org.apache.spark.sql.execution.columnar.{ColumnBatchIterator, ColumnTableScan}
import org.apache.spark.sql.execution.columnar.impl.{ColumnDelta, ColumnFormatEntry}
import org.apache.spark.sql.execution.metric.SQLMetric
import org.apache.spark.sql.execution.row.ResultSetTraversal
import org.apache.spark.sql.types._
import org.apache.spark.unsafe.Platform
import org.apache.spark.unsafe.types.UTF8String

/** sd_op / sd_type / sd_agg_fn values of include/snappy_gpu.h */
private[gpu] object Abi {
  final val VERSION = 2
  // sd_type
  final val BOOLEAN = 1; final val BYTE = 2; final val SHORT = 3; final val INT = 4; final val LONG = 5
  final val FLOAT = 6; final val DOUBLE = 7; final val DATE = 8; final val TIMESTAMP = 9; final val STRING = 10
  final val DECIMAL = 11
  // sd_op
  final val COL = 1; final val LIT = 2
  final val ADD = 10; final val SUB = 11; final val MUL = 12; final val DIV = 13; final val NEG = 14; final val CAST = 15
  final val EQ = 20; final val NE = 21; final val LT = 22; final val LE = 23; final val GT = 24; final val GE = 25
  final val AND = 30; final val OR = 31; final val NOT = 32; final val ISNULL = 33; final val ISNOTNULL = 34
  final val IN = 35; final val STARTSWITH = 36
  final val PAIR = 37   // (x, y) input of COVAR_POP / COVAR_SAMP / CORR
  final val GROUPING_SET = 38   // INT, a = one grouping-set mask; only in a GROUPING_ID node's list
  final val GROUPING_ID = 39    // INT, a = first of b GROUPING_SET nodes; only as the last grouping key
  // sd_agg_fn
  final val COUNT_STAR = 1; final val COUNT = 2; final val SUM = 3; final val AVG = 4; final val MIN = 5; final val MAX = 6
  // CentralMomentAgg: the child is DOUBLE (ImplicitCastInputTypes puts a Cast in front of any other numeric input)
  final val STDDEV_POP = 7; final val STDDEV_SAMP = 8; final val VAR_POP = 9; final val VAR_SAMP = 10; final val SKEWNESS = 11
  final val KURTOSIS = 12
  // Covariance / Corr: two DOUBLE children (ImplicitCastInputTypes casts them), sent as one PAIR node
  final val COVAR_POP = 13; final val COVAR_SAMP = 14; final val CORR = 15
  // First / Last: the row with the first / last scan position (the row buffer, then the column batches, rows in ordinal order)
  final val FIRST = 16; final val LAST = 17; final val FIRST_IGNORE_NULLS = 18; final val LAST_IGNORE_NULLS = 19
  // struct sizes / offsets (x86-64; jvm/abi_offsets.txt is generated from the ctypes mirror and checked by the tests)
  final val SIZEOF_COLUMN = 20; final val SIZEOF_EXPR = 20; final val SIZEOF_AGG = 8; final val SIZEOF_DESC = 104
  final val SIZEOF_LITERAL = 40
}

/** One literal slot of the plan: how to obtain THIS execution's value (ParamLiteral.value changes per execution of a
  * cached plan, core/.../catalyst/expressions/ParamLiteral.scala:244-330) and how to convert it for the C ABI. */
final case class LiteralSlot(expr: Expression, sdType: Int, decimalScale: Int,
    /** literal compared with Cast(dateColumn AS STRING) by upstream PromoteStrings: sent as DATE days */
    stringAsDate: Boolean)

/** Off-heap image of sd_plan_desc plus what the operator needs at run time. */
final class GpuPlanDesc(val address: Long, val scan: ColumnTableScan, val scanColumns: Array[Int] /* table ordinals */ ,
    val literals: Array[LiteralSlot], val partialSchema: StructType) {
  def numLiterals: Int = literals.length

  /** sd_literal[numLiterals] for this execution; the block (and the string bytes behind it) is owned by the returned
    * object and freed by the caller after sd_plan_set_literals (which copies) */
  def writeLiterals(): GpuPlanSerializer.NativeBlock = GpuPlanSerializer.writeLiterals(literals)

  def free(): Unit = Platform.freeMemory(address)
}

object GpuPlanSerializer {

  def numDevices: Int = java.lang.Integer.getInteger("snappydata.gpu.devices", 1)

  final class NativeBlock(val address: Long, val size: Long) { def free(): Unit = Platform.freeMemory(address) }

  private def sdType(dt: DataType): Option[Int] = dt match {
    case BooleanType => Some(Abi.BOOLEAN); case ByteType => Some(Abi.BYTE); case ShortType => Some(Abi.SHORT)
    case IntegerType => Some(Abi.INT); case LongType => Some(Abi.LONG); case FloatType => Some(Abi.FLOAT)
    case DoubleType => Some(Abi.DOUBLE); case DateType => Some(Abi.DATE); case TimestampType => Some(Abi.TIMESTAMP)
    case StringType => Some(Abi.STRING)
    // precision <= 18: int64 unscaled (enc/Uncompressed.scala:95-98); wider: [len][BigInteger bytes] records (:330-345)
    case _: DecimalType => Some(Abi.DECIMAL)
    case _ => None
  }
  private def decPS(dt: DataType): Int = dt match {
    case d: DecimalType => (d.precision << 8) | d.scale
    case _ => 0
  }

  private final class Unsupported(msg: String) extends RuntimeException(msg)

  /** Flattens expression trees into sd_expr[] (children before parents) with common nodes shared. */
  private final class Builder(scan: ColumnTableScan, aliases: Map[ExprId, Expression]) {
    val cols = new ArrayBuffer[(Int, Boolean, Int, Int, Int)]()        // type, nullable, table ordinal, scale, precision
    val colOfAttr = new scala.collection.mutable.HashMap[ExprId, Int]()
    val exprs = new ArrayBuffer[Array[Int]]()                            // op, type, a, b, c
    val literals = new ArrayBuffer[LiteralSlot]()
    private val memo = new scala.collection.mutable.HashMap[Expression, Int]()

    private def node(op: Int, t: Int, a: Int = 0, b: Int = 0, c: Int = 0): Int = {
      exprs += Array(op, t, a, b, c); exprs.length - 1
    }
    private def typeOf(e: Expression): Int =
      sdType(e.dataType).getOrElse(throw new Unsupported(s"type ${e.dataType} of $e"))

    private def column(a: AttributeReference): Int = colOfAttr.getOrElseUpdate(a.exprId, {
      // ColumnTableScan.output attribute -> 0-based table column (what getColumnLob takes, ColumnTableScan.scala:395-398)
      val ordinal = scan.relationSchema.fieldIndex(a.name)
      val (s, p) = a.dataType match { case d: DecimalType => (d.scale, d.precision); case _ => (0, 0) }
      cols += ((typeOf(a), a.nullable, ordinal, s, p)); cols.length - 1
    })

    private def literal(e: Expression, asDate: Boolean = false): Int = {
      val t = if (asDate) Abi.DATE else typeOf(e)
      literals += LiteralSlot(e, t, e.dataType match { case d: DecimalType => d.scale; case _ => 0 }, asDate)
      node(Abi.LIT, t, literals.length - 1, 0, if (asDate) 0 else decPS(e.dataType))
    }

    private def isLiteral(e: Expression): Boolean = e match {
      case _: Literal | _: DynamicReplacableConstant => true   // Literal, TokenLiteral, ParamLiteral, DynamicFoldableExpression
      case _ => false
    }

    /** upstream Spark 2.1 PromoteStrings turns `dateCol >= '1994-01-01'` into `Cast(dateCol, StringType) >= '1994-01-01'`
      * (SURVEY.md Appendix B.8); ISO dates order like their day numbers, so it is sent as an int-day compare */
    private object DateAsString {
      def unapply(e: Expression): Option[AttributeReference] = e match {
        case Cast(a: AttributeReference, StringType) if a.dataType == DateType => Some(a)
        case _ => None
      }
    }

    /** spark_grouping_id of GROUP BY ... WITH ROLLUP / CUBE / GROUPING SETS: the set nodes, then the GROUPING_ID node */
    def groupingId(masks: Seq[Int]): Int = {
      val first = exprs.length
      masks.foreach(m => node(Abi.GROUPING_SET, Abi.INT, m))
      node(Abi.GROUPING_ID, Abi.INT, first, masks.length)
    }

    /** the input of a two-input aggregate: a PAIR node over x and y (both DOUBLE) */
    def pair(x: Expression, y: Expression): Int = node(Abi.PAIR, Abi.DOUBLE, add(x), add(y))

    def add(e0: Expression): Int = memo.getOrElseUpdate(e0, e0 match {
      case a: AttributeReference if aliases.contains(a.exprId) => add(aliases(a.exprId))   // ProjectExec inlined
      case a: AttributeReference => node(Abi.COL, typeOf(a), column(a))
      case Alias(c, _) => add(c)
      case l if isLiteral(l) => literal(l)
      case Add(l, r) => node(Abi.ADD, typeOf(e0), add(l), add(r))
      case Subtract(l, r) => node(Abi.SUB, typeOf(e0), add(l), add(r))
      case Multiply(l, r) => node(Abi.MUL, typeOf(e0), add(l), add(r))
      case Divide(l, r) => node(Abi.DIV, typeOf(e0), add(l), add(r))
      case UnaryMinus(c) => node(Abi.NEG, typeOf(e0), add(c))
      case Cast(c, dt) if dt == c.dataType => add(c)
      case Cast(c, dt) => node(Abi.CAST, typeOf(e0), add(c), 0, decPS(dt))
      case cmp: BinaryComparison =>
        val op = cmp match {
          case _: EqualTo => Abi.EQ; case _: LessThan => Abi.LT; case _: LessThanOrEqual => Abi.LE
          case _: GreaterThan => Abi.GT; case _: GreaterThanOrEqual => Abi.GE
          case _ => throw new Unsupported(s"comparison $cmp")      // EqualNullSafe
        }
        (cmp.left, cmp.right) match {
          case (DateAsString(a), lit) if isLiteral(lit) => node(op, Abi.BOOLEAN, add(a), literal(lit, asDate = true))
          case (lit, DateAsString(a)) if isLiteral(lit) => node(op, Abi.BOOLEAN, literal(lit, asDate = true), add(a))
          case (l, r) => node(op, Abi.BOOLEAN, add(l), add(r))
        }
      case Not(EqualTo(l, r)) => node(Abi.NE, Abi.BOOLEAN, add(l), add(r))
      case And(l, r) => node(Abi.AND, Abi.BOOLEAN, add(l), add(r))
      case Or(l, r) => node(Abi.OR, Abi.BOOLEAN, add(l), add(r))
      case Not(c) => node(Abi.NOT, Abi.BOOLEAN, add(c))
      case IsNull(c) => node(Abi.ISNULL, Abi.BOOLEAN, add(c))
      case IsNotNull(c) => node(Abi.ISNOTNULL, Abi.BOOLEAN, add(c))
      case In(v, list) if list.nonEmpty && list.forall(isLiteral) =>
        val value = add(v)
        val first = literals.length
        list.foreach { l => literals += LiteralSlot(l, typeOf(v), decPS(v.dataType) & 0xff, stringAsDate = false) }
        node(Abi.IN, Abi.BOOLEAN, value, first, list.length)
      case StartsWith(l, r) if isLiteral(r) => node(Abi.STARTSWITH, Abi.BOOLEAN, add(l), literal(r))
      case other => throw new Unsupported(s"expression ${other.getClass.getSimpleName}: $other")
    })
  }

  /** GROUP BY ... WITH ROLLUP / WITH CUBE / GROUPING SETS as upstream Spark 2.1.1's ResolveGroupingAnalytics plans it (restated;
    * the fork's analyzer source is not at hand): ExpandExec(projections, output, ProjectExec(c ++ groupByAliases, ...)) under
    * the partial aggregate, where every projection is  c ++ (per GROUP BY key: its attribute | null literal) ++ Literal(mask)
    * and output = c ++ the keys' new instances ++ gid, the aggregate grouping by those n + 1 attributes.  The mask of a
    * projection must be the one its null literals spell in SnappyParser's convention (bit n-1-k set <=> key k absent,
    * core/SnappyParser.scala:564-571).  Returns (the n key attributes of Expand's child, the masks); None for any other Expand --
    * e.g. RewriteDistinctAggregates', whose projections null aggregate inputs, not keys. */
  private def groupingSets(agg: SnappyHashAggregateExec, e: ExpandExec): Option[(Seq[Attribute], Seq[Int])] = {
    val n = agg.groupingExpressions.length - 1
    val c = e.output.length - n - 1
    if (n < 1 || c < 0 || e.child.output.length != c + n || e.projections.isEmpty) return None
    val grouped = agg.groupingExpressions.map {
      case a: Attribute => Some(a.exprId)
      case _ => None
    }
    if (grouped != e.output.drop(c).map(a => Some(a.exprId))) return None
    if (e.output.last.dataType != IntegerType || e.output.last.nullable) return None
    val prefix = e.child.output.take(c).map(_.exprId)
    val keys = e.child.output.drop(c)
    val masks = e.projections.map { p =>
      if (p.length != c + n + 1) return None
      if (p.take(c).map { case a: Attribute => Some(a.exprId); case _ => None } != prefix.map(Some(_))) return None
      var mask = 0
      for (i <- 0 until n) p(c + i) match {
        case a: Attribute if a.exprId == keys(i).exprId =>
        case Literal(null, _) => mask |= 1 << (n - 1 - i)
        case _ => return None
      }
      p(c + n) match {
        case Literal(m: Int, IntegerType) if m == mask => mask
        case _ => return None
      }
    }
    if (masks.distinct.length != masks.length) None else Some((keys, masks))   // duplicate sets: refused by the library too
  }

  /** Some(desc) iff the fragment is SnappyHashAggregateExec(Partial) over [Project] [Filter] ColumnTableScan
    * (core/.../aggregate/SnappyHashAggregateExec.scala:72-80; planned at StoreDataSourceStrategy.scala:128-130,236-240)
    * with expressions the C ABI expresses and a plan the library accepts; anything else stays on the stock operators.
    * That is a PLANNING decision -- once a GPU plan is chosen its failures are exceptions, never a CPU fallback. */
  def tryBuild(agg: SnappyHashAggregateExec): Option[GpuPlanDesc] = {
    def unwrap(p: SparkPlan, filters: Seq[Expression], aliases: Map[ExprId, Expression])
        : Option[(ColumnTableScan, Seq[Expression], Map[ExprId, Expression])] = p match {
      case FilterExec(cond, child) => unwrap(child, filters :+ cond, aliases)
      case ProjectExec(list, child) =>
        unwrap(child, filters, aliases ++ list.collect { case a @ Alias(c, _) => a.exprId -> c })
      case scan: ColumnTableScan if scan.otherRDDs.isEmpty && !scan.isForSampleReservoirAsRegion =>
        Some((scan, filters, aliases))
      case _ => None
    }
    if (agg.hasDistinct || !agg.aggregateExpressions.forall(a => a.mode == Partial && !a.isDistinct)) return None
    // ROLLUP / CUBE / GROUPING SETS: Expand directly under the aggregate, in ResolveGroupingAnalytics' shape only
    val (below, sets) = agg.child match {
      case e: ExpandExec => groupingSets(agg, e) match {
        case Some(s) => (e.child, Some(s))
        case None => return None
      }
      case other => (other, None)
    }
    unwrap(below, Nil, Map.empty).flatMap { case (scan, filters, aliases) =>
      try {
        val b = new Builder(scan, aliases)
        val filter = if (filters.isEmpty) -1 else b.add(filters.reduce(And))
        // grouping sets: the GROUP BY keys (Expand's child projects them as aliases); spark_grouping_id follows below
        val groupKeys = sets match {
          case Some((attrs, _)) => attrs.map(b.add(_)).toArray
          case None => agg.groupingExpressions.map(b.add(_)).toArray
        }
        val aggs = agg.aggregateExpressions.map { ae =>
          ae.aggregateFunction match {
            case Count(Seq(l)) if l.foldable && l.eval(null) != null => (Abi.COUNT_STAR, -1)   // count(*) == count(1)
            case Count(Seq(c)) => (Abi.COUNT, b.add(c))
            case Sum(c) => (Abi.SUM, b.add(c))
            case Average(c) => (Abi.AVG, b.add(c))
            case Min(c) => (Abi.MIN, b.add(c))
            case Max(c) => (Abi.MAX, b.add(c))
            case m @ (StddevPop(_) | StddevSamp(_) | VariancePop(_) | VarianceSamp(_) | Skewness(_) | Kurtosis(_)) =>
              val c = m.children.head
              val fn = m match {
                case _: StddevPop => Abi.STDDEV_POP
                case _: StddevSamp => Abi.STDDEV_SAMP
                case _: VariancePop => Abi.VAR_POP
                case _: VarianceSamp => Abi.VAR_SAMP
                case _: Skewness => Abi.SKEWNESS
                case _ => Abi.KURTOSIS
              }
              (fn, b.add(c))
            case c @ (CovPopulation(_, _) | CovSample(_, _) | Corr(_, _)) =>
              val Seq(x, y) = c.children
              val fn = c match {
                case _: CovPopulation => Abi.COVAR_POP
                case _: CovSample => Abi.COVAR_SAMP
                case _ => Abi.CORR
              }
              (fn, b.pair(x, y))
            // first / first_value / last / last_value; Dataset.dropDuplicates(cols) is First(c) per other column
            case First(c, Literal(ignoreNulls: Boolean, BooleanType)) =>
              (if (ignoreNulls) Abi.FIRST_IGNORE_NULLS else Abi.FIRST, b.add(c))
            case Last(c, Literal(ignoreNulls: Boolean, BooleanType)) =>
              (if (ignoreNulls) Abi.LAST_IGNORE_NULLS else Abi.LAST, b.add(c))
            case f => throw new Unsupported(s"aggregate function ${f.prettyName}")
          }
        }.toArray
        // the set nodes come last, so that the scan's generated source is the plain GROUP BY's
        val keys = sets.fold(groupKeys)(s => groupKeys :+ b.groupingId(s._2))
        // make sure every scan column the kernel must read exists even when only count(*) is asked for
        val addr = write(b, filter, keys, aggs)
        // the library validates the plan (types, casts, limits) and compiles / finds its kernel: probe it once here
        val probe = try SnappyGpuNative.planCreate(addr) catch {
          case e: RuntimeException => Platform.freeMemory(addr); throw new Unsupported(e.getMessage)
        }
        SnappyGpuNative.planDestroy(probe)
        // rows that come back: UnsafeRow(groupingAttributes ++ aggregateBufferAttributes) = the partial aggregate's output
        val partialSchema = StructType(agg.output.map(a => StructField(a.name, a.dataType, a.nullable)))
        Some(new GpuPlanDesc(addr, scan, b.cols.map(_._3).toArray, b.literals.toArray, partialSchema))
      } catch {
        case _: Unsupported => None
      }
    }
  }

  /** sd_plan_desc + its arrays in ONE off-heap block; pointers are absolute addresses into the block */
  private def write(b: Builder, filter: Int, keys: Array[Int], aggs: Array[(Int, Int)]): Long = {
    def align8(x: Long): Long = (x + 7L) & ~7L
    val oCols = align8(Abi.SIZEOF_DESC)
    val oExprs = align8(oCols + b.cols.length * Abi.SIZEOF_COLUMN)
    val oKeys = align8(oExprs + b.exprs.length * Abi.SIZEOF_EXPR)
    val oAggs = align8(oKeys + keys.length * 4)
    val oLits = align8(oAggs + aggs.length * Abi.SIZEOF_AGG)
    val size = align8(oLits + b.literals.length * 4) + 8
    val base = Platform.allocateMemory(size)
    Platform.setMemory(base, 0.toByte, size)
    def i32(off: Long, v: Int): Unit = Platform.putInt(null, base + off, v)
    def ptr(off: Long, target: Long): Unit = Platform.putLong(null, base + off, base + target)
    i32(0, Abi.VERSION)
    i32(4, b.cols.length); ptr(8, oCols)
    i32(16, b.exprs.length); ptr(24, oExprs)
    i32(32, filter)
    i32(36, keys.length); ptr(40, oKeys)
    i32(48, aggs.length); ptr(56, oAggs)
    i32(64, 0); ptr(72, oKeys)                      // nproj = 0: aggregate plans do not project
    i32(80, b.literals.length); ptr(88, oLits)
    i32(96, 0)
    b.cols.zipWithIndex.foreach { case ((t, nullable, ord, scale, prec), i) =>
      val o = oCols + i * Abi.SIZEOF_COLUMN
      i32(o, t); i32(o + 4, if (nullable) 1 else 0); i32(o + 8, ord); i32(o + 12, scale); i32(o + 16, prec)
    }
    b.exprs.zipWithIndex.foreach { case (e, i) =>
      val o = oExprs + i * Abi.SIZEOF_EXPR
      i32(o, e(0)); i32(o + 4, e(1)); i32(o + 8, e(2)); i32(o + 12, e(3)); i32(o + 16, e(4))
    }
    keys.zipWithIndex.foreach { case (k, i) => i32(oKeys + 4 * i, k) }
    aggs.zipWithIndex.foreach { case ((fn, e), i) => i32(oAggs + 8 * i, fn); i32(oAggs + 8 * i + 4, e) }
    b.literals.zipWithIndex.foreach { case (l, i) => i32(oLits + 4 * i, l.sdType) }
    base
  }

  /** sd_literal[n] for this execution: {type:4, is_null:4, i:8, d:8, s:8, slen:4, pad:4}; string bytes follow the array, and
   *  so do the unscaled values of DECIMAL slots wider than 18 digits (BigInteger.toByteArray at the slot's scale) */
  def writeLiterals(literals: Array[LiteralSlot]): NativeBlock = {
    val values = literals.map { l =>
      l.expr match {
        case d: DynamicReplacableConstant => d.value     // ParamLiteral / TokenLiteral: the value bound for THIS execution
        case lit: Literal => lit.value
        case other => other.eval(null)
      }
    }
    val strings = values.zip(literals).map {
      case (s: UTF8String, l) if !l.stringAsDate => s.getBytes
      case (v: Decimal, l) => l.expr.dataType match {
        case d: DecimalType if d.precision > Decimal.MAX_LONG_DIGITS =>
          v.toJavaBigDecimal.setScale(d.scale).unscaledValue.toByteArray
        case _ => null
      }
      case _ => null
    }
    val head = literals.length.toLong * Abi.SIZEOF_LITERAL
    val size = head + strings.map(s => if (s eq null) 0 else s.length).sum + 8
    val base = Platform.allocateMemory(size)
    Platform.setMemory(base, 0.toByte, size)
    var tail = base + head
    var i = 0
    while (i < literals.length) {
      val o = base + i.toLong * Abi.SIZEOF_LITERAL
      val l = literals(i)
      Platform.putInt(null, o, l.sdType)
      values(i) match {
        case null => Platform.putInt(null, o + 4, 1)
        case s: UTF8String if l.stringAsDate =>          // '1994-01-01' against a DATE column: days since epoch
          val days = DateTimeUtils.stringToDate(s)
          if (days.isEmpty) Platform.putInt(null, o + 4, 1) else Platform.putLong(null, o + 8, days.get.toLong)
        case s: UTF8String =>
          val bytes = strings(i)
          Platform.copyMemory(bytes, Platform.BYTE_ARRAY_OFFSET, null, tail, bytes.length)
          Platform.putLong(null, o + 24, tail); Platform.putInt(null, o + 32, bytes.length)
          tail += bytes.length
        case v: Boolean => Platform.putLong(null, o + 8, if (v) 1L else 0L)
        case v: Byte => Platform.putLong(null, o + 8, v.toLong)
        case v: Short => Platform.putLong(null, o + 8, v.toLong)
        case v: Int => Platform.putLong(null, o + 8, v.toLong)          // INT and DATE
        case v: Long => Platform.putLong(null, o + 8, v)                // LONG and TIMESTAMP
        case v: Float => Platform.putDouble(null, o + 16, v.toDouble)
        case v: Double => Platform.putDouble(null, o + 16, v)
        case _: Decimal if strings(i) ne null =>         // DECIMAL(p > 18): its bytes, like a string literal's
          val bytes = strings(i)
          Platform.copyMemory(bytes, Platform.BYTE_ARRAY_OFFSET, null, tail, bytes.length)
          Platform.putLong(null, o + 24, tail); Platform.putInt(null, o + 32, bytes.length)
          tail += bytes.length
        case v: Decimal => Platform.putLong(null, o + 8, v.toUnscaledLong)   // at the slot's scale (Catalyst cast it to the column type)
        case other => throw new IllegalStateException(s"literal value $other of ${other.getClass}")
      }
      i += 1
    }
    new NativeBlock(base, size)
  }

  // direct buffers: the same call SharedUtils.toUnsafeRow makes (encoders/.../collection/SharedUtils.scala:68-78)
  private def address(buf: ByteBuffer): Long =
    if (buf.isDirect) UnsafeHolder.getDirectBufferAddress(buf) + buf.position() else 0L

  /**
   * One column batch.  `stats` is what colInput.next() returned (ColumnTableScan.scala:518-543).  Buffers are fetched
   * through the iterator's real API: getColumnLob(tableColumn) for values; deltas and the delete mask through
   * getColumnBuffer(columnIndex, throwIfMissing = false) with the region-key arithmetic of
   * ColumnDelta.deltaColumnIndex (encoders/.../impl/ColumnDelta.scala:300-301) and ColumnFormatEntry.DELETE_MASK_COL_INDEX
   * (.../ColumnFormatEntry.scala:87) -- exactly what getUpdatedColumnDecoder / getDeletedColumnDecoder do
   * (ColumnBatchIterator.scala:122-163).  The iterator retains every ColumnFormatValue it hands out until the next
   * moveNext() (:165-184), and sd_batch_submit has copied the bytes when it returns, so ownership is unchanged.
   */
  def submitBatch(plan: Long, it: ColumnBatchIterator, stats: ByteBuffer, desc: GpuPlanDesc): Unit = {
    val nCols = desc.scanColumns.length
    val nTableCols = desc.scan.relationSchema.length
    val numStatsFields = 1 + 3 * nTableCols                    // ColumnStatsSchema.numStatsColumns (ColumnEncoding.scala:1015-1036)
    val statsRow = SharedUtils.toUnsafeRow(stats, numStatsFields)
    var numRows = statsRow.getInt(0)                           // ColumnStatsSchema.COUNT_INDEX_IN_SCHEMA
    // old-format delta stats row: full stats may be obsolete -> no skipping for this batch (ColumnTableScan.scala:536-539)
    var hasUpdates = it.getCurrentDeltaStats ne null
    val skipAllowed = !hasUpdates
    if (numRows < 0) { hasUpdates = true; numRows = -numRows } // count < 0 marks delta updates (:524-528)

    val addrs = new Array[Long](nCols); val lens = new Array[Long](nCols); val heap = new Array[Array[Byte]](nCols)
    val heapOff = new Array[Int](nCols)
    val d0a = new Array[Long](nCols); val d0l = new Array[Long](nCols); val d0h = new Array[Array[Byte]](nCols)
    val d1a = new Array[Long](nCols); val d1l = new Array[Long](nCols); val d1h = new Array[Array[Byte]](nCols)
    val d0o = new Array[Int](nCols); val d1o = new Array[Int](nCols)
    def place(buf: ByteBuffer, i: Int, a: Array[Long], l: Array[Long], h: Array[Array[Byte]], off: Array[Int]): Unit = {
      l(i) = buf.remaining()
      if (buf.isDirect) a(i) = address(buf)
      else { h(i) = buf.array(); off(i) = buf.arrayOffset() + buf.position() }   // heap buffer: copied by the shim (no pinning)
    }
    var i = 0
    while (i < nCols) {
      val tableCol = desc.scanColumns(i)                       // 0-based, as getColumnLob takes it
      place(it.getColumnLob(tableCol), i, addrs, lens, heap, heapOff)
      if (hasUpdates) {
        val deltaPosition = ColumnDelta.deltaColumnIndex(tableCol, 0)
        val u0 = it.getColumnBuffer(deltaPosition, throwIfMissing = false)          // depth 0 (wins on equal position)
        val u1 = it.getColumnBuffer(deltaPosition - 1, throwIfMissing = false)      // depth 1
        if (u0 ne null) place(u0, i, d0a, d0l, d0h, d0o)
        if (u1 ne null) place(u1, i, d1a, d1l, d1h, d1o)
      }
      i += 1
    }
    val del = it.getColumnBuffer(ColumnFormatEntry.DELETE_MASK_COL_INDEX, throwIfMissing = false)
    val stHeap = if (!skipAllowed || stats.isDirect) null else stats.array()
    // throws RuntimeException(sd_last_error()) on a non-zero status
    SnappyGpuNative.batchSubmit(plan, numRows, nCols, addrs, lens, heap, heapOff,
      d0a, d0l, d0h, d0o, d1a, d1l, d1h, d1o,
      if ((del ne null) && del.isDirect) address(del) else 0L, if (del ne null) del.remaining().toLong else 0L,
      if ((del ne null) && !del.isDirect) del.array() else null,
      if ((del ne null) && !del.isDirect) del.arrayOffset() + del.position() else 0,
      if (skipAllowed && stats.isDirect) address(stats) else 0L, if (skipAllowed) stats.remaining().toLong else 0L,
      stHeap, if (stHeap ne null) stats.arrayOffset() + stats.position() else 0,
      nTableCols, it.getCurrentBucketId, it.getCurrentBatchId)
  }

  /**
   * Rows not yet rolled over into column batches: the first element of the partition iterator is a ResultSetTraversal
   * whose JDBC ResultSet the generated loop reads column by column with numBatchRows = 1
   * (ColumnTableScan.scala:236-241,572-588; core/.../row/RowFormatScanRDD.scala:446-456).  Here they are written as
   * UnsafeRows of the plan's scan columns, [int64 size][row]..., and handed over in chunks (sd_rows_submit).
   */
  def submitRowBuffer(plan: Long, rowInput: Iterator[_], desc: GpuPlanDesc): Long = {
    val rs = rowInput.asInstanceOf[ResultSetTraversal].rs
    val types = desc.scanColumns.map(ord => desc.scan.relationSchema(ord).dataType)
    val n = types.length
    val row = new UnsafeRow(n)
    val holder = new BufferHolder(row, 64)
    val writer = new UnsafeRowWriter(holder, n)
    var chunk = ByteBuffer.allocateDirect(1 << 20).order(ByteOrder.nativeOrder())
    var rowsInChunk = 0
    var total = 0L
    def flush(): Unit = if (rowsInChunk > 0) {
      SnappyGpuNative.rowsSubmit(plan, address(chunk.duplicate().position(0).asInstanceOf[ByteBuffer]), chunk.position().toLong, rowsInChunk)
      chunk.clear(); rowsInChunk = 0
    }
    while (rs.next()) {
      holder.reset(); writer.zeroOutNullBytes()
      var c = 0
      while (c < n) {
        val j = c + 1                                            // JDBC columns are 1-based, in scan-column order
        types(c) match {
          case BooleanType => val v = rs.getBoolean(j); if (rs.wasNull()) writer.setNullAt(c) else writer.write(c, v)
          case ByteType => val v = rs.getByte(j); if (rs.wasNull()) writer.setNullAt(c) else writer.write(c, v)
          case ShortType => val v = rs.getShort(j); if (rs.wasNull()) writer.setNullAt(c) else writer.write(c, v)
          case IntegerType => val v = rs.getInt(j); if (rs.wasNull()) writer.setNullAt(c) else writer.write(c, v)
          case LongType => val v = rs.getLong(j); if (rs.wasNull()) writer.setNullAt(c) else writer.write(c, v)
          case FloatType => val v = rs.getFloat(j); if (rs.wasNull()) writer.setNullAt(c) else writer.write(c, v)
          case DoubleType => val v = rs.getDouble(j); if (rs.wasNull()) writer.setNullAt(c) else writer.write(c, v)
          case DateType =>
            val v = rs.getDate(j); if (v eq null) writer.setNullAt(c) else writer.write(c, DateTimeUtils.fromJavaDate(v))
          case TimestampType =>
            val v = rs.getTimestamp(j); if (v eq null) writer.setNullAt(c) else writer.write(c, DateTimeUtils.fromJavaTimestamp(v))
          case StringType =>
            val v = rs.getString(j); if (v eq null) writer.setNullAt(c) else writer.write(c, UTF8String.fromString(v))
          case d: DecimalType =>
            val v = rs.getBigDecimal(j)
            if (v eq null) writer.setNullAt(c) else writer.write(c, Decimal(v, d.precision, d.scale), d.precision, d.scale)
          case other => throw new IllegalStateException(s"row buffer column type $other")
        }
        c += 1
      }
      val size = holder.totalSize()
      if (chunk.remaining() < 8 + size) {
        flush()
        if (chunk.capacity() < 8 + size) chunk = ByteBuffer.allocateDirect(2 * (8 + size)).order(ByteOrder.nativeOrder())
      }
      chunk.putLong(size.toLong)
      chunk.put(holder.buffer, 0, size)
      rowsInChunk += 1; total += 1
    }
    flush()
    total
  }

  /** sd_plan_finish -> rows of the partial aggregate's output schema: [int64 sizeInBytes][UnsafeRow] repeated; each row is
    * wrapped with UnsafeRow.pointTo over a copy of its bytes (rows outlive the native buffer). */
  def finishToUnsafeRows(plan: Long, desc: GpuPlanDesc, numOutputRows: SQLMetric): Iterator[InternalRow] = {
    var cap = 64L << 10
    var block = Platform.allocateMemory(cap)
    var len = SnappyGpuNative.planFinish(plan, block, cap)
    if (len < 0) {                                              // SD_ERR_OVERFLOW: -needed; the execution itself is complete
      Platform.freeMemory(block); cap = -len + 64; block = Platform.allocateMemory(cap)
      len = SnappyGpuNative.planFinish(plan, block, cap)
    }
    val n = desc.partialSchema.length
    val rows = new ArrayBuffer[InternalRow]()
    var pos = 0L
    while (pos + 8 <= len) {
      val size = Platform.getLong(null, block + pos).toInt
      val bytes = new Array[Byte](size)
      Platform.copyMemory(null, block + pos + 8, bytes, Platform.BYTE_ARRAY_OFFSET, size)
      val r = new UnsafeRow(n)
      r.pointTo(bytes, Platform.BYTE_ARRAY_OFFSET, size)
      rows += r
      pos += 8 + size
    }
    Platform.freeMemory(block)
    if (numOutputRows ne null) numOutputRows.add(rows.length)
    rows.iterator
  }
}
